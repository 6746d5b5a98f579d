/*
 * vqcuda_group.h — a device group: the owner of a multi-GPU world inside ONE process, part of the C-ABI of vqcuda.h.
 *
 * The band forms of the passes (the *_multi_signal calls, vq_specular_prefilter_ranges) store one rank's band into every rank's
 * buffers and meet their peers in the kernel's last CTA (VqPeerSignal). A group supplies what those calls need from outside the
 * kernels: peer access between the ranks' devices, one flag array per rank, each rank's order of destinations and the matching
 * signal, the row split of every band (DESIGN.md §6), and the arrival of a rank whose call was refused (the one launch here).
 *
 * Conventions are vqcuda.h's: every call returns 0 (VQ_OK) or a negative VqStatus with a vq_last_error() message; arguments are
 * checked before any device work. The band plans are host arithmetic and need no device.
 */
#ifndef VQCUDA_GROUP_H
#define VQCUDA_GROUP_H

#include "vqcuda.h"
#include "vqcuda_rendezvous.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct VqGroup VqGroup;

/* n_ranks (1..8) existing contexts, rank r = ctxs[r]. Enables peer access between every pair of DISTINCT devices (refused with
 * VQ_ERR_UNSUPPORTED, before anything is changed, if cudaDeviceCanAccessPeer says no; an already-enabled pair is fine). The same
 * device may appear more than once: that is a simulated world on one GPU. flag_arrays: NULL -> the group allocates rank r's array
 * of n_ranks zeroed words on rank r's device; else n_ranks caller-owned zeroed arrays that every rank's device can reach (e.g.
 * mapped pinned host memory), used as given. The contexts must outlive the group. Peer access is left enabled on destroy.
 * Refused with VQ_ERR_INVALID_ARG: a null `out` or `ctxs`, n_ranks outside 1..8, a null or repeated context, a null flag array. */
VQ_API int vq_group_create(VqContext* const* ctxs, int n_ranks, uint32_t* const* flag_arrays, VqGroup** out);
/* Frees the group and the flag arrays it allocated. The caller first ends every call that uses its signals. NULL is fine. */
VQ_API int vq_group_destroy(VqGroup* g);
/* Rank r's order of ranks: r first, then its peers rotated (r+1, r+2, ... mod n) in order[0..n_ranks-1]; order[n_ranks..7] = -1.
 * The destinations a rank passes to a band call are listed in this order, and vq_group_signal's flag arrays follow it. */
VQ_API int vq_group_rank_order(const VqGroup* g, int rank, int order[8]);
/* Rank r's VqPeerSignal at `epoch`: flags[k] = the flag array of rank order[k] (flags[0] its own), my_index = r, n_ranks. */
VQ_API int vq_group_signal(const VqGroup* g, int rank, uint32_t epoch, VqPeerSignal* out);

/* Rank `rank`'s arrival at `epoch` without its signalled call: stores `epoch` into word `rank` of every peer's flag array, as the
 * call's last CTA would, after all work enqueued earlier on `stream` (one launch on the rank's device). For a rank whose call of a
 * phase was refused after its peers' calls were enqueued: the peers finish instead of waiting for it. The result of that phase is
 * invalid. Refused: a null group, rank out of range. */
VQ_API int vq_group_arrive(const VqGroup* g, int rank, uint32_t epoch, void* stream);

/* The rendezvous policy of vqcuda_rendezvous.h on every rank's context: a deadline of `ns` (1..VQ_RENDEZVOUS_MAX_DEADLINE_NS) for
 * the signalled calls enqueued after this returns. Refused: a null group, ns outside the range. */
VQ_API int vq_group_set_rendezvous_deadline(const VqGroup* g, uint64_t ns);
/* vq_ctx_cancel_rendezvous on every rank's context (a host store each, no CUDA call). Refused: a null group, a rank whose context
 * has no registered deadline. */
VQ_API int vq_group_cancel(const VqGroup* g);
/* Rank `rank`'s rendezvous at `epoch` without a pass, after all work enqueued earlier on `stream`: one one-thread launch on the
 * rank's device that stores `epoch` into word `rank` of every peer's flag array and waits, under the rank's policy, until every
 * peer's word in its own array has reached `epoch`. Every rank's barrier at a fresh epoch is how a group meets again after a wait
 * gave up: once every rank's barrier has met its peers, every store of the earlier steps, a late peer's included, has landed.
 * A group of one rank launches nothing. Refused: a null group, rank out of range. */
VQ_API int vq_group_barrier(const VqGroup* g, int rank, uint32_t epoch, void* stream);

/* HOST. The rows [*row_begin, *row_end) of rank `rank` when n_rows rows are split over n_ranks ranks:
 *   even = 0: contiguous blocks whose sizes differ by at most one, rank r from floor(n_rows r / n) (the shading of a G-buffer,
 *             K2's (face, row) space, K4, the display frame);
 *   even = 1: inner boundaries on even rows, sizes differing by at most two, the larger shares first (the from-materials calls,
 *             whose 2x2 quads start on even rows).
 * A band may be empty when n_rows < n_ranks (or < 2 n_ranks with even = 1). Refused: null outputs, n_rows < 0, n_ranks outside
 * 1..8, rank outside [0, n_ranks), even not 0 or 1. */
VQ_API int vq_band_rows(int n_rows, int n_ranks, int rank, int even, int* row_begin, int* row_end);
/* HOST. The increasing, disjoint row ranges of the flattened (mip, face, row) space that rank `rank` gives
 * vq_specular_prefilter_ranges: every mip whose 6 (res >> m) rows divide by n_ranks (n_ranks > 1) is split into n_ranks equal
 * blocks and the rank takes block `rank`; every other mip is computed whole by every rank. Pairs [begin, end) go to
 * ranges[2i], ranges[2i+1]; *n_ranges receives their count (also when capacity, counted in pairs, is too small, which is refused).
 * Refused: res < 1, mips outside 1..vq_mip_level_count(res, res), n_ranks outside 1..8, rank outside [0, n_ranks), a null n_ranges,
 * a null ranges with capacity > 0, too small a capacity. */
VQ_API int vq_specular_rank_ranges(int res, int mips, int n_ranks, int rank, int* ranges, int capacity, int* n_ranges);

#ifdef __cplusplus
}
#endif
#endif /* VQCUDA_GROUP_H */
