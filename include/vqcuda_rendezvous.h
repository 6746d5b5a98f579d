/*
 * vqcuda_rendezvous.h — a deadline, a cancel and a status record for the in-kernel rendezvous of a context's signalled calls, part
 * of the C-ABI of vqcuda.h.
 *
 * Every call that takes a VqPeerSignal (vqcuda.h, vqcuda_prefilter_multi.h) ends in a rendezvous run by its kernel's last CTA: it
 * stores its epoch into the peers' flag arrays, then waits until every peer's word in its own array has reached the epoch. By
 * default a peer that never arrives fails the kernel after 20 s with a trap, which loses the process's CUDA context.
 *
 * A context that registers a deadline here changes that for its own calls: the wait ends when every peer has arrived, when the
 * deadline has passed since the rank's own arrival, or when the context's cancel word is set. A wait that gives up records the
 * failure in the context's status record and the kernel ends normally; the process, its context and the device stay usable.
 *   - A call that gave up has still stored its band into every destination and its epoch into every peer's flag array. The rank's
 *     own destinations hold its own band; what the peers' bands hold there is undefined.
 *   - The status is the only way to learn of a failure: a signalled call returns VQ_OK as soon as it is enqueued.
 *   - A late peer may still store its band into this rank's destinations after the wait has given up. Before a group of ranks
 *     goes on, it meets again at a fresh epoch (vq_group_barrier, vqcuda_group.h) and clears the status.
 *
 * Conventions are vqcuda.h's: every call returns 0 (VQ_OK) or a negative VqStatus with a vq_last_error() message; arguments are
 * checked before any device work.
 */
#ifndef VQCUDA_RENDEZVOUS_H
#define VQCUDA_RENDEZVOUS_H

#include "vqcuda.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The longest deadline a context may register: the unregistered wait's bound */
#define VQ_RENDEZVOUS_MAX_DEADLINE_NS 20000000000ull

/* A context's record of the rendezvous waits that gave up since the last clear. */
typedef struct VqRendezvousStatus {
    uint32_t failures;         /* waits that gave up (deadline or cancel) */
    uint32_t first_epoch;      /* the epoch of the first of them (failures > 0) */
    uint32_t last_epoch;       /* the epoch of the one recorded last (failures > 0) */
    uint32_t missing_mask;     /* bit j: rank j's word had not reached the epoch when a wait gave up (ORed over the failures) */
    uint32_t cancelled;        /* 1: at least one of them ended because of vq_ctx_cancel_rendezvous */
} VqRendezvousStatus;

/* Registers a deadline of `ns` nanoseconds (1..VQ_RENDEZVOUS_MAX_DEADLINE_NS) for the rendezvous of the signalled calls enqueued
 * on `ctx` after this call returns. A later call changes the deadline only and does not block.
 * The first call BLOCKS: it allocates the context's cancel word (mapped, pinned host memory) and its status record (device memory),
 * zeroes the record on a stream of its own, and loads the kernel of vq_ctx_rendezvous_clear. Loading a kernel waits for the kernels
 * running on the device, so make the first registration between steps, before any signalled call is in flight. Both allocations
 * are freed with the context.
 * Refused with VQ_ERR_INVALID_ARG: a null context, ns == 0, ns > VQ_RENDEZVOUS_MAX_DEADLINE_NS. */
VQ_API int vq_ctx_set_rendezvous_deadline(VqContext* ctx, uint64_t ns);
/* Sets the context's cancel word: every wait of `ctx` that is spinning, or that starts later, ends as cancelled until
 * vq_ctx_rendezvous_clear resets the word. A plain host store, no CUDA call: any thread may call it while the device is busy.
 * Refused with VQ_ERR_INVALID_ARG: a null context, a context with no registered deadline. */
VQ_API int vq_ctx_cancel_rendezvous(VqContext* ctx);
/* BLOCKS. Copies the status record into *out, ordered after all work enqueued on `stream` before this call, then waits for the
 * copy. A record with failures == 0 says every wait of that work met its peers. A context with no registered deadline has no
 * record: *out is all zeroes. Refused with VQ_ERR_INVALID_ARG: a null context, a null `out`. */
VQ_API int vq_ctx_rendezvous_status(VqContext* ctx, void* stream, VqRendezvousStatus* out);
/* Zeroes the status record and the cancel word, ordered on `stream` after the work enqueued on it before (does not block). A
 * context with no registered deadline has nothing to clear. Refused with VQ_ERR_INVALID_ARG: a null context. */
VQ_API int vq_ctx_rendezvous_clear(VqContext* ctx, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VQCUDA_RENDEZVOUS_H */
