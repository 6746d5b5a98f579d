// TEST INFRASTRUCTURE: a HOST build of the argument check vq_fsr_easu runs before it launches anything
// (vqengine_b200/csrc/vq_easu_check.cuh), so that tests/test_post_domain.py can sweep it on the CPU. Built by the test with
// g++ -O2 -ffp-contract=off; never linked into the product.
#include "../../vqengine_b200/csrc/vq_easu_check.cuh"

extern "C" {

// con0 = (scale x, scale y, bias x, bias y); `fused` selects the up path's tiling: 0 = easu_up_kernel's (EASU_UP_TILE, what
// vq_fsr_easu checks), 1 = post_fsr_up_kernel's (FUSED_UP_TILE, what vq_post_process checks). Returns the verdict (0 = accepted)
// and, in out3, {path, ncx, ncy}
int hostcheck_easu_check(const float con0[4], int in_w, int in_h, int out_w, int out_h, int fused, int* out3) {
    int ncx = 0, ncy = 0;
    const int v = vqeasu::check(con0, in_w, in_h, out_w, out_h, &ncx, &ncy, fused ? vqeasu::FUSED_UP_TILE : vqeasu::EASU_UP_TILE);
    out3[0] = vqeasu::path(con0, in_w, in_h, out_w, out_h);
    out3[1] = ncx;
    out3[2] = ncy;
    return v;
}

// floor(easu_pos(o)) for o = 0 .. n_out-1: the 'f' texel of every output pixel along one axis
void hostcheck_easu_f(float scale, float bias, int n_out, int* out) {
    for (int o = 0; o < n_out; ++o) out[o] = (int)floorf(vqeasu::pos(o, scale, bias));
}

}  // extern "C"
