// TEST INFRASTRUCTURE: a HOST build of the product's own per-pixel shadow math (vqengine_b200/csrc/vq_shadow_math.cuh with
// VQ_HOST_CHECK), so that tests/test_shadow_math_host.py can compare it with the oracle on the CPU. Built by the test with
// g++ -O2 -ffp-contract=off; never linked into the product.
#define VQ_HOST_CHECK 1
#include "../../vqengine_b200/csrc/vq_shadow_math.cuh"
#include <vector>

extern "C" {

// base: the pass without casters (what K1 produces for per_frame_without_casters); out = base + caster terms
void hostcheck_shade_casters(const VqPerFrameData* pf, const VqPerViewLightingData* pv, const VqShadowMaps* sm,
                             const float* pos, const float* nrm, const float* alb, const float* base, int n_pixels, float* out) {
    vqshadow::ShadowLights L;
    vqshadow::fill_shadow_lights(L, *pf, *pv, *sm);
    for (int i = 0; i < n_pixels; ++i) {
        auto ld = [&](const float* p) { vqshadow::Px4 r; r.x = p[4 * i]; r.y = p[4 * i + 1]; r.z = p[4 * i + 2]; r.w = p[4 * i + 3]; return r; };
        const vqshadow::Px4 o = vqshadow::shade_casters(L, ld(pos), ld(nrm), ld(alb), ld(base));
        out[4 * i] = o.x; out[4 * i + 1] = o.y; out[4 * i + 2] = o.z; out[4 * i + 3] = o.w;
    }
}
// the per-pixel PCF records the device kernel stores (5 bits per caster)
void hostcheck_pcf_records(const VqPerFrameData* pf, const VqPerViewLightingData* pv, const VqShadowMaps* sm,
                           const float* pos, const float* nrm, int n_pixels, unsigned long long* out) {
    vqshadow::ShadowLights L;
    vqshadow::fill_shadow_lights(L, *pf, *pv, *sm);
    for (int i = 0; i < n_pixels; ++i) {
        auto ld = [&](const float* p) { vqshadow::Px4 r; r.x = p[4 * i]; r.y = p[4 * i + 1]; r.z = p[4 * i + 2]; r.w = p[4 * i + 3]; return r; };
        out[i] = vqshadow::pcf_record(L, ld(pos), ld(nrm));
    }
}
// the same tap counts handed to an array instead of the record: [n_pixels][11], -1 where a slot is not reported
void hostcheck_pcf_counts(const VqPerFrameData* pf, const VqPerViewLightingData* pv, const VqShadowMaps* sm,
                          const float* pos, const float* nrm, int n_pixels, int* out) {
    vqshadow::ShadowLights L;
    vqshadow::fill_shadow_lights(L, *pf, *pv, *sm);
    for (int i = 0; i < n_pixels; ++i) {
        auto ld = [&](const float* p) { return vqshadow::v3(vqshadow::F(p[4 * i]), vqshadow::F(p[4 * i + 1]), vqshadow::F(p[4 * i + 2])); };
        vqshadow::ArraySink c;
        for (int k = 0; k < 11; ++k) c.c[k] = -1;
        vqshadow::caster_counts(L, ld(pos), ld(nrm), c);
        for (int k = 0; k < 11; ++k) out[11 * i + k] = c.c[k];
    }
}
void hostcheck_per_frame_without_casters(const VqPerFrameData* pf, VqPerFrameData* out) { *out = vqshadow::per_frame_without_casters(*pf); }

// the launcher's sequence (vq_depth_min_pyramid) with the kernels' texel function run in loops
int hostcheck_depth_min_pyramid(const float* depth, int pitch, int W, int H, float* levels, int n_levels) {
    if (n_levels < 1 || n_levels > vqshadow::depth_level_count(W, H)) return -1;
    for (int y = 0; y < H; ++y) for (int x = 0; x < W; ++x) levels[(size_t)y * W + x] = depth[(size_t)y * pitch + x];
    vqshadow::DepthLevelPlan plan[13];
    vqshadow::depth_pyramid_plan(W, H, n_levels, plan);
    std::vector<float> padA((size_t)((W + 1) / 2) * ((H + 1) / 2) + 1), padB(padA.size());
    const float* src = levels;
    for (int l = 1; l < n_levels; ++l) {
        const vqshadow::DepthLevelPlan& p = plan[l];
        float* pad = (l & 1) ? padA.data() : padB.data();
        for (int y = 0; y < p.ph; ++y)
            for (int x = 0; x < p.pw; ++x) {
                const float m = vqshadow::depth_min_texel(src, p.sw, p.sh, x, y);
                pad[(size_t)y * p.pw + x] = m;
                if (x < p.lw && y < p.lh) levels[p.out_offset + (size_t)y * p.lw + x] = m;
            }
        src = pad;
    }
    return vqshadow::depth_level_count(W, H);
}

}  // extern "C"
