// TEST INFRASTRUCTURE: a stand-alone driver around the host build of the PCF code (shadow_math_host.cpp), so that
// tests/test_pcf_ref.py can run it under AddressSanitizer / UndefinedBehaviorSanitizer without loading a sanitizer runtime into
// Python. Reads one scene from argv[1], writes the per-pixel tap counts ([n][11] int32, -1 = slot not reported) to argv[2].
//   input: VqPerFrameData, VqPerViewLightingData, int32 {cube_res, spot_w, spot_h, dir_w, dir_h, n_pixels}, then float32
//          cubes [5][6][res][res], spot maps [5][spot_h][spot_w], directional map [dir_h][dir_w], positions [n][4], normals [n][4]
#include "shadow_math_host.cpp"
#include <cstdio>
#include <vector>

template <class T> static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
    if (argc != 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 3;
    VqPerFrameData pf; VqPerViewLightingData pv; int d[6];
    if (!rd(f, &pf, 1) || !rd(f, &pv, 1) || !rd(f, d, 6)) return 4;
    const int res = d[0], sw = d[1], sh = d[2], dw = d[3], dh = d[4], n = d[5];
    std::vector<float> cubes((size_t)5 * 6 * res * res), spots((size_t)5 * sw * sh), dmap((size_t)dw * dh), pos((size_t)4 * n), nrm((size_t)4 * n);
    if (!rd(f, cubes.data(), cubes.size()) || !rd(f, spots.data(), spots.size()) || !rd(f, dmap.data(), dmap.size()) ||
        !rd(f, pos.data(), pos.size()) || !rd(f, nrm.data(), nrm.size())) return 5;
    fclose(f);
    VqShadowMaps sm;
    sm.point_cubes = cubes.data(); sm.point_res = res;
    sm.spot_maps = spots.data(); sm.spot_width = sw; sm.spot_height = sh;
    sm.directional_map = dmap.data(); sm.directional_width = dw; sm.directional_height = dh;
    std::vector<int> out((size_t)11 * n);
    hostcheck_pcf_counts(&pf, &pv, &sm, pos.data(), nrm.data(), n, out.data());
    FILE* o = fopen(argv[2], "wb");
    if (!o || fwrite(out.data(), sizeof(int), out.size(), o) != out.size()) return 6;
    fclose(o);
    return 0;
}
