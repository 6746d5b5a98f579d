// ORACLE — TEST INFRASTRUCTURE ONLY. Not part of the product; never linked into libvqcuda.
//
// oracle_frame.cpp — SURVEY §8(f).2 / (f).3: the data formats and the two streaming passes either side of the
// shading path, restated as scalar C++:
//   * Radiance .hdr (RGBE) decode, as Image::LoadFromFile reaches it: stbi_loadf(path, ..., 4)
//     (Libs/VQUtils/Source/Image.cpp:119-121) -> stbi__hdr_load / stbi__hdr_convert (vendored stb_image.h v2.xx,
//     Libs/VQUtils/Libs/stb/stb_image.h:6786-7010);
//   * Image::CalculateMaxLuminance (Image.cpp:43-86);
//   * .hdr encode, as Image::SaveToDisk reaches it: stbi_write_hdr(path, x, y, 4, data) (Image.cpp:210-213)
//     -> stbi_write_hdr_core / stbiw__write_hdr_scanline / stbiw__linear_to_rgbe (stb_image_write.h);
//   * Skydome PSMain (Shaders/Skydome.hlsl:35-56, drawn at SceneRendering.cpp:1821-1850);
//   * ApplyReflections CSMain (Shaders/ApplyReflections.hlsl:31-57).
// PINNED by the reference itself: oracle/_ref/libstbref.so compiles the reference's own stb_image.h /
// stb_image_write.h in place; tests/test_frame_oracle.py compares byte-for-byte / bit-for-bit.
#include "oracle.h"
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

namespace orc {

// stbi__hdr_convert with req_comp == 4 (stb_image.h): rgb * 2^(e-136), alpha 1; e == 0 -> (0,0,0,1)
float4 HdrConvert(const uint8_t rgbe[4]) {
    if (rgbe[3] != 0) {
        const float f1 = (float)std::ldexp(1.0f, (int)rgbe[3] - (int)(128 + 8));
        return {rgbe[0] * f1, rgbe[1] * f1, rgbe[2] * f1, 1.0f};
    }
    return {0.0f, 0.0f, 0.0f, 1.0f};
}

namespace {
struct Reader {   // stbi__context over memory: reads past the end return 0 (stbi__get8)
    const uint8_t* p; size_t n, i;
    bool eof() const { return i >= n; }
    int get8() { return i < n ? p[i++] : 0; }
};
// stbi__hdr_gettoken: one line without the '\n' (lines longer than 1023 are cut and the rest of the line skipped)
std::string gettoken(Reader& r) {
    std::string s;
    char c = (char)r.get8();
    while (!r.eof() && c != '\n') {
        s.push_back(c);
        if (s.size() == 1024 - 1) {
            while (!r.eof() && r.get8() != '\n') {}
            break;
        }
        c = (char)r.get8();
    }
    return s;
}
}  // namespace

// stbi__hdr_load with req_comp = 4. Returns 0 on success, otherwise the stb failure:
//   1 "not HDR", 2 "unsupported format", 3 "unsupported data layout", 4 "invalid decoded scanline length",
//   5 "bad RLE data", 6 "too large".
int HdrDecode(const uint8_t* file, size_t n, int* outW, int* outH, std::vector<float>* rgba) {
    Reader s{file, n, 0};
    const std::string id = gettoken(s);
    if (id != "#?RADIANCE" && id != "#?RGBE") return 1;
    bool valid = false;
    for (;;) {
        const std::string t = gettoken(s);
        if (t.empty()) break;
        if (t == "FORMAT=32-bit_rle_rgbe") valid = true;
    }
    if (!valid) return 2;
    const std::string res = gettoken(s);
    if (std::strncmp(res.c_str(), "-Y ", 3) != 0) return 3;
    char* end = nullptr;
    const int height = (int)std::strtol(res.c_str() + 3, &end, 10);
    while (*end == ' ') ++end;
    if (std::strncmp(end, "+X ", 3) != 0) return 3;
    const int width = (int)std::strtol(end + 3, nullptr, 10);
    *outW = width; *outH = height;
    if (width < 0 || height < 0 || (width && height && (uint64_t)width * (uint64_t)height > (1ull << 27))) return 6;
    rgba->assign((size_t)width * height * 4, 0.0f);
    float* out = rgba->data();
    auto put = [&](size_t texel, const uint8_t* rgbe) {
        const float4 v = HdrConvert(rgbe);
        out[texel * 4 + 0] = v.x; out[texel * 4 + 1] = v.y; out[texel * 4 + 2] = v.z; out[texel * 4 + 3] = v.w;
    };
    auto flat_from = [&](size_t firstTexel) {       // "main_decode_loop": 4 bytes per texel to the end of the image
        for (size_t t = firstTexel; t < (size_t)width * height; ++t) {
            uint8_t rgbe[4];
            for (int k = 0; k < 4; ++k) rgbe[k] = (uint8_t)s.get8();
            put(t, rgbe);
        }
    };
    if (width < 8 || width >= 32768) { flat_from(0); return 0; }
    std::vector<uint8_t> scan((size_t)width * 4);
    for (int j = 0; j < height; ++j) {
        const int c1 = s.get8(), c2 = s.get8();
        int len = s.get8();
        if (c1 != 2 || c2 != 2 || (len & 0x80)) {
            // not run-length encoded: these bytes are texel 0 and the rest of the image follows flat, restarting at
            // row 0 ("yes, this makes no sense", stb_image.h) — reproduced literally
            uint8_t rgbe[4] = {(uint8_t)c1, (uint8_t)c2, (uint8_t)len, (uint8_t)s.get8()};
            put(0, rgbe);
            flat_from(1);
            return 0;
        }
        len = (len << 8) | s.get8();
        if (len != width) return 4;
        for (int k = 0; k < 4; ++k) {
            int i = 0, nleft;
            while ((nleft = width - i) > 0) {
                // stb reads 0 past the end of the stream and would spin here forever on a truncated file
                // (count == 0 makes no progress); a stream that ends inside a scanline is reported as corrupt
                if (s.eof()) return 5;
                int count = s.get8();
                if (count > 128) {
                    const uint8_t value = (uint8_t)s.get8();
                    count -= 128;
                    if (count > nleft) return 5;
                    for (int z = 0; z < count; ++z) scan[(size_t)(i++) * 4 + k] = value;
                } else {
                    if (count > nleft) return 5;
                    // count == 0 is a no-op that consumes one byte (as in stb)
                    for (int z = 0; z < count; ++z) scan[(size_t)(i++) * 4 + k] = (uint8_t)s.get8();
                }
            }
        }
        for (int i = 0; i < width; ++i) put((size_t)j * width + i, &scan[(size_t)i * 4]);
    }
    return 0;
}

// Image.cpp:43-86: the value LoadFromFile stores in Image::MaxLuminance (the other running maxima are dead code)
float CalculateMaxLuminance(const float* rgba, int width, int height) {
    float MaxLuminance = 0.0f;
    for (int h = 0; h < height; ++h)
        for (int w = 0; w < width; ++w) {
            const float* p = rgba + ((size_t)w + (size_t)width * h) * 4;
            const float lum = 0.2126f * p[0] + 0.7152f * p[1] + 0.0722f * p[2];
            if (lum > MaxLuminance) MaxLuminance = lum;
        }
    return MaxLuminance;
}

// stbiw__linear_to_rgbe (stb_image_write.h). maxcomp is stbiw__max(r, stbiw__max(g, b)) with stbiw__max(a, b) = a > b ? a : b,
// so a NaN in r or g is ignored (the comparison is false and the other operand is taken) and a NaN in b is not. C leaves
// the (unsigned char) cast of a negative, NaN or huge product undefined; the bytes are pinned to the rule vqcuda.h states
// for vq_hdr_encode_rgbe: the low byte of the product truncated to int32 (NaN -> 0, saturated at the int32 range). frexp
// gives exponent 0 for +Inf and NaN (-Inf is below the cut-off); an exponent of 128 (maxcomp >= 2^127) wraps the byte to 0.
static uint8_t TruncByte(float x) {
    if (std::isnan(x)) return 0;
    if (x >= 2147483648.0f) return 0xff;
    if (x <= -2147483648.0f) return 0;
    return (uint8_t)((int32_t)x & 0xff);
}
void LinearToRgbe(uint8_t rgbe[4], const float linear[3]) {
    const float gb = linear[1] > linear[2] ? linear[1] : linear[2];
    const float maxcomp = linear[0] > gb ? linear[0] : gb;
    if (maxcomp < 1e-32f) { rgbe[0] = rgbe[1] = rgbe[2] = rgbe[3] = 0; return; }
    int exponent = 0;
    const float mant = (float)std::frexp(maxcomp, &exponent);
    if (!std::isfinite(maxcomp)) exponent = 0;
    const float normalize = mant * 256.0f / maxcomp;
    rgbe[0] = TruncByte(linear[0] * normalize);
    rgbe[1] = TruncByte(linear[1] * normalize);
    rgbe[2] = TruncByte(linear[2] * normalize);
    rgbe[3] = (uint8_t)((exponent + 128) & 0xff);
}

// stbi_write_hdr_core with comp = 4 (Image.cpp:212): header + one RLE (or flat) scanline per row
void HdrEncode(const float* rgba, int width, int height, std::vector<uint8_t>* file) {
    file->clear();
    if (width <= 0 || height <= 0 || !rgba) return;
    auto emit = [&](const void* p, size_t n) { const uint8_t* b = (const uint8_t*)p; file->insert(file->end(), b, b + n); };
    static const char header[] = "#?RADIANCE\n# Written by stb_image_write.h\nFORMAT=32-bit_rle_rgbe\n";
    emit(header, sizeof(header) - 1);
    char buffer[128];
    const int len = std::snprintf(buffer, sizeof(buffer), "EXPOSURE=          1.0000000000000\n\n-Y %d +X %d\n", height, width);
    emit(buffer, (size_t)len);
    std::vector<uint8_t> scratch((size_t)width * 4);
    for (int y = 0; y < height; ++y) {
        const float* scanline = rgba + (size_t)y * width * 4;
        if (width < 8 || width >= 32768) {
            for (int x = 0; x < width; ++x) {
                uint8_t rgbe[4]; const float lin[3] = {scanline[x * 4 + 0], scanline[x * 4 + 1], scanline[x * 4 + 2]};
                LinearToRgbe(rgbe, lin);
                emit(rgbe, 4);
            }
            continue;
        }
        for (int x = 0; x < width; ++x) {
            uint8_t rgbe[4]; const float lin[3] = {scanline[x * 4 + 0], scanline[x * 4 + 1], scanline[x * 4 + 2]};
            LinearToRgbe(rgbe, lin);
            for (int c = 0; c < 4; ++c) scratch[(size_t)x + (size_t)width * c] = rgbe[c];
        }
        const uint8_t scanlineheader[4] = {2, 2, (uint8_t)((width & 0xff00) >> 8), (uint8_t)(width & 0x00ff)};
        emit(scanlineheader, 4);
        for (int c = 0; c < 4; ++c) {
            const uint8_t* comp = &scratch[(size_t)width * c];
            int x = 0;
            while (x < width) {
                int r = x;                                   // find first run
                while (r + 2 < width) {
                    if (comp[r] == comp[r + 1] && comp[r] == comp[r + 2]) break;
                    ++r;
                }
                if (r + 2 >= width) r = width;
                while (x < r) {                              // dump up to first run
                    int l = r - x; if (l > 128) l = 128;
                    const uint8_t lb = (uint8_t)l; emit(&lb, 1); emit(&comp[x], (size_t)l);
                    x += l;
                }
                if (r + 2 < width) {                         // output the run
                    while (r < width && comp[r] == comp[x]) ++r;
                    while (x < r) {
                        int l = r - x; if (l > 127) l = 127;
                        const uint8_t lb = (uint8_t)(l + 128); emit(&lb, 1); emit(&comp[x], 1);
                        x += l;
                    }
                }
            }
        }
    }
}

// Skydome.hlsl:35-56 over a full-screen pixel grid. The engine rasterises a unit cube centred on the camera with
// matViewProj = skyCam.View * skyCam.Proj (Scene.cpp:573-584, camera at the origin); the interpolated
// CubemapLookDirection is proportional to the cube-surface point under the pixel, i.e. to the view ray, so per pixel:
//   ndc = pixel centre; ray = mul(float4(ndc, 1, 1), inverse(matViewProj)); dir = normalize(ray.xyz / ray.w)
// (row-vector convention, XMMATRIX). `invViewProj` is that inverse, computed by the caller in double and rounded.
float3 SkydomeLookDirection(const VqMatrix& invViewProj, int px, int py, int width, int height) {
    const float nx = ((float)px + 0.5f) / (float)width * 2.0f - 1.0f;
    const float ny = 1.0f - ((float)py + 0.5f) / (float)height * 2.0f;
    const float* m = invViewProj.m;                       // row-major: v' = v * M
    const float x = nx * m[0] + ny * m[4] + m[8]  + m[12];
    const float y = nx * m[1] + ny * m[5] + m[9]  + m[13];
    const float z = nx * m[2] + ny * m[6] + m[10] + m[14];
    const float w = nx * m[3] + ny * m[7] + m[11] + m[15];
    const float3 ray = {x / w, y / w, z / w};
    return normalize(ray);                                // VSMain: CubemapLookDirection = normalize(position.xyz) (:47)
}
float4 Skydome_PSMain(const Pyramid& texEquirectEnvironmentMap, const VqMatrix& invViewProj, int px, int py, int width, int height) {
    const float3 dir = normalize(SkydomeLookDirection(invViewProj, px, py, width, height));   // PSMain normalizes again (:53)
    const float2 uv = DirectionToEquirectUV(dir);
    const float4 c = SampleEquirectLevel(texEquirectEnvironmentMap, uv, 0.0f);
    return {c.x, c.y, c.z, 1.0f};
}

// ApplyReflections.hlsl:31-57; bv == nullptr is the variant without COMPOSITE_BOUNDING_VOLUMES
float4 ApplyReflections_CSMain(float4 SceneRadianceAndRoughness, float4 ReflectionRadiance, const float4* bv) {
    float3 FinalComposite = {SceneRadianceAndRoughness.x + ReflectionRadiance.x, SceneRadianceAndRoughness.y + ReflectionRadiance.y,
                             SceneRadianceAndRoughness.z + ReflectionRadiance.z};
    float FinalAlpha = SceneRadianceAndRoughness.w;
    if (bv) {
        const float a = bv->w, oma = 1.0f - bv->w;
        FinalComposite = {bv->x * a + FinalComposite.x * oma, bv->y * a + FinalComposite.y * oma, bv->z * a + FinalComposite.z * oma};
        FinalAlpha = a;
    }
    return {FinalComposite.x, FinalComposite.y, FinalComposite.z, FinalAlpha};
}

}  // namespace orc
