// AnyEdit's post-filter scores (AnyEdit_Collection/filter_tool/utils.py get_clip_score, get_directional_clip, get_L1_distance;
// DESIGN.md §10.10).
//   anysd_clip_preprocess_plan  host only: per image, the resized size (short side 224, long side int(224 * long / short)), the
//                               224 x 224 crop offsets (transformers' floor or torchvision's round-half-even) and Pillow's
//                               bicubic coefficients for the crop's columns and rows (pil_resample.cuh)
//   clip_preprocess_kernel      one CTA per image x band of output rows: the horizontal pass of the band's source rows as
//                               clipped uint8 in shared memory, the vertical pass, a per-channel fp16 table -> the patch rows
//                               of the vision tower's patch contraction (and optionally the crop's bytes)
//   l1_wrapped_kernel           sum of (a - b) mod 256 over the bytes of each pair, exact in 64 bits
//   postfilter_scores_kernel    one CTA per pair: exp(logit_scale) cos / 100, and the cosine of the feature differences
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "pil_resample.cuh"

namespace anysd {

namespace {

constexpr int CROP = 224, PREC = PIL_PREC, PRE_THREADS = 256, SMEM_MAX = 200 * 1024;

__device__ __forceinline__ int clip8(int s) {
    s >>= PREC;
    return s < 0 ? 0 : (s > 255 ? 255 : s);
}

__global__ void __launch_bounds__(PRE_THREADS) clip_preprocess_kernel(const uint8_t* const* __restrict__ images,
                                                                       const int* __restrict__ table, int R, int patch,
                                                                       const __half* __restrict__ lut, __half* __restrict__ rows,
                                                                       int kp, uint8_t* __restrict__ crop) {
    extern __shared__ uint8_t band[];  // horizontal pass of the band's source rows, [rows][224][3] clipped uint8
    __shared__ __half slut[3 * 256];
    const int b = blockIdx.y, oy0 = blockIdx.x * R, nr = min(R, CROP - oy0), tid = threadIdx.x;
    const int* g = table + b * CLIP_PRE_G;
    const int W = g[1], sx = g[3], sy = g[5];
    const int* tx = table + g[2];
    const int* ty = table + g[4];
    const uint8_t* src = images[b];
    const int y0 = ty[oy0 * sy], y1 = ty[(oy0 + nr - 1) * sy] + ty[(oy0 + nr - 1) * sy + 1];
    for (int i = tid; i < 3 * 256; i += PRE_THREADS) slut[i] = lut[i];
    for (int i = tid; i < (y1 - y0) * CROP; i += PRE_THREADS) {
        const int r = i / CROP, ox = i - r * CROP;
        const int* e = tx + ox * sx;
        const uint8_t* s = src + ((size_t)(y0 + r) * W + e[0]) * 3;
        int a0 = 1 << (PREC - 1), a1 = a0, a2 = a0;
        for (int k = 0; k < e[1]; ++k) {
            const int c = e[2 + k];
            a0 += s[3 * k] * c;
            a1 += s[3 * k + 1] * c;
            a2 += s[3 * k + 2] * c;
        }
        uint8_t* d = band + i * 3;
        d[0] = (uint8_t)clip8(a0), d[1] = (uint8_t)clip8(a1), d[2] = (uint8_t)clip8(a2);
    }
    __syncthreads();
    const int gp = CROP / patch, pp = patch * patch;
    for (int i = tid; i < nr * CROP; i += PRE_THREADS) {
        const int r = i / CROP, ox = i - r * CROP, oy = oy0 + r;
        const int* e = ty + oy * sy;
        const uint8_t* s = band + ((e[0] - y0) * CROP + ox) * 3;
        int a0 = 1 << (PREC - 1), a1 = a0, a2 = a0;
        for (int k = 0; k < e[1]; ++k) {
            const int c = e[2 + k];
            a0 += s[k * CROP * 3] * c;
            a1 += s[k * CROP * 3 + 1] * c;
            a2 += s[k * CROP * 3 + 2] * c;
        }
        const int v[3] = {clip8(a0), clip8(a1), clip8(a2)};
        if (crop) {
            uint8_t* d = crop + (((size_t)b * CROP + oy) * CROP + ox) * 3;
            d[0] = (uint8_t)v[0], d[1] = (uint8_t)v[1], d[2] = (uint8_t)v[2];
        }
        const int py = oy / patch, px = ox / patch;
        __half* row = rows + ((size_t)b * gp * gp + py * gp + px) * kp + (oy - py * patch) * patch + (ox - px * patch);
#pragma unroll
        for (int c = 0; c < 3; ++c) row[c * pp] = slut[c * 256 + v[c]];
    }
    // zero the padding columns [3 p^2, kp) of the patch rows that start in this band
    const int pad = kp - 3 * pp;
    if (pad > 0)
        for (int i = tid; i < nr * gp * pad; i += PRE_THREADS) {
            const int r = i / (gp * pad), rest = i - r * gp * pad, oy = oy0 + r;
            if (oy % patch) continue;
            rows[((size_t)b * gp * gp + (oy / patch) * gp + rest / pad) * kp + 3 * pp + rest % pad] = __float2half(0.0f);
        }
}

constexpr int L1_THREADS = 256, L1_CHUNK = L1_THREADS * 16 * 8;  // bytes per CTA

__global__ void __launch_bounds__(L1_THREADS) l1_wrapped_kernel(const uint8_t* const* __restrict__ a, const uint8_t* const* __restrict__ b,
                                                               const long long* __restrict__ nbytes, unsigned long long* __restrict__ out) {
    const int p = blockIdx.y;
    const long long n = nbytes[p], start = (long long)blockIdx.x * L1_CHUNK;
    if (start >= n) return;
    const long long end = min(n, start + (long long)L1_CHUNK);
    const uint8_t *pa = a[p], *pb = b[p];
    unsigned long long s = 0;
    if ((((uintptr_t)pa | (uintptr_t)pb) & 15) == 0) {
        const long long nv = (end - start) / 16;
        const uint4* va = reinterpret_cast<const uint4*>(pa + start);
        const uint4* vb = reinterpret_cast<const uint4*>(pb + start);
        unsigned int t = 0;  // at most 8 vectors x 16 bytes x 255 per thread
        for (long long i = threadIdx.x; i < nv; i += L1_THREADS) {
            const uint4 x = va[i], y = vb[i];
            t += __vsadu4(__vsub4(x.x, y.x), 0u) + __vsadu4(__vsub4(x.y, y.y), 0u) + __vsadu4(__vsub4(x.z, y.z), 0u) +
                 __vsadu4(__vsub4(x.w, y.w), 0u);
        }
        s = t;
        for (long long i = start + nv * 16 + threadIdx.x; i < end; i += L1_THREADS) s += (uint8_t)(pa[i] - pb[i]);
    } else {
        for (long long i = start + threadIdx.x; i < end; i += L1_THREADS) s += (uint8_t)(pa[i] - pb[i]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __shared__ unsigned long long red[L1_THREADS / 32];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < L1_THREADS / 32; ++w) s += red[w];
        atomicAdd(out + p, s);
    }
}

constexpr int SC_THREADS = 256;

__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int w = 0; w < SC_THREADS / 32; ++w) t += red[w];
    return t;
}

__global__ void __launch_bounds__(SC_THREADS) postfilter_scores_kernel(const float* __restrict__ img_h, const float* __restrict__ txt_h,
                                                                        int E1, float logit_scale, const float* __restrict__ img_a,
                                                                        const float* __restrict__ img_b, const float* __restrict__ txt_a,
                                                                        const float* __restrict__ txt_b, int E2, float* __restrict__ out) {
    __shared__ float red[SC_THREADS / 32];
    const int p = blockIdx.x;
    if (img_h) {
        float d = 0.f, ni = 0.f, nt = 0.f;
        for (int i = threadIdx.x; i < E1; i += SC_THREADS) {
            const float x = img_h[(size_t)p * E1 + i], y = txt_h[(size_t)p * E1 + i];
            d += x * y, ni += x * x, nt += y * y;
        }
        d = block_sum(d, red), ni = block_sum(ni, red), nt = block_sum(nt, red);
        if (threadIdx.x == 0) out[p * 2] = expf(logit_scale) * (d / (sqrtf(ni) * sqrtf(nt))) / 100.0f;
    }
    if (img_a) {
        float d = 0.f, ni = 0.f, nt = 0.f;
        for (int i = threadIdx.x; i < E2; i += SC_THREADS) {
            const size_t o = (size_t)p * E2 + i;
            const float x = img_b[o] - img_a[o], y = txt_b[o] - txt_a[o];
            d += x * y, ni += x * x, nt += y * y;
        }
        d = block_sum(d, red), ni = block_sum(ni, red), nt = block_sum(nt, red);
        // an unchanged pair (or caption) has a zero difference: directional 0, which no threshold accepts
        if (threadIdx.x == 0) out[p * 2 + 1] = (ni == 0.f || nt == 0.f) ? 0.0f : d / (sqrtf(ni) * sqrtf(nt));
    }
}

}  // namespace

}  // namespace anysd

using namespace anysd;

extern "C" {

int anysd_clip_preprocess_plan(const int* hw, int B, int channels, int crop_mode, int patch, int* table, long long* table_ints,
                               int* rows_per_cta, int* smem_bytes) {
    ANYSD_REQUIRE(hw && table_ints && rows_per_cta && smem_bytes, ANYSD_EINVAL, "clip_preprocess_plan: null pointer");
    ANYSD_REQUIRE(B >= 1 && B <= 65535, ANYSD_EINVAL, "clip_preprocess_plan: bad batch %d", B);
    ANYSD_REQUIRE(channels == 3, ANYSD_EINVAL, "clip_preprocess_plan: %d channels; the CLIP preprocessors take RGB (3)", channels);
    ANYSD_REQUIRE(crop_mode == CLIP_CROP_FLOOR || crop_mode == CLIP_CROP_ROUND, ANYSD_EINVAL,
                  "clip_preprocess_plan: unknown crop mode %d", crop_mode);
    ANYSD_REQUIRE(patch == 14 || patch == 32, ANYSD_EUNSUPPORTED, "clip_preprocess_plan: patch size %d (14 or 32)", patch);
    std::vector<int> t((size_t)B * CLIP_PRE_G, 0);
    int span_rows[5] = {0, 0, 0, 0, 0};  // the largest band of source rows for 16, 8, 4, 2, 1 output rows per CTA
    for (int b = 0; b < B; ++b) {
        const int H = hw[2 * b], W = hw[2 * b + 1];
        ANYSD_REQUIRE(H >= 1 && W >= 1 && (long long)H * W * 3 < (1LL << 31), ANYSD_EINVAL,
                      "clip_preprocess_plan: image %d is %d x %d", b, H, W);
        // get_resize_output_image_size / torchvision Resize: short side 224, long side int(224 * long / short) in float
        int rh, rw;
        if (W <= H) {
            rw = CROP;
            rh = (int)((double)CROP * H / W);
        } else {
            rh = CROP;
            rw = (int)((double)CROP * W / H);
        }
        ANYSD_REQUIRE(rh >= CROP && rw >= CROP, ANYSD_EINVAL, "clip_preprocess_plan: image %d resizes to %d x %d", b, rh, rw);
        int top, left;
        if (crop_mode == CLIP_CROP_FLOOR) {  // transformers image_transforms.center_crop
            top = (rh - CROP) / 2, left = (rw - CROP) / 2;
        } else {  // torchvision center_crop: int(round((h - 224) / 2)), half to even
            top = (int)nearbyint((rh - CROP) / 2.0), left = (int)nearbyint((rw - CROP) / 2.0);
        }
        int* g = &t[(size_t)b * CLIP_PRE_G];
        g[0] = H, g[1] = W;
        g[2] = (int)t.size();
        const int kx = pil_axis_coeffs(PIL_BICUBIC, W, rw, left, CROP, nullptr);
        pil_axis_coeffs(PIL_BICUBIC, W, rw, left, CROP, &t);
        g = &t[(size_t)b * CLIP_PRE_G];
        g[3] = 2 + kx;
        g[4] = (int)t.size();
        const int ky = pil_axis_coeffs(PIL_BICUBIC, H, rh, top, CROP, nullptr);
        pil_axis_coeffs(PIL_BICUBIC, H, rh, top, CROP, &t);
        g = &t[(size_t)b * CLIP_PRE_G];
        g[5] = 2 + ky;
        ANYSD_REQUIRE(t.size() < (1u << 31), ANYSD_EINVAL, "clip_preprocess_plan: table too large");
        const int* ty = &t[g[4]];
        for (int j = 0; j < 5; ++j) {
            const int R = 16 >> j;
            for (int oy0 = 0; oy0 < CROP; oy0 += R) {
                const int last = (std::min(oy0 + R, CROP) - 1) * g[5];
                span_rows[j] = std::max(span_rows[j], ty[last] + ty[last + 1] - ty[oy0 * g[5]]);
            }
        }
    }
    int j = 0;
    while (j < 4 && span_rows[j] * CROP * 3 > SMEM_MAX) ++j;
    ANYSD_REQUIRE(span_rows[j] * CROP * 3 <= SMEM_MAX, ANYSD_EUNSUPPORTED,
                  "clip_preprocess_plan: one output row needs %d source rows (downscale too large)", span_rows[j]);
    *rows_per_cta = 16 >> j;
    *smem_bytes = span_rows[j] * CROP * 3;
    if (table) {
        ANYSD_REQUIRE(*table_ints >= (long long)t.size(), ANYSD_EINVAL, "clip_preprocess_plan: table has %lld ints, needs %zu",
                      *table_ints, t.size());
        memcpy(table, t.data(), t.size() * sizeof(int));
    }
    *table_ints = (long long)t.size();
    return ANYSD_OK;
}

int anysd_clip_preprocess_u8(const void* images, const void* table, int B, int patch, int rows_per_cta, int smem_bytes, const void* lut,
                             void* rows, void* crop_u8, anysd_stream_t stream) {
    ANYSD_REQUIRE(images && table && lut && rows, ANYSD_EINVAL, "clip_preprocess: null pointer");
    ANYSD_REQUIRE(B >= 1 && B <= 65535, ANYSD_EINVAL, "clip_preprocess: bad batch %d", B);
    ANYSD_REQUIRE(patch == 14 || patch == 32, ANYSD_EUNSUPPORTED, "clip_preprocess: patch size %d (14 or 32)", patch);
    ANYSD_REQUIRE(rows_per_cta >= 1 && rows_per_cta <= 16 && smem_bytes >= 0 && smem_bytes <= SMEM_MAX, ANYSD_EINVAL,
                  "clip_preprocess: bad plan (%d rows per CTA, %d bytes)", rows_per_cta, smem_bytes);
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(clip_preprocess_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX);
        attr = true;
    }
    const int kp = (3 * patch * patch + 7) / 8 * 8;
    clip_preprocess_kernel<<<dim3(cdiv(CROP, rows_per_cta), B), PRE_THREADS, smem_bytes, (cudaStream_t)stream>>>(
        (const uint8_t* const*)images, (const int*)table, rows_per_cta, patch, (const __half*)lut, (__half*)rows, kp, (uint8_t*)crop_u8);
    return check_launch("clip_preprocess");
}

int anysd_l1_wrapped_u8(const void* a, const void* b, const void* nbytes, int B, long long max_bytes, void* out, anysd_stream_t stream) {
    ANYSD_REQUIRE(a && b && nbytes && out, ANYSD_EINVAL, "l1_wrapped: null pointer");
    ANYSD_REQUIRE(B >= 1 && B <= 65535 && max_bytes >= 1, ANYSD_EINVAL, "l1_wrapped: bad dims B=%d max_bytes=%lld", B, max_bytes);
    ANYSD_REQUIRE(max_bytes / L1_CHUNK < (1LL << 31) - 1, ANYSD_EINVAL, "l1_wrapped: image too large");
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemsetAsync(out, 0, sizeof(unsigned long long) * B, st) != cudaSuccess) return check_launch("l1_wrapped memset");
    l1_wrapped_kernel<<<dim3(cdiv(max_bytes, L1_CHUNK), B), L1_THREADS, 0, st>>>(
        (const uint8_t* const*)a, (const uint8_t* const*)b, (const long long*)nbytes, (unsigned long long*)out);
    return check_launch("l1_wrapped");
}

int anysd_postfilter_scores_f32(const float* img_h, const float* txt_h, int E1, float logit_scale, const float* img_a, const float* img_b,
                                const float* txt_a, const float* txt_b, int E2, int B, float* out, anysd_stream_t stream) {
    ANYSD_REQUIRE(out && (img_h || img_a), ANYSD_EINVAL, "postfilter_scores: null pointer");
    ANYSD_REQUIRE(!img_h || (txt_h && E1 >= 1), ANYSD_EINVAL, "postfilter_scores: CLIP-H features need txt_h and E1 >= 1");
    ANYSD_REQUIRE(!img_a || (img_b && txt_a && txt_b && E2 >= 1), ANYSD_EINVAL,
                  "postfilter_scores: directional features need img_a, img_b, txt_a, txt_b and E2 >= 1");
    ANYSD_REQUIRE(B >= 1 && B <= (1 << 30), ANYSD_EINVAL, "postfilter_scores: bad batch %d", B);
    postfilter_scores_kernel<<<B, SC_THREADS, 0, (cudaStream_t)stream>>>(img_h, txt_h, E1, logit_scale, img_a, img_b, txt_a, txt_b, E2,
                                                                         out);
    return check_launch("postfilter_scores");
}

}  // extern "C"
