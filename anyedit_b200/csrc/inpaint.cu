// AnyEdit's inpainting edits (local_pipeline_tool.py background_change / replace through StableDiffusionInpaintPipeline;
// DESIGN.md §10.11).  All of it is integer arithmetic except the masked image, which is the processor's float32 formula.
//   anysd_pil_resize_plan   host only: per image Pillow's coefficients of both axes (pil_resample.cuh) for LANCZOS, BICUBIC,
//                           NEAREST, or a mode "1" image (0/1 bytes, NEAREST, then convert("L"): 0/255)
//   pil_resize_kernel       one CTA per image x band of output rows: the horizontal pass of the band's source rows as clipped
//                           uint8 in shared memory, then the vertical pass -> the output bytes; images of any sizes in one launch
//   inpaint_prepare_kernel  one thread per pixel of the 8x-latent-sized RGB and mask bytes: the masked image x / 255 * 2 - 1
//                           (0 where mask >= 128) as the encoder's fp16 NHWC input, the nearest-sampled fp32 mask latent and the
//                           per-request count of mask pixels
//   background_mask_kernel  per 32 x 32 tile of a BGR mask: OpenCV's 8-bit GaussianBlur((5, 5), 0) (BORDER_REFLECT_101), BGR2GRAY,
//                           == 0 -> uint8 0/1, and the per-request count of ones; images of any sizes in one launch
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "pil_resample.cuh"

namespace anysd {

namespace {

constexpr int RS_THREADS = 256, RS_SMEM_MAX = 200 * 1024, RS_MAX_SIDE = 32767;

__device__ __forceinline__ int clip8_22(int s) {
    s >>= PIL_PREC;
    return s < 0 ? 0 : (s > 255 ? 255 : s);
}

// table row of image b: (H, W, OH, OW, x entries offset, x stride, y entries offset, y stride)
template <int C>
__global__ void __launch_bounds__(RS_THREADS) pil_resize_kernel(const uint8_t* const* __restrict__ src, uint8_t* const* __restrict__ dst,
                                                                const int* __restrict__ table, int R) {
    extern __shared__ uint8_t band[];  // [source rows][OW][C]
    const int b = blockIdx.y, tid = threadIdx.x;
    const int* g = table + b * PIL_RESIZE_G;
    const int W = g[1], OH = g[2], OW = g[3], sx = g[5], sy = g[7];
    const int oy0 = blockIdx.x * R;
    if (oy0 >= OH) return;
    const int nr = min(R, OH - oy0);
    const int* tx = table + g[4];
    const int* ty = table + g[6];
    const uint8_t* s0 = src[b];
    uint8_t* d0 = dst[b];
    const int y0 = ty[oy0 * sy], y1 = ty[(oy0 + nr - 1) * sy] + ty[(oy0 + nr - 1) * sy + 1];
    for (int i = tid; i < (y1 - y0) * OW; i += RS_THREADS) {
        const int r = i / OW, ox = i - r * OW;
        const int* e = tx + ox * sx;
        const uint8_t* s = s0 + ((size_t)(y0 + r) * W + e[0]) * C;
        int a[C];
#pragma unroll
        for (int c = 0; c < C; ++c) a[c] = 1 << (PIL_PREC - 1);
        for (int k = 0; k < e[1]; ++k) {
            const int w = e[2 + k];
#pragma unroll
            for (int c = 0; c < C; ++c) a[c] += s[C * k + c] * w;
        }
#pragma unroll
        for (int c = 0; c < C; ++c) band[i * C + c] = (uint8_t)clip8_22(a[c]);
    }
    __syncthreads();
    for (int i = tid; i < nr * OW; i += RS_THREADS) {
        const int r = i / OW, ox = i - r * OW, oy = oy0 + r;
        const int* e = ty + oy * sy;
        const uint8_t* s = band + ((size_t)(e[0] - y0) * OW + ox) * C;
        int a[C];
#pragma unroll
        for (int c = 0; c < C; ++c) a[c] = 1 << (PIL_PREC - 1);
        for (int k = 0; k < e[1]; ++k) {
            const int w = e[2 + k];
#pragma unroll
            for (int c = 0; c < C; ++c) a[c] += s[(size_t)k * OW * C + c] * w;
        }
        uint8_t* d = d0 + ((size_t)oy * OW + ox) * C;
#pragma unroll
        for (int c = 0; c < C; ++c) d[c] = (uint8_t)clip8_22(a[c]);
    }
}

constexpr int PREP_THREADS = 256;

// ldc fp16 channels per pixel (a multiple of 8): the 3 image channels, then zeros (the encoder's padded input rows)
__global__ void __launch_bounds__(PREP_THREADS) inpaint_prepare_kernel(const uint8_t* __restrict__ img, const uint8_t* __restrict__ mask,
                                                                       int H, int W, int ldc, __half* __restrict__ masked,
                                                                       float* __restrict__ mask_latent, int* __restrict__ counts) {
    const int b = blockIdx.y;
    const int p = blockIdx.x * PREP_THREADS + threadIdx.x;
    const int HW = H * W;
    bool on = false;
    if (p < HW) {
        const size_t q = (size_t)b * HW + p;
        on = mask[q] >= 128;  // VaeImageProcessor binarize: byte / 255 >= 0.5
        const float keep = on ? 0.0f : 1.0f;
        const uint8_t* s = img + q * 3;
        __half v[8];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float x = __fdiv_rn((float)s[c], 255.0f);           // pil_to_numpy: float32 / 255
            v[c] = __float2half_rn(__fsub_rn(__fmul_rn(2.0f, x), 1.0f) * keep);   // normalize, then image * (mask < 0.5)
        }
#pragma unroll
        for (int c = 3; c < 8; ++c) v[c] = __float2half_rn(0.0f);
        uint4* d = reinterpret_cast<uint4*>(masked + q * ldc);
        d[0] = *reinterpret_cast<const uint4*>(v);
        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
        for (int j = 1; j < ldc / 8; ++j) d[j] = z;
        const int y = p / W, x = p - y * W;
        if ((y & 7) == 0 && (x & 7) == 0)  // F.interpolate(mask, (H / 8, W / 8)), nearest: mask[8i, 8j]
            mask_latent[((size_t)b * (H / 8) + (y >> 3)) * (W / 8) + (x >> 3)] = on ? 1.0f : 0.0f;
    }
    const int n = __popc(__ballot_sync(0xffffffffu, on));
    __shared__ int red[PREP_THREADS / 32];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < PREP_THREADS / 32; ++w) t += red[w];
        if (t) atomicAdd(counts + b, t);
    }
}

constexpr int BT = 32, BHALO = 2, BIN = BT + 2 * BHALO, BM_THREADS = 256;

// OpenCV's borderInterpolate for BORDER_REFLECT_101 (any offset, any length >= 1)
__device__ __forceinline__ int reflect101_any(int p, int len) {
    if (len == 1) return 0;
    while ((unsigned)p >= (unsigned)len) p = p < 0 ? -p : 2 * len - 2 - p;
    return p;
}

// hw: per image (H, W).  GaussianBlur((5, 5), 0) of 8-bit images: sigma 0 selects OpenCV's fixed kernel [1 4 6 4 1] / 16 on both
// axes, in 8.8 fixed point rows and 16.16 columns with one rounding: (sum_ij w_i w_j p_ij + 128) >> 8, exact in integers.
__global__ void __launch_bounds__(BM_THREADS) background_mask_kernel(const uint8_t* const* __restrict__ src, uint8_t* const* __restrict__ dst,
                                                                     const int* __restrict__ hw, int* __restrict__ counts) {
    __shared__ uint8_t in[BIN][BIN][3];
    __shared__ int rowsum[BIN][BT][3];
    const int b = blockIdx.z, H = hw[2 * b], W = hw[2 * b + 1];
    const int x0 = blockIdx.x * BT, y0 = blockIdx.y * BT, tid = threadIdx.x;
    if (x0 >= W || y0 >= H) return;
    const uint8_t* im = src[b];
    for (int i = tid; i < BIN * BIN; i += BM_THREADS) {
        const int ly = i / BIN, lx = i - ly * BIN;
        const int y = reflect101_any(y0 - BHALO + ly, H), x = reflect101_any(x0 - BHALO + lx, W);
        const uint8_t* p = im + ((size_t)y * W + x) * 3;
        in[ly][lx][0] = p[0], in[ly][lx][1] = p[1], in[ly][lx][2] = p[2];
    }
    __syncthreads();
    for (int i = tid; i < BIN * BT; i += BM_THREADS) {
        const int ly = i / BT, lx = i - ly * BT;
#pragma unroll
        for (int c = 0; c < 3; ++c)
            rowsum[ly][lx][c] = in[ly][lx][c] + 4 * in[ly][lx + 1][c] + 6 * in[ly][lx + 2][c] + 4 * in[ly][lx + 3][c] + in[ly][lx + 4][c];
    }
    __syncthreads();
    int n = 0;
    for (int i = tid; i < BT * BT; i += BM_THREADS) {
        const int ly = i / BT, lx = i - ly * BT, y = y0 + ly, x = x0 + lx;
        if (y >= H || x >= W) continue;
        int v[3];
#pragma unroll
        for (int c = 0; c < 3; ++c)
            v[c] = (rowsum[ly][lx][c] + 4 * rowsum[ly + 1][lx][c] + 6 * rowsum[ly + 2][lx][c] + 4 * rowsum[ly + 3][lx][c] +
                    rowsum[ly + 4][lx][c] + 128) >> 8;
        const int grey = (v[0] * 3735 + v[1] * 19235 + v[2] * 9798 + (1 << 14)) >> 15;  // BGR2GRAY (as sketch.cu)
        dst[b][(size_t)y * W + x] = grey == 0;
        n += grey == 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    __shared__ int red[BM_THREADS / 32];
    if ((tid & 31) == 0) red[tid >> 5] = n;
    __syncthreads();
    if (tid == 0) {
        int t = 0;
        for (int w = 0; w < BM_THREADS / 32; ++w) t += red[w];
        if (t) atomicAdd(counts + b, t);
    }
}

}  // namespace

}  // namespace anysd

using namespace anysd;

extern "C" {

int anysd_pil_resize_plan(const int* sizes, const int* filters, int B, int channels, int* table, long long* table_ints, int* rows_per_cta,
                          int* smem_bytes, int* bands) {
    ANYSD_REQUIRE(sizes && filters && table_ints && rows_per_cta && smem_bytes && bands, ANYSD_EINVAL, "pil_resize_plan: null pointer");
    ANYSD_REQUIRE(B >= 1 && B <= 65535, ANYSD_EINVAL, "pil_resize_plan: bad batch %d", B);
    ANYSD_REQUIRE(channels == 1 || channels == 3, ANYSD_EUNSUPPORTED, "pil_resize_plan: %d channels (1: L, 3: RGB)", channels);
    std::vector<int> t((size_t)B * PIL_RESIZE_G, 0);
    int span_rows[5] = {0, 0, 0, 0, 0};  // the largest band of source rows x output width for 16, 8, 4, 2, 1 output rows per CTA
    long long span_bytes[5] = {0, 0, 0, 0, 0};
    int max_bands[5] = {0, 0, 0, 0, 0};
    for (int b = 0; b < B; ++b) {
        const int H = sizes[4 * b], W = sizes[4 * b + 1], OH = sizes[4 * b + 2], OW = sizes[4 * b + 3], f = filters[b];
        ANYSD_REQUIRE(H >= 1 && W >= 1 && OH >= 1 && OW >= 1 && H <= RS_MAX_SIDE && W <= RS_MAX_SIDE && OH <= RS_MAX_SIDE &&
                          OW <= RS_MAX_SIDE,
                      ANYSD_EINVAL, "pil_resize_plan: image %d is %d x %d -> %d x %d (sides 1 .. %d)", b, H, W, OH, OW, RS_MAX_SIDE);
        ANYSD_REQUIRE(f == PIL_RESAMPLE_NEAREST || f == PIL_RESAMPLE_LANCZOS || f == PIL_RESAMPLE_BICUBIC || f == PIL_RESAMPLE_MODE1,
                      ANYSD_EUNSUPPORTED, "pil_resize_plan: image %d has filter %d (NEAREST 0, LANCZOS 1, BICUBIC 3, mode-1 16)", b, f);
        ANYSD_REQUIRE(f != PIL_RESAMPLE_MODE1 || channels == 1, ANYSD_EINVAL, "pil_resize_plan: a mode \"1\" image has one channel");
        int* g = &t[(size_t)b * PIL_RESIZE_G];
        g[0] = H, g[1] = W, g[2] = OH, g[3] = OW;
        int kx = 1, ky = 1;
        g[4] = (int)t.size();
        if (f == PIL_RESAMPLE_NEAREST || f == PIL_RESAMPLE_MODE1) {
            pil_axis_nearest(W, OW, &t, f == PIL_RESAMPLE_MODE1 ? 255 : 1);  // convert("L") of mode "1": 1 -> 255
        } else {
            kx = pil_axis_coeffs((PilFilter)f, W, OW, 0, OW, nullptr);
            pil_axis_coeffs((PilFilter)f, W, OW, 0, OW, &t);
        }
        const int oy = (int)t.size();
        if (f == PIL_RESAMPLE_NEAREST || f == PIL_RESAMPLE_MODE1) {
            pil_axis_nearest(H, OH, &t);
        } else {
            ky = pil_axis_coeffs((PilFilter)f, H, OH, 0, OH, nullptr);
            pil_axis_coeffs((PilFilter)f, H, OH, 0, OH, &t);
        }
        ANYSD_REQUIRE(t.size() < (1u << 31), ANYSD_EINVAL, "pil_resize_plan: table too large");
        g = &t[(size_t)b * PIL_RESIZE_G];
        g[5] = 2 + kx, g[6] = oy, g[7] = 2 + ky;
        const int* ty = &t[oy];
        for (int j = 0; j < 5; ++j) {
            const int R = 16 >> j;
            max_bands[j] = std::max(max_bands[j], (OH + R - 1) / R);
            for (int oy0 = 0; oy0 < OH; oy0 += R) {
                const int last = (std::min(oy0 + R, OH) - 1) * g[7];
                const int rows = ty[last] + ty[last + 1] - ty[oy0 * g[7]];
                span_rows[j] = std::max(span_rows[j], rows);
                span_bytes[j] = std::max(span_bytes[j], (long long)rows * OW * channels);
            }
        }
    }
    int j = 0;
    while (j < 4 && span_bytes[j] > RS_SMEM_MAX) ++j;
    ANYSD_REQUIRE(span_bytes[j] <= RS_SMEM_MAX, ANYSD_EUNSUPPORTED,
                  "pil_resize_plan: one output row needs %lld bytes of source rows (over %d)", span_bytes[j], RS_SMEM_MAX);
    *rows_per_cta = 16 >> j;
    *smem_bytes = (int)span_bytes[j];
    *bands = max_bands[j];
    if (table) {
        ANYSD_REQUIRE(*table_ints >= (long long)t.size(), ANYSD_EINVAL, "pil_resize_plan: table has %lld ints, needs %zu", *table_ints,
                      t.size());
        memcpy(table, t.data(), t.size() * sizeof(int));
    }
    *table_ints = (long long)t.size();
    return ANYSD_OK;
}

int anysd_pil_resize_u8(const void* src, const void* dst, const void* table, int B, int channels, int rows_per_cta, int smem_bytes,
                        int bands, anysd_stream_t stream) {
    ANYSD_REQUIRE(src && dst && table, ANYSD_EINVAL, "pil_resize: null pointer");
    ANYSD_REQUIRE(B >= 1 && B <= 65535 && bands >= 1, ANYSD_EINVAL, "pil_resize: bad batch %d / %d bands", B, bands);
    ANYSD_REQUIRE(channels == 1 || channels == 3, ANYSD_EUNSUPPORTED, "pil_resize: %d channels (1 or 3)", channels);
    ANYSD_REQUIRE(rows_per_cta >= 1 && rows_per_cta <= 16 && smem_bytes >= 0 && smem_bytes <= RS_SMEM_MAX, ANYSD_EINVAL,
                  "pil_resize: bad plan (%d rows per CTA, %d bytes)", rows_per_cta, smem_bytes);
    static bool attr_done[64];  // per device (function attributes are per-device)
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!attr_done[dev]) {
        cudaFuncSetAttribute(pil_resize_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, RS_SMEM_MAX);
        cudaFuncSetAttribute(pil_resize_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, RS_SMEM_MAX);
        attr_done[dev] = true;
    }
    const dim3 grid(bands, B);
    cudaStream_t st = (cudaStream_t)stream;
    if (channels == 3)
        pil_resize_kernel<3><<<grid, RS_THREADS, smem_bytes, st>>>((const uint8_t* const*)src, (uint8_t* const*)dst, (const int*)table,
                                                                     rows_per_cta);
    else
        pil_resize_kernel<1><<<grid, RS_THREADS, smem_bytes, st>>>((const uint8_t* const*)src, (uint8_t* const*)dst, (const int*)table,
                                                                     rows_per_cta);
    return check_launch("pil_resize");
}

int anysd_inpaint_prepare(const void* img, const void* mask, int B, int H, int W, int ldc, void* masked_f16, float* mask_latent,
                          int* counts, anysd_stream_t stream) {
    ANYSD_REQUIRE(img && mask && masked_f16 && mask_latent && counts, ANYSD_EINVAL, "inpaint_prepare: null pointer");
    ANYSD_REQUIRE(B >= 1 && B <= 65535 && H >= 8 && W >= 8 && H % 8 == 0 && W % 8 == 0 && (long long)H * W < (1LL << 30), ANYSD_EINVAL,
                  "inpaint_prepare: bad dims B=%d %d x %d (sides multiples of 8)", B, H, W);
    ANYSD_REQUIRE(ldc >= 8 && ldc % 8 == 0 && (uintptr_t)masked_f16 % 16 == 0, ANYSD_EINVAL,
                  "inpaint_prepare: the fp16 rows need a multiple of 8 channels (got %d) and 16-byte alignment", ldc);
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemsetAsync(counts, 0, sizeof(int) * B, st) != cudaSuccess) return check_launch("inpaint_prepare memset");
    inpaint_prepare_kernel<<<dim3(cdiv((long long)H * W, PREP_THREADS), B), PREP_THREADS, 0, st>>>(
        (const uint8_t*)img, (const uint8_t*)mask, H, W, ldc, (__half*)masked_f16, mask_latent, counts);
    return check_launch("inpaint_prepare");
}

int anysd_background_mask_u8(const void* src, const void* dst, const void* hw, int B, int max_h, int max_w, int* counts,
                             anysd_stream_t stream) {
    ANYSD_REQUIRE(src && dst && hw && counts, ANYSD_EINVAL, "background_mask: null pointer");
    ANYSD_REQUIRE(B >= 1 && B <= 65535 && max_h >= 1 && max_w >= 1 && (long long)max_h * max_w < (1LL << 31), ANYSD_EINVAL,
                  "background_mask: bad dims B=%d, largest %d x %d", B, max_h, max_w);
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemsetAsync(counts, 0, sizeof(int) * B, st) != cudaSuccess) return check_launch("background_mask memset");
    background_mask_kernel<<<dim3(cdiv(max_w, BT), cdiv(max_h, BT), B), BM_THREADS, 0, st>>>(
        (const uint8_t* const*)src, (uint8_t* const*)dst, (const int*)hw, counts);
    return check_launch("background_mask");
}

}  // extern "C"
