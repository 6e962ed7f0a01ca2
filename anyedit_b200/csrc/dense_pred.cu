// Dense-prediction helpers of the Depth Anything V2 DPT head (depth_anything_v2/dpt.py, util/blocks.py); the convolutions and
// projections of the head run on anysd_gemm_f16.
//   resize_bilinear_ac   F.interpolate(mode="bilinear", align_corners=True) at any (H, W) -> (Ho, Wo), NHWC fp16 (C % 8 == 0,
//                        16-byte vectors) with an optional fp16 addend of the output's shape folded in before the one rounding,
//                        and a single-channel fp32 form (infer_image's resize to the raw image size)
//   relu                 y = max(x, 0) as a copy: ResidualConvUnit needs x (its residual) and relu(x) (its conv input)
//   depth_to_space       ConvTranspose2d(kernel = stride = r) as one contraction: [B*gh*gw, (ky, kx, co)] -> [B, r gh, r gw, co]
#include "common.cuh"

namespace anysd {

// Source coordinate of output index o along one axis, as ATen computes it for align_corners=True in fp32
// (area_pixel_compute_scale / area_pixel_compute_source_index, UpSampleBilinear2d): src = o * (in - 1) / (out - 1).
struct Tap {
    int i0, i1;
    float l0, l1;
};
__device__ __forceinline__ Tap bl_tap(int o, float scale, int in) {
    const float src = scale * (float)o;
    Tap t;
    t.i0 = (int)src;
    if (t.i0 > in - 1) t.i0 = in - 1;
    t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
    t.l1 = src - (float)t.i0;
    t.l0 = 1.0f - t.l1;
    return t;
}
static inline float bl_scale(int in, int out) { return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.0f; }

__global__ void resize_bilinear_ac_f16_kernel(const uint4* __restrict__ x, const uint4* __restrict__ add, uint4* __restrict__ y, int H,
                                              int W, int Ho, int Wo, int CV, float sh, float sw, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(i % CV);
        long long r = i / CV;
        const int ox = (int)(r % Wo);
        r /= Wo;
        const int oy = (int)(r % Ho);
        const long long n = r / Ho;
        const Tap ty = bl_tap(oy, sh, H), tx = bl_tap(ox, sw, W);
        const uint4* img = x + n * H * W * CV + cv;
        float a[8], b[8], c[8], d[8], o[8];
        unpack8(img[((long long)ty.i0 * W + tx.i0) * CV], a);
        unpack8(img[((long long)ty.i0 * W + tx.i1) * CV], b);
        unpack8(img[((long long)ty.i1 * W + tx.i0) * CV], c);
        unpack8(img[((long long)ty.i1 * W + tx.i1) * CV], d);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = ty.l0 * (tx.l0 * a[j] + tx.l1 * b[j]) + ty.l1 * (tx.l0 * c[j] + tx.l1 * d[j]);
        if (add != nullptr) {
            float e[8];
            unpack8(add[i], e);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] += e[j];
        }
        y[i] = pack8(o);
    }
}

__global__ void resize_bilinear_ac_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, int Ho, int Wo, float sh,
                                              float sw, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % Wo);
        const long long r = i / Wo;
        const int oy = (int)(r % Ho);
        const long long n = r / Ho;
        const Tap ty = bl_tap(oy, sh, H), tx = bl_tap(ox, sw, W);
        const float* img = x + n * H * W;
        y[i] = ty.l0 * (tx.l0 * img[ty.i0 * W + tx.i0] + tx.l1 * img[ty.i0 * W + tx.i1]) +
               ty.l1 * (tx.l0 * img[ty.i1 * W + tx.i0] + tx.l1 * img[ty.i1 * W + tx.i1]);
    }
}

__global__ void relu_f16_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long long nvec) {
    // per fp16 lane: sign bit set -> +0, else x unchanged (exact; -0 and negative infinities become +0)
    auto relu2 = [](uint32_t w) { return w & ~(((w >> 15) & 0x00010001u) * 0xFFFFu); };
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        const uint4 u = x[i];
        y[i] = make_uint4(relu2(u.x), relu2(u.y), relu2(u.z), relu2(u.w));
    }
}

// out[b, y r + ky, x r + kx, c] = g[(b gh + y) gw + x, (ky r + kx) C + c], 8 channels per thread
__global__ void depth_to_space_f16_kernel(const uint4* __restrict__ g, uint4* __restrict__ out, int gh, int gw, int r, int CV,
                                          long long total) {
    const int Wo = gw * r, Ho = gh * r;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(i % CV);
        long long t = i / CV;
        const int X = (int)(t % Wo);
        t /= Wo;
        const int Y = (int)(t % Ho);
        const long long b = t / Ho;
        const int y = Y / r, ky = Y - y * r, x = X / r, kx = X - x * r;
        out[i] = g[((b * gh + y) * gw + x) * ((long long)r * r * CV) + (ky * r + kx) * CV + cv];
    }
}

static int dp_grid(long long n, int block = 256, int per_sm = 8) {
    long long g = (n + block - 1) / block;
    const long long cap = (long long)sm_count() * per_sm;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace anysd

using namespace anysd;

extern "C" {

int anysd_resize_bilinear_ac_f16(const void* x, const void* addend, void* y, int N, int H, int W, int C, int Ho, int Wo,
                                 anysd_stream_t stream) {
    ANYSD_REQUIRE(x && y, ANYSD_EINVAL, "resize_bilinear: null pointer");
    ANYSD_REQUIRE(N > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 8 == 0, ANYSD_EINVAL,
                  "resize_bilinear: bad dims N=%d %dx%d -> %dx%d C=%d (C must be a multiple of 8)", N, H, W, Ho, Wo, C);
    ANYSD_REQUIRE((uintptr_t)x % 16 == 0 && (uintptr_t)y % 16 == 0 && (uintptr_t)addend % 16 == 0, ANYSD_EINVAL,
                  "resize_bilinear: x, y and addend must be 16-byte aligned");
    const long long total = (long long)N * Ho * Wo * (C / 8);
    resize_bilinear_ac_f16_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>(
        (const uint4*)x, (const uint4*)addend, (uint4*)y, H, W, Ho, Wo, C / 8, bl_scale(H, Ho), bl_scale(W, Wo), total);
    return check_launch("resize_bilinear_f16");
}

int anysd_resize_bilinear_ac_f32(const float* x, float* y, int N, int H, int W, int Ho, int Wo, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && y, ANYSD_EINVAL, "resize_bilinear_f32: null pointer");
    ANYSD_REQUIRE(N > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, ANYSD_EINVAL, "resize_bilinear_f32: bad dims N=%d %dx%d -> %dx%d", N, H,
                  W, Ho, Wo);
    const long long total = (long long)N * Ho * Wo;
    resize_bilinear_ac_f32_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>(x, y, H, W, Ho, Wo, bl_scale(H, Ho), bl_scale(W, Wo),
                                                                                     total);
    return check_launch("resize_bilinear_f32");
}

int anysd_relu_f16(const void* x, void* y, long long n, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && y && n > 0 && n % 8 == 0, ANYSD_EINVAL, "relu: bad args (n %% 8 == 0)");
    ANYSD_REQUIRE((uintptr_t)x % 16 == 0 && (uintptr_t)y % 16 == 0, ANYSD_EINVAL, "relu: x and y must be 16-byte aligned");
    relu_f16_kernel<<<dp_grid(n / 8), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, (uint4*)y, n / 8);
    return check_launch("relu");
}

int anysd_depth_to_space_f16(const void* g, void* out, int B, int gh, int gw, int r, int C, anysd_stream_t stream) {
    ANYSD_REQUIRE(g && out, ANYSD_EINVAL, "depth_to_space: null pointer");
    ANYSD_REQUIRE(B > 0 && gh > 0 && gw > 0 && r > 0 && C > 0 && C % 8 == 0, ANYSD_EINVAL,
                  "depth_to_space: bad dims B=%d %dx%d r=%d C=%d (C must be a multiple of 8)", B, gh, gw, r, C);
    ANYSD_REQUIRE((uintptr_t)g % 16 == 0 && (uintptr_t)out % 16 == 0, ANYSD_EINVAL, "depth_to_space: pointers must be 16-byte aligned");
    const long long total = (long long)B * gh * r * gw * r * (C / 8);
    depth_to_space_f16_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)g, (uint4*)out, gh, gw, r, C / 8, total);
    return check_launch("depth_to_space");
}

}  // extern "C"
