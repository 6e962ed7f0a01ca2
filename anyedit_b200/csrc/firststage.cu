// First-stage (autoencoder) helpers, SURVEY.md 8f rank 1 -- everything else of the VAE runs on the UNet's kernels.
//   softmax_rows   the single-head d = C attention of AttnBlock (ldm/modules/diffusionmodules/model.py:176-203) at C = 512 is
//                  wider than the wgmma attention kernel takes (O in registers for d <= 160): it runs as two contractions around a
//                  row softmax -- S = q k^T (fp32) -> P = softmax(S * C^-0.5) (fp16) -> O = P v.
//   gaussian       DiagonalGaussianDistribution (ldm/modules/distributions/distributions.py:24-62): clamp, std, sample.
#include "common.cuh"

namespace anysd {

// one CTA per row; three sweeps over the row (max, sum, write) -- the row (<= 64 KB) stays in L1/L2 between them
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ S, long long ld_s, __half* __restrict__ P, long long ld_p,
                                                           int n, float scale_log2) {
    const float* s = S + (size_t)blockIdx.x * ld_s;
    __half* p = P + (size_t)blockIdx.x * ld_p;
    __shared__ float red[8];
    __shared__ float bcast;
    float m = -INFINITY;
    for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, s[i]);
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = red[0];
        for (int w = 1; w < 8; ++w) t = fmaxf(t, red[w]);
        bcast = t;
    }
    __syncthreads();
    m = bcast * scale_log2;
    float sum = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) sum += exp2f(fmaf(s[i], scale_log2, -m));
    sum = warp_sum(sum);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += red[w];
        bcast = 1.0f / t;
    }
    __syncthreads();
    const float inv = bcast;
    for (int i = threadIdx.x; i < n; i += blockDim.x) p[i] = __float2half_rn(exp2f(fmaf(s[i], scale_log2, -m)) * inv);
}

// moments fp32 NCHW [B, 2Z, HW] -> mean | clamp(logvar, -30, 20); sample = mean + exp(0.5 logvar) * noise (noise NULL: mode)
__global__ void gaussian_posterior_kernel(const float* __restrict__ mom, const float* __restrict__ noise, float* __restrict__ sample,
                                          float* __restrict__ logvar_out, float scale, long long zhw, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / zhw, r = i - b * zhw;
        const float mean = mom[b * 2 * zhw + r];
        float lv = mom[b * 2 * zhw + zhw + r];
        lv = fminf(fmaxf(lv, -30.0f), 20.0f);
        if (logvar_out) logvar_out[i] = lv;
        if (sample) {
            const float v = noise ? __fadd_rn(mean, __fmul_rn(expf(0.5f * lv), noise[i])) : mean;
            sample[i] = scale == 1.0f ? v : __fmul_rn(scale, v);
        }
    }
}

}  // namespace anysd

using namespace anysd;

static int fs_grid(long long n) {
    long long g = (n + 255) / 256;
    const long long cap = (long long)sm_count() * 8;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

extern "C" {

int anysd_softmax_rows_f32(const float* S, long long ld_s, void* P, long long ld_p, int rows, int n, float scale, anysd_stream_t stream) {
    ANYSD_REQUIRE(S && P && rows > 0 && n > 0 && ld_s >= n && ld_p >= n, ANYSD_EINVAL, "softmax_rows: bad args");
    softmax_rows_kernel<<<rows, 256, 0, (cudaStream_t)stream>>>(S, ld_s, (__half*)P, ld_p, n, scale * 1.4426950408889634f);
    return check_launch("softmax_rows");
}

int anysd_gaussian_posterior_f32(const float* moments, const float* noise, float* sample, float* logvar, float scale, int B,
                                 long long z_hw, anysd_stream_t stream) {
    ANYSD_REQUIRE(moments && (sample || logvar) && B > 0 && z_hw > 0, ANYSD_EINVAL, "gaussian_posterior: bad args");
    const long long total = (long long)B * z_hw;
    gaussian_posterior_kernel<<<fs_grid(total), 256, 0, (cudaStream_t)stream>>>(moments, noise, sample, logvar, scale, z_hw, total);
    return check_launch("gaussian_posterior");
}
}
