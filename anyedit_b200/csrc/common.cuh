// Shared device/host helpers for the anysd_b200 kernels (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/anysd_b200.h"

namespace anysd {

// ---- error plumbing (thread-local message, negative return codes) -----------------------
void set_error(const char* fmt, ...);
int check_launch(const char* what);

#define ANYSD_REQUIRE(cond, code, ...)                 \
    do {                                               \
        if (!(cond)) {                                 \
            ::anysd::set_error(__VA_ARGS__);           \
            return (code);                             \
        }                                              \
    } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

int sm_count();

// ---- small device helpers ---------------------------------------------------------------
__device__ __forceinline__ float silu_f(float v) { return v / (1.0f + __expf(-v)); }
__device__ __forceinline__ float gelu_erf_f(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f)); }
// QuickGELU of the OpenAI CLIP towers (transformers activations.py: x * sigmoid(1.702 x))
__device__ __forceinline__ float quick_gelu_f(float v) { return v / (1.0f + __expf(-1.702f * v)); }
// epilogue activations of anysd_gemm_params::act other than GEGLU: 1 SiLU, 3 GELU (erf), 4 QuickGELU, 6 ReLU
__device__ __forceinline__ float act_f(float v, int act) {
    return act == 1 ? silu_f(v) : (act == 3 ? gelu_erf_f(v) : (act == 4 ? quick_gelu_f(v) : (act == 6 ? fmaxf(v, 0.0f) : v)));
}

// Exact (erf) GELU  x Phi(x)  in 11 instructions: Phi(x) = 1 / (1 + 2^(-x P(x^2))) with a cubic P fitted (minimax on the ABSOLUTE
// error of x Phi(x), x^2 clamped at 36 -- beyond it the logistic is saturated either way) to |err| < 1.2e-5 for all x: 1/40 of the
// fp16 spacing at unit magnitude, 1/7 of it at the minimum of GELU (-0.17).  Used by the fp16-output epilogues of gemm_wgmma.cu
// (the GEGLU contractions are issue-bound there) and by the fused feed-forward (feedforward_wgmma.cu);
// tests/test_gpu_ops.py::test_gelu_epilogue_accuracy pins the bound against torch's erf GELU.
__device__ __forceinline__ float p_gelu(float v) {
    const float t = fminf(v * v, 36.0f);
    float q = fmaf(t, 2.483638929e-05f, 7.36060983e-04f);
    q = fmaf(q, t, -0.10598272654f);
    q = fmaf(q, t, -2.30164716054f);
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * q));          // 2^(-x P(x^2))
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return v * r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

struct __align__(16) half8 {
    __half2 a, b, c, d;
};

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 t = __half22float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    return u;
}

// One LayerNorm row held by LPR lanes, lane l holding the row's 8-element vectors l, l + LPR, .. (f[i] = vector
// l + i LPR, valid while < CV; s its sum, added in order while loading): the xor-shuffle tree LPR / 2 .. 1, two-pass exact variance
// (layernorm_row_stats), then f becomes the normalised output (layernorm_row_apply).  layernorm_kernel (norm.cu) and the
// fused cross-attention block (xattn_block_wgmma.cu) both call these, so their LayerNorms are one expression.
template <int LPR, int VPL>
__device__ __forceinline__ void layernorm_row_stats(const float (&f)[VPL][8], float s, int l, int CV, float eps,
                                                    float& mean, float& rstd) {
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float inv_c = 1.0f / (float)(CV * 8);
    // rounded on its own: with CV a compile-time constant the compiler would otherwise fuse s * inv_c into each f - mean
    mean = __fmul_rn(s, inv_c);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i)
        if (l + i * LPR < CV) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float d = f[i][j] - mean;
                q += d * d;
            }
        }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    rstd = rsqrtf(q * inv_c + eps);
}
template <int LPR, int VPL>
__device__ __forceinline__ void layernorm_row_apply(float (&f)[VPL][8], int l, int CV, const float* __restrict__ gamma,
                                                    const float* __restrict__ beta, float mean, float rstd) {
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        const int v = l + i * LPR;
        if (v < CV) {
            const float4* g4 = reinterpret_cast<const float4*>(gamma + v * 8);
            const float4* b4 = reinterpret_cast<const float4*>(beta + v * 8);
            float4 g0 = __ldg(g4), g1 = __ldg(g4 + 1), b0 = __ldg(b4), b1 = __ldg(b4 + 1);
            float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
            float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int j = 0; j < 8; ++j) f[i][j] = (f[i][j] - mean) * rstd * gg[j] + bb[j];
        }
    }
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

// cp.async 16B with zero-fill when !valid (src must still be a legal address)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
// D(16x8,f32) += A(16x16,f16,row) * B(16x8,f16,col)
__device__ __forceinline__ void mma_16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

}  // namespace anysd
