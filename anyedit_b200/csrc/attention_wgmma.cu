// Hopper-native attention: S = Q K^T and O += P V on wgmma with register accumulators, operands staged by TMA,
// online softmax in fp32 on the accumulator fragment.  Replaces the n x n score tensor of the reference's eager
// CrossAttention (ldm/modules/attention.py:171-193).
//
//   CTA = 128 query rows of one (batch, head), 384 threads: warpgroup 0 is the TMA producer (Q once, then a 3-stage ring
//   of (K, V) tiles of BKV rows, 128-byte swizzle) and hands its registers to consumer warpgroups 1 and 2 (setmaxnreg
//   24 / 240), which own 64 query rows each.
//   Per kv tile: S [64 x BKV] = Q K^T (both operands in shared memory, K-extent d_ext = ceil16(d)); online softmax in
//   base 2 (a score row lives in the 4 lanes of a quad; keys past n_kv masked in the last, partial tile); P rounded to
//   fp16 and kept in registers as the A operand of O [64 x d_ext] += P V, V consumed as an MN-major B operand straight
//   from its row-major tile.
//   Schedule: the products of tile j are S_j and P_{j-1} V_{j-1}, issued back to back; the softmax of S_j runs while
//   P_{j-1} V_{j-1} is still on the tensor cores.  The two consumer warpgroups take turns issuing (named barriers 1 and
//   2), so one warpgroup's exponentials run under the other's products.
//   d % 16 == 8 needs the head stride padded to >= ceil16(d) with zero columns (anyedit_b200.unet packs q/k/v that way).
//   aux_cols operands (anysd_attn_params::aux_cols) arrive with q pre-scaled by scale * log2(e); their extra padding
//   columns multiply zeros here, so they run with a unit scale (the UNIT instances: no scale multiply at all).
//   Exponent arithmetic: p = ex2(round(s * scale_log2) - m) with the maximum m of the rounded scaled scores, and the
//   denominator summed from the unrounded fp32 p in a fixed order.
#include <cuda.h>
#include <math.h>
#include <stdlib.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace anysd {

constexpr int AW_BQ = 128, AW_ATOM = 128 * 128, AW_ST = 2;     // Q atom: 128 rows x 64 halves; AW_ST: backward ring
constexpr int AW_THREADS = 384, AW_KV_ST = 3;                  // forward: producer + 2 consumer warpgroups, (K, V) ring

struct AwArgs {
    __half* out;
    long long obs;
    int ldo;
    int n_q, n_kv, d, hs;              // hs = head stride (elements) inside q/k/v rows
    float scale_log2;
    const float* gate;
    int gate_stride, accumulate;
    float* lse;                        // optional [B, heads, n_q]: base-2 log-sum-exp of every score row
};

__device__ __forceinline__ void aw_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void aw_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void aw_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void aw_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void aw_tma_2d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ float aw_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t aw_pack(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
// Issue turns of the two consumer warpgroups: warpgroup c waits on named barrier 1 + c before it issues its products, and
// then arrives on the other one's barrier (both barriers count the 256 consumer threads).
__device__ __forceinline__ void aw_turn_wait(int c) { asm volatile("bar.sync %0, 256;" ::"r"(1 + c) : "memory"); }
__device__ __forceinline__ void aw_turn_pass(int c) { asm volatile("bar.arrive %0, 256;" ::"r"(2 - c) : "memory"); }

template <int DP, int BKV>
struct AwCfg {
    static constexpr int NA = (DP + 63) / 64;                 // 64-column atoms per row
    static constexpr int KV_ATOM = BKV * 128;                 // bytes of one [BKV x 64] K or V atom
    static constexpr int STAGE_BYTES = 2 * NA * KV_ATOM;      // K then V
    static constexpr int SMEM = NA * AW_ATOM + AW_KV_ST * STAGE_BYTES + 1024 + 128;
    static_assert(SMEM <= 227 * 1024, "attention (wgmma): shared memory");
};

// UNIT: aux_cols operands (q pre-scaled, unit scale), where the scale multiplies below fold away
template <int DP, int BKV, bool UNIT>
__global__ void __launch_bounds__(AW_THREADS, 1)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmV, const AwArgs p) {
    using Cfg = AwCfg<DP, BKV>;
    constexpr int NA = Cfg::NA, KV_ATOM = Cfg::KV_ATOM, ST = AW_KV_ST;
    extern __shared__ unsigned char aw_smem_raw[];
    const uint32_t raw = smem_u32(aw_smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;              // 128-byte swizzled tiles want 1024-byte alignment
    const uint32_t kv_off = NA * AW_ATOM;
    const uint32_t bars = base + kv_off + ST * Cfg::STAGE_BYTES;
    // barriers: 0 q_full | 1.. kv_full | 1 + ST.. kv_empty
    auto BAR = [&](int i) { return bars + 8u * i; };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * AW_BQ;
    const int nt = (p.n_kv + BKV - 1) / BKV;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmQ) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmK) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmV) : "memory");
        aw_init(BAR(0), 1);
        for (int s = 0; s < ST; ++s) {
            aw_init(BAR(1 + s), 1);
            aw_init(BAR(1 + ST + s), 8);                        // one arrive per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 4) {
        // ===== TMA producer warpgroup: one thread issues the loads =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;" ::: "memory");
        if (warp == 0 && lane == 0) {
            const int col0 = h * p.hs;
            aw_expect_tx(BAR(0), NA * AW_ATOM);
            for (int a = 0; a < NA; ++a) aw_tma_2d(base + a * AW_ATOM, &tmQ, BAR(0), col0 + a * 64, b * p.n_q + q0);
            for (int j = 0; j < nt; ++j) {
                const int s = j % ST;
                aw_wait(BAR(1 + ST + s), (((uint32_t)j / ST) & 1) ^ 1);
                aw_expect_tx(BAR(1 + s), Cfg::STAGE_BYTES);
                const uint32_t kb = base + kv_off + s * Cfg::STAGE_BYTES, vb = kb + NA * KV_ATOM;
                for (int a = 0; a < NA; ++a) aw_tma_2d(kb + a * KV_ATOM, &tmK, BAR(1 + s), col0 + a * 64, b * p.n_kv + j * BKV);
                for (int a = 0; a < NA; ++a) aw_tma_2d(vb + a * KV_ATOM, &tmV, BAR(1 + s), col0 + a * 64, b * p.n_kv + j * BKV);
            }
        }
        return;
    }

    // ===== two consumer warpgroups, 64 query rows each; this thread: rows r0 and r0 + 8 of the warp's 16 =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;" ::: "memory");
    const int wg = __shfl_sync(0xffffffffu, (warp >> 2) - 1, 0);   // warp-uniform to the compiler: keeps wgmma unserialized
    const int wq = warp & 3, q4 = lane & 3;
    const uint32_t qa = base + wg * 64 * 128;
    const float c = UNIT ? 1.0f : p.scale_log2;                // > 0 (attention_wg_supported)
    float o[DP / 2];
#pragma unroll
    for (int i = 0; i < DP / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float sc[BKV / 2];                                          // S_j, then its exponentials
    uint32_t pa[BKV / 16][4];                                   // P_{j-1} in the A-operand register layout of m64k16
    auto issue_s = [&](int j) {                                 // S_j = Q K_j^T
        const uint32_t kb = base + kv_off + (j % ST) * Cfg::STAGE_BYTES;
#pragma unroll
        for (int k = 0; k < DP / 16; ++k)
            Wgmma<BKV>::ss(sc, wg_desc(qa + (k >> 2) * AW_ATOM + (k & 3) * 32, 16, 1024),
                           wg_desc(kb + (k >> 2) * KV_ATOM + (k & 3) * 32, 16, 1024), k > 0);
        wg_commit();
    };
    auto issue_pv = [&](int j) {                                // O += P_j V_j
        const uint32_t vb = base + kv_off + (j % ST) * Cfg::STAGE_BYTES + NA * KV_ATOM;
#pragma unroll
        for (int kk = 0; kk < BKV / 16; ++kk) Wgmma<DP>::rs_t(o, pa[kk], wg_desc(vb + kk * 2048, KV_ATOM, 1024), 1);
        wg_commit();
    };
    auto release = [&](int j) {                                 // after O += P_j V_j has completed: K/V stage free
#pragma unroll
        for (int i = 0; i < DP / 2; ++i) wg_fence_regs(o[i]);
        __syncwarp();
        if (lane == 0) aw_arrive(BAR(1 + ST + j % ST));
    };
    // online softmax (base 2) of the completed S_j: sc becomes its exponentials, corr the factor of the running sums.
    // The compiler turns the mask of the last, partial tile into a select per element on every tile; measured on the H100,
    // a second softmax body without it was slower (larger loop), so the mask stays inline.
    auto softmax = [&](int j, float (&corr)[2]) {
#pragma unroll
        for (int i = 0; i < BKV / 2; ++i) wg_fence_regs(sc[i]);
        const int kv_left = p.n_kv - j * BKV;
        if (kv_left < BKV) {                                    // keys past n_kv
#pragma unroll
            for (int i = 0; i < BKV / 8; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (8 * i + 2 * q4 + (e & 1) >= kv_left) sc[4 * i + e] = -INFINITY;
        }
        // row maxima of the unscaled scores: c > 0 and rounding is monotone, so max(s) c rounds to the maximum of the rounded s c
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < BKV / 8; ++i)
#pragma unroll
            for (int e = 0; e < 4; ++e) mx[e >> 1] = fmaxf(mx[e >> 1], sc[4 * i + e]);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r] * c);
            corr[r] = aw_ex2(m_run[r] - m_new);                // first tile: ex2(-inf) = 0
            m_run[r] = m_new;
            l_run[r] *= corr[r];
        }
        // p = 2^(round(s c) - m): the scaled score is rounded before the maximum is subtracted (no FFMA), so every p
        // keeps the bits of scaling the score row first
#pragma unroll
        for (int kk = 0; kk < BKV / 16; ++kk) {
            float* t = sc + 8 * kk;
#pragma unroll
            for (int e = 0; e < 8; ++e) t[e] = aw_ex2((UNIT ? t[e] : __fmul_rn(t[e], c)) - m_run[(e >> 1) & 1]);
            l_run[0] += (t[0] + t[1]) + (t[4] + t[5]);
            l_run[1] += (t[2] + t[3]) + (t[6] + t[7]);
        }
    };
    // once O += P_{j-1} V_{j-1} has completed: O rescaled to the new row maxima, P_j packed as the next A operand
    auto rescale_pack = [&](const float (&corr)[2]) {
#pragma unroll
        for (int i = 0; i < DP / 8; ++i) {
            o[4 * i] *= corr[0];
            o[4 * i + 1] *= corr[0];
            o[4 * i + 2] *= corr[1];
            o[4 * i + 3] *= corr[1];
        }
#pragma unroll
        for (int kk = 0; kk < BKV / 16; ++kk) {
            const float* t = sc + 8 * kk;
            pa[kk][0] = aw_pack(t[0], t[1]);
            pa[kk][1] = aw_pack(t[2], t[3]);
            pa[kk][2] = aw_pack(t[4], t[5]);
            pa[kk][3] = aw_pack(t[6], t[7]);
        }
    };

    // Turn order: warpgroup 0 takes the first turn without waiting, and warpgroup 1 passes no turn after its last one, so
    // every bar.sync meets exactly one bar.arrive.
    aw_wait(BAR(0), 0);
    float corr[2];
    aw_wait(BAR(1), 0);
    if (wg == 1) aw_turn_wait(wg);
    wg_fence();
    issue_s(0);
    aw_turn_pass(wg);
    wg_wait<0>();
    softmax(0, corr);
    rescale_pack(corr);
    for (int j = 1; j < nt; ++j) {
        aw_wait(BAR(1 + j % ST), ((uint32_t)j / ST) & 1);
        aw_turn_wait(wg);
        wg_fence();
        issue_s(j);
        issue_pv(j - 1);
        aw_turn_pass(wg);
        wg_wait<1>();                                           // S_j done; P_{j-1} V_{j-1} still running
        softmax(j, corr);
        wg_wait<0>();
        release(j - 1);
        rescale_pack(corr);
    }
    aw_turn_wait(wg);
    wg_fence();
    issue_pv(nt - 1);
    wg_wait<0>();
    if (wg == 0) aw_turn_pass(wg);
    release(nt - 1);

    // ---- epilogue: O / l -> fp16 -> global ----
    const float g = p.gate ? p.gate[(size_t)b * p.gate_stride] : 1.0f;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float l = l_run[r];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const int qr = q0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * r;
        if (qr >= p.n_q) continue;
        if (p.lse != nullptr && q4 == 0) p.lse[((size_t)b * gridDim.y + h) * p.n_q + qr] = m_run[r] + log2f(l);
        const float inv = g / l;
        __half* orow = p.out + (size_t)b * p.obs + (size_t)qr * p.ldo + (size_t)h * p.d;
#pragma unroll
        for (int i = 0; i < DP / 8; ++i) {
            const int col = 8 * i + 2 * q4;
            if (col >= p.d) break;
            float v0 = o[4 * i + 2 * r] * inv, v1 = o[4 * i + 2 * r + 1] * inv;
            __half2* dst = reinterpret_cast<__half2*>(orow + col);
            if (p.accumulate) {
                const float2 prev = __half22float2(*dst);
                v0 += prev.x;
                v1 += prev.y;
            }
            *dst = __floats2half2_rn(v0, v1);
        }
    }
}

// ---- host ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFnA)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFnA a_get_encode() {
    static EncodeTiledFnA fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qr) == cudaSuccess &&
            qr == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFnA)f;
    }
    return fn;
}
// 2-D fp16 map with a 64-column (128-byte, swizzled) box
static bool a_map(CUtensorMap* tm, const void* ptr, uint64_t width, uint64_t rows, uint64_t ld, uint32_t box_rows) {
    cuuint64_t dims[2] = {width, rows};
    cuuint64_t strides[1] = {ld * 2};
    cuuint32_t box[2] = {64, box_rows};
    cuuint32_t es[2] = {1, 1};
    return a_get_encode()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

bool attention_wg_supported(const anysd_attn_params* q) {
    const int hs = q->head_stride > 0 ? q->head_stride : q->d;
    const int d_ext = (q->d + 15) / 16 * 16;
    if (d_ext > hs && q->heads > 1) return false;              // K-extent would reach into the next head's columns
    if (q->d % 8 != 0 || d_ext > 160) return false;
    if (q->aux_cols && (q->d % 16 != 8 || hs < q->d + 8)) return false;
    if (!q->aux_cols && !(q->scale > 0.f)) return false;       // the kernel takes the row maximum before scaling
    if (q->ld_q % 8 || q->ld_k % 8 || q->ld_v % 8 || q->ld_o % 8) return false;
    if (((uintptr_t)q->q % 16) || ((uintptr_t)q->k % 16) || ((uintptr_t)q->v % 16) || ((uintptr_t)q->out % 16)) return false;
    // batches must be stacked rows of one matrix (what the UNet produces): batch stride = n * ld
    if (q->q_batch_stride != (long long)q->n_q * q->ld_q || q->k_batch_stride != (long long)q->n_kv * q->ld_k ||
        q->v_batch_stride != (long long)q->n_kv * q->ld_v)
        return false;
    if ((q->o_batch_stride % 8) != 0) return false;
    return a_get_encode() != nullptr;
}

template <int DP>
static int aw_launch(const anysd_attn_params* q, const AwArgs& a, cudaStream_t st) {
    // kv tile: 128 rows while the S and O fragments fit the registers next to each other, 64 for the wide heads
    constexpr int BKV = DP <= 64 ? 128 : 64;
    using Cfg = AwCfg<DP, BKV>;
    const int hs = a.hs;
    CUtensorMap tmQ, tmK, tmV;
    // valid columns from the slice pointer (aux_cols: the last head's padding columns are operands too)
    const uint64_t width = q->aux_cols ? (uint64_t)q->heads * hs : (uint64_t)(q->heads - 1) * hs + q->d;
    const bool ok = a_map(&tmQ, q->q, width, (uint64_t)q->B * q->n_q, q->ld_q, AW_BQ) &&
                    a_map(&tmK, q->k, width, (uint64_t)q->B * q->n_kv, q->ld_k, BKV) &&
                    a_map(&tmV, q->v, width, (uint64_t)q->B * q->n_kv, q->ld_v, BKV);
    if (!ok) {
        set_error("attention (wgmma): cuTensorMapEncodeTiled failed (B=%d n_q=%d n_kv=%d d=%d)", q->B, q->n_q, q->n_kv, q->d);
        return ANYSD_ECUDA;
    }
    static bool done[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(attention_wgmma_kernel<DP, BKV, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(attention_wgmma_kernel<DP, BKV, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
        if (e != cudaSuccess) {
            set_error("attention (wgmma): smem opt-in failed: %s", cudaGetErrorString(e));
            return ANYSD_ECUDA;
        }
        done[dev] = true;
    }
    dim3 grid(cdiv(q->n_q, AW_BQ), q->heads, q->B);
    if (q->aux_cols) attention_wgmma_kernel<DP, BKV, true><<<grid, AW_THREADS, Cfg::SMEM, st>>>(tmQ, tmK, tmV, a);
    else attention_wgmma_kernel<DP, BKV, false><<<grid, AW_THREADS, Cfg::SMEM, st>>>(tmQ, tmK, tmV, a);
    return check_launch("attention (wgmma)");
}

int launch_attention_wg(const anysd_attn_params* q, cudaStream_t st) {
    AwArgs a;
    a.out = (__half*)q->out;
    a.obs = q->o_batch_stride;
    a.ldo = q->ld_o;
    a.n_q = q->n_q; a.n_kv = q->n_kv; a.d = q->d;
    a.hs = q->head_stride > 0 ? q->head_stride : q->d;
    a.scale_log2 = q->aux_cols ? 1.0f : q->scale * 1.4426950408889634f;
    a.gate = q->gate; a.gate_stride = q->gate_stride; a.accumulate = q->accumulate;
    a.lse = q->lse;
    switch ((q->d + 15) / 16 * 16) {
        case 16: return aw_launch<16>(q, a, st);
        case 32: return aw_launch<32>(q, a, st);
        case 48: return aw_launch<48>(q, a, st);
        case 64: return aw_launch<64>(q, a, st);
        case 80: return aw_launch<80>(q, a, st);
        case 96: return aw_launch<96>(q, a, st);
        case 112: return aw_launch<112>(q, a, st);
        case 128: return aw_launch<128>(q, a, st);
        case 144: return aw_launch<144>(q, a, st);
        default: return aw_launch<160>(q, a, st);
    }
}

// ===== backward (train.py:694-709 through attention.py:163-194) =============================================================
// The forward's base-2 log-sum-exp (anysd_attn_params::lse) makes the probabilities one exp2 away: no log-sum-exp pass.
//   bwd_prep_kernel       D = dO . O per (query, head), and dO re-laid into the padded head layout of q / k / v (its padding
//                         columns are K-extent of dO V^T and must be zero: with aux_cols V carries 1.0 there).
//   bwd_wgmma_kernel<DQ>  CTA = 128 query rows (Q, dO resident), 64-key tiles of (K, V) streamed: S = Q K^T, dP = dO V^T,
//                         dS = c P (dP - D) in registers, dQ += dS K (dS as register A operand, K as MN-major B).
//   bwd_wgmma_kernel<DKV> CTA = 128 key rows (K, V resident), 64-query tiles of (Q, dO) streamed, every product transposed so that
//                         key rows are the M dimension: S^T = K Q^T, dP^T = V dO^T, dV += P^T dO, dK += dS^T Q.
// No cross-CTA reduction, no atomics: deterministic.  Shapes: ceil16(d) <= 64 == head stride, n_q and n_kv multiples of 128,
// stacked batches, no gate (anything else runs the mma.sync kernels of attention_bwd.cu).
constexpr int BW_THREADS = 288, BW_RES = 128, BW_STR = 64;
constexpr int BW_RES_ATOM = BW_RES * 128, BW_STR_ATOM = BW_STR * 128;

struct BwArgs {
    __half* dq; __half* dk; __half* dv;
    long long dqbs, dkbs, dvbs;
    int lddq, lddk, lddv;
    int n_q, n_kv, d, hs;
    float c_nat, c_log2;
    const float* lse;       // [B, heads, n_q] base-2 log-sum-exp of the forward
    const float* D;         // [B, heads, n_q]
    int accumulate_dq;
};

// one thread per (row, head): d / 8 16-byte vectors of dO and O in, hs / 8 vectors out (zeros behind column d)
__global__ void bwd_prep_kernel(const __half* __restrict__ dout, long long dobs, int lddo, const __half* __restrict__ o, long long obs,
                                int ldo, __half* __restrict__ dpad, float* __restrict__ D, int B, int n_q, int heads, int d, int hs) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)B * n_q * heads;
    if (t >= total) return;
    const int h = (int)(t % heads);
    const long long r = t / heads;
    const int b = (int)(r / n_q), i = (int)(r % n_q);
    const uint4* g = reinterpret_cast<const uint4*>(dout + (size_t)b * dobs + (size_t)i * lddo + (size_t)h * d);
    const uint4* oo = reinterpret_cast<const uint4*>(o + (size_t)b * obs + (size_t)i * ldo + (size_t)h * d);
    uint4* dst = reinterpret_cast<uint4*>(dpad + ((size_t)r * heads + h) * hs);
    float acc = 0.f;
    for (int v = 0; v < d / 8; ++v) {
        const uint4 a = __ldg(g + v), c = __ldg(oo + v);
        float fa[8], fc[8];
        unpack8(a, fa);
        unpack8(c, fc);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc = fmaf(fa[k], fc[k], acc);
        dst[v] = a;
    }
    for (int v = d / 8; v < hs / 8; ++v) dst[v] = make_uint4(0u, 0u, 0u, 0u);
    D[((size_t)b * heads + h) * n_q + i] = acc;
}

// DQ: resident (R1, R2) = (Q, dO), streamed (S1, S2) = (K, V).  !DQ: resident = (K, V), streamed = (Q, dO).
template <int DP, bool DQ>
__global__ void __launch_bounds__(BW_THREADS, 1)
bwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmR1, const __grid_constant__ CUtensorMap tmR2,
                 const __grid_constant__ CUtensorMap tmS1, const __grid_constant__ CUtensorMap tmS2, const BwArgs p) {
    extern __shared__ unsigned char bw_smem_raw[];
    const uint32_t raw = smem_u32(bw_smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    constexpr uint32_t STAGE = 2 * BW_STR_ATOM;
    const uint32_t str_off = 2 * BW_RES_ATOM;
    const uint32_t bars = base + str_off + AW_ST * STAGE;
    auto BAR = [&](int i) { return bars + 8u * i; };     // 0 resident | 1.. stream full | 1 + AW_ST.. stream empty

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.z, h = blockIdx.y, heads = gridDim.y;
    const int n_res = DQ ? p.n_q : p.n_kv, n_str = DQ ? p.n_kv : p.n_q;
    const int r0 = blockIdx.x * BW_RES;
    const int nt = n_str / BW_STR;

    if (threadIdx.x == 0) {
        aw_init(BAR(0), 1);
        for (int s = 0; s < AW_ST; ++s) {
            aw_init(BAR(1 + s), 1);
            aw_init(BAR(1 + AW_ST + s), 8);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            const int col0 = h * p.hs;
            aw_expect_tx(BAR(0), 2 * BW_RES_ATOM);
            aw_tma_2d(base, &tmR1, BAR(0), col0, b * n_res + r0);
            aw_tma_2d(base + BW_RES_ATOM, &tmR2, BAR(0), col0, b * n_res + r0);
            for (int j = 0; j < nt; ++j) {
                const int s = j % AW_ST;
                aw_wait(BAR(1 + AW_ST + s), (((uint32_t)j / AW_ST) & 1) ^ 1);
                aw_expect_tx(BAR(1 + s), STAGE);
                const uint32_t sb = base + str_off + s * STAGE;
                aw_tma_2d(sb, &tmS1, BAR(1 + s), col0, b * n_str + j * BW_STR);
                aw_tma_2d(sb + BW_STR_ATOM, &tmS2, BAR(1 + s), col0, b * n_str + j * BW_STR);
            }
        }
        return;
    }

    const int wg = warp >> 2, wq = warp & 3, q4 = lane & 3;
    const uint32_t a1 = base + wg * 64 * 128, a2 = a1 + BW_RES_ATOM;
    const size_t sbase = ((size_t)b * heads + h) * p.n_q;      // lse / D of this (batch, head)
    float acc1[DP / 2], acc2[DP / 2];                            // DQ: dQ | !DQ: dK, dV
#pragma unroll
    for (int i = 0; i < DP / 2; ++i) acc1[i] = acc2[i] = 0.f;
    // DQ: this thread's two query rows carry their log-sum-exp and D
    float lse_r[2] = {0.f, 0.f}, D_r[2] = {0.f, 0.f};
    if (DQ) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int qr = r0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * r;
            lse_r[r] = __ldg(p.lse + sbase + qr);
            D_r[r] = __ldg(p.D + sbase + qr);
        }
    }
    aw_wait(BAR(0), 0);
    for (int j = 0; j < nt; ++j) {
        const int s = j % AW_ST;
        // !DQ: the streamed tile's query columns carry the log-sum-exp and D (loads in flight while the tile lands)
        float2 lse_c[BW_STR / 8], D_c[BW_STR / 8];
        if (!DQ) {
#pragma unroll
            for (int i = 0; i < BW_STR / 8; ++i) {
                const size_t qc = sbase + (size_t)j * BW_STR + 8 * i + 2 * q4;
                lse_c[i] = __ldg(reinterpret_cast<const float2*>(p.lse + qc));
                D_c[i] = __ldg(reinterpret_cast<const float2*>(p.D + qc));
            }
        }
        aw_wait(BAR(1 + s), ((uint32_t)j / AW_ST) & 1);
        const uint32_t s1 = base + str_off + s * STAGE, s2 = s1 + BW_STR_ATOM;
        float x[BW_STR / 2], y[BW_STR / 2];                     // S (or S^T) and dP (or dP^T)
        wg_fence();
#pragma unroll
        for (int k = 0; k < DP / 16; ++k)
            Wgmma<BW_STR>::ss(x, wg_desc(a1 + k * 32, 16, 1024), wg_desc(s1 + k * 32, 16, 1024), k > 0);
#pragma unroll
        for (int k = 0; k < DP / 16; ++k)
            Wgmma<BW_STR>::ss(y, wg_desc(a2 + k * 32, 16, 1024), wg_desc(s2 + k * 32, 16, 1024), k > 0);
        wg_commit();
        wg_wait<0>();
#pragma unroll
        for (int i = 0; i < BW_STR / 2; ++i) {
            wg_fence_regs(x[i]);
            wg_fence_regs(y[i]);
        }
        // element 4 i + 2 hh + e: row (lane / 4 + 8 hh) of the warp's 16, column 8 i + 2 (lane % 4) + e of the tile
        uint32_t pa[BW_STR / 16][4], da[BW_STR / 16][4];        // P (or P^T) and dS (or dS^T) as fp16 A operands
#pragma unroll
        for (int kk = 0; kk < BW_STR / 16; ++kk) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {                       // A register q: column block i = 2 kk + q / 2, row half hh = q % 2
                const int i = 2 * kk + (q >> 1), hh = q & 1, t = 4 * i + 2 * hh;
                const float l0 = DQ ? lse_r[hh] : lse_c[i].x, l1 = DQ ? lse_r[hh] : lse_c[i].y;
                const float d0 = DQ ? D_r[hh] : D_c[i].x, d1 = DQ ? D_r[hh] : D_c[i].y;
                const float p0 = aw_ex2(fmaf(x[t], p.c_log2, -l0)), p1 = aw_ex2(fmaf(x[t + 1], p.c_log2, -l1));
                pa[kk][q] = aw_pack(p0, p1);
                da[kk][q] = aw_pack(p.c_nat * p0 * (y[t] - d0), p.c_nat * p1 * (y[t + 1] - d1));
            }
        }
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < BW_STR / 16; ++kk) {
            if (DQ) {
                Wgmma<DP>::rs_t(acc1, da[kk], wg_desc(s1 + kk * 2048, BW_STR_ATOM, 1024), 1);       // dQ += dS K
            } else {
                Wgmma<DP>::rs_t(acc1, da[kk], wg_desc(s1 + kk * 2048, BW_STR_ATOM, 1024), 1);       // dK += dS^T Q
                Wgmma<DP>::rs_t(acc2, pa[kk], wg_desc(s2 + kk * 2048, BW_STR_ATOM, 1024), 1);       // dV += P^T dO
            }
        }
        wg_commit();
        wg_wait<0>();
#pragma unroll
        for (int i = 0; i < DP / 2; ++i) {
            wg_fence_regs(acc1[i]);
            wg_fence_regs(acc2[i]);
        }
        __syncwarp();
        if (lane == 0) aw_arrive(BAR(1 + AW_ST + s));
    }

    // ---- epilogue: fp16 rows, padding columns written as zeros ----
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = r0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * r;
#pragma unroll
        for (int i = 0; i < DP / 8; ++i) {
            const int col = 8 * i + 2 * q4;
            const bool in = col < p.d;
            if (DQ) {
                __half2* dst = reinterpret_cast<__half2*>(p.dq + (size_t)b * p.dqbs + (size_t)row * p.lddq + (size_t)h * p.hs + col);
                float v0 = in ? acc1[4 * i + 2 * r] : 0.f, v1 = in ? acc1[4 * i + 2 * r + 1] : 0.f;
                if (p.accumulate_dq && in) {
                    const float2 prev = __half22float2(*dst);
                    v0 += prev.x;
                    v1 += prev.y;
                }
                *dst = __floats2half2_rn(v0, v1);
            } else {
                *reinterpret_cast<__half2*>(p.dk + (size_t)b * p.dkbs + (size_t)row * p.lddk + (size_t)h * p.hs + col) =
                    __floats2half2_rn(in ? acc1[4 * i + 2 * r] : 0.f, in ? acc1[4 * i + 2 * r + 1] : 0.f);
                *reinterpret_cast<__half2*>(p.dv + (size_t)b * p.dvbs + (size_t)row * p.lddv + (size_t)h * p.hs + col) =
                    __floats2half2_rn(in ? acc2[4 * i + 2 * r] : 0.f, in ? acc2[4 * i + 2 * r + 1] : 0.f);
            }
        }
    }
}

bool attention_bwd_wg_supported(const anysd_attn_bwd_params* q) {
    static const char* off = getenv("ANYSD_ATTN_BWD");
    if (off && off[0] == 'm') return false;                     // ANYSD_ATTN_BWD=mma: the mma.sync kernels (A/B switch)
    const int hs = q->head_stride > 0 ? q->head_stride : q->d;
    const int d_ext = (q->d + 15) / 16 * 16;
    if (q->lse == nullptr || q->out == nullptr || q->dout_padded == nullptr || q->gate != nullptr || q->d_gate != nullptr) return false;
    if (d_ext > 64 || hs != d_ext || q->d % 8 != 0) return false;
    if (q->n_q % BW_RES != 0 || q->n_kv % BW_RES != 0) return false;
    if (q->ld_q % 8 || q->ld_k % 8 || q->ld_v % 8 || q->ld_dq % 8 || (q->dk && (q->ld_dk % 8 || q->ld_dv % 8))) return false;
    if (((uintptr_t)q->q % 16) || ((uintptr_t)q->k % 16) || ((uintptr_t)q->v % 16) || ((uintptr_t)q->dq % 16) ||
        ((uintptr_t)q->dout_padded % 16) || (q->dk && (((uintptr_t)q->dk % 16) || ((uintptr_t)q->dv % 16))))
        return false;
    if (q->q_batch_stride != (long long)q->n_q * q->ld_q || q->k_batch_stride != (long long)q->n_kv * q->ld_k ||
        q->v_batch_stride != (long long)q->n_kv * q->ld_v)
        return false;
    if ((q->dq_batch_stride % 8) || (q->dk && ((q->dk_batch_stride % 8) || (q->dv_batch_stride % 8)))) return false;
    return a_get_encode() != nullptr;
}

template <int DP>
static int bw_launch(const anysd_attn_bwd_params* q, const BwArgs& a, __half* dpad, cudaStream_t st) {
    const int hs = a.hs;
    const uint64_t width = (uint64_t)q->heads * hs, rq = (uint64_t)q->B * q->n_q, rk = (uint64_t)q->B * q->n_kv, ldp = width;
    CUtensorMap tmQ, tmDO, tmK, tmV, tmQs, tmDOs, tmKs, tmVs;    // resident 128-row tiles / streamed 64-row tiles
    const bool ok = a_map(&tmQ, q->q, width, rq, q->ld_q, BW_RES) && a_map(&tmDO, dpad, width, rq, ldp, BW_RES) &&
                    a_map(&tmK, q->k, width, rk, q->ld_k, BW_RES) && a_map(&tmV, q->v, width, rk, q->ld_v, BW_RES) &&
                    a_map(&tmQs, q->q, width, rq, q->ld_q, BW_STR) && a_map(&tmDOs, dpad, width, rq, ldp, BW_STR) &&
                    a_map(&tmKs, q->k, width, rk, q->ld_k, BW_STR) && a_map(&tmVs, q->v, width, rk, q->ld_v, BW_STR);
    if (!ok) {
        set_error("attention_bwd (wgmma): cuTensorMapEncodeTiled failed (B=%d n_q=%d n_kv=%d d=%d)", q->B, q->n_q, q->n_kv, q->d);
        return ANYSD_ECUDA;
    }
    const int smem = 2 * BW_RES_ATOM + AW_ST * 2 * BW_STR_ATOM + 1024 + 128;
    static bool done[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(bwd_wgmma_kernel<DP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(bwd_wgmma_kernel<DP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) {
            set_error("attention_bwd (wgmma): smem opt-in failed: %s", cudaGetErrorString(e));
            return ANYSD_ECUDA;
        }
        done[dev] = true;
    }
    bwd_wgmma_kernel<DP, true><<<dim3(q->n_q / BW_RES, q->heads, q->B), BW_THREADS, smem, st>>>(tmQ, tmDO, tmKs, tmVs, a);
    int rc = check_launch("attention_bwd dq (wgmma)");
    if (rc || q->dk == nullptr) return rc;
    bwd_wgmma_kernel<DP, false><<<dim3(q->n_kv / BW_RES, q->heads, q->B), BW_THREADS, smem, st>>>(tmK, tmV, tmQs, tmDOs, a);
    return check_launch("attention_bwd dk/dv (wgmma)");
}

int launch_attention_bwd_wg(const anysd_attn_bwd_params* q, cudaStream_t st) {
    const int hs = q->head_stride > 0 ? q->head_stride : q->d;
    BwArgs a;
    a.dq = (__half*)q->dq; a.dk = (__half*)q->dk; a.dv = (__half*)q->dv;
    a.dqbs = q->dq_batch_stride; a.dkbs = q->dk_batch_stride; a.dvbs = q->dv_batch_stride;
    a.lddq = q->ld_dq; a.lddk = q->ld_dk; a.lddv = q->ld_dv;
    a.n_q = q->n_q; a.n_kv = q->n_kv; a.d = q->d; a.hs = hs;
    a.c_nat = q->qk_scale; a.c_log2 = q->qk_scale * 1.4426950408889634f;
    a.lse = q->lse;
    float* D = (float*)q->workspace;                            // [B, heads, n_q] (the workspace holds twice that)
    a.D = D;
    a.accumulate_dq = q->accumulate_dq;
    __half* dpad = (__half*)q->dout_padded;
    const long long total = (long long)q->B * q->n_q * q->heads;
    bwd_prep_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const __half*)q->d_out, q->do_batch_stride, q->ld_do, (const __half*)q->out,
                                                                     q->o_batch_stride, q->ld_o, dpad, D, q->B, q->n_q, q->heads, q->d, hs);
    int rc = check_launch("attention_bwd (prep)");
    if (rc) return rc;
    switch (hs) {
        case 16: return bw_launch<16>(q, a, dpad, st);
        case 32: return bw_launch<32>(q, a, dpad, st);
        case 48: return bw_launch<48>(q, a, dpad, st);
        default: return bw_launch<64>(q, a, dpad, st);
    }
}

}  // namespace anysd
