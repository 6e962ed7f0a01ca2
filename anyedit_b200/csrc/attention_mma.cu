// Flash-style attention, first-generation path: mma.sync m16n8k16, online softmax in fp32,
// K/V tiles double-buffered with cp.async.  Never materialises the n x n score matrix the
// reference's eager CrossAttention builds (ldm/modules/attention.py:171-193).
// One CTA = 64 query rows of one (batch, head); 4 warps x 16 rows; KV tiles of 64.
// Head dims 40 / 64 / 80 / 160 (any multiple of 8 up to 160 via the padded template sizes).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace anysd {

int launch_attention_wg(const anysd_attn_params* q, const int* kv_batch, cudaStream_t st);
bool attention_wg_supported(const anysd_attn_params* q);

constexpr int ATT_BQ = 64, ATT_BKV = 64, ATT_THREADS = 128;

struct AttnArgs {
    const __half* q; const __half* k; const __half* v; __half* out;
    long long qbs, kbs, vbs, obs;
    int ldq, ldk, ldv, ldo;
    int n_q, n_kv, d, hs;
    float scale_log2;
    const float* gate;
    int gate_stride, accumulate;
    const int* kv_batch;                      // optional [B]: query batch b reads the K/V of batch kv_batch[b]
};

__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

template <int DP>   // padded head dim, multiple of 16
__global__ void __launch_bounds__(ATT_THREADS) attention_mma_kernel(const AttnArgs p) {
    constexpr int LDS = DP + 8;               // smem row stride in halves (odd multiple of 16 bytes)
    constexpr int CH = DP / 8;                // 16-byte chunks per row
    constexpr int TILE = ATT_BKV * LDS;       // halves per tile
    extern __shared__ __align__(128) __half att_smem[];
    __half* sQ = att_smem;
    __half* sK = sQ + ATT_BQ * LDS;
    __half* sV = sK + 2 * TILE;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * ATT_BQ;
    const int dch = p.d / 8;                  // real chunks per row
    const __half* qg = p.q + (size_t)b * p.qbs + (size_t)h * p.hs;
    const int kvb = p.kv_batch ? __ldg(p.kv_batch + b) : b;
    const __half* kg = p.k + (size_t)kvb * p.kbs + (size_t)h * p.hs;
    const __half* vg = p.v + (size_t)kvb * p.vbs + (size_t)h * p.hs;

    auto load_tile = [&](const __half* g, int ld, int row0, int nrows, __half* s) {
        for (int i = tid; i < ATT_BKV * CH; i += ATT_THREADS) {
            const int r = i / CH, c = i - r * CH;
            const bool ok = (row0 + r) < nrows && c < dch;
            const __half* src = g + (size_t)(ok ? (row0 + r) : 0) * ld + (ok ? c * 8 : 0);
            cp_async16(smem_u32(s + r * LDS + c * 8), src, ok);
        }
    };

    load_tile(qg, p.ldq, q0, p.n_q, sQ);
    load_tile(kg, p.ldk, 0, p.n_kv, sK);
    load_tile(vg, p.ldv, 0, p.n_kv, sV);
    cp_async_commit();

    const int nt = (p.n_kv + ATT_BKV - 1) / ATT_BKV;
    uint32_t qf[DP / 16][4];
    float o[DP / 8][4];
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    for (int t = 0; t < nt; ++t) {
        const int buf = t & 1;
        if (t + 1 < nt) {
            load_tile(kg, p.ldk, (t + 1) * ATT_BKV, p.n_kv, sK + (buf ^ 1) * TILE);
            load_tile(vg, p.ldv, (t + 1) * ATT_BKV, p.n_kv, sV + (buf ^ 1) * TILE);
        }
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        if (t == 0) {
#pragma unroll
            for (int ks = 0; ks < DP / 16; ++ks) {
                const __half* a = sQ + (warp * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8;
                ldmatrix_x4(qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], smem_u32(a));
            }
        }
        const __half* kt = sK + buf * TILE;
        const __half* vt = sV + buf * TILE;

        // ---- S = Q K^T (16 x 64 per warp) ----
        float s[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < DP / 16; ++ks) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                uint32_t b0, b1, b2, b3;
                const __half* a = kt + (j * 16 + (lane & 7) + ((lane >> 4) << 3)) * LDS + ks * 16 + ((lane >> 3) & 1) * 8;
                ldmatrix_x4(b0, b1, b2, b3, smem_u32(a));
                mma_16816(s[2 * j], qf[ks], b0, b1);
                mma_16816(s[2 * j + 1], qf[ks], b2, b3);
            }
        }
        // ---- scale, mask, online softmax ----
        const int kv_left = p.n_kv - t * ATT_BKV;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int col = j * 8 + (lane & 3) * 2 + (e & 1);
                float v = s[j][e] * p.scale_log2;
                v = (col < kv_left) ? v : -INFINITY;
                s[j][e] = v;
                mx[e >> 1] = fmaxf(mx[e >> 1], v);
            }
        }
        float corr[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);
            corr[r] = ex2(m_run[r] - m_new);
            m_run[r] = m_new;
            l_run[r] *= corr[r];
        }
#pragma unroll
        for (int i = 0; i < DP / 8; ++i) {
            o[i][0] *= corr[0]; o[i][1] *= corr[0];
            o[i][2] *= corr[1]; o[i][3] *= corr[1];
        }
        uint32_t pf[4][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float p0 = ex2(s[j][0] - m_run[0]), p1 = ex2(s[j][1] - m_run[0]);
            const float p2 = ex2(s[j][2] - m_run[1]), p3 = ex2(s[j][3] - m_run[1]);
            l_run[0] += p0 + p1;
            l_run[1] += p2 + p3;
            __half2 h01 = __floats2half2_rn(p0, p1), h23 = __floats2half2_rn(p2, p3);
            pf[j >> 1][(j & 1) * 2 + 0] = *reinterpret_cast<uint32_t*>(&h01);
            pf[j >> 1][(j & 1) * 2 + 1] = *reinterpret_cast<uint32_t*>(&h23);
        }
        // ---- O += P V ----
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int dn = 0; dn < DP / 16; ++dn) {
                uint32_t b0, b1, b2, b3;
                const __half* a = vt + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + dn * 16 + (lane >> 4) * 8;
                ldmatrix_x4_trans(b0, b1, b2, b3, smem_u32(a));
                mma_16816(o[2 * dn], pf[kk], b0, b1);
                mma_16816(o[2 * dn + 1], pf[kk], b2, b3);
            }
        }
        __syncthreads();   // everyone done with buf before it is refilled two iterations later
    }
    cp_async_wait<0>();

    // ---- finalise ----
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float l = l_run[r];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv[r] = 1.0f / l;
    }
    const float g = p.gate ? p.gate[(size_t)b * p.gate_stride] : 1.0f;
    __half* og = p.out + (size_t)b * p.obs + (size_t)h * p.d;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = q0 + warp * 16 + (lane >> 2) + r * 8;
        if (row >= p.n_q) continue;
#pragma unroll
        for (int i = 0; i < DP / 8; ++i) {
            const int col = i * 8 + (lane & 3) * 2;
            if (col >= p.d) continue;
            float v0 = o[i][r * 2] * inv[r] * g, v1 = o[i][r * 2 + 1] * inv[r] * g;
            __half2* dst = reinterpret_cast<__half2*>(og + (size_t)row * p.ldo + col);
            if (p.accumulate) {
                float2 prev = __half22float2(*dst);
                v0 += prev.x;
                v1 += prev.y;
            }
            *dst = __floats2half2_rn(v0, v1);
        }
    }
}

template <int DP>
static int launch_attn(const AttnArgs& a, int B, int heads, cudaStream_t st) {
    constexpr int LDS = DP + 8;
    const int smem = (ATT_BQ + 4 * ATT_BKV) * LDS * (int)sizeof(__half);
    static bool done[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!done[dev]) {
        cudaFuncSetAttribute(attention_mma_kernel<DP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        done[dev] = true;
    }
    dim3 grid(cdiv(a.n_q, ATT_BQ), heads, B);
    attention_mma_kernel<DP><<<grid, ATT_THREADS, smem, st>>>(a);
    return check_launch("attention (mma.sync)");
}

int launch_attention_mma(const anysd_attn_params* q, const int* kv_batch, cudaStream_t st) {
    AttnArgs a;
    a.q = (const __half*)q->q; a.k = (const __half*)q->k; a.v = (const __half*)q->v; a.out = (__half*)q->out;
    a.qbs = q->q_batch_stride; a.kbs = q->k_batch_stride; a.vbs = q->v_batch_stride; a.obs = q->o_batch_stride;
    a.ldq = q->ld_q; a.ldk = q->ld_k; a.ldv = q->ld_v; a.ldo = q->ld_o;
    a.n_q = q->n_q; a.n_kv = q->n_kv; a.d = q->d;
    a.hs = q->head_stride > 0 ? q->head_stride : q->d;
    a.scale_log2 = q->scale * 1.4426950408889634f;
    a.gate = q->gate; a.gate_stride = q->gate_stride; a.accumulate = q->accumulate;
    a.kv_batch = kv_batch;
    const int dp = (q->d + 15) / 16 * 16;
    switch (dp) {
        case 16: return launch_attn<16>(a, q->B, q->heads, st);
        case 32: return launch_attn<32>(a, q->B, q->heads, st);
        case 48: return launch_attn<48>(a, q->B, q->heads, st);
        case 64: return launch_attn<64>(a, q->B, q->heads, st);
        case 80: return launch_attn<80>(a, q->B, q->heads, st);
        case 96: return launch_attn<96>(a, q->B, q->heads, st);
        case 128: return launch_attn<128>(a, q->B, q->heads, st);
        case 160: return launch_attn<160>(a, q->B, q->heads, st);
        default:
            set_error("attention: head dim %d not supported (multiples of 8 up to 160, padded to 16/32/48/64/80/96/128/160)", q->d);
            return ANYSD_EUNSUPPORTED;
    }
}

}  // namespace anysd

using namespace anysd;

static int attention_run(const anysd_attn_params* p, const int* kv_batch, anysd_stream_t stream) {
    ANYSD_REQUIRE(p != nullptr, ANYSD_EINVAL, "attention: null params");
    ANYSD_REQUIRE(p->q && p->k && p->v && p->out, ANYSD_EINVAL, "attention: null pointer");
    ANYSD_REQUIRE(p->B > 0 && p->heads > 0 && p->n_q > 0 && p->n_kv > 0, ANYSD_EINVAL, "attention: bad sizes");
    ANYSD_REQUIRE(p->d > 0 && p->d % 8 == 0 && p->d <= 160, ANYSD_EUNSUPPORTED,
                  "attention: head dim %d must be a multiple of 8, at most 160", p->d);
    ANYSD_REQUIRE(p->ld_q % 8 == 0 && p->ld_k % 8 == 0 && p->ld_v % 8 == 0 && p->ld_o % 2 == 0, ANYSD_EINVAL,
                  "attention: leading dims must be multiples of 8");
    ANYSD_REQUIRE(p->q_batch_stride % 8 == 0 && p->k_batch_stride % 8 == 0 && p->v_batch_stride % 8 == 0, ANYSD_EINVAL,
                  "attention: batch strides must be multiples of 8");
    ANYSD_REQUIRE(((uintptr_t)p->q % 16) == 0 && ((uintptr_t)p->k % 16) == 0 && ((uintptr_t)p->v % 16) == 0 &&
                      ((uintptr_t)p->out % 4) == 0,
                  ANYSD_EINVAL, "attention: q/k/v must be 16-byte aligned");
    ANYSD_REQUIRE(p->heads <= 65535 && p->B <= 65535, ANYSD_EINVAL, "attention: grid too large");
    ANYSD_REQUIRE(p->head_stride == 0 || (p->head_stride >= p->d && p->head_stride % 8 == 0), ANYSD_EINVAL,
                  "attention: head_stride must be 0 or a multiple of 8 >= d");
    ANYSD_REQUIRE(((uintptr_t)kv_batch % 4) == 0, ANYSD_EINVAL, "attention: kv_batch must be 4-byte aligned");
    // wgmma kernel whenever its layout constraints hold; ANYSD_ATTN=mma|wgmma is a test/debug switch.
    static const char* force = getenv("ANYSD_ATTN");
    const bool want_wg = !force || !strcmp(force, "wgmma");
    if (want_wg && attention_wg_supported(p)) return launch_attention_wg(p, kv_batch, (cudaStream_t)stream);
    ANYSD_REQUIRE(p->lse == nullptr, ANYSD_EUNSUPPORTED, "attention: the log-sum-exp output needs the wgmma kernel");
    ANYSD_REQUIRE(!p->aux_cols, ANYSD_EUNSUPPORTED,
                  "attention: aux_cols needs the wgmma kernel (d %% 16 == 8, head_stride >= d + 8, stacked batches)");
    return launch_attention_mma(p, kv_batch, (cudaStream_t)stream);
}

extern "C" int anysd_attention_f16(const anysd_attn_params* p, anysd_stream_t stream) {
    return attention_run(p, nullptr, stream);
}

extern "C" int anysd_attention_kvmap_f16(const anysd_attn_params* p, const int* kv_batch, anysd_stream_t stream) {
    return attention_run(p, kv_batch, stream);
}
