// Attention backward (SURVEY.md a24: the training step back-propagates through CrossAttention.forward,
// attention.py:163-194, to reach the adapter experts).  First-generation tensor-core path: mma.sync m16n8k16,
// flash-style recomputation -- the n x n probabilities are never stored; the forward keeps nothing but q, k, v.
//
//   s_ij = c (q_i . k_j)          c = qk_scale (natural-log units; the caller passes scale, or ln 2 when q is
//   p_ij = exp(s_ij - lse_i)          already multiplied by scale*log2(e) -- the aux_cols packing)
//   dp_ij = g_b (dO_i . v_j)      g_b = optional per-sample gate of the forward (expert sum)
//   D_i  = sum_j p_ij dp_ij       (= dO_i . O_i without needing O)
//   ds_ij = c p_ij (dp_ij - D_i)
//   dq_i = sum_j ds_ij k_j ;  dk_j = sum_i ds_ij q_i ;  dv_j = g_b sum_i p_ij dO_i ;  dg_b = sum_ij p_ij (dO_i . v_j)
//
// Two kernels, no cross-CTA reduction:
//   attn_bwd_dq_kernel : CTA = 64 query rows; pass 0 row max / sum -> lse, pass 1 D, pass 2 dq.  Writes lse (base 2)
//                        and D to the workspace.
//   attn_bwd_dkv_kernel: CTA = 64 key rows; every product is formed transposed (S^T = K Q^T, dP^T = V dO^T) so that
//                        key rows are the M dimension of every mma and P^T / dS^T are A operands straight from
//                        registers.  Head dims above 96 accumulate dk/dv in two column halves (register budget).
#include <math.h>

#include "common.cuh"

namespace anysd {

constexpr int AB_T = 64, AB_THREADS = 128;

struct BwdArgs {
    const __half* q; const __half* k; const __half* v; const __half* dout;
    __half* dq; __half* dk; __half* dv;
    long long qbs, kbs, vbs, dobs, dqbs, dkbs, dvbs;
    int ldq, ldk, ldv, lddo, lddq, lddk, lddv;
    int n_q, n_kv, d, hs, heads;
    float c_nat, c_log2;                 // qk_scale, qk_scale * log2(e)
    const float* gate; int gate_stride; float* dgate;
    int accumulate_dq;
    float* lse; float* D;                // [B, heads, n_q]
    const __half* o; long long obs; int ldo;   // optional: this attention's own (ungated) forward output -> D = dO . O
    int sets, set_stride, gate_set_stride;     // expert streams: blockIdx.z = b * sets + e; K/V/dK/dV of set e sit e*set_stride columns on
};

__device__ __forceinline__ float b_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

// rows [row0, row0 + AB_T) x DP columns of a head slice -> smem (zero fill outside nrows / d)
template <int DP>
__device__ __forceinline__ void b_load_tile(const __half* g, int ld, int row0, int nrows, int dch, __half* s) {
    constexpr int LDS = DP + 8, CH = DP / 8;
    for (int i = threadIdx.x; i < AB_T * CH; i += AB_THREADS) {
        const int r = i / CH, c = i - r * CH;
        const bool ok = (row0 + r) < nrows && c < dch;
        const __half* src = g + (size_t)(ok ? (row0 + r) : 0) * ld + (ok ? c * 8 : 0);
        cp_async16(smem_u32(s + r * LDS + c * 8), src, ok);
    }
}

// acc[T/8][4] (16 x T) = A(16 x DP, rows a_row0.. of sA) * B^T, B = T rows of sB (both K-contiguous, "row.col")
template <int DP, int T>
__device__ __forceinline__ void b_mma_nt(float (*acc)[4], const __half* sA, int a_row0, const __half* sB, int lane) {
    constexpr int LDS = DP + 8;
#pragma unroll
    for (int j = 0; j < T / 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < DP / 16; ++ks) {
        uint32_t af[4];
        ldmatrix_x4(af[0], af[1], af[2], af[3], smem_u32(sA + (a_row0 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8));
#pragma unroll
        for (int j = 0; j < T / 16; ++j) {
            uint32_t b0, b1, b2, b3;
            const __half* a = sB + (j * 16 + (lane & 7) + ((lane >> 4) << 3)) * LDS + ks * 16 + ((lane >> 3) & 1) * 8;
            ldmatrix_x4(b0, b1, b2, b3, smem_u32(a));
            mma_16816(acc[2 * j], af, b0, b1);
            mma_16816(acc[2 * j + 1], af, b2, b3);
        }
    }
}

// acc[NC/8][4] (16 x NC) += A(16 x T, register fragments af[T/16][4]) * B, B = T rows x NC columns of sB starting at col0
template <int DP, int T, int NC>
__device__ __forceinline__ void b_mma_nn(float (*acc)[4], const uint32_t (*af)[4], const __half* sB, int col0, int lane) {
    constexpr int LDS = DP + 8;
#pragma unroll
    for (int kk = 0; kk < T / 16; ++kk) {
#pragma unroll
        for (int dn = 0; dn < NC / 16; ++dn) {
            uint32_t b0, b1, b2, b3;
            const __half* a = sB + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + col0 + dn * 16 + (lane >> 4) * 8;
            ldmatrix_x4_trans(b0, b1, b2, b3, smem_u32(a));
            mma_16816(acc[2 * dn], af[kk], b0, b1);
            mma_16816(acc[2 * dn + 1], af[kk], b2, b3);
        }
    }
}

template <int DP>
__global__ void __launch_bounds__(AB_THREADS) attn_bwd_dq_kernel(const BwdArgs p) {
    constexpr int LDS = DP + 8, TILE = AB_T * LDS;
    extern __shared__ __align__(128) __half ab_smem[];
    __half* sQ = ab_smem;
    __half* sdO = sQ + TILE;
    __half* sK = sdO + TILE;
    __half* sV = sK + TILE;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * AB_T;
    const int dch = p.d / 8;
    const __half* qg = p.q + (size_t)b * p.qbs + (size_t)h * p.hs;
    const __half* kg = p.k + (size_t)b * p.kbs + (size_t)h * p.hs;
    const __half* vg = p.v + (size_t)b * p.vbs + (size_t)h * p.hs;
    const __half* og = p.dout + (size_t)b * p.dobs + (size_t)h * p.d;
    const float g = p.gate ? p.gate[(size_t)b * p.gate_stride] : 1.0f;
    const int nt = (p.n_kv + AB_T - 1) / AB_T;

    b_load_tile<DP>(qg, p.ldq, q0, p.n_q, dch, sQ);
    b_load_tile<DP>(og, p.lddo, q0, p.n_q, dch, sdO);
    cp_async_commit();

    // ---- pass 0: log-sum-exp (base 2) of every row ----
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    for (int t = 0; t < nt; ++t) {
        __syncthreads();
        b_load_tile<DP>(kg, p.ldk, t * AB_T, p.n_kv, dch, sK);
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
        float s[AB_T / 8][4];
        b_mma_nt<DP, AB_T>(s, sQ, warp * 16, sK, lane);
        const int kv_left = p.n_kv - t * AB_T;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int j = 0; j < AB_T / 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int col = j * 8 + (lane & 3) * 2 + (e & 1);
                const float v = col < kv_left ? s[j][e] * p.c_log2 : -INFINITY;
                s[j][e] = v;
                mx[e >> 1] = fmaxf(mx[e >> 1], v);
            }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);
            l_run[r] *= b_ex2(m_run[r] - m_new);
            m_run[r] = m_new;
        }
#pragma unroll
        for (int j = 0; j < AB_T / 8; ++j) {
            l_run[0] += b_ex2(s[j][0] - m_run[0]) + b_ex2(s[j][1] - m_run[0]);
            l_run[1] += b_ex2(s[j][2] - m_run[1]) + b_ex2(s[j][3] - m_run[1]);
        }
    }
    float lse[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float l = l_run[r];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        lse[r] = m_run[r] + log2f(l);
    }

    // ---- pass 1: D_raw_i = sum_j p_ij (dO_i . v_j)   (= dO_i . O_i: one smem pass when the caller kept O) ----
    float d_raw[2] = {0.f, 0.f};
    if (p.o != nullptr) {
        __syncthreads();
        b_load_tile<DP>(p.o + (size_t)b * p.obs + (size_t)h * p.d, p.ldo, q0, p.n_q, dch, sK);
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int lr = warp * 16 + (lane >> 2) + r * 8;
            for (int c = (lane & 3) * 2; c < p.d; c += 8) {
                const float2 a2 = __half22float2(*reinterpret_cast<const __half2*>(sdO + lr * LDS + c));
                const float2 o2 = __half22float2(*reinterpret_cast<const __half2*>(sK + lr * LDS + c));
                d_raw[r] += a2.x * o2.x + a2.y * o2.y;
            }
        }
    } else
    for (int t = 0; t < nt; ++t) {
        __syncthreads();
        b_load_tile<DP>(kg, p.ldk, t * AB_T, p.n_kv, dch, sK);
        b_load_tile<DP>(vg, p.ldv, t * AB_T, p.n_kv, dch, sV);
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
        float s[AB_T / 8][4], dp[AB_T / 8][4];
        b_mma_nt<DP, AB_T>(s, sQ, warp * 16, sK, lane);
        b_mma_nt<DP, AB_T>(dp, sdO, warp * 16, sV, lane);
        const int kv_left = p.n_kv - t * AB_T;
#pragma unroll
        for (int j = 0; j < AB_T / 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int col = j * 8 + (lane & 3) * 2 + (e & 1);
                const float pr = col < kv_left ? b_ex2(s[j][e] * p.c_log2 - lse[e >> 1]) : 0.f;
                d_raw[e >> 1] += pr * dp[j][e];
            }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        d_raw[r] += __shfl_xor_sync(0xffffffffu, d_raw[r], 1);
        d_raw[r] += __shfl_xor_sync(0xffffffffu, d_raw[r], 2);
    }
    const float Dg[2] = {g * d_raw[0], g * d_raw[1]};
    {
        const size_t base = ((size_t)b * p.heads + h) * p.n_q;
        float dg_part = 0.f;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int row = q0 + warp * 16 + (lane >> 2) + r * 8;
            if (row < p.n_q) {
                if ((lane & 3) == 0) {
                    p.lse[base + row] = lse[r];
                    p.D[base + row] = Dg[r];
                    dg_part += d_raw[r];
                }
            }
        }
        if (p.dgate) {
            dg_part = warp_sum(dg_part);
            if (lane == 0 && dg_part != 0.f) atomicAdd(p.dgate + (size_t)b * p.gate_stride, dg_part);
        }
    }

    // ---- pass 2: dq_i = sum_j ds_ij k_j ----
    float dq[DP / 8][4];
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
    for (int t = 0; t < nt; ++t) {
        __syncthreads();
        b_load_tile<DP>(kg, p.ldk, t * AB_T, p.n_kv, dch, sK);
        b_load_tile<DP>(vg, p.ldv, t * AB_T, p.n_kv, dch, sV);
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
        float s[AB_T / 8][4], dp[AB_T / 8][4];
        b_mma_nt<DP, AB_T>(s, sQ, warp * 16, sK, lane);
        b_mma_nt<DP, AB_T>(dp, sdO, warp * 16, sV, lane);
        const int kv_left = p.n_kv - t * AB_T;
        uint32_t dsf[AB_T / 16][4];
#pragma unroll
        for (int j = 0; j < AB_T / 8; ++j) {
            float ds[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int col = j * 8 + (lane & 3) * 2 + (e & 1);
                const float pr = col < kv_left ? b_ex2(s[j][e] * p.c_log2 - lse[e >> 1]) : 0.f;
                ds[e] = p.c_nat * pr * (g * dp[j][e] - Dg[e >> 1]);
            }
            dsf[j >> 1][(j & 1) * 2 + 0] = pack_h2(ds[0], ds[1]);
            dsf[j >> 1][(j & 1) * 2 + 1] = pack_h2(ds[2], ds[3]);
        }
        b_mma_nn<DP, AB_T, DP>(dq, dsf, sK, 0, lane);
    }
    __half* dqg = p.dq + (size_t)b * p.dqbs + (size_t)h * p.hs;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = q0 + warp * 16 + (lane >> 2) + r * 8;
        if (row >= p.n_q) continue;
#pragma unroll
        for (int i = 0; i < DP / 8; ++i) {
            const int col = i * 8 + (lane & 3) * 2;
            if (col >= p.hs) continue;
            float v0 = dq[i][r * 2], v1 = dq[i][r * 2 + 1];
            if (col >= p.d) v0 = v1 = 0.f;                     // padding columns of the head stay exact zeros
            __half2* dst = reinterpret_cast<__half2*>(dqg + (size_t)row * p.lddq + col);
            if (p.accumulate_dq) {
                const float2 prev = __half22float2(*dst);
                v0 += prev.x;
                v1 += prev.y;
            }
            *dst = __floats2half2_rn(v0, v1);
        }
    }
}

// PACK (expert streams with <= 16 tokens per expert, launch_experts): the 64 key rows of the CTA are FOUR experts' 16 token slots
// -- warp w owns expert 4 blockIdx.z' + w: its own gate, log-sum-exp / D rows and output rows -- instead of one expert's 16 tokens
// and 48 idle rows: a quarter of the CTAs for the same tile products.
template <int DP, int DC, bool PACK = false>
__global__ void __launch_bounds__(AB_THREADS) attn_bwd_dkv_kernel(const BwdArgs p) {
    constexpr int LDS = DP + 8, TILE = AB_T * LDS;
    extern __shared__ __align__(128) __half ab_smem[];
    __half* sK = ab_smem;
    __half* sV = sK + TILE;
    __half* sQ = sV + TILE;
    __half* sdO = sQ + TILE;
    float* s_lse = reinterpret_cast<float*>(sdO + TILE);       // PACK: [4][AB_T] each
    float* s_D = s_lse + (PACK ? 4 : 1) * AB_T;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int egroups = PACK ? (p.sets + 3) / 4 : 1;
    const int e = PACK ? (blockIdx.z % egroups) * 4 + warp : (p.sets > 1 ? blockIdx.z % p.sets : 0);       // PACK: this warp's expert
    const int b = PACK ? blockIdx.z / egroups : (p.sets > 1 ? blockIdx.z / p.sets : blockIdx.z);
    const bool e_ok = !PACK || e < p.sets;
    const int h = blockIdx.y, k0 = blockIdx.x * AB_T;
    const int dch = p.d / 8;
    const __half* qg = p.q + (size_t)b * p.qbs + (size_t)h * p.hs;
    const __half* kg = p.k + (size_t)b * p.kbs + (size_t)h * p.hs + (size_t)e * p.set_stride;
    const __half* vg = p.v + (size_t)b * p.vbs + (size_t)h * p.hs + (size_t)e * p.set_stride;
    const __half* og = p.dout + (size_t)b * p.dobs + (size_t)h * p.d;
    const float g = (p.gate && e_ok) ? p.gate[(size_t)b * p.gate_stride + (size_t)e * p.gate_set_stride] : (e_ok ? 1.0f : 0.f);
    const size_t sbase = (((size_t)b * p.heads + h) * p.sets + (e_ok ? e : 0)) * p.n_q;
    const int nqt = (p.n_q + AB_T - 1) / AB_T;

    if (PACK) {
        // key slot r of the tile = token r % 16 of expert 4 z' + r / 16 (zero when the expert or the token does not exist)
        constexpr int CH = DP / 8;
        const int e0 = (blockIdx.z % egroups) * 4;
        const __half* kb = p.k + (size_t)b * p.kbs + (size_t)h * p.hs;
        const __half* vb = p.v + (size_t)b * p.vbs + (size_t)h * p.hs;
        for (int i = tid; i < AB_T * CH; i += AB_THREADS) {
            const int r = i / CH, c = i - r * CH;
            const int ee = e0 + (r >> 4), tok = r & 15;
            const bool ok = ee < p.sets && tok < p.n_kv && c < dch;
            const size_t off = ok ? (size_t)ee * p.set_stride + (size_t)tok * p.ldk + c * 8 : 0;
            cp_async16(smem_u32(sK + r * LDS + c * 8), kb + off, ok);
            cp_async16(smem_u32(sV + r * LDS + c * 8), vb + (ok ? (size_t)ee * p.set_stride + (size_t)tok * p.ldv + c * 8 : 0), ok);
        }
    } else {
        b_load_tile<DP>(kg, p.ldk, k0, p.n_kv, dch, sK);
        b_load_tile<DP>(vg, p.ldv, k0, p.n_kv, dch, sV);
    }
    cp_async_commit();

    for (int c0 = 0; c0 < DP; c0 += DC) {
        float dk[DC / 8][4], dv[DC / 8][4];
#pragma unroll
        for (int i = 0; i < DC / 8; ++i) {
            dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
            dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
        }
        for (int t = 0; t < nqt; ++t) {
            __syncthreads();
            b_load_tile<DP>(qg, p.ldq, t * AB_T, p.n_q, dch, sQ);
            b_load_tile<DP>(og, p.lddo, t * AB_T, p.n_q, dch, sdO);
            cp_async_commit();
            if (PACK) {                                               // every warp stages its own expert's rows
                for (int c = lane; c < AB_T; c += 32) {
                    const int row = t * AB_T + c;
                    s_lse[warp * AB_T + c] = (row < p.n_q && e_ok) ? p.lse[sbase + row] : INFINITY;
                    s_D[warp * AB_T + c] = (row < p.n_q && e_ok) ? p.D[sbase + row] : 0.f;
                }
            } else if (tid < AB_T) {
                const int row = t * AB_T + tid;
                s_lse[tid] = row < p.n_q ? p.lse[sbase + row] : INFINITY;     // exp2(x - inf) = 0: padded queries vanish
                s_D[tid] = row < p.n_q ? p.D[sbase + row] : 0.f;
            }
            cp_async_wait<0>();
            __syncthreads();
            float st[AB_T / 8][4], dpt[AB_T / 8][4];
            b_mma_nt<DP, AB_T>(st, sK, warp * 16, sQ, lane);        // S^T: key rows x query columns
            b_mma_nt<DP, AB_T>(dpt, sV, warp * 16, sdO, lane);      // dP^T (without the gate)
            uint32_t pf[AB_T / 16][4], dsf[AB_T / 16][4];
#pragma unroll
            for (int j = 0; j < AB_T / 8; ++j) {
                float pr[4], ds[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int col = j * 8 + (lane & 3) * 2 + (e & 1);
                    pr[e] = b_ex2(st[j][e] * p.c_log2 - s_lse[(PACK ? warp * AB_T : 0) + col]);
                    ds[e] = p.c_nat * pr[e] * (g * dpt[j][e] - s_D[(PACK ? warp * AB_T : 0) + col]);
                }
                pf[j >> 1][(j & 1) * 2 + 0] = pack_h2(pr[0], pr[1]);
                pf[j >> 1][(j & 1) * 2 + 1] = pack_h2(pr[2], pr[3]);
                dsf[j >> 1][(j & 1) * 2 + 0] = pack_h2(ds[0], ds[1]);
                dsf[j >> 1][(j & 1) * 2 + 1] = pack_h2(ds[2], ds[3]);
            }
            b_mma_nn<DP, AB_T, DC>(dv, pf, sdO, c0, lane);          // dv += P^T dO
            b_mma_nn<DP, AB_T, DC>(dk, dsf, sQ, c0, lane);          // dk += dS^T Q
        }
        __half* dkg = p.dk + (size_t)b * p.dkbs + (size_t)h * p.hs + (size_t)(e_ok ? e : 0) * p.set_stride;
        __half* dvg = p.dv + (size_t)b * p.dvbs + (size_t)h * p.hs + (size_t)(e_ok ? e : 0) * p.set_stride;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int row = PACK ? (lane >> 2) + r * 8 : k0 + warp * 16 + (lane >> 2) + r * 8;      // PACK: token index inside the warp's expert
            if (row >= p.n_kv || !e_ok) continue;
#pragma unroll
            for (int i = 0; i < DC / 8; ++i) {
                const int col = c0 + i * 8 + (lane & 3) * 2;
                if (col >= p.hs) continue;
                const bool real = col < p.d;
                *reinterpret_cast<__half2*>(dkg + (size_t)row * p.lddk + col) =
                    __floats2half2_rn(real ? dk[i][r * 2] : 0.f, real ? dk[i][r * 2 + 1] : 0.f);
                *reinterpret_cast<__half2*>(dvg + (size_t)row * p.lddv + col) =
                    __floats2half2_rn(real ? g * dv[i][r * 2] : 0.f, real ? g * dv[i][r * 2 + 1] : 0.f);
            }
        }
    }
}

// ---- expert streams: sum_e g_e Attn(q, K_e, V_e) with every expert's few visual tokens in ONE key tile ------------
// (oracle/anysd_oracle.py cross_extra; ip_adapter/attention_processor.py:160-176).  One launch per layer instead of E:
// the CTA keeps its 64 query rows and walks the experts; each expert has its own softmax, complete inside the tile,
// so P is normalised and gated BEFORE the P.V product and the output / dq accumulators simply add over experts.
struct ExpArgs {
    const __half* q; const __half* kv; const __half* dout;
    __half* out; __half* dq;
    long long qbs, kvbs, obs, dobs, dqbs;
    int ldq, ldkv, ldo, lddo, lddq;
    int n_q, n_kv, d, hs, heads, E, set_stride, v_off;
    float c_nat, c_log2;
    const float* gates; float* dgates; int gate_b_stride;
    float* lse; float* D;                // [B, heads, E, n_q]
};

template <int DP, bool BWD>
__global__ void __launch_bounds__(AB_THREADS) expert_attn_kernel(const ExpArgs p) {
    constexpr int LDS = DP + 8, TILE = AB_T * LDS;
    extern __shared__ __align__(128) __half ab_smem[];
    __half* sQ = ab_smem;
    __half* sK = sQ + TILE;
    __half* sV = sK + TILE;
    __half* sdO = sV + TILE;             // BWD only
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * AB_T;
    const int dch = p.d / 8;
    const __half* qg = p.q + (size_t)b * p.qbs + (size_t)h * p.hs;
    b_load_tile<DP>(qg, p.ldq, q0, p.n_q, dch, sQ);
    if (BWD) b_load_tile<DP>(p.dout + (size_t)b * p.dobs + (size_t)h * p.d, p.lddo, q0, p.n_q, dch, sdO);
    cp_async_commit();
    float acc[DP / 8][4];                // forward: O;  backward: dq
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    for (int e = 0; e < p.E; ++e) {
        const __half* kg = p.kv + (size_t)b * p.kvbs + (size_t)e * p.set_stride + (size_t)h * p.hs;
        __syncthreads();
        b_load_tile<DP>(kg, p.ldkv, 0, p.n_kv, dch, sK);
        b_load_tile<DP>(kg + p.v_off, p.ldkv, 0, p.n_kv, dch, sV);
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
        const float g = p.gates[(size_t)b * p.gate_b_stride + e];
        float s[AB_T / 8][4];
        b_mma_nt<DP, AB_T>(s, sQ, warp * 16, sK, lane);
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int j = 0; j < AB_T / 8; ++j)
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const int col = j * 8 + (lane & 3) * 2 + (t & 1);
                const float v = col < p.n_kv ? s[j][t] * p.c_log2 : -INFINITY;
                s[j][t] = v;
                mx[t >> 1] = fmaxf(mx[t >> 1], v);
            }
        float l[2] = {0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        }
#pragma unroll
        for (int j = 0; j < AB_T / 8; ++j)
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                s[j][t] = b_ex2(s[j][t] - mx[t >> 1]);          // masked columns: exp2(-inf) = 0
                l[t >> 1] += s[j][t];
            }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
            l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
        }
        const float inv[2] = {1.0f / l[0], 1.0f / l[1]};
        uint32_t af[AB_T / 16][4];
        if (!BWD) {
#pragma unroll
            for (int j = 0; j < AB_T / 8; ++j) {
                af[j >> 1][(j & 1) * 2 + 0] = pack_h2(s[j][0] * inv[0] * g, s[j][1] * inv[0] * g);
                af[j >> 1][(j & 1) * 2 + 1] = pack_h2(s[j][2] * inv[1] * g, s[j][3] * inv[1] * g);
            }
            b_mma_nn<DP, AB_T, DP>(acc, af, sV, 0, lane);       // O += (g / l) P V
        } else {
            float dp[AB_T / 8][4];
            b_mma_nt<DP, AB_T>(dp, sdO, warp * 16, sV, lane);
            float d_raw[2] = {0.f, 0.f};
#pragma unroll
            for (int j = 0; j < AB_T / 8; ++j)
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    s[j][t] *= inv[t >> 1];                       // p_ij
                    d_raw[t >> 1] += s[j][t] * dp[j][t];
                }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                d_raw[r] += __shfl_xor_sync(0xffffffffu, d_raw[r], 1);
                d_raw[r] += __shfl_xor_sync(0xffffffffu, d_raw[r], 2);
            }
            const size_t base = (((size_t)b * p.heads + h) * p.E + e) * p.n_q;
            float dg_part = 0.f;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int row = q0 + warp * 16 + (lane >> 2) + r * 8;
                if (row < p.n_q && (lane & 3) == 0) {
                    p.lse[base + row] = mx[r] + log2f(l[r]);
                    p.D[base + row] = g * d_raw[r];
                    dg_part += d_raw[r];
                }
            }
            dg_part = warp_sum(dg_part);
            if (lane == 0 && dg_part != 0.f) atomicAdd(p.dgates + (size_t)b * p.gate_b_stride + e, dg_part);
#pragma unroll
            for (int j = 0; j < AB_T / 8; ++j) {
                float ds[4];
#pragma unroll
                for (int t = 0; t < 4; ++t) ds[t] = p.c_nat * g * s[j][t] * (dp[j][t] - d_raw[t >> 1]);
                af[j >> 1][(j & 1) * 2 + 0] = pack_h2(ds[0], ds[1]);
                af[j >> 1][(j & 1) * 2 + 1] = pack_h2(ds[2], ds[3]);
            }
            b_mma_nn<DP, AB_T, DP>(acc, af, sK, 0, lane);       // dq += dS K
        }
    }
    // accumulate onto the text attention's output / dq
    __half* og = BWD ? p.dq + (size_t)b * p.dqbs + (size_t)h * p.hs : p.out + (size_t)b * p.obs + (size_t)h * p.d;
    const int ld = BWD ? p.lddq : p.ldo;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = q0 + warp * 16 + (lane >> 2) + r * 8;
        if (row >= p.n_q) continue;
#pragma unroll
        for (int i = 0; i < DP / 8; ++i) {
            const int col = i * 8 + (lane & 3) * 2;
            if (col >= p.d) continue;
            __half2* dst = reinterpret_cast<__half2*>(og + (size_t)row * ld + col);
            const float2 prev = __half22float2(*dst);
            *dst = __floats2half2_rn(prev.x + acc[i][r * 2], prev.y + acc[i][r * 2 + 1]);
        }
    }
}

// ---- expert streams with at most 16 tokens each (AnySD: 16 visual tokens per expert, 11 experts) ---------------------------
// The kernel above spends a full 64-key tile, a K/V load and two CTA barriers on every expert.  Here ALL experts' keys and values
// of the (batch, head) are staged once -- expert e in key slots [16 e, 16 e + 16), unused slots zero -- and a 64-key tile of the
// products covers FOUR experts: each expert's softmax is a segment of 16 columns (two n8 fragments), normalised and gated
// before P.V, so the accumulator simply adds over all keys.  Same arithmetic per expert as above (fp32 softmax, fp16 P),
// 3 tile passes instead of 11 for E = 11.
template <int DP, bool BWD>
__global__ void __launch_bounds__(AB_THREADS) expert_attn16_kernel(const ExpArgs p, int groups, int qtiles) {
    constexpr int LDS = DP + 8, TILE = AB_T * LDS, CH = DP / 8;
    extern __shared__ __align__(128) __half ab_smem[];
    __half* sQ = ab_smem;
    __half* sdO = sQ + TILE;             // BWD only (the slot exists either way)
    __half* sK = sdO + TILE;
    __half* sV = sK + groups * TILE;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, h = blockIdx.y;
    int q0 = blockIdx.x * qtiles * AB_T;                         // the CTA walks `qtiles` query tiles: K/V are staged once for all of them
    const int dch = p.d / 8;
    b_load_tile<DP>(p.q + (size_t)b * p.qbs + (size_t)h * p.hs, p.ldq, q0, p.n_q, dch, sQ);
    if (BWD) b_load_tile<DP>(p.dout + (size_t)b * p.dobs + (size_t)h * p.d, p.lddo, q0, p.n_q, dch, sdO);
    const __half* kvg = p.kv + (size_t)b * p.kvbs + (size_t)h * p.hs;
    for (int i = tid; i < groups * AB_T * CH; i += AB_THREADS) {
        const int row = i / CH, c = i - row * CH;
        const int e = row >> 4, r = row & 15;
        const bool ok = e < p.E && r < p.n_kv && c < dch;
        const __half* src = kvg + (ok ? (size_t)e * p.set_stride + (size_t)r * p.ldkv + c * 8 : 0);
        cp_async16(smem_u32(sK + row * LDS + c * 8), src, ok);
        cp_async16(smem_u32(sV + row * LDS + c * 8), src + (ok ? p.v_off : 0), ok);
    }
    cp_async_commit();
    for (int qt = 0; qt < qtiles && q0 < p.n_q; ++qt, q0 += AB_T) {
    if (qt > 0) {
        __syncthreads();                 // every warp is through with the previous query tile
        b_load_tile<DP>(p.q + (size_t)b * p.qbs + (size_t)h * p.hs, p.ldq, q0, p.n_q, dch, sQ);
        if (BWD) b_load_tile<DP>(p.dout + (size_t)b * p.dobs + (size_t)h * p.d, p.lddo, q0, p.n_q, dch, sdO);
        cp_async_commit();
    }
    cp_async_wait<0>();
    __syncthreads();
    float acc[DP / 8][4];                // forward: O;  backward: dq
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    for (int g4 = 0; g4 < groups; ++g4) {
        float s[AB_T / 8][4];
        b_mma_nt<DP, AB_T>(s, sQ, warp * 16, sK + g4 * TILE, lane);
        float dp[AB_T / 8][4];
        if (BWD) b_mma_nt<DP, AB_T>(dp, sdO, warp * 16, sV + g4 * TILE, lane);
        uint32_t af[AB_T / 16][4];
#pragma unroll
        for (int el = 0; el < 4; ++el) {
            const int e = g4 * 4 + el;
            const bool valid = e < p.E;
            const float g = valid ? p.gates[(size_t)b * p.gate_b_stride + e] : 0.f;
            float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int jj = 0; jj < 2; ++jj)
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const int col = jj * 8 + (lane & 3) * 2 + (t & 1);
                    const float v = (valid && col < p.n_kv) ? s[2 * el + jj][t] * p.c_log2 : -INFINITY;
                    s[2 * el + jj][t] = v;
                    mx[t >> 1] = fmaxf(mx[t >> 1], v);
                }
            float l[2] = {0.f, 0.f};
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
                if (!valid) mx[r] = 0.f;                           // an empty slot group: every p = exp2(-inf) = 0, no NaN
            }
#pragma unroll
            for (int jj = 0; jj < 2; ++jj)
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    s[2 * el + jj][t] = b_ex2(s[2 * el + jj][t] - mx[t >> 1]);
                    l[t >> 1] += s[2 * el + jj][t];
                }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
                l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
            }
            const float inv[2] = {valid ? 1.0f / l[0] : 0.f, valid ? 1.0f / l[1] : 0.f};
            if (!BWD) {
#pragma unroll
                for (int jj = 0; jj < 2; ++jj) {
                    const int j = 2 * el + jj;
                    af[j >> 1][(j & 1) * 2 + 0] = pack_h2(s[j][0] * inv[0] * g, s[j][1] * inv[0] * g);
                    af[j >> 1][(j & 1) * 2 + 1] = pack_h2(s[j][2] * inv[1] * g, s[j][3] * inv[1] * g);
                }
            } else {
                float d_raw[2] = {0.f, 0.f};
#pragma unroll
                for (int jj = 0; jj < 2; ++jj)
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        s[2 * el + jj][t] *= inv[t >> 1];             // p_ij
                        d_raw[t >> 1] += s[2 * el + jj][t] * dp[2 * el + jj][t];
                    }
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    d_raw[r] += __shfl_xor_sync(0xffffffffu, d_raw[r], 1);
                    d_raw[r] += __shfl_xor_sync(0xffffffffu, d_raw[r], 2);
                }
                float dg_part = 0.f;
                if (valid) {
                    const size_t base = (((size_t)b * p.heads + h) * p.E + e) * p.n_q;
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const int row = q0 + warp * 16 + (lane >> 2) + r * 8;
                        if (row < p.n_q && (lane & 3) == 0) {
                            p.lse[base + row] = mx[r] + log2f(l[r]);
                            p.D[base + row] = g * d_raw[r];
                            dg_part += d_raw[r];
                        }
                    }
                }
                dg_part = warp_sum(dg_part);
                if (valid && lane == 0 && dg_part != 0.f) atomicAdd(p.dgates + (size_t)b * p.gate_b_stride + e, dg_part);
#pragma unroll
                for (int jj = 0; jj < 2; ++jj) {
                    const int j = 2 * el + jj;
                    float ds[4];
#pragma unroll
                    for (int t = 0; t < 4; ++t) ds[t] = p.c_nat * g * s[j][t] * (dp[j][t] - d_raw[t >> 1]);
                    af[j >> 1][(j & 1) * 2 + 0] = pack_h2(ds[0], ds[1]);
                    af[j >> 1][(j & 1) * 2 + 1] = pack_h2(ds[2], ds[3]);
                }
            }
        }
        if (!BWD) b_mma_nn<DP, AB_T, DP>(acc, af, sV + g4 * TILE, 0, lane);      // O += sum over the group's experts (g / l) P V
        else b_mma_nn<DP, AB_T, DP>(acc, af, sK + g4 * TILE, 0, lane);            // dq += dS K
    }
    __half* og = BWD ? p.dq + (size_t)b * p.dqbs + (size_t)h * p.hs : p.out + (size_t)b * p.obs + (size_t)h * p.d;
    const int ld = BWD ? p.lddq : p.ldo;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = q0 + warp * 16 + (lane >> 2) + r * 8;
        if (row >= p.n_q) continue;
#pragma unroll
        for (int i = 0; i < DP / 8; ++i) {
            const int col = i * 8 + (lane & 3) * 2;
            if (col >= p.d) continue;
            __half2* dst = reinterpret_cast<__half2*>(og + (size_t)row * ld + col);
            const float2 prev = __half22float2(*dst);
            *dst = __floats2half2_rn(prev.x + acc[i][r * 2], prev.y + acc[i][r * 2 + 1]);
        }
    }
    }                                    // query tiles
}

template <int DP>
static int launch_experts(const ExpArgs& a, const BwdArgs* dkv, int B, cudaStream_t st) {
    constexpr int LDS = DP + 8;
    constexpr int DC = DP > 96 ? DP / 2 : DP;
    const int smem = 4 * AB_T * LDS * (int)sizeof(__half) + 2 * AB_T * (int)sizeof(float);
    static bool done[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!done[dev]) {
        cudaFuncSetAttribute(expert_attn_kernel<DP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(expert_attn_kernel<DP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(attn_bwd_dkv_kernel<DP, DC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        done[dev] = true;
    }
    dim3 grid(cdiv(a.n_q, AB_T), a.heads, B);
    // few tokens per expert: all experts staged once, four per key tile (expert_attn16_kernel); ANYSD_EXPERT16=0 switches it off
    static const char* e16 = getenv("ANYSD_EXPERT16");
    const int groups = (a.E + 3) / 4;
    const int smem16 = (2 + 2 * groups) * AB_T * LDS * (int)sizeof(__half);
    const bool use16 = a.n_kv <= 16 && smem16 <= 200 * 1024 && !(e16 && e16[0] == '0');
    if (use16) {
        static int set16[64];
        if (set16[dev] < smem16) {
            cudaFuncSetAttribute(expert_attn16_kernel<DP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem16);
            cudaFuncSetAttribute(expert_attn16_kernel<DP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem16);
            set16[dev] = smem16;
        }
    }
    // query tiles per CTA: 1 (staging the 37 KB of K/V once for several query tiles did not pay on the project's earlier GPU; not
    // re-measured on the H100).  ANYSD_EXPERT_QT overrides.
    static const char* qt_env = getenv("ANYSD_EXPERT_QT");
    const int qtiles = (use16 && qt_env && atoi(qt_env) > 0) ? atoi(qt_env) : 1;
    const dim3 grid16(cdiv(a.n_q, AB_T * qtiles), a.heads, B);
    if (dkv == nullptr) {
        if (use16) expert_attn16_kernel<DP, false><<<grid16, AB_THREADS, smem16, st>>>(a, groups, qtiles);
        else expert_attn_kernel<DP, false><<<grid, AB_THREADS, smem, st>>>(a);
        return check_launch("expert attention");
    }
    if (use16) expert_attn16_kernel<DP, true><<<grid16, AB_THREADS, smem16, st>>>(a, groups, qtiles);
    else expert_attn_kernel<DP, true><<<grid, AB_THREADS, smem, st>>>(a);
    int rc = check_launch("expert attention backward (dq)");
    if (rc) return rc;
    if (use16) {
        const int smem_p = 4 * AB_T * LDS * (int)sizeof(__half) + 8 * AB_T * (int)sizeof(float);
        static int setp[64];
        if (!setp[dev]) {
            cudaFuncSetAttribute(attn_bwd_dkv_kernel<DP, DC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_p);
            setp[dev] = 1;
        }
        attn_bwd_dkv_kernel<DP, DC, true><<<dim3(1, a.heads, B * groups), AB_THREADS, smem_p, st>>>(*dkv);
    } else {
        attn_bwd_dkv_kernel<DP, DC><<<dim3(cdiv(a.n_kv, AB_T), a.heads, B * a.E), AB_THREADS, smem, st>>>(*dkv);
    }
    return check_launch("expert attention backward (dk, dv)");
}

template <int DP>
static int launch_bwd(const BwdArgs& a, int B, cudaStream_t st, bool need_dkv) {
    constexpr int LDS = DP + 8;
    constexpr int DC = DP > 96 ? DP / 2 : DP;
    const int smem = 4 * AB_T * LDS * (int)sizeof(__half) + 2 * AB_T * (int)sizeof(float);
    static bool done[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!done[dev]) {
        cudaFuncSetAttribute(attn_bwd_dq_kernel<DP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(attn_bwd_dkv_kernel<DP, DC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        done[dev] = true;
    }
    attn_bwd_dq_kernel<DP><<<dim3(cdiv(a.n_q, AB_T), a.heads, B), AB_THREADS, smem, st>>>(a);
    int rc = check_launch("attention backward (dq)");
    if (rc || !need_dkv) return rc;
    attn_bwd_dkv_kernel<DP, DC><<<dim3(cdiv(a.n_kv, AB_T), a.heads, B), AB_THREADS, smem, st>>>(a);
    return check_launch("attention backward (dk, dv)");
}

}  // namespace anysd

using namespace anysd;

namespace anysd {
bool attention_bwd_wg_supported(const anysd_attn_bwd_params* q);
int launch_attention_bwd_wg(const anysd_attn_bwd_params* q, cudaStream_t st);
}

extern "C" size_t anysd_attention_bwd_workspace_bytes(int B, int heads, int n_q) {
    if (B <= 0 || heads <= 0 || n_q <= 0) return 0;
    return (size_t)2 * B * heads * n_q * sizeof(float);
}

extern "C" int anysd_attention_bwd_f16(const anysd_attn_bwd_params* p, anysd_stream_t stream) {
    ANYSD_REQUIRE(p != nullptr, ANYSD_EINVAL, "attention_bwd: null params");
    ANYSD_REQUIRE(p->q && p->k && p->v && p->d_out && p->dq && p->workspace, ANYSD_EINVAL, "attention_bwd: null pointer");
    ANYSD_REQUIRE((p->dk == nullptr) == (p->dv == nullptr), ANYSD_EINVAL, "attention_bwd: dk and dv go together");
    ANYSD_REQUIRE(p->B > 0 && p->heads > 0 && p->n_q > 0 && p->n_kv > 0, ANYSD_EINVAL, "attention_bwd: bad sizes");
    ANYSD_REQUIRE(p->d > 0 && p->d % 8 == 0 && p->d <= 160, ANYSD_EUNSUPPORTED,
                  "attention_bwd: head dim %d must be a multiple of 8, at most 160", p->d);
    const int hs = p->head_stride > 0 ? p->head_stride : p->d;
    const int dp = (p->d + 15) / 16 * 16;
    ANYSD_REQUIRE(hs % 8 == 0 && hs >= p->d && hs <= dp, ANYSD_EINVAL,
                  "attention_bwd: head_stride %d must be a multiple of 8 in [d, ceil16(d)]", hs);
    ANYSD_REQUIRE(p->ld_q % 8 == 0 && p->ld_k % 8 == 0 && p->ld_v % 8 == 0 && p->ld_do % 8 == 0 && p->ld_dq % 2 == 0 &&
                      (!p->dk || (p->ld_dk % 2 == 0 && p->ld_dv % 2 == 0)),
                  ANYSD_EINVAL, "attention_bwd: leading dims must be multiples of 8 (inputs) / 2 (outputs)");
    ANYSD_REQUIRE(p->q_batch_stride % 8 == 0 && p->k_batch_stride % 8 == 0 && p->v_batch_stride % 8 == 0 &&
                      p->do_batch_stride % 8 == 0,
                  ANYSD_EINVAL, "attention_bwd: batch strides must be multiples of 8");
    ANYSD_REQUIRE(((uintptr_t)p->q % 16) == 0 && ((uintptr_t)p->k % 16) == 0 && ((uintptr_t)p->v % 16) == 0 &&
                      ((uintptr_t)p->d_out % 16) == 0 && ((uintptr_t)p->dq % 4) == 0,
                  ANYSD_EINVAL, "attention_bwd: pointers must be 16-byte aligned");
    ANYSD_REQUIRE(p->workspace_bytes >= anysd_attention_bwd_workspace_bytes(p->B, p->heads, p->n_q), ANYSD_EINVAL,
                  "attention_bwd: workspace too small");
    ANYSD_REQUIRE(p->heads <= 65535 && p->B <= 65535, ANYSD_EINVAL, "attention_bwd: grid too large");
    ANYSD_REQUIRE(p->out == nullptr || (p->gate == nullptr && p->ld_o % 8 == 0 && ((uintptr_t)p->out % 16) == 0 && p->o_batch_stride % 8 == 0),
                  ANYSD_EINVAL, "attention_bwd: `out` must be the un-gated output of this attention, 16-byte aligned, ld_o %% 8 == 0");
    // wgmma kernels when the forward's log-sum-exp came along and the shape allows (attention_wgmma.cu)
    if (attention_bwd_wg_supported(p)) return launch_attention_bwd_wg(p, (cudaStream_t)stream);
    BwdArgs a;
    a.q = (const __half*)p->q; a.k = (const __half*)p->k; a.v = (const __half*)p->v; a.dout = (const __half*)p->d_out;
    a.dq = (__half*)p->dq; a.dk = (__half*)p->dk; a.dv = (__half*)p->dv;
    a.qbs = p->q_batch_stride; a.kbs = p->k_batch_stride; a.vbs = p->v_batch_stride; a.dobs = p->do_batch_stride;
    a.dqbs = p->dq_batch_stride; a.dkbs = p->dk_batch_stride; a.dvbs = p->dv_batch_stride;
    a.ldq = p->ld_q; a.ldk = p->ld_k; a.ldv = p->ld_v; a.lddo = p->ld_do; a.lddq = p->ld_dq; a.lddk = p->ld_dk; a.lddv = p->ld_dv;
    a.n_q = p->n_q; a.n_kv = p->n_kv; a.d = p->d; a.hs = hs; a.heads = p->heads;
    a.c_nat = p->qk_scale; a.c_log2 = p->qk_scale * 1.4426950408889634f;
    a.gate = p->gate; a.gate_stride = p->gate_stride; a.dgate = p->d_gate;
    a.accumulate_dq = p->accumulate_dq;
    a.lse = (float*)p->workspace; a.D = a.lse + (size_t)p->B * p->heads * p->n_q;
    ANYSD_REQUIRE(p->out == nullptr || (p->gate == nullptr && p->ld_o % 8 == 0 && ((uintptr_t)p->out % 16) == 0 && p->o_batch_stride % 8 == 0),
                  ANYSD_EINVAL, "attention_bwd: `out` must be the un-gated output of this attention, 16-byte aligned, ld_o %% 8 == 0");
    a.o = (const __half*)p->out; a.obs = p->o_batch_stride; a.ldo = p->ld_o;
    a.sets = 1; a.set_stride = 0; a.gate_set_stride = 0;
    cudaStream_t st = (cudaStream_t)stream;
    const bool need = p->dk != nullptr;
    switch (dp) {
        case 16: return launch_bwd<16>(a, p->B, st, need);
        case 32: return launch_bwd<32>(a, p->B, st, need);
        case 48: return launch_bwd<48>(a, p->B, st, need);
        case 64: return launch_bwd<64>(a, p->B, st, need);
        case 80: return launch_bwd<80>(a, p->B, st, need);
        case 96: return launch_bwd<96>(a, p->B, st, need);
        case 128: return launch_bwd<128>(a, p->B, st, need);
        case 160: return launch_bwd<160>(a, p->B, st, need);
        default:
            set_error("attention_bwd: head dim %d not supported", p->d);
            return ANYSD_EUNSUPPORTED;
    }
}

extern "C" size_t anysd_expert_attention_bwd_workspace_bytes(int B, int heads, int E, int n_q) {
    if (B <= 0 || heads <= 0 || E <= 0 || n_q <= 0) return 0;
    return (size_t)2 * B * heads * E * n_q * sizeof(float);
}

static int expert_common(const anysd_expert_attn_params* p, bool bwd, ExpArgs& a) {
    ANYSD_REQUIRE(p != nullptr && p->q && p->kv && p->gates, ANYSD_EINVAL, "expert_attention: null pointer");
    ANYSD_REQUIRE(p->B > 0 && p->heads > 0 && p->n_q > 0 && p->E > 0 && p->n_kv > 0 && p->n_kv <= AB_T, ANYSD_EUNSUPPORTED,
                  "expert_attention: every expert's tokens must fit one key tile (n_kv <= %d, got %d)", AB_T, p->n_kv);
    ANYSD_REQUIRE(p->d > 0 && p->d % 8 == 0 && p->d <= 160, ANYSD_EUNSUPPORTED, "expert_attention: head dim %d", p->d);
    const int hs = p->head_stride > 0 ? p->head_stride : p->d;
    ANYSD_REQUIRE(hs % 8 == 0 && hs >= p->d, ANYSD_EINVAL, "expert_attention: bad head_stride");
    ANYSD_REQUIRE(p->ld_q % 8 == 0 && p->ld_kv % 8 == 0 && p->set_stride % 8 == 0 && p->v_offset % 8 == 0 && p->ld_o % 2 == 0, ANYSD_EINVAL,
                  "expert_attention: leading dims / offsets must be multiples of 8");
    ANYSD_REQUIRE(((uintptr_t)p->q % 16) == 0 && ((uintptr_t)p->kv % 16) == 0, ANYSD_EINVAL, "expert_attention: 16-byte alignment");
    ANYSD_REQUIRE(p->heads <= 65535 && (long long)p->B * p->E <= 65535, ANYSD_EINVAL, "expert_attention: grid too large");
    a.q = (const __half*)p->q; a.kv = (const __half*)p->kv; a.out = (__half*)p->out;
    a.qbs = (long long)p->n_q * p->ld_q; a.kvbs = (long long)p->n_kv * p->ld_kv; a.obs = (long long)p->n_q * p->ld_o;
    a.ldq = p->ld_q; a.ldkv = p->ld_kv; a.ldo = p->ld_o;
    a.n_q = p->n_q; a.n_kv = p->n_kv; a.d = p->d; a.hs = hs; a.heads = p->heads; a.E = p->E;
    a.set_stride = p->set_stride; a.v_off = p->v_offset;
    a.c_nat = p->qk_scale; a.c_log2 = p->qk_scale * 1.4426950408889634f;
    a.gates = p->gates; a.gate_b_stride = p->gate_b_stride;
    a.dout = nullptr; a.dq = nullptr; a.dgates = nullptr; a.lse = a.D = nullptr; a.dobs = a.dqbs = 0; a.lddo = a.lddq = 0;
    (void)bwd;
    return ANYSD_OK;
}

#define ANYSD_EXP_DISPATCH(CALL)                                                               \
    switch ((p->d + 15) / 16 * 16) {                                                           \
        case 16: return CALL(16); case 32: return CALL(32); case 48: return CALL(48);          \
        case 64: return CALL(64); case 80: return CALL(80); case 96: return CALL(96);          \
        case 128: return CALL(128); case 160: return CALL(160);                                \
        default: set_error("expert_attention: head dim %d not supported", p->d); return ANYSD_EUNSUPPORTED; \
    }

extern "C" int anysd_expert_attention_f16(const anysd_expert_attn_params* p, anysd_stream_t stream) {
    ExpArgs a;
    int rc = expert_common(p, false, a);
    if (rc) return rc;
    ANYSD_REQUIRE(p->out != nullptr, ANYSD_EINVAL, "expert_attention: null out");
#define ANYSD_CALL(DPV) launch_experts<DPV>(a, nullptr, p->B, (cudaStream_t)stream)
    ANYSD_EXP_DISPATCH(ANYSD_CALL)
#undef ANYSD_CALL
}

extern "C" int anysd_expert_attention_bwd_f16(const anysd_expert_attn_params* p, const void* d_out, int ld_do, void* dq, int ld_dq,
                                              void* dkv, float* d_gates, void* workspace, size_t workspace_bytes,
                                              anysd_stream_t stream) {
    ExpArgs a;
    int rc = expert_common(p, true, a);
    if (rc) return rc;
    ANYSD_REQUIRE(d_out && dq && dkv && d_gates && workspace, ANYSD_EINVAL, "expert_attention_bwd: null pointer");
    ANYSD_REQUIRE(ld_do % 8 == 0 && ld_dq % 2 == 0 && ((uintptr_t)d_out % 16) == 0, ANYSD_EINVAL, "expert_attention_bwd: bad strides");
    ANYSD_REQUIRE(workspace_bytes >= anysd_expert_attention_bwd_workspace_bytes(p->B, p->heads, p->E, p->n_q), ANYSD_EINVAL,
                  "expert_attention_bwd: workspace too small");
    const int dp = (p->d + 15) / 16 * 16;
    ANYSD_REQUIRE(a.hs <= dp, ANYSD_EINVAL, "expert_attention_bwd: head_stride must be <= ceil16(d)");
    a.dout = (const __half*)d_out; a.lddo = ld_do; a.dobs = (long long)p->n_q * ld_do;
    a.dq = (__half*)dq; a.lddq = ld_dq; a.dqbs = (long long)p->n_q * ld_dq;
    a.dgates = d_gates;
    a.lse = (float*)workspace; a.D = a.lse + (size_t)p->B * p->heads * p->E * p->n_q;
    BwdArgs k;
    k.q = a.q; k.k = a.kv; k.v = a.kv + p->v_offset; k.dout = a.dout;
    k.dq = nullptr; k.dk = (__half*)dkv; k.dv = (__half*)dkv + p->v_offset;
    k.qbs = a.qbs; k.kbs = a.kvbs; k.vbs = a.kvbs; k.dobs = a.dobs; k.dqbs = 0; k.dkbs = a.kvbs; k.dvbs = a.kvbs;
    k.ldq = a.ldq; k.ldk = a.ldkv; k.ldv = a.ldkv; k.lddo = ld_do; k.lddq = 0; k.lddk = a.ldkv; k.lddv = a.ldkv;
    k.n_q = a.n_q; k.n_kv = a.n_kv; k.d = a.d; k.hs = a.hs; k.heads = a.heads;
    k.c_nat = a.c_nat; k.c_log2 = a.c_log2;
    k.gate = a.gates; k.gate_stride = a.gate_b_stride; k.dgate = nullptr; k.accumulate_dq = 0;
    k.lse = a.lse; k.D = a.D; k.o = nullptr; k.obs = 0; k.ldo = 0;
    k.sets = p->E; k.set_stride = p->set_stride; k.gate_set_stride = 1;
#define ANYSD_CALL(DPV) launch_experts<DPV>(a, &k, p->B, (cudaStream_t)stream)
    ANYSD_EXP_DISPATCH(ANYSD_CALL)
#undef ANYSD_CALL
}
