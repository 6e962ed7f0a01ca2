// GroupNorm(+SiLU) on NHWC fp16 and LayerNorm on token rows.  HBM-bound kernels:
// 16-byte vector loads/stores, fp32 statistics, warp-shuffle / smem reductions.
//
// GroupNorm: the image is cut into chunks of GN_U * R rows; each thread owns ONE 8-channel vector column and issues
// its row loads at once, so per-channel partial sums live in registers; one smem fold per chunk writes per-(chunk,
// group) {sum, sumsq} partials.  Default = one cooperative launch (gn_fused_kernel: partials | grid barrier | fold in
// double + streaming y = silu(a*x + b)); gn_stats_kernel + gn_apply_kernel run the same chunks as two launches.
// The input may be the channel concat of two tensors (x2 != nullptr): columns < C1/8 come from x1.
#include "common.cuh"

namespace anysd {

constexpr int GN_MAX_SPLITS = 64;
constexpr int GN_U = 8;            // 16-byte loads a thread keeps in flight

// x * sigmoid(x) with two MUFU ops (ex2, rcp) instead of an IEEE division: ~1e-7 relative, far below the fp16 store
// (inline PTX: __fdividef / __expf expand to ~11 instructions with range checks; this is FMUL, MUFU.EX2, FADD, MUFU.RCP, FMUL)
__device__ __forceinline__ float silu_fast(float v) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * -1.4426950408889634f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return v * r;
}

struct GnGeom {
    int CV;    // 8-channel vectors per row (C/8)
    int CV1;   // vectors that come from x1
    int R;     // rows walked in parallel by one block
    int T;     // threads per block = CV * R
};

static GnGeom gn_geom(int C1, int C2) {
    GnGeom g;
    g.CV = (C1 + C2) / 8;
    g.CV1 = C1 / 8;
    g.R = 512 / g.CV;
    if (g.R < 1) g.R = 1;
    g.T = g.CV * g.R;
    return g;
}

// partial {sum, sumsq} of logical chunk (n, s) -> partials[((n * S + s) * G + g) * 2]; all threads of the block take part
__device__ __forceinline__ void gn_stats_block(const uint4* __restrict__ x1, const uint4* __restrict__ x2, int CV, int CV1, int R,
                                               int HW, int rows_per_block, int S, int G, int cpg, int n, int s,
                                               float* __restrict__ partials, float* sm) {
    const int cv = threadIdx.x % CV, r = threadIdx.x / CV;
    const int C = CV * 8;
    const int row0 = s * rows_per_block;
    int row1 = row0 + rows_per_block;
    if (row1 > HW) row1 = HW;
    const bool first = cv < CV1;
    const int CV2 = CV - CV1;
    const uint4* base = first ? (x1 + (size_t)n * HW * CV1 + cv) : (x2 + (size_t)n * HW * CV2 + (cv - CV1));
    const int stride = first ? CV1 : CV2;

    float sum[8], sq[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) sum[j] = sq[j] = 0.f;
    // GN_U independent 16-byte loads in flight per thread, predicated: a chunk is normally ONE such batch (the host
    // sizes rows_per_block = GN_U * R), so a thread never chains dependent memory latencies.
    for (int row = row0 + r; row < row1; row += GN_U * R) {
        uint4 v[GN_U];
#pragma unroll
        for (int u = 0; u < GN_U; ++u) {
            const int rr = row + u * R;
            v[u] = rr < row1 ? __ldg(base + (size_t)rr * stride) : make_uint4(0u, 0u, 0u, 0u);
        }
#pragma unroll
        for (int u = 0; u < GN_U; ++u) {
            float f[8];
            unpack8(v[u], f);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                sum[j] += f[j];
                sq[j] += f[j] * f[j];
            }
        }
    }
    float* ssum = sm;
    float* ssq = sm + (size_t)R * C;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        ssum[(size_t)r * C + j * CV + cv] = sum[j];   // [r][j][cv]: conflict-free
        ssq[(size_t)r * C + j * CV + cv] = sq[j];
    }
    __syncthreads();
    // fold 1: one thread per channel slot sums the R row-lanes (R loads), result back into row-lane 0
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
        float a = 0.f, b = 0.f;
        for (int rr = 0; rr < R; ++rr) {
            a += ssum[(size_t)rr * C + i];
            b += ssq[(size_t)rr * C + i];
        }
        ssum[i] = a;
        ssq[i] = b;
    }
    __syncthreads();
    // fold 2: thread g < G sums its group's cpg channels
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
        float a = 0.f, b = 0.f;
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
            const int idx = (c & 7) * CV + (c >> 3);
            a += ssum[idx];
            b += ssq[idx];
        }
        float* p = partials + (((size_t)n * S + s) * G + g) * 2;
        p[0] = a;
        p[1] = b;
    }
}

// The S partials of image n folded in a fixed order, in double: deterministic, independent of which block runs it.
__device__ __forceinline__ void gn_fold(const float* __restrict__ partials, int n, int S, int G, int g, int HW, int cpg, float eps,
                                        float& mean_out, float& rstd_out) {
    double a = 0.0, b = 0.0;
    const float* p = partials + ((size_t)n * S * G + g) * 2;
    for (int i = 0; i < S; ++i) {
        a += (double)__ldcg(p + (size_t)i * G * 2);
        b += (double)__ldcg(p + (size_t)i * G * 2 + 1);
    }
    const double cnt = (double)HW * cpg;
    const double mean = a / cnt;
    double var = b / cnt - mean * mean;
    if (var < 0.0) var = 0.0;
    mean_out = (float)mean;
    rstd_out = (float)(1.0 / sqrt(var + (double)eps));
}

__global__ void __launch_bounds__(512, 2) gn_stats_kernel(const uint4* __restrict__ x1, const uint4* __restrict__ x2, int CV, int CV1, int R,
                                int HW, int rows_per_block, int G, int cpg, float eps, float* __restrict__ partials,
                                float* __restrict__ meanrstd, unsigned int* __restrict__ counters) {
    extern __shared__ float sm[];  // [R][CV*8] sums, then [R][CV*8] squares
    const int n = blockIdx.y;
    gn_stats_block(x1, x2, CV, CV1, R, HW, rows_per_block, gridDim.x, G, cpg, n, blockIdx.x, partials, sm);
    // The last block of image n to finish folds the S partials into mean / rstd, so the apply pass starts streaming
    // at once.
    __shared__ bool is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int done = atomicAdd(&counters[n], 1u);
        is_last = (done == gridDim.x - 1);
        if (is_last) counters[n] = 0;                 // re-arm for the next launch (stream-ordered)
    }
    __syncthreads();
    if (is_last) {
        __threadfence();
        for (int g = threadIdx.x; g < G; g += blockDim.x) {
            float m, rs;
            gn_fold(partials, n, gridDim.x, G, g, HW, cpg, eps, m, rs);
            meanrstd[((size_t)n * G + g) * 2] = m;
            meanrstd[((size_t)n * G + g) * 2 + 1] = rs;
        }
    }
}

// y = [silu](x * a + b) over the rows of logical chunk (n, s); s_mean / s_rstd: this image's statistics in smem
// COEF_SMEM: per-channel a = rstd*gamma, b = beta - mean*a were staged in shared memory (coef[0..C) = a, coef[C..2C) = b)
// by the caller and are read per use (frees 16 registers for loads in flight); otherwise they are built here.
template <bool COEF_SMEM, bool PIPE = false, int U = GN_U>
__device__ __forceinline__ void gn_apply_block(const uint4* __restrict__ x1, const uint4* __restrict__ x2, int CV, int CV1, int R,
                                               int HW, int rows_per_block, int cpg, int n, int s, const float* s_mean,
                                               const float* s_rstd, const float* __restrict__ gamma,
                                               const float* __restrict__ beta, int fuse_silu, uint4* __restrict__ y,
                                               const float* coef) {
    const int cv = threadIdx.x % CV, r = threadIdx.x / CV;
    float ca[8], cb[8];
    if (!COEF_SMEM) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = cv * 8 + j;
            const int g = c / cpg;
            const float a = s_rstd[g] * gamma[c];
            ca[j] = a;
            cb[j] = beta[c] - s_mean[g] * a;
        }
    }
    const int row0 = s * rows_per_block;
    int row1 = row0 + rows_per_block;
    if (row1 > HW) row1 = HW;
    const bool first = cv < CV1;
    const int CV2 = CV - CV1;
    const uint4* base = first ? (x1 + (size_t)n * HW * CV1 + cv) : (x2 + (size_t)n * HW * CV2 + (cv - CV1));
    const int stride = first ? CV1 : CV2;
    uint4* out = y + (size_t)n * HW * CV + cv;
    // Software pipeline over batches of GN_U rows per thread: the loads of batch k+1 are in flight while batch k goes
    // through the FMA / MUFU / pack / store stretch, so a CTA never sits with an empty memory pipe (a chunk of one batch --
    // the statistics chunking -- degenerates to load, compute, store).
    const int step = U * R;
    auto load = [&](uint4 (&v)[U], int row) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int rr = row + u * R;
            v[u] = rr < row1 ? __ldg(base + (size_t)rr * stride) : make_uint4(0u, 0u, 0u, 0u);
        }
    };
    auto process = [&](uint4 (&v)[U], int row) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int rr = row + u * R;
            float f[8];
            unpack8(v[u], f);
            if (COEF_SMEM) {
                const float4* a4 = reinterpret_cast<const float4*>(coef + cv * 8);
                const float4* b4 = reinterpret_cast<const float4*>(coef + CV * 8 + cv * 8);
                const float4 a0 = a4[0], a1 = a4[1], b0 = b4[0], b1 = b4[1];
                ca[0] = a0.x; ca[1] = a0.y; ca[2] = a0.z; ca[3] = a0.w; ca[4] = a1.x; ca[5] = a1.y; ca[6] = a1.z; ca[7] = a1.w;
                cb[0] = b0.x; cb[1] = b0.y; cb[2] = b0.z; cb[3] = b0.w; cb[4] = b1.x; cb[5] = b1.y; cb[6] = b1.z; cb[7] = b1.w;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float t = fmaf(f[j], ca[j], cb[j]);
                f[j] = fuse_silu ? silu_fast(t) : t;
            }
            if (rr < row1) out[(size_t)rr * CV] = pack8(f);
        }
    };
    if (PIPE) {
        uint4 va[U], vb[U];
        int row = row0 + r;
        load(va, row);
        for (; row < row1; row += 2 * step) {
            load(vb, row + step);
            process(va, row);
            load(va, row + 2 * step);
            process(vb, row + step);
        }
    } else {
        uint4 va[U];
        for (int row = row0 + r; row < row1; row += step) {
            load(va, row);
            process(va, row);
        }
    }
}

__global__ void __launch_bounds__(512, 2) gn_apply_kernel(const uint4* __restrict__ x1, const uint4* __restrict__ x2, int CV, int CV1, int R,
                                int HW, int rows_per_block, int G, int cpg, const float* __restrict__ meanrstd,
                                const float* __restrict__ gamma, const float* __restrict__ beta, int fuse_silu,
                                uint4* __restrict__ y) {
    __shared__ float s_mean[64], s_rstd[64];
    const int n = blockIdx.y;
    if (threadIdx.x < G) {
        s_mean[threadIdx.x] = meanrstd[((size_t)n * G + threadIdx.x) * 2];
        s_rstd[threadIdx.x] = meanrstd[((size_t)n * G + threadIdx.x) * 2 + 1];
    }
    __syncthreads();
    gn_apply_block<false>(x1, x2, CV, CV1, R, HW, rows_per_block, cpg, n, blockIdx.x, s_mean, s_rstd, gamma, beta, fuse_silu, y, nullptr);
}

// ---- statistics that arrive from the producing contraction's epilogue (anysd_gemm_params::stats) ----------------------
// stats1 [*, S, C1, 2] (+ stats2 [*, S, C2, 2] for a channel concat): {sum, sum of squares} per (image, 32-row slab, channel).
// One CTA per (group, image): the S * cpg cells of the group are dealt to the threads in a fixed order, accumulated in double
// and combined by a fixed smem tree -- deterministic and independent of the batch, like gn_fold.
// Apply pass of the epilogue-statistics path: chunks of several row batches (the pass is elementwise, so its chunking is
// free of the statistics' order constraints), per-channel a = rstd * gamma, b = beta - mean * a staged in shared memory.
__global__ void __launch_bounds__(512, 2) gn_apply_coef_kernel(const uint4* __restrict__ x, int CV, int R, int HW, int rows_per_block, int G,
                                                               int cpg, const float* __restrict__ meanrstd, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, int fuse_silu, uint4* __restrict__ y) {
    extern __shared__ float coef[];                      // a[0..C) | b[0..C)
    const int n = blockIdx.y, C = CV * 8;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int g = c / cpg;
        const float a = meanrstd[((size_t)n * G + g) * 2 + 1] * gamma[c];
        coef[c] = a;
        coef[C + c] = beta[c] - meanrstd[((size_t)n * G + g) * 2] * a;
    }
    __syncthreads();
    gn_apply_block<true, true, 4>(x, nullptr, CV, CV, R, HW, rows_per_block, cpg, n, blockIdx.x, nullptr, nullptr, gamma, beta, fuse_silu, y, coef);
}

__global__ void __launch_bounds__(128) gn_finalize_kernel(const float2* __restrict__ stats1, int C1, const float2* __restrict__ stats2, int C2,
                                                          int S, int HW, int cpg, float eps, float* __restrict__ meanrstd) {
    const int g = blockIdx.x, n = blockIdx.y, G = gridDim.x;
    double a = 0.0, b = 0.0;
    // thread t takes slabs t, t + 128, ...; the group's cpg channels of one slab are adjacent (cpg * 8 bytes): the loads of a
    // slab are issued together (independent), the additions follow in channel order -- a fixed order per thread
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        for (int c0 = 0; c0 < cpg; c0 += 8) {
            float2 v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = g * cpg + c0 + j;
                v[j] = make_float2(0.f, 0.f);
                if (c0 + j < cpg)
                    v[j] = c < C1 ? __ldg(stats1 + ((size_t)n * S + s) * C1 + c) : __ldg(stats2 + ((size_t)n * S + s) * C2 + (c - C1));
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                a += (double)v[j].x;
                b += (double)v[j].y;
            }
        }
    }
    __shared__ double ra[128], rb[128];
    ra[threadIdx.x] = a;
    rb[threadIdx.x] = b;
    __syncthreads();
    for (int o = 64; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) {
            ra[threadIdx.x] += ra[threadIdx.x + o];
            rb[threadIdx.x] += rb[threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double cnt = (double)HW * cpg;
        const double mean = ra[0] / cnt;
        double var = rb[0] / cnt - mean * mean;
        if (var < 0.0) var = 0.0;
        meanrstd[((size_t)n * G + g) * 2] = (float)mean;
        meanrstd[((size_t)n * G + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
    }
}

// One launch instead of two (cooperative: every CTA resident).  The N*S logical chunks -- the SAME chunks, thread
// mapping and fold order as the two-kernel path, so every output bit is identical and independent of the batch size
// and of the physical grid -- are dealt round-robin to the CTAs: phase 1 writes chunk partials, a sense-reversing
// grid barrier (bar[0] arrivals, bar[1] generation) separates the phases, phase 2 folds the image statistics and
// streams y; its reads of x hit L2 (the whole activation was read moments ago: <= 63 MB at the bench shapes).
struct GnFusedArgs {
    const uint4* x1; const uint4* x2;
    int CV, CV1, R, HW, rows_per_block, S, N, G, cpg;
    float eps;
    float* partials;
    const float* gamma; const float* beta;
    int fuse_silu;
    uint4* y;
    unsigned int* bar;
};

__global__ void __launch_bounds__(512, 2) gn_fused_kernel(const GnFusedArgs a) {
    extern __shared__ float sm[];
    __shared__ float s_mean[64], s_rstd[64];
    const int chunks = a.N * a.S;
    for (int ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
        gn_stats_block(a.x1, a.x2, a.CV, a.CV1, a.R, a.HW, a.rows_per_block, a.S, a.G, a.cpg, ch / a.S, ch % a.S, a.partials, sm);
        __syncthreads();                                  // sm is reused by the next chunk
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        volatile unsigned int* gen = a.bar + 1;
        const unsigned int g0 = *gen;
        __threadfence();
        if (atomicAdd(a.bar, 1u) == gridDim.x - 1) {
            a.bar[0] = 0;                                 // re-arm (the next launch is stream-ordered behind this one)
            __threadfence();
            atomicAdd(a.bar + 1, 1u);
        } else {
            while (*gen == g0) __nanosleep(32);
        }
        __threadfence();
    }
    __syncthreads();
    int cur_n = -1;
    for (int ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
        const int n = ch / a.S;
        if (n != cur_n) {
            __syncthreads();                              // previous chunk's readers of s_mean / s_rstd are done
            if (threadIdx.x < a.G) gn_fold(a.partials, n, a.S, a.G, threadIdx.x, a.HW, a.cpg, a.eps, s_mean[threadIdx.x], s_rstd[threadIdx.x]);
            __syncthreads();
            const int C = a.CV * 8;
            for (int c = threadIdx.x; c < C; c += blockDim.x) {      // sm (the stats scratch) now holds a[0..C) | b[0..C)
                const int g = c / a.cpg;
                const float ca = s_rstd[g] * a.gamma[c];
                sm[c] = ca;
                sm[C + c] = a.beta[c] - s_mean[g] * ca;
            }
            __syncthreads();
            cur_n = n;
        }
        gn_apply_block<true>(a.x1, a.x2, a.CV, a.CV1, a.R, a.HW, a.rows_per_block, a.cpg, n, ch % a.S, s_mean, s_rstd, a.gamma, a.beta,
                             a.fuse_silu, a.y, sm);
    }
}

// ---- GroupNorm(+SiLU), register-resident (small maps: one read, one write, one plain launch) -------------------------------
// One CTA per (image, span of `gpc` whole groups that is a whole number of 16-byte channel vectors, VC of them); a CTA is
// VC x RL threads (RL = 32 or 64 row lanes), thread (rl, vl) owns the vector column vl of rows rl, rl + RL, ... -- at most V of
// them (V <= 8: maps of up to 8 RL pixels), all loaded up front and KEPT IN REGISTERS until the store.  Moments are exact
// two-pass sums (mean, then centred squares: no E[x^2] - mean^2 cancellation) folded in a fixed order: thread -> 8 row lanes ->
// group (one warp, lane-strided + shuffle tree).  The decomposition is a function of (C, HW, G) only, so every output bit is
// independent of the batch.  Against the cooperative statistics + apply kernel: no second read of x, no grid barrier.
// A cluster version of the same kernel (up to 16 CTAs per span splitting the rows, partials exchanged through distributed shared
// memory) was built for the large maps and was slower than the epilogue-statistics path -- two cluster barriers + the remote
// reads are latency that two resident CTAs per SM cannot hide -- so it is not kept.
struct GnResArgs {
    const uint4* x1; const uint4* x2; uint4* y;
    const float* gamma; const float* beta;
    int CV1, CV2, HW, VC, RL, cpg, gpc, fuse_silu;
    float eps, inv_cnt;
};

template <int V>
__global__ void __maxnreg__(V <= 4 ? 64 : 96) gn_res_kernel(const GnResArgs a) {
    extern __shared__ __align__(16) float gnr_sm[];
    const int VC = a.VC, RL = a.RL, CW = VC * 8, P = RL / 8, gpc = a.gpc, cpg = a.cpg;
    float* part = gnr_sm;                       // [RL][CW] per-thread channel partials
    float* part2 = part + RL * CW;              // [P][CW]  after the fold over 8 row lanes
    float* chm = part2 + P * CW;                // [CW] per channel: mean of its group
    float* cha = chm + CW;                      // [CW] rstd * gamma
    float* chb = cha + CW;                      // [CW] beta - mean * rstd * gamma
    float* gsum = chb + CW;                     // [gpc] group sums of the current pass
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const int vl = tid % VC, rl = tid / VC;
    const int n = blockIdx.y;
    const int gv = blockIdx.x * VC + vl;                         // global vector column (a vector never straddles x1 | x2)
    const bool first = gv < a.CV1;
    const uint4* src = first ? a.x1 + (size_t)n * a.HW * a.CV1 + gv : a.x2 + (size_t)n * a.HW * a.CV2 + (gv - a.CV1);
    const int xs = first ? a.CV1 : a.CV2, CV = a.CV1 + a.CV2;
    uint4 d[V];
#pragma unroll
    for (int k = 0; k < V; ++k) {
        const int r = rl + k * RL;
        d[k] = r < a.HW ? __ldg(src + r * xs) : make_uint4(0u, 0u, 0u, 0u);
    }

    // per-thread 8-channel partials -> per-group sums in gsum[g]
    auto fold = [&](const float* v8) {
        float4* pw = reinterpret_cast<float4*>(part + rl * CW + vl * 8);
        pw[0] = make_float4(v8[0], v8[1], v8[2], v8[3]);
        pw[1] = make_float4(v8[4], v8[5], v8[6], v8[7]);
        __syncthreads();
        {
            const int c = tid % CW, p = tid / CW;               // blockDim = VC * RL = CW * P threads exactly
            float t = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) t += part[(p * 8 + i) * CW + c];
            part2[p * CW + c] = t;
        }
        __syncthreads();
        for (int g = warp; g < gpc; g += nwarps) {
            float t = 0.f;
            for (int i = lane; i < cpg * P; i += 32) t += part2[(i / cpg) * CW + g * cpg + (i % cpg)];
            t = warp_sum(t);
            if (lane == 0) gsum[g] = t;
        }
        __syncthreads();
    };

    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) {
        float f[8];
        unpack8(d[k], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];             // rows beyond HW hold zeros
    }
    fold(acc);
    if (tid < CW) chm[tid] = gsum[tid / cpg] * a.inv_cnt;
    __syncthreads();
    {
        const float4 m0 = *reinterpret_cast<const float4*>(chm + vl * 8), m1 = *reinterpret_cast<const float4*>(chm + vl * 8 + 4);
        const float m8[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
        for (int k = 0; k < V; ++k) {
            if (rl + k * RL < a.HW) {
                float f[8];
                unpack8(d[k], f);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float c = f[j] - m8[j];
                    acc[j] = fmaf(c, c, acc[j]);
                }
            }
        }
    }
    fold(acc);
    if (tid < CW) {
        const float rstd = rsqrtf(gsum[tid / cpg] * a.inv_cnt + a.eps);
        const float ga = __ldg(a.gamma + blockIdx.x * CW + tid) * rstd;
        cha[tid] = ga;
        chb[tid] = __ldg(a.beta + blockIdx.x * CW + tid) - chm[tid] * ga;
    }
    __syncthreads();
    {
        const float4 a0 = *reinterpret_cast<const float4*>(cha + vl * 8), a1 = *reinterpret_cast<const float4*>(cha + vl * 8 + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(chb + vl * 8), b1 = *reinterpret_cast<const float4*>(chb + vl * 8 + 4);
        const float a8[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float b8[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        uint4* dst = a.y + (size_t)n * a.HW * CV + gv;
#pragma unroll
        for (int k = 0; k < V; ++k) {
            const int r = rl + k * RL;
            if (r < a.HW) {
                float f[8], o[8];
                unpack8(d[k], f);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float z = fmaf(f[j], a8[j], b8[j]);
                    o[j] = a.fuse_silu ? silu_fast(z) : z;
                }
                dst[r * CV] = pack8(o);
            }
        }
    }
}

// Geometry of the register-resident kernel for (C1 + C2 channels, HW pixels, G groups), or false when it does not apply.
struct GnResPlan { int VC, RL, gpc, V; };
static bool gn_res_plan(int C1, int C2, int HW, int G, GnResPlan* pl) {
    static const char* env = getenv("ANYSD_GN_RES");
    if (env && env[0] == '0') return false;
    const int C = C1 + C2;
    if (G <= 0 || C % G != 0 || C1 % 8 != 0 || C2 % 8 != 0 || HW <= 0) return false;
    const int cpg = C / G;
    int gpc = 1;
    while ((gpc * cpg) % 8 != 0) ++gpc;
    const int VC = gpc * cpg / 8;
    if (G % gpc != 0 || VC > 16) return false;
    const int RL = VC * 64 <= 512 ? 64 : 32;
    const int v = cdiv(HW, RL);
    if (v > 8) return false;
    int V = 1;
    while (V < v) V <<= 1;
    pl->VC = VC; pl->RL = RL; pl->gpc = gpc; pl->V = V;
    return true;
}

static int launch_gn_res(const GnResPlan& pl, const void* x1, int C1, const void* x2, int C2, const float* gamma, const float* beta, void* y,
                         int N, int HW, int G, float eps, int fuse_silu, cudaStream_t st) {
    GnResArgs a;
    a.x1 = (const uint4*)x1; a.x2 = (const uint4*)x2; a.y = (uint4*)y;
    a.gamma = gamma; a.beta = beta;
    a.CV1 = C1 / 8; a.CV2 = C2 / 8; a.HW = HW; a.VC = pl.VC; a.RL = pl.RL; a.cpg = (C1 + C2) / G; a.gpc = pl.gpc;
    a.fuse_silu = fuse_silu; a.eps = eps;
    a.inv_cnt = 1.0f / ((float)HW * (float)a.cpg);
    const int CW = pl.VC * 8;
    const dim3 grid((unsigned)(G / pl.gpc), (unsigned)N);
    const unsigned T = (unsigned)(pl.VC * pl.RL);
    const size_t smem = (size_t)(pl.RL * CW + pl.RL / 8 * CW + 3 * CW + pl.gpc) * sizeof(float);
    switch (pl.V) {
        case 1: gn_res_kernel<1><<<grid, T, smem, st>>>(a); break;
        case 2: gn_res_kernel<2><<<grid, T, smem, st>>>(a); break;
        case 4: gn_res_kernel<4><<<grid, T, smem, st>>>(a); break;
        default: gn_res_kernel<8><<<grid, T, smem, st>>>(a); break;
    }
    return check_launch("groupnorm (resident)");
}

// ---- LayerNorm: LPR lanes per token row (8 / 16 / 32), VPL 16-byte vectors per lane held in registers ---------
// C = 320 / 640 / 1280 map to LPR = 8 / 16 / 32 with exactly 5 vectors per lane: a warp then normalises
// 4 / 2 / 1 rows at once with 5 independent 16-byte loads in flight per lane (the one-warp-per-row version left
// 24 of 32 lanes with a single load at C = 320).  Two-pass exact variance from registers.
template <int LPR, int VPL>
__global__ void layernorm_kernel(const uint4* __restrict__ x, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, uint4* __restrict__ y, long long M, int CV, float eps) {
    constexpr int RPW = 32 / LPR;                       // rows per warp
    const int lane = threadIdx.x & 31;
    const int sub = lane / LPR, l = lane % LPR;
    const long long row = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + sub;
    const bool row_ok = row < M;
    const uint4* xr = x + (row_ok ? row : 0) * CV;
    float f[VPL][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        const int v = l + i * LPR;
        if (v < CV) {
            uint4 u = __ldg(xr + v);
            unpack8(u, f[i]);
#pragma unroll
            for (int j = 0; j < 8; ++j) s += f[i][j];
        }
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float inv_c = 1.0f / (float)(CV * 8);
    const float mean = s * inv_c;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        const int v = l + i * LPR;
        if (v < CV) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float d = f[i][j] - mean;
                q += d * d;
            }
        }
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q * inv_c + eps);
    if (!row_ok) return;
    uint4* yr = y + row * CV;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        const int v = l + i * LPR;
        if (v < CV) {
            const float4* g4 = reinterpret_cast<const float4*>(gamma + v * 8);
            const float4* b4 = reinterpret_cast<const float4*>(beta + v * 8);
            float4 g0 = __ldg(g4), g1 = __ldg(g4 + 1), b0 = __ldg(b4), b1 = __ldg(b4 + 1);
            float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
            float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = (f[i][j] - mean) * rstd * gg[j] + bb[j];
            yr[v] = pack8(o);
        }
    }
}

}  // namespace anysd

using namespace anysd;

extern "C" {

int anysd_groupnorm_resident(int C1, int C2, int HW, int G) {
    GnResPlan pl;
    return gn_res_plan(C1, C2 < 0 ? 0 : C2, HW, G, &pl) ? 1 : 0;
}

size_t anysd_groupnorm_workspace_bytes(int N, int G, int C) {
    (void)C;
    if (N <= 0 || G <= 0) return 0;
    // partials [N, 64, G, 2] | mean/rstd [N, G, 2] | per-image completion counters [N] (must be zero on first use:
    // the caller zero-fills the workspace once; every launch re-arms them)
    // | grid barrier of the one-launch path {arrivals, generation}
    return (size_t)N * GN_MAX_SPLITS * G * 2 * sizeof(float) + (size_t)N * G * 2 * sizeof(float) + (size_t)N * sizeof(unsigned int) +
           2 * sizeof(unsigned int);
}

int anysd_groupnorm_nhwc_f16(const void* x1, int C1, const void* x2, int C2, const float* gamma, const float* beta,
                             void* y, int N, int HW, int G, float eps, int fuse_silu, void* workspace,
                             size_t workspace_bytes, anysd_stream_t stream) {
    ANYSD_REQUIRE(x1 && gamma && beta && y && workspace, ANYSD_EINVAL, "groupnorm: null pointer");
    if (x2 == nullptr) C2 = 0;
    const int C = C1 + C2;
    ANYSD_REQUIRE(N > 0 && HW > 0 && G > 0 && G <= 64 && C1 > 0 && C2 >= 0, ANYSD_EINVAL, "groupnorm: bad shape");
    ANYSD_REQUIRE(C % G == 0 && C1 % 8 == 0 && C2 % 8 == 0, ANYSD_EINVAL,
                  "groupnorm: C=%d must divide into G=%d groups and both sources must be multiples of 8 channels", C, G);
    ANYSD_REQUIRE(C / 8 <= 1024, ANYSD_EINVAL, "groupnorm: C=%d too large", C);
    ANYSD_REQUIRE(workspace_bytes >= anysd_groupnorm_workspace_bytes(N, G, C), ANYSD_EINVAL,
                  "groupnorm: workspace too small (%zu bytes)", workspace_bytes);
    const int cpg = C / G;
    {
        // geometry-only decision (the same kernel whatever the batch): the register-resident kernel wherever it applies
        GnResPlan pl;
        if (gn_res_plan(C1, C2, HW, G, &pl))
            return launch_gn_res(pl, x1, C1, x2, C2, gamma, beta, y, N, HW, G, eps, fuse_silu, (cudaStream_t)stream);
    }
    const GnGeom g = gn_geom(C1, C2);
    // The spatial split depends on the image geometry only (never on N): the summation order, and hence
    // every output bit, is independent of how many samples share the batch.  >= 8 row-steps per block.
    // A chunk is one batch of GN_U row-steps per thread (more only when that would exceed GN_MAX_SPLITS chunks).
    const int batch = GN_U * g.R;
    const int rpb = batch * cdiv(HW, (long long)batch * GN_MAX_SPLITS);
    const int S = cdiv(HW, rpb);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = (size_t)2 * g.R * C * sizeof(float);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(gn_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        ANYSD_REQUIRE(e == cudaSuccess, ANYSD_ECUDA, "groupnorm: smem opt-in failed: %s", cudaGetErrorString(e));
    }
    float* partials = (float*)workspace;
    float* meanrstd = partials + (size_t)N * GN_MAX_SPLITS * G * 2;
    unsigned int* counters = (unsigned int*)(meanrstd + (size_t)N * G * 2);
    // One cooperative launch when the device can hold a useful grid (ANYSD_GN_FUSED=0 forces the two-kernel path,
    // which produces the same bits).
    static const char* fused_env = getenv("ANYSD_GN_FUSED");
    if (!(fused_env && fused_env[0] == '0')) {
        static thread_local int occ_T = -1, occ_smem = -1, occ = 0, occ_dev = -1;
        int dev = 0;
        cudaGetDevice(&dev);
        if (occ_T != g.T || occ_smem != (int)smem || occ_dev != dev) {
            if (smem > 48 * 1024) cudaFuncSetAttribute(gn_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            occ = 0;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gn_fused_kernel, g.T, smem) != cudaSuccess) occ = 0;
            occ_T = g.T; occ_smem = (int)smem; occ_dev = dev;
        }
        long long P = (long long)occ * sm_count();
        if (P > (long long)N * S) P = (long long)N * S;
        if (P >= 1) {
            GnFusedArgs fa;
            fa.x1 = (const uint4*)x1; fa.x2 = (const uint4*)x2;
            fa.CV = g.CV; fa.CV1 = g.CV1; fa.R = g.R; fa.HW = HW; fa.rows_per_block = rpb; fa.S = S; fa.N = N; fa.G = G; fa.cpg = cpg;
            fa.eps = eps; fa.partials = partials; fa.gamma = gamma; fa.beta = beta; fa.fuse_silu = fuse_silu; fa.y = (uint4*)y;
            fa.bar = counters + N;
            void* kargs[] = {(void*)&fa};
            cudaError_t e = cudaLaunchCooperativeKernel((const void*)gn_fused_kernel, dim3((unsigned)P), dim3(g.T), kargs, smem, st);
            ANYSD_REQUIRE(e == cudaSuccess, ANYSD_ECUDA, "groupnorm (fused): launch failed: %s", cudaGetErrorString(e));
            return check_launch("groupnorm (fused)");
        }
    }
    gn_stats_kernel<<<dim3(S, N), g.T, smem, st>>>((const uint4*)x1, (const uint4*)x2, g.CV, g.CV1, g.R, HW, rpb, G, cpg, eps,
                                                   partials, meanrstd, counters);
    int rc = check_launch("groupnorm stats");
    if (rc) return rc;
    gn_apply_kernel<<<dim3(S, N), g.T, 0, st>>>((const uint4*)x1, (const uint4*)x2, g.CV, g.CV1, g.R, HW, rpb, G, cpg,
                                                meanrstd, gamma, beta, fuse_silu, (uint4*)y);
    return check_launch("groupnorm apply");
}

int anysd_groupnorm_apply_nhwc_f16(const void* x, int C, const float* stats1, int C1, const float* stats2, int S, const float* gamma,
                                   const float* beta, void* y, int N, int HW, int G, float eps, int fuse_silu, void* workspace,
                                   size_t workspace_bytes, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && stats1 && gamma && beta && y && workspace, ANYSD_EINVAL, "groupnorm_apply: null pointer");
    ANYSD_REQUIRE(N > 0 && HW > 0 && G > 0 && G <= 64 && C > 0 && C % G == 0 && C % 8 == 0 && C / 8 <= 1024, ANYSD_EINVAL,
                  "groupnorm_apply: bad shape N=%d HW=%d C=%d G=%d", N, HW, C, G);
    ANYSD_REQUIRE(C1 > 0 && C1 <= C && (C1 == C) == (stats2 == nullptr), ANYSD_EINVAL,
                  "groupnorm_apply: stats2 must be given exactly when the first source covers fewer than C channels");
    ANYSD_REQUIRE(S > 0 && S * 32 == HW, ANYSD_EINVAL, "groupnorm_apply: S=%d slabs of 32 rows must cover HW=%d", S, HW);
    ANYSD_REQUIRE(workspace_bytes >= anysd_groupnorm_workspace_bytes(N, G, C), ANYSD_EINVAL, "groupnorm_apply: workspace too small");
    const GnGeom g = gn_geom(C, 0);
    const int cpg = C / G;
    const int batch = 4 * g.R;                            // the apply kernel keeps 2 x 4 loads in flight per thread
    // chunk = up to 8 row batches (software-pipelined inside the CTA) while the grid still fills the machine twice over
    int nb = 8;
    while (nb > 1 && (long long)N * cdiv(HW, (long long)batch * nb) < 2LL * sm_count()) nb >>= 1;
    const int rpb = batch * nb;
    const int Sx = cdiv(HW, rpb);
    cudaStream_t st = (cudaStream_t)stream;
    float* meanrstd = (float*)workspace + (size_t)N * GN_MAX_SPLITS * G * 2;
    gn_finalize_kernel<<<dim3(G, N), 128, 0, st>>>((const float2*)stats1, C1, (const float2*)stats2, C - C1, S, HW, cpg, eps, meanrstd);
    int rc = check_launch("groupnorm finalize");
    if (rc) return rc;
    gn_apply_coef_kernel<<<dim3(Sx, N), g.T, (size_t)2 * C * sizeof(float), st>>>((const uint4*)x, g.CV, g.R, HW, rpb, G, cpg, meanrstd, gamma,
                                                                                  beta, fuse_silu, (uint4*)y);
    return check_launch("groupnorm apply");
}

int anysd_layernorm_f16(const void* x, const float* gamma, const float* beta, void* y, long long M, int C, float eps,
                        anysd_stream_t stream) {
    ANYSD_REQUIRE(x && gamma && beta && y && M > 0, ANYSD_EINVAL, "layernorm: bad args");
    ANYSD_REQUIRE(C > 0 && C % 8 == 0 && C / 8 <= 256, ANYSD_EINVAL, "layernorm: C=%d must be a multiple of 8 and <= 2048", C);
    const int CV = C / 8, warps = 8;
    cudaStream_t st = (cudaStream_t)stream;
    const uint4* xi = (const uint4*)x;
    uint4* yo = (uint4*)y;
#define ANYSD_LN(LPR, VPL)                                                                                     \
    layernorm_kernel<LPR, VPL><<<cdiv(M, (long long)warps * (32 / LPR)), warps * 32, 0, st>>>(xi, gamma, beta, yo, M, CV, eps)
    if (CV <= 8 * 5) {
        if (CV <= 8) ANYSD_LN(8, 1);
        else if (CV <= 16) ANYSD_LN(8, 2);
        else if (CV <= 24) ANYSD_LN(8, 3);
        else ANYSD_LN(8, 5);
    } else if (CV <= 16 * 5) {
        ANYSD_LN(16, 5);
    } else if (CV <= 32 * 5) {
        ANYSD_LN(32, 5);
    } else {
        ANYSD_LN(32, 8);
    }
#undef ANYSD_LN
    return check_launch("layernorm");
}
}
