// Persistent wgmma contraction: every dense contraction and 3x3 implicit-GEMM conv of the path whose layout
// constraints hold (anysd_gemm_f16 selects it; gemm_mma.cu takes the rest).
//
//   * one CTA per SM, static round-robin over work units (a 128 x BN output tile, or a K range of one with split-K),
//     n-tile fastest so that the CTAs running concurrently share A rows and weight tiles in L2;
//   * warp 0: TMA producer (2-D map for token matrices, 4-D NHWC map for conv patches: the conv's zero padding is the
//     map's out-of-bounds fill), a ring of STAGES x (16 KB A + BN x 128 B of B), 128-byte swizzle;
//   * warpgroups 1 and 2: 64 rows of the tile each, wgmma m64nBNk16 into register accumulators while the producer
//     already streams the next unit's operands; the epilogue works on the accumulator fragment in place: bias or
//     folded LayerNorm, time-embedding row add, SiLU / GELU / QuickGELU / GEGLU, residual, fp16 or fp32 stores,
//     GroupNorm statistics (per 32-row slab and channel) and LayerNorm row statistics (per 64-column slab) of the output.
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace anysd {

constexpr int G_BM = 128, G_BK = 64, G_THREADS = 384;
constexpr int G_A_BYTES = G_BM * G_BK * 2;          // 16 KB

template <int BN>
struct GCfg {
    static constexpr int STAGE_BYTES = G_A_BYTES + BN * G_BK * 2;
    static constexpr int RED_BYTES = 8 * BN * 8;    // per consumer warp: BN x {sum, sum of squares} (GroupNorm statistics)
    static constexpr int PAR_BYTES = 2 * 2 * BN * 4;  // per consumer warpgroup: the unit's bias and folded-LayerNorm column sums
    static constexpr int FIT = (212 * 1024 - RED_BYTES - PAR_BYTES) / STAGE_BYTES;
    static constexpr int STAGES = FIT > 6 ? 6 : FIT;
    static constexpr int SMEM = STAGES * STAGE_BYTES + RED_BYTES + PAR_BYTES + 1024 + 256;
};

struct GArgs {
    const float* bias;
    const float* rowadd;
    const __half* residual;
    void* out;
    int M, N, ldo, ldr, ld_rowadd, rows_per_batch;
    int act, out_f16;
    int num_kb, tiles_m, tiles_n, num_tiles;
    // conv geometry
    int Nimg, Ho, Wo;
    int BW, BH, NB, tiles_w, tiles_h;
    int kb_per_tap, stride;
    int pad_lo;              // zero rows / columns before the image: 1 (pad 1 on every side) or 0 (right / bottom padding only)
    // per-(32-row slab, channel) {sum, sum of squares} of the OUTPUT for the consumer's GroupNorm (anysd_gemm_params::stats)
    float* stats;
    int stats_hw, stats_spi, stats_nimg;     // rows per image, slabs per image (= hw / 32), image slots in the buffer
    // split-K (few output tiles, long K): a work unit = (tile, k-range); every unit dumps its raw fp32 accumulators, the
    // LAST unit of a tile to arrive (per 32-row slab, atomic counter) adds the partials in split order -- a fixed order, so
    // the result does not depend on the arrival order -- and runs the normal epilogue
    int splits, kb_per_split, num_units;
    float* sk_ws;                            // [tile][split][128 rows][bn] fp32
    unsigned int* sk_cnt;                    // [tile][4 slabs], zero between launches
    // LayerNorm around the contraction (anysd_gemm_params::row_stats / ln_stats, dense only):
    //   producer side: per-row {sum, sum of squares} of the OUTPUT per 64-column slab -> row_stats[slab][M] (float2)
    //   consumer side: A is the un-normalised x, W carries gamma, out = rstd_m (acc - mean_m colsum_n) + bias_n
    float* row_stats;
    const float* ln_stats;                   // [ln_slabs][M] float2 = the producer's row_stats
    const float* ln_colsum;                  // [N]
    int ln_slabs;
    float ln_eps, ln_inv_k;
};

__device__ __forceinline__ void g_bar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void g_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void g_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void g_wait(uint32_t bar, uint32_t parity) {
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
__device__ __forceinline__ void g_tma_2d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void g_tma_4d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
// named barrier of the two warps that share a 32-row slab (ids 1..4), of one consumer warpgroup (ids 5, 6)
__device__ __forceinline__ void g_pair_bar(int id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void g_wg_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// Exact (erf) GELU  x Phi(x)  in 11 instructions: Phi(x) = 1 / (1 + 2^(-x P(x^2))) with a cubic P fitted (minimax on the ABSOLUTE
// error of x Phi(x), x^2 clamped at 36 -- beyond it the logistic is saturated either way) to |err| < 1.2e-5 for all x: 1/40 of the
// fp16 spacing at unit magnitude, 1/7 of it at the minimum of GELU (-0.17).  Used by the fp16-output epilogues (the GEGLU
// contractions are issue-bound there); tests/test_gpu_ops.py::test_gelu_epilogue_accuracy pins the bound against torch's erf GELU.
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

struct TileCoord {
    int nt;              // column tile (first column nt * BN)
    int m0;              // dense: first row
    int tw, th, tn;      // conv: patch indices
};

template <bool CONV>
__device__ __forceinline__ TileCoord tile_coord(const GArgs& p, int tile) {
    TileCoord c;
    const int mt = tile / p.tiles_n;
    c.nt = tile - mt * p.tiles_n;
    c.m0 = mt * G_BM;
    c.tw = c.th = c.tn = 0;
    if (CONV) {
        c.tw = mt % p.tiles_w;
        c.th = (mt / p.tiles_w) % p.tiles_h;
        c.tn = mt / (p.tiles_w * p.tiles_h);
    }
    return c;
}

template <int BN, bool CONV>
__global__ void __launch_bounds__(G_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GArgs p) {
    using Cfg = GCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ unsigned char g_smem_raw[];
    const uint32_t raw = smem_u32(g_smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char* smem = g_smem_raw + (base - raw);
    float2* red = reinterpret_cast<float2*>(smem + STAGES * Cfg::STAGE_BYTES);
    float* par = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES + Cfg::RED_BYTES);
    const uint32_t bars = base + STAGES * Cfg::STAGE_BYTES + Cfg::RED_BYTES + Cfg::PAR_BYTES;
    volatile int* sk_flag = reinterpret_cast<volatile int*>(smem + STAGES * Cfg::STAGE_BYTES + Cfg::RED_BYTES + Cfg::PAR_BYTES + 16 * STAGES);
    auto full_bar = [&](int s) { return bars + 8u * s; };
    auto empty_bar = [&](int s) { return bars + 8u * (STAGES + s); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
        for (int s = 0; s < STAGES; ++s) {
            g_bar_init(full_bar(s), 1);
            g_bar_init(empty_bar(s), 8);      // one arrive per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 4) {
        // ===== producer warpgroup: one thread issues the TMA loads, running ahead across unit boundaries =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (warp == 0 && lane == 0) {
            uint32_t g = 0;
            for (int unit = blockIdx.x; unit < p.num_units; unit += gridDim.x) {
                const int tile = unit / p.splits;
                const int kb0 = (unit - tile * p.splits) * p.kb_per_split;
                const int kb1 = kb0 + p.kb_per_split < p.num_kb ? kb0 + p.kb_per_split : p.num_kb;
                const TileCoord c = tile_coord<CONV>(p, tile);
                const int n0 = c.nt * BN;
                for (int kb = kb0; kb < kb1; ++kb, ++g) {
                    const int s = g % STAGES;
                    g_wait(empty_bar(s), ((g / STAGES) & 1) ^ 1);
                    const uint32_t sa = base + s * Cfg::STAGE_BYTES, sb = sa + G_A_BYTES;
                    g_expect_tx(full_bar(s), Cfg::STAGE_BYTES);
                    if (CONV) {
                        const int tap = kb / p.kb_per_tap;
                        const int c0 = (kb - tap * p.kb_per_tap) * G_BK;
                        const int ky = tap / 3, kx = tap - ky * 3;
                        g_tma_4d(sa, &tmA, full_bar(s), c0, c.tw * p.BW * p.stride + kx - p.pad_lo,
                                 c.th * p.BH * p.stride + ky - p.pad_lo, c.tn * p.NB);
                    } else {
                        g_tma_2d(sa, &tmA, full_bar(s), kb * G_BK, c.m0);
                    }
                    g_tma_2d(sb, &tmB, full_bar(s), kb * G_BK, n0);
                }
            }
        }
        return;
    }

    // ===== consumer warpgroups =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int wg = (warp >> 2) - 1;                       // rows 64 wg .. 64 wg + 63 of the tile
    const int wq = warp & 3;                              // rows 16 wq .. of the warpgroup's 64
    const int ew = wg * 4 + wq;                           // consumer warp 0..7
    const int slab = ew >> 1;                             // 32-row slab of the tile (two warps)
    const int rl0 = wg * 64 + wq * 16 + (lane >> 2);      // this thread's tile rows: rl0, rl0 + 8
    const int q4 = lane & 3;
    const bool ln_in = !CONV && p.ln_stats != nullptr;
    const bool row_st = !CONV && p.row_stats != nullptr;
    // the unit's bias / column sums reach the epilogue through shared memory, loaded before the mainloop: read straight from
    // global memory inside the epilogue they would cost one L2 round trip per 8-column step
    float* s_bias = par + wg * 2 * BN;
    float* s_cs = s_bias + BN;
    const int wtid = threadIdx.x & 127;
    float acc[BN / 2];
    uint32_t g = 0;
    for (int unit = blockIdx.x; unit < p.num_units; unit += gridDim.x) {
        const int tile = unit / p.splits;
        const int kb0 = (unit - tile * p.splits) * p.kb_per_split;
        const int kb1 = kb0 + p.kb_per_split < p.num_kb ? kb0 + p.kb_per_split : p.num_kb;
        const TileCoord c = tile_coord<CONV>(p, tile);
        const int n0 = c.nt * BN;
        float pb[2], pc[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int j = wtid + 128 * r, col = n0 + j;
            pb[r] = (j < BN && col < p.N && p.bias != nullptr) ? __ldg(p.bias + col) : 0.f;
            pc[r] = (j < BN && col < p.N && ln_in) ? __ldg(p.ln_colsum + col) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        for (int kb = kb0; kb < kb1; ++kb, ++g) {
            const int s = g % STAGES;
            g_wait(full_bar(s), (g / STAGES) & 1);
            const uint32_t sa = base + s * Cfg::STAGE_BYTES + wg * 64 * 128, sb = base + s * Cfg::STAGE_BYTES + G_A_BYTES;
            wg_fence();
#pragma unroll
            for (int k = 0; k < G_BK / 16; ++k) Wgmma<BN>::ss(acc, wg_desc(sa + 32 * k, 16, 1024), wg_desc(sb + 32 * k, 16, 1024), 1);
            wg_commit();
            wg_wait<1>();                                 // the previous k-block's products have read their stage
            if (kb > kb0) {
                __syncwarp();
                if (lane == 0) g_arrive(empty_bar((g - 1) % STAGES));
            }
        }
        wg_wait<0>();
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) wg_fence_regs(acc[i]);
        if (kb1 > kb0) {
            __syncwarp();
            if (lane == 0) g_arrive(empty_bar((g - 1) % STAGES));
        }
        g_wg_bar(5 + wg);                                 // the previous unit's epilogue is done with s_bias / s_cs
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (wtid + 128 * r < BN) {
                s_bias[wtid + 128 * r] = pb[r];
                s_cs[wtid + 128 * r] = pc[r];
            }
        }
        g_wg_bar(5 + wg);

        // ---- split-K: dump this unit's raw accumulators; the slab's last unit adds all partials in split order ----
        if (p.splits > 1) {
            const int ks = unit - tile * p.splits;
            const float* wst = p.sk_ws + (size_t)tile * p.splits * (G_BM * BN);
            float* mine = p.sk_ws + ((size_t)tile * p.splits + ks) * (G_BM * BN);
#pragma unroll
            for (int i = 0; i < BN / 8; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    __stcg(reinterpret_cast<float2*>(mine + (size_t)(rl0 + 8 * h) * BN + 8 * i + 2 * q4),
                           make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]));
            __threadfence();                              // partials visible before the arrival is counted
            g_pair_bar(1 + slab);
            if ((ew & 1) == 0 && lane == 0) {
                unsigned int* cnt = p.sk_cnt + (size_t)tile * 4 + slab;
                const unsigned int old = atomicAdd(cnt, 1u);
                if (old == (unsigned)p.splits - 1) *cnt = 0;   // re-arm for the next launch (stream-ordered)
                sk_flag[slab] = old == (unsigned)p.splits - 1;
            }
            g_pair_bar(1 + slab);
            const bool last = sk_flag[slab] != 0;
            g_pair_bar(1 + slab);                         // the flag is read before the next unit may rewrite it
            if (!last) continue;                          // another unit finishes this slab
            __threadfence();                              // ... and the other units' partials visible to the adder
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            for (int k2 = 0; k2 < p.splits; ++k2) {
#pragma unroll
                for (int i = 0; i < BN / 8; ++i)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float2 f = __ldcg(reinterpret_cast<const float2*>(wst + (size_t)k2 * (G_BM * BN) +
                                                                                 (size_t)(rl0 + 8 * h) * BN + 8 * i + 2 * q4));
                        acc[4 * i + 2 * h] += f.x;
                        acc[4 * i + 2 * h + 1] += f.y;
                    }
            }
        }

        // ---- this thread's two output rows ----
        size_t pix[2];
        bool valid[2];
        int img[2];
        float ln_nm[2] = {0.f, 0.f}, ln_rs[2] = {1.f, 1.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = rl0 + 8 * h;
            if (CONV) {
                const int x = r % p.BW, y = (r / p.BW) % p.BH, n = r / (p.BW * p.BH);
                const int X = c.tw * p.BW + x, Y = c.th * p.BH + y, I = c.tn * p.NB + n;
                valid[h] = X < p.Wo && Y < p.Ho && I < p.Nimg;
                pix[h] = ((size_t)I * p.Ho + Y) * p.Wo + X;
                img[h] = I < p.Nimg ? I : p.Nimg - 1;
            } else {
                const int m = c.m0 + r;
                valid[h] = m < p.M;
                pix[h] = (size_t)m;
                img[h] = (m < p.M ? m : p.M - 1) / p.rows_per_batch;
                if (ln_in) {                              // row moments folded slab by slab in index order, combined in double
                    const float2* sp2 = reinterpret_cast<const float2*>(p.ln_stats) + (m < p.M ? m : p.M - 1);
                    float s1 = 0.f, s2 = 0.f;
                    for (int sl = 0; sl < p.ln_slabs; ++sl) {
                        const float2 f = __ldg(sp2 + (size_t)sl * p.M);
                        s1 += f.x;
                        s2 += f.y;
                    }
                    const double mean = (double)s1 * (double)p.ln_inv_k;
                    double var = (double)s2 * (double)p.ln_inv_k - mean * mean;
                    if (var < 0.0) var = 0.0;
                    ln_nm[h] = -(float)mean;
                    ln_rs[h] = rsqrtf((float)var + p.ln_eps);
                }
            }
        }
        auto store2 = [&](int h, int ocol, float a, float b) {      // GEGLU outputs (residual read here)
            if (valid[h]) {
                if (p.residual != nullptr) {
                    const float2 r = __half22float2(*reinterpret_cast<const __half2*>(p.residual + pix[h] * p.ldr + ocol));
                    a += r.x;
                    b += r.y;
                }
                if (p.out_f16) *reinterpret_cast<__half2*>((__half*)p.out + pix[h] * p.ldo + ocol) = __floats2half2_rn(a, b);
                else *reinterpret_cast<float2*>((float*)p.out + pix[h] * p.ldo + ocol) = make_float2(a, b);
            }
        };

        float rs1[2] = {0.f, 0.f}, rs2[2] = {0.f, 0.f};
        // The column steps run as a rolled loop over chunks of CH: unrolled over all BN / 8 steps, every feature path of the
        // epilogue would be replicated per step (tens of thousands of instructions that miss the instruction cache on every
        // unit).  The chunk's accumulators are selected with static indices so that they stay in registers.
        constexpr int CH = 4;
        constexpr int UNROLL = BN <= 64 ? BN / 8 / CH : 1;   // (BN = 64: two chunks, unrolled -- rolled, ptxas serialises the wgmma)
#pragma unroll UNROLL
        for (int i0 = 0; i0 < BN / 8; i0 += CH) {
            if (n0 + 8 * i0 >= p.N) break;                // N % 8 == 0: warp-uniform
            float a[CH][4];
#pragma unroll
            for (int u = 0; u < CH; ++u)
#pragma unroll
                for (int e = 0; e < 4; ++e) a[u][e] = acc[4 * u + e];
#pragma unroll
            for (int k = CH; k < BN / 8; k += CH)         // selects, not branches: no divergent accumulator access
#pragma unroll
                for (int u = 0; u < CH; ++u)
#pragma unroll
                    for (int e = 0; e < 4; ++e) a[u][e] = k == i0 ? acc[4 * (k + u) + e] : a[u][e];
            float2 ra[CH][2];                             // row adds and residuals of the chunk, in flight at once
            __half2 rr[CH][2];
#pragma unroll
            for (int u = 0; u < CH; ++u) {
                const int cw = n0 + 8 * (i0 + u) + 2 * q4;
                const bool in = cw < p.N;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    ra[u][h] = (in && p.rowadd != nullptr)
                                   ? __ldg(reinterpret_cast<const float2*>(p.rowadd + (size_t)img[h] * p.ld_rowadd + cw))
                                   : make_float2(0.f, 0.f);
                    rr[u][h] = (in && valid[h] && p.residual != nullptr && p.act != 2)
                                   ? *reinterpret_cast<const __half2*>(p.residual + pix[h] * p.ldr + cw)
                                   : __floats2half2_rn(0.f, 0.f);
                }
            }
#pragma unroll
        for (int u = 0; u < CH; ++u) {
            const int i = i0 + u;
            if (n0 + 8 * i >= p.N) break;
            const int col = n0 + 8 * i + 2 * q4;          // accumulator columns col, col + 1
            float v[2][2];
            const float2 bb = *reinterpret_cast<const float2*>(s_bias + 8 * i + 2 * q4);
            if (ln_in) {
                const float2 cs = *reinterpret_cast<const float2*>(s_cs + 8 * i + 2 * q4);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    v[h][0] = fmaf(ln_rs[h], fmaf(ln_nm[h], cs.x, a[u][2 * h]), bb.x);
                    v[h][1] = fmaf(ln_rs[h], fmaf(ln_nm[h], cs.y, a[u][2 * h + 1]), bb.y);
                }
            } else {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    v[h][0] = a[u][2 * h] + bb.x;
                    v[h][1] = a[u][2 * h + 1] + bb.y;
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                v[h][0] += ra[u][h].x;
                v[h][1] += ra[u][h].y;
            }
            if (p.act == 2) {
                // GEGLU: (a, gate) column pairs -> one output at column col / 2; neighbouring lanes swap so that each
                // stores two adjacent outputs (the even lane of row rl0, the odd lane of row rl0 + 8)
                float gv[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) gv[h] = v[h][0] * (p.out_f16 ? p_gelu(v[h][1]) : gelu_erf_f(v[h][1]));
                const float recv = __shfl_xor_sync(0xffffffffu, (lane & 1) ? gv[0] : gv[1], 1);
                const int h = lane & 1;
                const int ocol = (col >> 1) - h;
                if (h) store2(1, ocol, recv, gv[1]);
                else store2(0, ocol, gv[0], recv);
                continue;
            }
            if (p.act != 0) {
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        v[h][e] = p.act == 1 ? silu_f(v[h][e])
                                             : (p.act == 3 ? (p.out_f16 ? p_gelu(v[h][e]) : gelu_erf_f(v[h][e])) : quick_gelu_f(v[h][e]));
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float2 r = __half22float2(rr[u][h]);
                v[h][0] += r.x;
                v[h][1] += r.y;
                if (valid[h]) {
                    if (p.out_f16) *reinterpret_cast<__half2*>((__half*)p.out + pix[h] * p.ldo + col) = __floats2half2_rn(v[h][0], v[h][1]);
                    else *reinterpret_cast<float2*>((float*)p.out + pix[h] * p.ldo + col) = make_float2(v[h][0], v[h][1]);
                }
            }
            if (p.stats != nullptr) {
                // GroupNorm statistics of what was just produced (fp32, before the fp16 rounding): per channel over the
                // warp's 16 rows (fixed shuffle tree), the slab's two warps combined below in warp order
                float a0 = v[0][0] + v[1][0], a1 = v[0][1] + v[1][1];
                float b0 = v[0][0] * v[0][0] + v[1][0] * v[1][0], b1 = v[0][1] * v[0][1] + v[1][1] * v[1][1];
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
                    a0 += __shfl_xor_sync(0xffffffffu, a0, o);
                    a1 += __shfl_xor_sync(0xffffffffu, a1, o);
                    b0 += __shfl_xor_sync(0xffffffffu, b0, o);
                    b1 += __shfl_xor_sync(0xffffffffu, b1, o);
                }
                if (lane < 4) {
                    red[ew * BN + 8 * i + 2 * lane] = make_float2(a0, b0);
                    red[ew * BN + 8 * i + 2 * lane + 1] = make_float2(a1, b1);
                }
            }
            if (row_st) {                                 // one cell per (64-column slab, row)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    rs1[h] += v[h][0] + v[h][1];
                    rs2[h] = fmaf(v[h][0], v[h][0], fmaf(v[h][1], v[h][1], rs2[h]));
                }
                if ((i & 7) == 7) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        rs1[h] += __shfl_xor_sync(0xffffffffu, rs1[h], 1);
                        rs2[h] += __shfl_xor_sync(0xffffffffu, rs2[h], 1);
                        rs1[h] += __shfl_xor_sync(0xffffffffu, rs1[h], 2);
                        rs2[h] += __shfl_xor_sync(0xffffffffu, rs2[h], 2);
                        if (q4 == 0 && valid[h])
                            reinterpret_cast<float2*>(p.row_stats)[(size_t)((n0 >> 6) + (i >> 3)) * p.M + pix[h]] =
                                make_float2(rs1[h], rs2[h]);
                        rs1[h] = rs2[h] = 0.f;
                    }
                }
            }
        }
        }
        if (p.stats != nullptr) {
            g_pair_bar(1 + slab);
            if ((ew & 1) == 0) {
                int simg, sii;
                if (CONV) {
                    const int ppi = p.BW * p.BH;                           // patch pixels per image (multiple of 32)
                    simg = c.tn * p.NB + (slab * 32) / ppi;
                    sii = (c.th * p.tiles_w + c.tw) * (ppi >> 5) + (((slab * 32) % ppi) >> 5);
                } else {
                    const int r0 = c.m0 + slab * 32;
                    simg = r0 / p.stats_hw;
                    sii = (r0 - simg * p.stats_hw) >> 5;
                    if (r0 >= p.M) simg = p.stats_nimg;
                }
                if (simg < p.stats_nimg) {
                    for (int j = lane; j < BN && n0 + j < p.N; j += 32) {
                        const float2 x0 = red[ew * BN + j], x1 = red[(ew + 1) * BN + j];
                        reinterpret_cast<float2*>(p.stats)[((size_t)simg * p.stats_spi + sii) * p.N + n0 + j] =
                            make_float2(x0.x + x1.x, x0.y + x1.y);
                    }
                }
            }
            g_pair_bar(1 + slab);                         // read before the next tile's statistics overwrite it
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFnP)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFnP p_get_encode() {
    static EncodeTiledFnP fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qr) == cudaSuccess &&
            qr == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFnP)f;
    }
    return fn;
}

// Encoded tensor maps are kept in a small direct-mapped table keyed by everything that goes into the encoding: a sampling
// loop launches the same few hundred (pointer, shape) combinations over and over (the caching allocator hands the same
// blocks back), and cuTensorMapEncodeTiled is a few microseconds of host time per map.
struct PMapKey {
    const void* ptr;
    uint64_t d0, d1, d2, d3, ld;
    uint32_t b0, b1, b2, b3, es, rank;
    bool operator==(const PMapKey& o) const {
        return ptr == o.ptr && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && d3 == o.d3 && ld == o.ld && b0 == o.b0 && b1 == o.b1 &&
               b2 == o.b2 && b3 == o.b3 && es == o.es && rank == o.rank;
    }
};
struct PMapSlot {
    PMapKey key;
    CUtensorMap map;
    bool valid;
};
constexpr int P_MAP_SLOTS = 4096;
static thread_local PMapSlot* p_map_table = nullptr;
static PMapSlot* p_map_slot(const PMapKey& k) {
    if (p_map_table == nullptr) p_map_table = (PMapSlot*)calloc(P_MAP_SLOTS, sizeof(PMapSlot));
    uint64_t h = (uint64_t)(uintptr_t)k.ptr * 0x9E3779B97F4A7C15ull;
    h ^= (k.d0 * 31 + k.d1) * 0xC2B2AE3D27D4EB4Full + (k.d2 * 131 + k.d3 * 17 + k.ld) * 0x165667B19E3779F9ull;
    h ^= ((uint64_t)k.b0 << 40) ^ ((uint64_t)k.b1 << 28) ^ ((uint64_t)k.b2 << 16) ^ ((uint64_t)k.b3 << 4) ^ k.es ^ ((uint64_t)k.rank << 60);
    return p_map_table ? &p_map_table[(h >> 20) % P_MAP_SLOTS] : nullptr;
}

static bool p_map_2d(CUtensorMap* tm, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t bi, uint32_t bo) {
    const PMapKey key = {ptr, inner, outer, 0, 0, ld, bi, bo, 0, 0, 1, 2};
    PMapSlot* slot = p_map_slot(key);
    if (slot && slot->valid && slot->key == key) {
        *tm = slot->map;
        return true;
    }
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {ld * 2};
    cuuint32_t box[2] = {bi, bo};
    cuuint32_t es[2] = {1, 1};
    const bool ok = p_get_encode()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    if (ok && slot) {
        slot->key = key;
        slot->map = *tm;
        slot->valid = true;
    }
    return ok;
}
// NHWC tensor [N, H, W, C] with row pitch ld (elements per pixel), box 64 x BW x BH x NB, element stride s in W/H
// (cuTensorMapEncodeTiled: "to load N elements along a dimension, boxDim = N * elementStrides")
static bool p_map_nhwc(CUtensorMap* tm, const void* ptr, int N, int H, int W, int C, int ld, int BW, int BH, int NB, int s) {
    const PMapKey key = {ptr, (uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)N, (uint64_t)ld, 64u, (uint32_t)BW, (uint32_t)BH, (uint32_t)NB,
                         (uint32_t)s, 4};
    PMapSlot* slot = p_map_slot(key);
    if (slot && slot->valid && slot->key == key) {
        *tm = slot->map;
        return true;
    }
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)W * ld * 2, (cuuint64_t)H * W * ld * 2};
    cuuint32_t box[4] = {64u, (cuuint32_t)(BW * s), (cuuint32_t)(BH * s), (cuuint32_t)NB};
    cuuint32_t es[4] = {1, (cuuint32_t)s, (cuuint32_t)s, 1};
    const bool ok = p_get_encode()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, es,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    if (ok && slot) {
        slot->key = key;
        slot->map = *tm;
        slot->valid = true;
    }
    return ok;
}

// rectangular patch of 128 output pixels (BW x BH x NB, all powers of two): prefer extents that divide the image exactly
// (64->64x2, 32->32x4, 16->16x8, 8->8x8x2, 96->32x4, 48->16x8, 24->8x8x2), otherwise the smallest power of two that covers
// it (the overshoot is TMA out-of-bounds fill + masked rows).
static int p_pow2_ceil(int v) {
    int r = 1;
    while (r < v) r <<= 1;
    return r;
}
static int p_pick_extent(int len, int cap) {
    int lim = p_pow2_ceil(len);
    if (lim > cap) lim = cap;
    for (int c = lim; c >= 4; c >>= 1)
        if (len % c == 0) return c;
    return lim;
}

// nearest-neighbour x2 (F.interpolate(scale_factor=2, mode="nearest"), openaimodel.py:110-115) on NHWC fp16, materialised
// into the caller's workspace in front of an upsampling conv
__global__ void upsample2x_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int H, int W, int CV, long long total) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(i % CV);
        long long r = i / CV;
        const int ox = (int)(r % (2 * W));
        r /= (2 * W);
        const int oy = (int)(r % (2 * H));
        const long long n = r / (2 * H);
        dst[i] = __ldg(src + ((n * H + (oy >> 1)) * W + (ox >> 1)) * CV + cv);
    }
}

int launch_upsample2x(const __half* src, __half* dst, int N, int H, int W, int C, cudaStream_t st) {
    const long long total = (long long)N * 4 * H * W * (C / 8);
    int grid = (int)((total + 255) / 256);
    if (grid > sm_count() * 16) grid = sm_count() * 16;
    upsample2x_kernel<<<grid, 256, 0, st>>>((const uint4*)src, (uint4*)dst, H, W, C / 8, total);
    return check_launch("upsample2x");
}

static void p_conv_patch(const anysd_gemm_params* q, int* Ho, int* Wo, int* BW, int* BH, int* NB) {
    const int Hin = q->H << q->upsample, Win = q->Wd << q->upsample;
    *Ho = q->conv_pad ? (Hin - 2) / 2 + 1 : (Hin - 1) / q->stride + 1;
    *Wo = q->conv_pad ? (Win - 2) / 2 + 1 : (Win - 1) / q->stride + 1;
    *BW = p_pick_extent(*Wo, 128);
    *BH = p_pick_extent(*Ho, 128 / *BW);
    *NB = 128 / (*BW * *BH);
}

// GroupNorm statistics from the epilogue: possible when every 32-row slab of the output lies inside one image and the
// conv patches tile the image exactly.  Returns the slabs per image (rows_per_batch / 32), 0 when not possible.
int wg_stats_slabs(const anysd_gemm_params* q) {
    if (q->act == 2 || q->out_dtype != ANYSD_F16) return 0;
    const int hw = q->rows_per_batch;
    if (hw <= 0 || hw % 32 != 0 || q->M % hw != 0) return 0;
    if (q->conv) {
        int Ho, Wo, BW, BH, NB;
        p_conv_patch(q, &Ho, &Wo, &BW, &BH, &NB);
        if (Ho * Wo != hw || (BW * BH) % 32 != 0 || Wo % BW != 0 || Ho % BH != 0) return 0;
    }
    return hw / 32;
}

// K split: a function of the PER-IMAGE geometry only -- never of the batch -- because splitting changes the fp32 summation
// order: a layer either always runs as `splits` ordered partial sums or never does, so every output bit stays independent
// of how many images share the batch (and of the grid).  Layers with at most one 128-row tile per image (8x8 maps and
// smaller) and a very long K are the ones that leave most SMs idle at sampling batch sizes; the partial dump and the ordered
// add only pay off for the longest of them: 3 partials from 256 k-blocks on, convs only.  This rule was fitted on the project's
// earlier GPU (tests/diag_splitk.py) and is inherited unchanged; it has not been re-fitted for this kernel on the H100.
// ANYSD_GEMM_SPLITK=0|n forces a count (experiments).
static int p_geometry_splits(const anysd_gemm_params* q, int num_kb) {
    static const char* force_sk = getenv("ANYSD_GEMM_SPLITK");
    if (q->act == 2 || q->out_dtype != ANYSD_F16 || q->row_stats != nullptr || q->ln_stats != nullptr) return 1;
    int rows_per_image = q->rows_per_batch;
    if (q->conv) {
        int Ho, Wo, BW, BH, NB;
        p_conv_patch(q, &Ho, &Wo, &BW, &BH, &NB);
        rows_per_image = Ho * Wo;
    }
    if (rows_per_image <= 0 || rows_per_image > G_BM) return 1;
    if (force_sk) {
        const int f = atoi(force_sk);
        return (f <= 1 || num_kb / f < 8) ? 1 : (f > 8 ? 8 : f);
    }
    return (q->conv && num_kb >= 256) ? 3 : 1;
}

// Tile width 256 / 192 / 128 / 64.  Cost model = scheduling rounds of the work units (tiles x splits) on the SMs x per-unit
// time ~ (bn + 270) x (k-blocks of the unit + 8 when split: the partial dump and the ordered add): deep levels otherwise leave
// most of the machine idle while every busy SM streams a full K operand pair through its L2 port; mid levels suffer from
// wave quantisation.  The per-tile constant 270 is inherited from the project's earlier GPU and kernel and has not been re-fitted
// for this kernel on the H100 (only the SM count is the H100's).  ANYSD_GEMM_BN forces a width.
static void p_select(const anysd_gemm_params* q, int tiles_m, int num_kb, int* bn_out, int* splits_out) {
    static const char* force_bn = getenv("ANYSD_GEMM_BN");
    const int sp = splits_out ? p_geometry_splits(q, num_kb) : 1;
    int bn = 256;
    double best = -1;
    static const int widths[4] = {256, 192, 128, 64};     // 192 balances N = 320 (192 + 128) and divides 960 / 1920
    for (int wi = 0; wi < 4; ++wi) {
        const int w = widths[wi];
        if (force_bn && atoi(force_bn) != w) continue;
        const long units = (long)tiles_m * cdiv(q->N, w) * sp;
        const long slots = sm_count();
        const long rounds = (units + slots - 1) / slots;
        const double cost = (double)rounds * (w + 270) * ((double)cdiv(num_kb, sp) + (sp > 1 ? 8.0 : 0.0));
        if (best < 0 || cost < best) { best = cost; bn = w; }
    }
    *bn_out = bn;
    if (splits_out) *splits_out = sp;
}
static size_t p_splitk_bytes(int tiles_m, int N, int bn, int splits) {
    if (splits <= 1) return 0;
    return (size_t)tiles_m * cdiv(N, bn) * splits * G_BM * bn * sizeof(float);
}

static void p_tiles(const anysd_gemm_params* q, int* tiles_m, int* num_kb) {
    if (q->conv) {
        int Ho, Wo, BW, BH, NB;
        p_conv_patch(q, &Ho, &Wo, &BW, &BH, &NB);
        *tiles_m = cdiv(Wo, BW) * cdiv(Ho, BH) * cdiv(q->Nimg, NB);
        *num_kb = 9 * (q->Cin / G_BK);
    } else {
        *tiles_m = cdiv(q->M, G_BM);
        *num_kb = cdiv(q->K, G_BK);
    }
}

// scratch the caller should provide for this contraction to run split-K (0: the schedule does not split it)
size_t wg_splitk_bytes(const anysd_gemm_params* q) {
    int tiles_m, num_kb, bn, splits;
    p_tiles(q, &tiles_m, &num_kb);
    p_select(q, tiles_m, num_kb, &bn, &splits);
    return p_splitk_bytes(tiles_m, q->N, bn, splits);
}

// LayerNorm around a contraction (row_stats output / ln_stats input): NULL when this kernel can do it, else the reason.
static const char* wg_ln_unsupported(const anysd_gemm_params* q) {
    if (q->conv) return "dense contractions only";
    if (q->out_dtype != ANYSD_F16) return "fp16 output only";
    if (q->row_stats != nullptr) {
        if (q->act != 0) return "row statistics need act = 0";
        if (q->N % 64 != 0) return "row statistics need N % 64 == 0";
        if ((uintptr_t)q->row_stats % 8) return "row_stats must be 8-byte aligned";
    }
    if (q->ln_stats != nullptr) {
        if (q->K % 64 != 0) return "folded LayerNorm needs K % 64 == 0";
        if (q->bias == nullptr || q->ln_colsum == nullptr) return "folded LayerNorm needs bias (beta W^T + b) and ln_colsum";
        if (((uintptr_t)q->ln_stats % 8) || ((uintptr_t)q->ln_colsum % 16)) return "ln_stats / ln_colsum misaligned";
        if (q->N % 32 != 0) return "folded LayerNorm needs N % 32 == 0";
        if (q->act != 0 && q->act != 1 && q->act != 2) return "folded LayerNorm: act must be 0, 1 or 2";
    }
    return nullptr;
}

bool wg_supported(const anysd_gemm_params* q) {
    if (q->N % 8 != 0 || q->K % 8 != 0) return false;
    if (q->act == 2 && q->N % 16 != 0) return false;
    const int n_out = q->act == 2 ? q->N / 2 : q->N;
    if (((uintptr_t)q->out % 16) || q->ldo % 8 != 0 || n_out % 4 != 0) return false;
    if (q->residual && (((uintptr_t)q->residual % 16) || q->ldr % 8 != 0)) return false;
    if (q->bias && ((uintptr_t)q->bias % 16)) return false;
    if (q->rowadd && (((uintptr_t)q->rowadd % 16) || q->ld_rowadd % 4 != 0)) return false;
    if (q->conv) {
        if (q->Cin % G_BK != 0) return false;
        if (q->upsample) {
            const size_t need = (size_t)q->Nimg * (2 * q->H) * (2 * q->Wd) * q->Cin * sizeof(__half);
            if (q->workspace == nullptr || q->workspace_bytes < need || ((uintptr_t)q->workspace % 16)) return false;
        }
    }
    return p_get_encode() != nullptr;
}

template <int BN, bool CONV>
static int p_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const GArgs& a, cudaStream_t st) {
    static bool done[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(gemm_wgmma_kernel<BN, CONV>, cudaFuncAttributeMaxDynamicSharedMemorySize, GCfg<BN>::SMEM);
        if (e != cudaSuccess) {
            set_error("wgmma gemm: smem opt-in failed: %s", cudaGetErrorString(e));
            return ANYSD_ECUDA;
        }
        done[dev] = true;
    }
    int grid = sm_count();
    if (grid > a.num_units) grid = a.num_units;
    gemm_wgmma_kernel<BN, CONV><<<grid, G_THREADS, GCfg<BN>::SMEM, st>>>(tmA, tmB, a);
    return check_launch(CONV ? "conv3x3 (wgmma)" : "gemm (wgmma)");
}

template <bool CONV>
static int p_launch_bn(int bn, const CUtensorMap& tmA, const CUtensorMap& tmB, const GArgs& a, cudaStream_t st) {
    switch (bn) {
        case 256: return p_launch<256, CONV>(tmA, tmB, a, st);
        case 192: return p_launch<192, CONV>(tmA, tmB, a, st);
        case 128: return p_launch<128, CONV>(tmA, tmB, a, st);
        default: return p_launch<64, CONV>(tmA, tmB, a, st);
    }
}

int launch_gemm_wg(const anysd_gemm_params* q, cudaStream_t st) {
    GArgs a;
    a.stats = nullptr;
    a.stats_hw = a.stats_spi = a.stats_nimg = 0;
    if (q->stats != nullptr) {
        a.stats_spi = wg_stats_slabs(q);
        if (a.stats_spi == 0 || q->stats_images <= 0) {
            set_error("gemm: output statistics requested for a shape that cannot produce them (M=%d rows_per_batch=%d conv=%d act=%d); "
                      "query anysd_gemm_stats_slabs first", q->M, q->rows_per_batch, q->conv, q->act);
            return ANYSD_EUNSUPPORTED;
        }
        a.stats = q->stats;
        a.stats_hw = q->rows_per_batch;
        a.stats_nimg = q->stats_images;
    }
    a.row_stats = q->row_stats;
    a.ln_stats = q->ln_stats;
    a.ln_colsum = q->ln_colsum;
    a.ln_slabs = q->K / 64;
    a.ln_eps = q->ln_eps;
    a.ln_inv_k = 1.0f / (float)q->K;
    if (q->row_stats != nullptr || q->ln_stats != nullptr) {
        const char* why = wg_ln_unsupported(q);
        if (why) {
            set_error("gemm: LayerNorm fold / row statistics: %s (M=%d N=%d K=%d act=%d)", why, q->M, q->N, q->K, q->act);
            return ANYSD_EUNSUPPORTED;
        }
        if (q->stats != nullptr || q->act >= 3) {
            set_error("gemm: LayerNorm fold / row statistics cannot be combined with GroupNorm statistics or GELU epilogues");
            return ANYSD_EUNSUPPORTED;
        }
    }
    a.bias = q->bias;
    a.rowadd = q->rowadd;
    a.residual = (const __half*)q->residual;
    a.out = q->out;
    a.M = q->M;
    a.N = q->N;
    a.ldo = q->ldo;
    a.ldr = q->ldr;
    a.ld_rowadd = q->ld_rowadd;
    a.rows_per_batch = q->rows_per_batch > 0 ? q->rows_per_batch : 1;
    a.act = q->act;
    a.out_f16 = q->out_dtype == ANYSD_F16;
    a.Nimg = q->Nimg;
    a.BW = a.BH = a.NB = a.tiles_w = a.tiles_h = 1;
    a.kb_per_tap = 1;
    a.stride = q->conv ? q->stride : 1;
    a.pad_lo = (q->conv && q->conv_pad) ? 0 : 1;
    a.Ho = a.Wo = 0;
    CUtensorMap tmA, tmB;
    bool ok = true;
    p_tiles(q, &a.tiles_m, &a.num_kb);
    if (q->conv) {
        const void* img = q->A;
        int Hin = q->H, Win = q->Wd;
        if (q->upsample) {
            int rc = launch_upsample2x((const __half*)q->A, (__half*)q->workspace, q->Nimg, q->H, q->Wd, q->Cin, st);
            if (rc) return rc;
            img = q->workspace;
            Hin *= 2;
            Win *= 2;
        }
        p_conv_patch(q, &a.Ho, &a.Wo, &a.BW, &a.BH, &a.NB);
        a.tiles_w = cdiv(a.Wo, a.BW);
        a.tiles_h = cdiv(a.Ho, a.BH);
        a.kb_per_tap = q->Cin / G_BK;
        ok = ok && p_map_nhwc(&tmA, img, q->Nimg, Hin, Win, q->Cin, q->Cin, a.BW, a.BH, a.NB, a.stride);
    } else {
        ok = ok && p_map_2d(&tmA, q->A, (uint64_t)q->K, (uint64_t)q->M, (uint64_t)q->lda, G_BK, G_BM);
    }
    int bn = 256, splits = 1;
    p_select(q, a.tiles_m, a.num_kb, &bn, &splits);
    const size_t sk_need = p_splitk_bytes(a.tiles_m, q->N, bn, splits);
    if (splits > 1 && (q->splitk_workspace == nullptr || q->splitk_workspace_bytes < sk_need || q->splitk_counters == nullptr ||
                       (size_t)a.tiles_m * cdiv(q->N, bn) * 4 * sizeof(unsigned int) > q->splitk_counters_bytes)) {
        splits = 1;                                   // no scratch from the caller: the plain schedule
        p_select(q, a.tiles_m, a.num_kb, &bn, nullptr);
    }
    a.tiles_n = cdiv(q->N, bn);
    ok = ok && p_map_2d(&tmB, q->W, (uint64_t)q->K, (uint64_t)q->N, (uint64_t)q->ldw, G_BK, bn);
    if (!ok) {
        set_error("wgmma gemm: cuTensorMapEncodeTiled failed (M=%d N=%d K=%d conv=%d)", q->M, q->N, q->K, q->conv);
        return ANYSD_ECUDA;
    }
    a.num_tiles = a.tiles_m * a.tiles_n;
    a.splits = splits;
    a.kb_per_split = cdiv(a.num_kb, splits);
    a.num_units = a.num_tiles * splits;
    a.sk_ws = (float*)q->splitk_workspace;
    a.sk_cnt = (unsigned int*)q->splitk_counters;
    return q->conv ? p_launch_bn<true>(bn, tmA, tmB, a, st) : p_launch_bn<false>(bn, tmA, tmB, a, st);
}

}  // namespace anysd
