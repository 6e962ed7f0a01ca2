// The span of a 320-channel transformer block (attention.py BasicTransformerBlock) from the self-attention's output
// projection to the feed-forward's LayerNorm as ONE kernel.  Per 128-row tile, a1 the self-attention output and t the
// block input (both fp16 [M, 320]):
//
//   t2  = a1 Wo1^T + bo1 + t                   written (the residual of t3)
//   l2  = LayerNorm2(t2)                       shared memory only
//   q_h = l2 Wq_h^T         h = 0 .. 7         48 padded columns per head, scale * log2(e) folded into Wq; registers only
//   o_h = softmax(q_h K_h^T) V_h               the tile's image's context K/V (aux_cols operands, <= 80 keys)
//   t3  = concat_h(o_h) Wo2^T + bo2 + t2       written
//   l3  = LayerNorm3(t3)                       written (the input of the fused feed-forward)
//
// Structure (feedforward_wgmma.cu's): persistent CTAs over 128-row tiles, 384 threads; warpgroup 0 is the TMA producer
// (24 registers), consumer warpgroups 1 and 2 (240 registers) own 64 rows of the tile each.  Shared memory:
//   X   [128 x 320] fp16 (5 swizzled atoms of 64 columns, 80 KB): a1 from TMA; each warpgroup overwrites its 64-row half
//       with t2, LayerNorm 2 rewrites it in place as l2, and after the last head it holds t3 for LayerNorm 3;
//   A2  [128 x 320] fp16 (80 KB): the attention output, the A operand of Wo2;
//   one ring of 2 x 30 KB weight slots carrying, in order per tile: Wo1 as [192 x 64] + [128 x 64] pieces per k-block,
//   per head Wq_h [48 x 320] then K_h + V_h (80 keys x one 64-column atom each), and Wo2 like Wo1.
// q_h needs no buffer: its m64n48 accumulator, rounded to fp16, is already the register A fragment of the k16 steps of
// S = q_h K_h^T (the identity attention_wgmma.cu uses for P).
//
// Bit identity with the launches it replaces (gemm + bias + residual, layernorm, gemm, attention, gemm + bias +
// residual, layernorm; tests/test_gpu_xattn_block.py):
//   * every product keeps the k order of the contraction it replaces (K = 320 in order; the keys in order);
//   * the contraction epilogues repeat gemm_wgmma.cu's order: acc + bias, + 0 for the absent row add, + residual, one
//     fp16 rounding (to_q: no bias, no residual -- acc + 0);
//   * the softmax is attention_wgmma_kernel<48, 128, true>'s for a single, masked key tile: unit scale, keys past the
//     context masked, row maximum and sums over the same columns in the same order.  S covers 80 key columns instead
//     of 128; the 48 it leaves out are masked there, so they only add exact zeros to the row sums and to P V;
//   * both LayerNorms are layernorm_kernel<8, 5>'s: 8 lanes per row, lane l holding 16-byte vectors l, l + 8, .., l + 32,
//     through the same layernorm_row_stats / layernorm_row_apply (common.cuh).
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace anysd {

constexpr int XB_C = 320, XB_BM = 128, XB_THREADS = 384;
constexpr int XB_HEADS = 8, XB_D = 40, XB_HS = 48, XB_KEYS = 80;
constexpr int XB_KA = XB_C / 64;                                   // 5 atoms of 64 columns along C
constexpr int XB_X_ATOM = XB_BM * 128;                             // [128 rows x 64 halves] = 16 KB
constexpr int XB_X_BYTES = XB_KA * XB_X_ATOM;                      // 80 KB
constexpr int XB_WA = 192, XB_WB = XB_C - XB_WA;                   // output-column pieces of Wo1 / Wo2
constexpr int XB_WQ_ATOM = XB_HS * 128;                            // [48 rows x 64 halves] = 6 KB
constexpr int XB_KV_ATOM = XB_KEYS * 128;                          // [80 keys x 64 halves] = 10 KB
constexpr int XB_SLOT = XB_KA * XB_WQ_ATOM;                        // 30 KB: the largest item (Wq_h)
static_assert(XB_WA * 128 <= XB_SLOT && 2 * XB_KV_ATOM <= XB_SLOT, "cross-attention block: ring slot");
constexpr int XB_A2_OFF = XB_X_BYTES;
constexpr int XB_RING_OFF = XB_A2_OFF + XB_X_BYTES;
constexpr int XB_BAR_OFF = XB_RING_OFF + 2 * XB_SLOT;
constexpr int XB_SMEM = XB_BAR_OFF + 8 * 8 + 1024;                 // + alignment slack for the 1024-byte swizzle atoms
static_assert(XB_SMEM <= 227 * 1024, "cross-attention block: shared memory");

struct XbArgs {
    const __half* t;         // block input (residual of t2)
    const float *bo1, *ln2_w, *ln2_b, *bo2, *ln3_w, *ln3_b;
    __half *t2, *t3, *l3;
    int n, L, num_tiles;     // rows per image, context length, 128-row tiles
    float eps;
};

__device__ __forceinline__ void xb_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void xb_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void xb_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void xb_wait(uint32_t bar, uint32_t parity) {
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
__device__ __forceinline__ void xb_tma_2d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ float xb_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t xb_pack(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
// generic-proxy shared-memory writes -> later wgmma / TMA (async proxy) accesses
__device__ __forceinline__ void xb_fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// the 128 threads of consumer warpgroup wg (named barriers 1 and 2)
__device__ __forceinline__ void xb_wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }
// byte offset of (row, column pair 2k) inside a [rows x 320] tile of 128-byte swizzled 64-column atoms of atom_bytes
__device__ __forceinline__ uint32_t xb_swz(int row, int col, int atom_bytes) {
    return (col >> 6) * atom_bytes + row * 128 + ((((col >> 3) & 7) ^ (row & 7)) << 4) + (col & 7) * 2;
}

__global__ void __launch_bounds__(XB_THREADS, 1)
xattn_block_wgmma_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmWo1a,
                         const __grid_constant__ CUtensorMap tmWo1b, const __grid_constant__ CUtensorMap tmWq,
                         const __grid_constant__ CUtensorMap tmKV, const __grid_constant__ CUtensorMap tmWo2a,
                         const __grid_constant__ CUtensorMap tmWo2b, const XbArgs p) {
    extern __shared__ unsigned char xb_smem_raw[];
    const uint32_t raw = smem_u32(xb_smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char* smem = xb_smem_raw + (base - raw);
    // barriers: 0 x_full | 1 x_empty | 2, 3 slot_full | 4, 5 slot_empty
    const uint32_t bars = base + XB_BAR_OFF;
    auto BAR = [&](int i) { return bars + 8u * i; };
    auto slot = [&](uint32_t c) { return base + XB_RING_OFF + (c & 1) * XB_SLOT; };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmWo1a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmWo1b) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmWq) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmKV) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmWo2a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmWo2b) : "memory");
        // full barriers take the producer's expect_tx, empty ones one arrive per consumer warp
        for (int i = 0; i < 6; ++i) xb_init(BAR(i), (i == 1 || i >= 4) ? 8 : 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 4) {
        // ===== TMA producer: one thread; the a1 tile, then the tile's 36 ring items in consumption order =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;" ::: "memory");
        if (warp == 0 && lane == 0) {
            uint32_t c = 0;
            auto push = [&](uint32_t bytes) {             // claims the next slot; returns its address
                const int s = c & 1;
                xb_wait(BAR(4 + s), ((c >> 1) & 1) ^ 1);
                xb_expect_tx(BAR(2 + s), bytes);
                return slot(c++);
            };
            auto push_wo = [&](const CUtensorMap* ta, const CUtensorMap* tb) {
                for (int kb = 0; kb < XB_KA; ++kb) {
                    uint32_t d = push(XB_WA * 128);
                    xb_tma_2d(d, ta, BAR(2 + ((c - 1) & 1)), kb * 64, 0);
                    d = push(XB_WB * 128);
                    xb_tma_2d(d, tb, BAR(2 + ((c - 1) & 1)), kb * 64, XB_WA);
                }
            };
            int it = 0;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
                const int img = tile * XB_BM / p.n;
                xb_wait(BAR(1), (it & 1) ^ 1);
                xb_expect_tx(BAR(0), XB_X_BYTES);
                for (int a = 0; a < XB_KA; ++a) xb_tma_2d(base + a * XB_X_ATOM, &tmX, BAR(0), a * 64, tile * XB_BM);
                push_wo(&tmWo1a, &tmWo1b);
                for (int h = 0; h < XB_HEADS; ++h) {
                    uint32_t d = push(XB_SLOT);
                    for (int a = 0; a < XB_KA; ++a) xb_tma_2d(d + a * XB_WQ_ATOM, &tmWq, BAR(2 + ((c - 1) & 1)), a * 64, h * XB_HS);
                    d = push(2 * XB_KV_ATOM);
                    xb_tma_2d(d, &tmKV, BAR(2 + ((c - 1) & 1)), h * XB_HS, img * p.L);
                    xb_tma_2d(d + XB_KV_ATOM, &tmKV, BAR(2 + ((c - 1) & 1)), XB_HEADS * XB_HS + h * XB_HS, img * p.L);
                }
                push_wo(&tmWo2a, &tmWo2b);
            }
        }
        return;
    }

    // ===== consumer warpgroups: rows 64 wg .. 64 wg + 63 of every tile; this thread: rows r, r + 8 of the warp's 16 =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;" ::: "memory");
    const int wg = __shfl_sync(0xffffffffu, (warp >> 2) - 1, 0);   // warp-uniform to the compiler: keeps wgmma unserialized
    const int wq = warp & 3, q4 = lane & 3, wtid = threadIdx.x - 128 * (wg + 1);
    const uint32_t xa = base + wg * 64 * 128, a2a = base + XB_A2_OFF + wg * 64 * 128;
    unsigned char* xs_g = smem + wg * 64 * 128;                     // generic pointers to the warpgroup's halves
    unsigned char* a2_g = smem + XB_A2_OFF + wg * 64 * 128;
    float o[XB_C / 2];                                              // [64 x 320]: element 4 i + 2 h + e at column 8 i + 2 q + e
    uint32_t c = 0;

    auto take = [&]() { xb_wait(BAR(2 + (c & 1)), (c >> 1) & 1); };
    auto give = [&](uint32_t cc) {
        __syncwarp();
        if (lane == 0) xb_arrive(BAR(4 + (cc & 1)));
    };
    // o = A W^T over K = 320 in order, A = the warpgroup's half of X or A2, W streamed as 192- and 128-row pieces
    auto product_wo = [&](uint32_t a_base) {
#pragma unroll
        for (int i = 0; i < XB_C / 2; ++i) o[i] = 0.f;
        wg_fence();
#pragma unroll 1
        for (int kb = 0; kb < XB_KA; ++kb) {
            take();
#pragma unroll
            for (int k = 0; k < 4; ++k)
                Wgmma<XB_WA>::ss(o, wg_desc(a_base + kb * XB_X_ATOM + k * 32, 16, 1024), wg_desc(slot(c) + k * 32, 16, 1024), 1);
            wg_commit();
            if (kb > 0) {
                wg_wait<1>();
                give(c - 1);
            }
            ++c;
            take();
#pragma unroll
            for (int k = 0; k < 4; ++k)
                Wgmma<XB_WB>::ss(o + XB_WA / 2, wg_desc(a_base + kb * XB_X_ATOM + k * 32, 16, 1024),
                                 wg_desc(slot(c) + k * 32, 16, 1024), 1);
            wg_commit();
            wg_wait<1>();
            give(c - 1);
            ++c;
        }
        wg_wait<0>();
        give(c - 1);
#pragma unroll
        for (int i = 0; i < XB_C / 2; ++i) wg_fence_regs(o[i]);
    };
    // (o + bias) + 0, + residual, one fp16 rounding (gemm_wgmma.cu's act-0 order): written to dst and into the X half
    auto epilogue_wo = [&](int tile, const float* bias, const __half* res, __half* dst) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int rr = wq * 16 + (lane >> 2) + 8 * h;
            const size_t m = (size_t)tile * XB_BM + wg * 64 + rr;
            const __half* rrow = res + m * XB_C + 2 * q4;
            __half* orow = dst + m * XB_C + 2 * q4;
            constexpr int G = 8;
#pragma unroll
            for (int i0 = 0; i0 < XB_C / 8; i0 += G) {
                __half2 rv[G];
#pragma unroll
                for (int u = 0; u < G; ++u) rv[u] = *reinterpret_cast<const __half2*>(rrow + 8 * (i0 + u));
#pragma unroll
                for (int u = 0; u < G; ++u) {
                    const int i = i0 + u;
                    const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + 8 * i + 2 * q4));
                    float v0 = o[4 * i + 2 * h] + bb.x, v1 = o[4 * i + 2 * h + 1] + bb.y;
                    v0 += 0.f;
                    v1 += 0.f;
                    const float2 r = __half22float2(rv[u]);
                    v0 += r.x;
                    v1 += r.y;
                    const __half2 hv = __floats2half2_rn(v0, v1);
                    *reinterpret_cast<__half2*>(orow + 8 * i) = hv;
                    *reinterpret_cast<__half2*>(xs_g + xb_swz(rr, 8 * i + 2 * q4, XB_X_ATOM)) = hv;
                }
            }
        }
    };
    // LayerNorm of the X half's 64 rows, 8 lanes per row (16 rows per pass): in place, or to global when out != nullptr
    auto layernorm = [&](int tile, const float* gamma, const float* beta, __half* out) {
        const int l = wtid & 7;
#pragma unroll 1
        for (int pass = 0; pass < 4; ++pass) {
            const int rr = pass * 16 + (wtid >> 3);
            float f[5][8];
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 5; ++i) {
                unpack8(*reinterpret_cast<const uint4*>(xs_g + xb_swz(rr, 8 * (l + 8 * i), XB_X_ATOM)), f[i]);
#pragma unroll
                for (int j = 0; j < 8; ++j) s += f[i][j];
            }
            float mean, rstd;
            layernorm_row_stats<8, 5>(f, s, l, XB_C / 8, p.eps, mean, rstd);
            layernorm_row_apply<8, 5>(f, l, XB_C / 8, gamma, beta, mean, rstd);
#pragma unroll
            for (int i = 0; i < 5; ++i) {
                const uint4 u = pack8(f[i]);
                if (out != nullptr)
                    *reinterpret_cast<uint4*>(out + ((size_t)tile * XB_BM + wg * 64 + rr) * XB_C + 8 * (l + 8 * i)) = u;
                else
                    *reinterpret_cast<uint4*>(xs_g + xb_swz(rr, 8 * (l + 8 * i), XB_X_ATOM)) = u;
            }
        }
    };

    int it = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
        xb_wait(BAR(0), it & 1);
        // ---- t2 = a1 Wo1^T + bo1 + t; l2 = LayerNorm2(t2) in place ----
        product_wo(xa);
        epilogue_wo(tile, p.bo1, p.t, p.t2);
        xb_wg_sync(wg);
        layernorm(tile, p.ln2_w, p.ln2_b, nullptr);
        xb_fence_async();
        xb_wg_sync(wg);

        // ---- per head: q_h = l2 Wq_h^T, o_h = softmax(q_h K_h^T) V_h into A2 ----
#pragma unroll 1
        for (int hh = 0; hh < XB_HEADS; ++hh) {
            float qc[XB_HS / 2];
#pragma unroll
            for (int i = 0; i < XB_HS / 2; ++i) qc[i] = 0.f;
            take();
            wg_fence();
#pragma unroll
            for (int k = 0; k < XB_C / 16; ++k)
                Wgmma<XB_HS>::ss(qc, wg_desc(xa + (k >> 2) * XB_X_ATOM + (k & 3) * 32, 16, 1024),
                                 wg_desc(slot(c) + (k >> 2) * XB_WQ_ATOM + (k & 3) * 32, 16, 1024), 1);
            wg_commit();
            wg_wait<0>();
            give(c);
            ++c;
            // to_q epilogue: acc + 0 (no bias, no row add, no residual), one fp16 rounding; k16 step s of S takes
            // accumulator column blocks 2 s and 2 s + 1
            uint32_t qa[XB_HS / 16][4];
#pragma unroll
            for (int i = 0; i < XB_HS / 2; ++i) {
                wg_fence_regs(qc[i]);
                qc[i] += 0.f;
            }
#pragma unroll
            for (int s = 0; s < XB_HS / 16; ++s) {
                const float* t = qc + 8 * s;
                qa[s][0] = xb_pack(t[0], t[1]);
                qa[s][1] = xb_pack(t[2], t[3]);
                qa[s][2] = xb_pack(t[4], t[5]);
                qa[s][3] = xb_pack(t[6], t[7]);
            }
            take();
            const uint32_t kb = slot(c), vb = kb + XB_KV_ATOM;
            float sc[XB_KEYS / 2];
            wg_fence();
#pragma unroll
            for (int k = 0; k < XB_HS / 16; ++k) Wgmma<XB_KEYS>::rs(sc, qa[k], wg_desc(kb + k * 32, 16, 1024), k > 0);
            wg_commit();
            wg_wait<0>();
            // softmax of the single, masked key tile (attention_wgmma_kernel, UNIT): p = ex2(s - m), sums in its order
#pragma unroll
            for (int i = 0; i < XB_KEYS / 2; ++i) wg_fence_regs(sc[i]);
#pragma unroll
            for (int i = 0; i < XB_KEYS / 8; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (8 * i + 2 * q4 + (e & 1) >= p.L) sc[4 * i + e] = -INFINITY;
            float mx[2] = {-INFINITY, -INFINITY}, lr[2] = {0.f, 0.f};
#pragma unroll
            for (int i = 0; i < XB_KEYS / 8; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e) mx[e >> 1] = fmaxf(mx[e >> 1], sc[4 * i + e]);
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            }
            uint32_t pa[XB_KEYS / 16][4];
#pragma unroll
            for (int kk = 0; kk < XB_KEYS / 16; ++kk) {
                float* t = sc + 8 * kk;
#pragma unroll
                for (int e = 0; e < 8; ++e) t[e] = xb_ex2(t[e] - mx[(e >> 1) & 1]);
                lr[0] += (t[0] + t[1]) + (t[4] + t[5]);
                lr[1] += (t[2] + t[3]) + (t[6] + t[7]);
                pa[kk][0] = xb_pack(t[0], t[1]);
                pa[kk][1] = xb_pack(t[2], t[3]);
                pa[kk][2] = xb_pack(t[4], t[5]);
                pa[kk][3] = xb_pack(t[6], t[7]);
            }
            float oh[XB_HS / 2];
#pragma unroll
            for (int i = 0; i < XB_HS / 2; ++i) oh[i] = 0.f;
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < XB_KEYS / 16; ++kk)
                Wgmma<XB_HS>::rs_t(oh, pa[kk], wg_desc(vb + kk * 2048, XB_KV_ATOM, 1024), 1);
            wg_commit();
            wg_wait<0>();
#pragma unroll
            for (int i = 0; i < XB_HS / 2; ++i) wg_fence_regs(oh[i]);
            give(c);
            ++c;
            // O / l -> fp16 -> columns 40 hh .. 40 hh + 39 of the A2 half
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                float l = lr[r];
                l += __shfl_xor_sync(0xffffffffu, l, 1);
                l += __shfl_xor_sync(0xffffffffu, l, 2);
                const float inv = 1.0f / l;
                const int rr = wq * 16 + (lane >> 2) + 8 * r;
#pragma unroll
                for (int i = 0; i < XB_D / 8; ++i)
                    *reinterpret_cast<__half2*>(a2_g + xb_swz(rr, hh * XB_D + 8 * i + 2 * q4, XB_X_ATOM)) =
                        __floats2half2_rn(oh[4 * i + 2 * r] * inv, oh[4 * i + 2 * r + 1] * inv);
            }
        }
        xb_fence_async();
        xb_wg_sync(wg);

        // ---- t3 = a2 Wo2^T + bo2 + t2 (t2 re-read from global: written by this same thread); l3 = LayerNorm3(t3) ----
        product_wo(a2a);
        epilogue_wo(tile, p.bo2, p.t2, p.t3);
        xb_wg_sync(wg);
        layernorm(tile, p.ln3_w, p.ln3_b, p.l3);
        xb_fence_async();
        __syncwarp();
        if (lane == 0) xb_arrive(BAR(1));                           // X free for the next tile's a1
    }
}

// ---- host side ---------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFnX)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFnX x_get_encode() {
    static EncodeTiledFnX fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qr) == cudaSuccess &&
            qr == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFnX)f;
    }
    return fn;
}
// 2-D fp16 map [rows, width] with row pitch ld, 64-column (128-byte, swizzled) box of box_rows rows
static bool x_map(CUtensorMap* tm, const void* ptr, uint64_t width, uint64_t rows, uint64_t ld, uint32_t box_rows) {
    cuuint64_t dims[2] = {width, rows};
    cuuint64_t strides[1] = {ld * 2};
    cuuint32_t box[2] = {64, box_rows};
    cuuint32_t es[2] = {1, 1};
    return x_get_encode()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace anysd

using namespace anysd;

extern "C" int anysd_xattn_block_f16(const void* a1, const void* t, const void* wo1, const float* bo1, const float* ln2_w,
                                     const float* ln2_b, const void* wq, const void* kv, int ld_kv, const void* wo2,
                                     const float* bo2, const float* ln3_w, const float* ln3_b, void* t2, void* t3, void* l3,
                                     int M, int n, int L, int C, int heads, int d, int hs, int aux_cols, float eps,
                                     anysd_stream_t stream) {
    ANYSD_REQUIRE(a1 && t && wo1 && bo1 && ln2_w && ln2_b && wq && kv && wo2 && bo2 && ln3_w && ln3_b && t2 && t3 && l3,
                  ANYSD_EINVAL, "xattn_block: null pointer");
    ANYSD_REQUIRE(M > 0 && n > 0 && L > 0 && M % n == 0, ANYSD_EINVAL, "xattn_block: bad M=%d n=%d L=%d", M, n, L);
    ANYSD_REQUIRE(C == XB_C && heads == XB_HEADS && d == XB_D && hs == XB_HS, ANYSD_EUNSUPPORTED,
                  "xattn_block: only C = %d as %d heads of %d (stride %d) (got C=%d heads=%d d=%d hs=%d)", XB_C, XB_HEADS,
                  XB_D, XB_HS, C, heads, d, hs);
    ANYSD_REQUIRE(aux_cols, ANYSD_EUNSUPPORTED, "xattn_block: only aux_cols heads");
    ANYSD_REQUIRE(n % XB_BM == 0, ANYSD_EUNSUPPORTED, "xattn_block: rows per image n=%d must be a multiple of %d", n, XB_BM);
    ANYSD_REQUIRE(L <= XB_KEYS, ANYSD_EUNSUPPORTED, "xattn_block: context of %d tokens (at most %d)", L, XB_KEYS);
    ANYSD_REQUIRE(ld_kv >= 2 * heads * hs && ld_kv % 8 == 0, ANYSD_EINVAL, "xattn_block: ld_kv=%d", ld_kv);
    const void* ptrs[] = {a1, t, wo1, bo1, ln2_w, ln2_b, wq, kv, wo2, bo2, ln3_w, ln3_b, t2, t3, l3};
    for (const void* q : ptrs) ANYSD_REQUIRE(((uintptr_t)q % 16) == 0, ANYSD_EINVAL, "xattn_block: pointers must be 16-byte aligned");
    ANYSD_REQUIRE(x_get_encode() != nullptr, ANYSD_ECUDA, "xattn_block: cuTensorMapEncodeTiled unavailable");
    const int B = M / n;
    CUtensorMap tmX, tmWo1a, tmWo1b, tmWq, tmKV, tmWo2a, tmWo2b;
    const bool ok = x_map(&tmX, a1, XB_C, (uint64_t)M, XB_C, XB_BM) && x_map(&tmWo1a, wo1, XB_C, XB_C, XB_C, XB_WA) &&
                    x_map(&tmWo1b, wo1, XB_C, XB_C, XB_C, XB_WB) && x_map(&tmWq, wq, XB_C, XB_HEADS * XB_HS, XB_C, XB_HS) &&
                    x_map(&tmKV, kv, 2 * XB_HEADS * XB_HS, (uint64_t)B * L, ld_kv, XB_KEYS) &&
                    x_map(&tmWo2a, wo2, XB_C, XB_C, XB_C, XB_WA) && x_map(&tmWo2b, wo2, XB_C, XB_C, XB_C, XB_WB);
    ANYSD_REQUIRE(ok, ANYSD_ECUDA, "xattn_block: cuTensorMapEncodeTiled failed (M=%d L=%d)", M, L);
    static bool done[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(xattn_block_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, XB_SMEM);
        ANYSD_REQUIRE(e == cudaSuccess, ANYSD_ECUDA, "xattn_block: smem opt-in failed: %s", cudaGetErrorString(e));
        done[dev] = true;
    }
    XbArgs a;
    a.t = (const __half*)t;
    a.bo1 = bo1; a.ln2_w = ln2_w; a.ln2_b = ln2_b; a.bo2 = bo2; a.ln3_w = ln3_w; a.ln3_b = ln3_b;
    a.t2 = (__half*)t2; a.t3 = (__half*)t3; a.l3 = (__half*)l3;
    a.n = n; a.L = L; a.num_tiles = M / XB_BM; a.eps = eps;
    int grid = sm_count();
    if (grid > a.num_tiles) grid = a.num_tiles;
    xattn_block_wgmma_kernel<<<grid, XB_THREADS, XB_SMEM, (cudaStream_t)stream>>>(tmX, tmWo1a, tmWo1b, tmWq, tmKV, tmWo2a,
                                                                                  tmWo2b, a);
    return check_launch("xattn_block (wgmma)");
}
