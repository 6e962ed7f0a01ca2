// The 320-channel GEGLU feed-forward of a transformer block (attention.py FeedForward: Linear(C, 8C) -> GEGLU ->
// Linear(4C, C), plus the block's residual) as ONE kernel whose 1280-wide hidden activations never leave the SM:
//
//   out = residual + W2 GEGLU(W1 x + b1) + b2,   x = norm3(t) [M, 320] fp16, out [M, 320] fp16.
//
// The structure is the attention forward's (attention_wgmma.cu) with the softmax replaced by bias + GEGLU and no running
// maximum:
//   * persistent CTAs over 128-row tiles, 384 threads: warpgroup 0 is the TMA producer (24 registers), consumer warpgroups
//     1 and 2 (240 registers) own 64 rows of the tile each;
//   * the x tile is loaded once per tile (5 k-blocks of 64 columns, 80 KB); the hidden dimension streams in chunks of 32
//     GEGLU outputs: 64 rows of the permuted ff1 pack (40 KB, 2-slot ring) and the matching 32 rows of W2^T (20 KB, 2-slot
//     ring of its own, since it is read one chunk later than the ff1 rows);
//   * per chunk: S [64 x 64] = x W1_chunk^T (20 x m64n64k16, both operands in shared memory), bias + GEGLU on the fragment,
//     rounded to fp16 in registers as the A operand of O [64 x 320] += P W2_chunk (2 k16 steps x m64n192 + m64n128, W2^T
//     an MN-major B operand).  S of chunk j and P V of chunk j - 1 are issued back to back, the GEGLU of j runs while the
//     latter is on the tensor cores, and the two consumer warpgroups take turns issuing (named barriers 1 and 2);
//   * epilogue: O + b2 + residual, rounded to fp16, plain fragment stores.
//
// No shuffles: unet.py permutes the interleaved (a, gate) rows of ff1 within each chunk of 32 outputs so that the pair a
// thread's S fragment holds at column step i is hidden unit 16 floor(i / 4) + [2q, 2q + 1, 2q + 8, 2q + 9][i % 4] (q = lane
// % 4): the GEGLU results of steps 4s .. 4s + 3 are then exactly the register A fragment of k16 step s in natural hidden
// order.  Both products keep the k order of the two contractions they replace (x over K = 320; the hidden units in order),
// and the epilogues repeat gemm_wgmma.cu's operation order (acc + bias, + 0 from the absent row add, then GEGLU / + residual),
// so the result is that of layernorm -> gemm(act 2) -> gemm(+ residual) bit for bit (tests/test_gpu_geglu_ff.py).
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace anysd {

constexpr int FF_C = 320, FF_HID = 4 * FF_C, FF_BM = 128, FF_THREADS = 384;
constexpr int FF_CH = 32;                                 // GEGLU outputs per chunk
constexpr int FF_NCH = FF_HID / FF_CH;                    // 40 chunks
constexpr int FF_KA = FF_C / 64;                          // 5 atoms of 64 columns along C
constexpr int FF_X_ATOM = FF_BM * 128;                    // [128 rows x 64 halves] = 16 KB
constexpr int FF_W1_ATOM = 2 * FF_CH * 128;               // [64 rows x 64 halves] = 8 KB
constexpr int FF_W2_ATOM = FF_CH * 128;                   // [32 rows x 64 halves] = 4 KB
constexpr int FF_X_BYTES = FF_KA * FF_X_ATOM, FF_W1_BYTES = FF_KA * FF_W1_ATOM, FF_W2_BYTES = FF_KA * FF_W2_ATOM;
constexpr int FF_W1_OFF = FF_X_BYTES;
constexpr int FF_W2_OFF = FF_W1_OFF + 2 * FF_W1_BYTES;
constexpr int FF_B1_OFF = FF_W2_OFF + 2 * FF_W2_BYTES;    // fp32 [2 * hidden] permuted ff1 bias
constexpr int FF_B2_OFF = FF_B1_OFF + 2 * FF_HID * 4;     // fp32 [C]
constexpr int FF_BAR_OFF = FF_B2_OFF + FF_C * 4;
constexpr int FF_SMEM = FF_BAR_OFF + 16 * 8 + 1024;       // + alignment slack for the 1024-byte swizzle atoms
static_assert(FF_SMEM <= 227 * 1024, "fused feed-forward: shared memory");

struct FfArgs {
    const float* b1;         // [2 * hidden], permuted like the ff1 rows
    const float* b2;         // [C]
    const __half* residual;
    __half* out;
    int M, ldr, ldo, num_tiles;
};

__device__ __forceinline__ void ff_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void ff_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void ff_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void ff_wait(uint32_t bar, uint32_t parity) {
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
__device__ __forceinline__ void ff_tma_2d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ uint32_t ff_pack(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
// issue turns of the two consumer warpgroups, as in attention_wgmma.cu: warpgroup c waits on named barrier 1 + c before it
// issues its products and then arrives on the other one's (both barriers count the 256 consumer threads)
__device__ __forceinline__ void ff_turn_wait(int c) { asm volatile("bar.sync %0, 256;" ::"r"(1 + c) : "memory"); }
__device__ __forceinline__ void ff_turn_pass(int c) { asm volatile("bar.arrive %0, 256;" ::"r"(2 - c) : "memory"); }

__global__ void __launch_bounds__(FF_THREADS, 1)
geglu_ff_wgmma_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW1,
                      const __grid_constant__ CUtensorMap tmW2, const FfArgs p) {
    extern __shared__ unsigned char ff_smem_raw[];
    const uint32_t raw = smem_u32(ff_smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char* smem = ff_smem_raw + (base - raw);
    float* s_b1 = reinterpret_cast<float*>(smem + FF_B1_OFF);
    float* s_b2 = reinterpret_cast<float*>(smem + FF_B2_OFF);
    // barriers: 0 x_full | 1 x_empty | 2, 3 w1_full | 4, 5 w1_empty | 6, 7 w2_full | 8, 9 w2_empty
    const uint32_t bars = base + FF_BAR_OFF;
    auto BAR = [&](int i) { return bars + 8u * i; };
    const uint32_t xs = base;
    auto w1s = [&](int s) { return base + FF_W1_OFF + s * FF_W1_BYTES; };
    auto w2s = [&](int s) { return base + FF_W2_OFF + s * FF_W2_BYTES; };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    for (int i = threadIdx.x; i < 2 * FF_HID; i += FF_THREADS) s_b1[i] = __ldg(p.b1 + i);
    for (int i = threadIdx.x; i < FF_C; i += FF_THREADS) s_b2[i] = p.b2 != nullptr ? __ldg(p.b2 + i) : 0.f;
    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW1) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW2) : "memory");
        // full barriers take the producer's expect_tx, empty ones one arrive per consumer warp
        for (int i = 0; i < 10; ++i) ff_init(BAR(i), (i == 1 || i == 4 || i == 5 || i == 8 || i == 9) ? 8 : 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 4) {
        // ===== TMA producer: one thread; x once per tile, then the chunks' ff1 rows and W2^T rows in ring order =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;" ::: "memory");
        if (warp == 0 && lane == 0) {
            uint32_t c = 0;
            int it = 0;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
                ff_wait(BAR(1), (it & 1) ^ 1);
                ff_expect_tx(BAR(0), FF_X_BYTES);
                for (int a = 0; a < FF_KA; ++a) ff_tma_2d(xs + a * FF_X_ATOM, &tmX, BAR(0), a * 64, tile * FF_BM);
                for (int j = 0; j < FF_NCH; ++j, ++c) {
                    const int s = c & 1;
                    const uint32_t ph = ((c >> 1) & 1) ^ 1;
                    ff_wait(BAR(4 + s), ph);
                    ff_expect_tx(BAR(2 + s), FF_W1_BYTES);
                    for (int a = 0; a < FF_KA; ++a) ff_tma_2d(w1s(s) + a * FF_W1_ATOM, &tmW1, BAR(2 + s), a * 64, j * 2 * FF_CH);
                    ff_wait(BAR(8 + s), ph);
                    ff_expect_tx(BAR(6 + s), FF_W2_BYTES);
                    for (int a = 0; a < FF_KA; ++a) ff_tma_2d(w2s(s) + a * FF_W2_ATOM, &tmW2, BAR(6 + s), a * 64, j * FF_CH);
                }
            }
        }
        return;
    }

    // ===== consumer warpgroups: rows 64 wg .. 64 wg + 63 of every tile; this thread: rows r, r + 8 of the warp's 16 =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;" ::: "memory");
    const int wg = __shfl_sync(0xffffffffu, (warp >> 2) - 1, 0);   // warp-uniform to the compiler: keeps wgmma unserialized
    const int wq = warp & 3, q4 = lane & 3;
    const uint32_t xa = xs + wg * 64 * 128;
    float o[FF_C / 2];                                    // O [64 x 320]: element 4 i + 2 h + e at column 8 i + 2 q + e
    float sc[2 * FF_CH / 2];                              // S [64 x 64] of the current chunk, then its GEGLU values
    uint32_t pa[2][4];                                    // P of the previous chunk: the A fragments of its two k16 steps

    auto issue_s = [&](int s) {                           // S = x W1_chunk^T, k order 0 .. 319
#pragma unroll
        for (int i = 0; i < 2 * FF_CH / 2; ++i) sc[i] = 0.f;
        wg_fence();
#pragma unroll
        for (int k = 0; k < FF_C / 16; ++k)
            Wgmma<64>::ss(sc, wg_desc(xa + (k >> 2) * FF_X_ATOM + (k & 3) * 32, 16, 1024),
                          wg_desc(w1s(s) + (k >> 2) * FF_W1_ATOM + (k & 3) * 32, 16, 1024), 1);
        wg_commit();
    };
    auto issue_pv = [&](int s) {                          // O += P W2_chunk: columns 0..191 and 192..319, hidden units in order
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
            Wgmma<192>::rs_t(o, pa[kk], wg_desc(w2s(s) + kk * 2048, FF_W2_ATOM, 1024), 1);
            Wgmma<128>::rs_t(o + 96, pa[kk], wg_desc(w2s(s) + 3 * FF_W2_ATOM + kk * 2048, FF_W2_ATOM, 1024), 1);
        }
        wg_commit();
    };
    auto release = [&](int bar) {
        __syncwarp();
        if (lane == 0) ff_arrive(BAR(bar));
    };
    // bias + GEGLU of the completed S in place, in gemm_wgmma.cu's order: (acc + bias) + 0, then a * p_gelu(gate)
    auto geglu = [&](int j) {
#pragma unroll
        for (int i = 0; i < 2 * FF_CH / 2; ++i) wg_fence_regs(sc[i]);
        const float* b1 = s_b1 + j * 2 * FF_CH + 2 * q4;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float2 bb = *reinterpret_cast<const float2*>(b1 + 8 * i);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float a = sc[4 * i + 2 * h] + bb.x, g = sc[4 * i + 2 * h + 1] + bb.y;
                a += 0.f;
                g += 0.f;
                sc[4 * i + 2 * h] = a * p_gelu(g);
            }
        }
    };
    auto pack = [&]() {                                   // steps 4s .. 4s + 3 -> k16 step s (see the header comment)
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const float* t = sc + 16 * s;                 // GEGLU value of step i, row h at t[4 (i - 4 s) + 2 h]
            pa[s][0] = ff_pack(t[0], t[4]);
            pa[s][1] = ff_pack(t[2], t[6]);
            pa[s][2] = ff_pack(t[8], t[12]);
            pa[s][3] = ff_pack(t[10], t[14]);
        }
    };

    // Turn order: warpgroup 1 hands warpgroup 0 the CTA's first turn up front and passes no turn after its last one, so
    // every bar.sync meets exactly one bar.arrive.
    if (wg == 1) ff_turn_pass(wg);
    uint32_t c = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
#pragma unroll
        for (int i = 0; i < FF_C / 2; ++i) o[i] = 0.f;
        ff_wait(BAR(0), it & 1);
        // chunk 0: S alone
        ff_wait(BAR(2 + (c & 1)), (c >> 1) & 1);
        ff_turn_wait(wg);
        issue_s(c & 1);
        ff_turn_pass(wg);
        wg_wait<0>();
        release(4 + (c & 1));                             // ff1 rows of the chunk read
        geglu(0);
        pack();
        ++c;
        // chunks 1 ..: S of this chunk and P V of the previous one
        for (int j = 1; j < FF_NCH; ++j, ++c) {
            const int s = c & 1;
            ff_wait(BAR(2 + s), (c >> 1) & 1);
            ff_wait(BAR(6 + (s ^ 1)), ((c - 1) >> 1) & 1);
            ff_turn_wait(wg);
            issue_s(s);
            issue_pv(s ^ 1);
            ff_turn_pass(wg);
            wg_wait<1>();                                 // S done; P V of the previous chunk may still run
            release(4 + s);
            if (j == FF_NCH - 1) release(1);              // the x tile is read for the last time
            geglu(j);
            wg_wait<0>();
#pragma unroll
            for (int i = 0; i < FF_C / 2; ++i) wg_fence_regs(o[i]);
            release(8 + (s ^ 1));                         // W2^T rows of the previous chunk read
            pack();
        }
        const int sl = (c - 1) & 1;
        ff_wait(BAR(6 + sl), ((c - 1) >> 1) & 1);
        ff_turn_wait(wg);
        wg_fence();
        issue_pv(sl);
        if (wg == 0 || tile + (int)gridDim.x < p.num_tiles) ff_turn_pass(wg);
        wg_wait<0>();
#pragma unroll
        for (int i = 0; i < FF_C / 2; ++i) wg_fence_regs(o[i]);
        release(8 + sl);

        // ---- epilogue: (O + b2) + 0, + residual, one fp16 rounding (gemm_wgmma.cu's act-0 order) ----
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = tile * FF_BM + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
            if (m >= p.M) continue;
            const __half* rrow = p.residual + (size_t)m * p.ldr + 2 * q4;
            __half* orow = p.out + (size_t)m * p.ldo + 2 * q4;
            constexpr int G = 8;                          // residual loads in flight at once
#pragma unroll
            for (int i0 = 0; i0 < FF_C / 8; i0 += G) {
                __half2 rr[G];
#pragma unroll
                for (int u = 0; u < G; ++u) rr[u] = *reinterpret_cast<const __half2*>(rrow + 8 * (i0 + u));
#pragma unroll
                for (int u = 0; u < G; ++u) {
                    const int i = i0 + u;
                    const float2 bb = *reinterpret_cast<const float2*>(s_b2 + 8 * i + 2 * q4);
                    float v0 = o[4 * i + 2 * h] + bb.x, v1 = o[4 * i + 2 * h + 1] + bb.y;
                    v0 += 0.f;
                    v1 += 0.f;
                    const float2 r = __half22float2(rr[u]);
                    v0 += r.x;
                    v1 += r.y;
                    *reinterpret_cast<__half2*>(orow + 8 * i) = __floats2half2_rn(v0, v1);
                }
            }
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFnF)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFnF f_get_encode() {
    static EncodeTiledFnF fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qr) == cudaSuccess &&
            qr == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFnF)f;
    }
    return fn;
}
// 2-D fp16 map [rows, C] with row pitch ld, 64-column (128-byte, swizzled) box of box_rows rows
static bool f_map(CUtensorMap* tm, const void* ptr, uint64_t rows, uint64_t ld, uint32_t box_rows) {
    cuuint64_t dims[2] = {(cuuint64_t)FF_C, rows};
    cuuint64_t strides[1] = {ld * 2};
    cuuint32_t box[2] = {64, box_rows};
    cuuint32_t es[2] = {1, 1};
    return f_get_encode()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace anysd

using namespace anysd;

extern "C" int anysd_geglu_ff_f16(const void* x, int ldx, const void* w1, const float* b1, const void* w2t, const float* b2,
                                  const void* residual, int ldr, void* out, int ldo, int M, int C, int hidden,
                                  anysd_stream_t stream) {
    ANYSD_REQUIRE(x && w1 && b1 && w2t && residual && out, ANYSD_EINVAL, "geglu_ff: null pointer");
    ANYSD_REQUIRE(M > 0, ANYSD_EINVAL, "geglu_ff: bad M=%d", M);
    ANYSD_REQUIRE(C == FF_C && hidden == FF_HID, ANYSD_EUNSUPPORTED,
                  "geglu_ff: only C = %d with hidden = %d (got C=%d hidden=%d)", FF_C, FF_HID, C, hidden);
    ANYSD_REQUIRE(ldx >= C && ldr >= C && ldo >= C && ldx % 8 == 0 && ldr % 8 == 0 && ldo % 8 == 0, ANYSD_EINVAL,
                  "geglu_ff: ldx=%d ldr=%d ldo=%d must be multiples of 8 and >= C", ldx, ldr, ldo);
    ANYSD_REQUIRE(((uintptr_t)x % 16) == 0 && ((uintptr_t)w1 % 16) == 0 && ((uintptr_t)w2t % 16) == 0 &&
                      ((uintptr_t)residual % 16) == 0 && ((uintptr_t)out % 16) == 0 && ((uintptr_t)b1 % 16) == 0 &&
                      ((uintptr_t)b2 % 16) == 0,
                  ANYSD_EINVAL, "geglu_ff: x, w1, w2t, residual, out, b1, b2 must be 16-byte aligned");
    ANYSD_REQUIRE(f_get_encode() != nullptr, ANYSD_ECUDA, "geglu_ff: cuTensorMapEncodeTiled unavailable");
    CUtensorMap tmX, tmW1, tmW2;
    const bool ok = f_map(&tmX, x, (uint64_t)M, (uint64_t)ldx, FF_BM) && f_map(&tmW1, w1, 2 * FF_HID, FF_C, 2 * FF_CH) &&
                    f_map(&tmW2, w2t, FF_HID, FF_C, FF_CH);
    ANYSD_REQUIRE(ok, ANYSD_ECUDA, "geglu_ff: cuTensorMapEncodeTiled failed (M=%d)", M);
    static bool done[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(geglu_ff_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FF_SMEM);
        ANYSD_REQUIRE(e == cudaSuccess, ANYSD_ECUDA, "geglu_ff: smem opt-in failed: %s", cudaGetErrorString(e));
        done[dev] = true;
    }
    FfArgs a;
    a.b1 = b1;
    a.b2 = b2;
    a.residual = (const __half*)residual;
    a.out = (__half*)out;
    a.M = M;
    a.ldr = ldr;
    a.ldo = ldo;
    a.num_tiles = cdiv(M, FF_BM);
    int grid = sm_count();
    if (grid > a.num_tiles) grid = a.num_tiles;
    geglu_ff_wgmma_kernel<<<grid, FF_THREADS, FF_SMEM, (cudaStream_t)stream>>>(tmX, tmW1, tmW2, a);
    return check_launch("geglu_ff (wgmma)");
}
