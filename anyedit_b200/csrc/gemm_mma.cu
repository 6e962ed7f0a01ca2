// Dense / implicit-GEMM contraction, first-generation path: mma.sync m16n8k16 fed by a 4-stage
// cp.async pipeline with XOR-swizzled shared memory.  One template serves nn.Linear / 1x1 conv
// (dense A rows) and 3x3 conv (A gathered from the NHWC image: stride 1|2, optional nearest-x2
// upsample folded into the gather coordinates, zero-fill halo through cp.async src-size 0).
// Epilogue (fp32): + bias[n] + rowadd[m / rows_per_batch, n] -> x col_scale[n] -> activation | GEGLU | SwiGLU -> + residual
// -> fp16|fp32.
//
// This is the correctness baseline the wgmma kernel (gemm_wgmma.cu) is validated against;
// the dispatch in anysd_gemm_f16 prefers wgmma wherever its shape constraints hold.
#include "common.cuh"

namespace anysd {

constexpr int BM = 128, BN = 128, BK = 32, STAGES = 4, GEMM_THREADS = 256;
constexpr int A_STAGE_BYTES = BM * BK * 2, B_STAGE_BYTES = BN * BK * 2;
constexpr int GEMM_SMEM = STAGES * (A_STAGE_BYTES + B_STAGE_BYTES);

struct GemmArgs {
    const __half* A;
    const __half* W;
    const float* bias;
    const float* rowadd;
    const __half* residual;
    void* out;
    int M, N, K;
    int lda, ldw, ldo, ldr, ld_rowadd;
    int rows_per_batch;
    int act, out_f16;
    // conv
    int H, Wd, Cin, Ho, Wo, stride, up;
    const float* col_scale;
};

// byte offset of 16-byte chunk `cc` (0..3) of row `r` inside a [rows][32 halves] tile
__device__ __forceinline__ int swz(int r, int cc) { return r * 64 + ((cc ^ ((r >> 1) & 3)) << 4); }

template <bool CONV>
__global__ void __launch_bounds__(GEMM_THREADS, 2) gemm_mma_kernel(const GemmArgs p) {
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t sA = smem_u32(smem);
    const uint32_t sB = sA + STAGES * A_STAGE_BYTES;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 2, wn = warp & 3;          // 2 x 4 warps -> warp tile 64 x 32
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

    // ---- per-thread load assignment: rows (tid>>2) and (tid>>2)+64, 16B chunk (tid&3) -------
    const int lr = tid >> 2, lc = tid & 3;
    const __half* a_row[2];
    bool a_ok[2];
    int a_oy[2], a_ox[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int m = m0 + lr + i * 64;
        a_ok[i] = m < p.M;
        if (CONV) {
            const int mm = a_ok[i] ? m : 0;
            const int hw = p.Ho * p.Wo;
            const int img = mm / hw, rem = mm - img * hw;
            a_oy[i] = rem / p.Wo;
            a_ox[i] = rem - a_oy[i] * p.Wo;
            a_row[i] = p.A + (size_t)img * p.H * p.Wd * p.Cin;
        } else {
            a_row[i] = p.A + (size_t)(a_ok[i] ? m : 0) * p.lda;
            a_oy[i] = a_ox[i] = 0;
        }
    }
    const __half* b_row[2];
    bool b_ok[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int n = n0 + lr + i * 64;
        b_ok[i] = n < p.N;
        b_row[i] = p.W + (size_t)(b_ok[i] ? n : 0) * p.ldw;
    }
    const int KT = (p.K + BK - 1) / BK;

    auto load_stage = [&](int kt, int stage) {
        const int k = kt * BK + lc * 8;
        const bool k_ok = k < p.K;
        int dy = 0, dx = 0, ci = 0;
        if (CONV) {
            const int tap = k / p.Cin;
            ci = k - tap * p.Cin;
            dy = tap / 3;
            dx = tap - dy * 3;
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int r = lr + i * 64;
            const __half* src;
            bool ok = a_ok[i] && k_ok;
            if (CONV) {
                const int iy = a_oy[i] * p.stride + dy - 1, ix = a_ox[i] * p.stride + dx - 1;
                const int Hl = p.H << p.up, Wl = p.Wd << p.up;
                ok = ok && iy >= 0 && iy < Hl && ix >= 0 && ix < Wl;
                const int sy = ok ? (iy >> p.up) : 0, sx = ok ? (ix >> p.up) : 0;
                src = a_row[i] + ((size_t)sy * p.Wd + sx) * p.Cin + (ok ? ci : 0);
            } else {
                src = a_row[i] + (ok ? k : 0);
            }
            cp_async16(sA + stage * A_STAGE_BYTES + swz(r, lc), src, ok);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int r = lr + i * 64;
            const bool ok = b_ok[i] && k_ok;
            cp_async16(sB + stage * B_STAGE_BYTES + swz(r, lc), b_row[i] + (ok ? k : 0), ok);
        }
    };

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < KT) load_stage(s, s);
        cp_async_commit();
    }

    for (int kt = 0; kt < KT; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {
            const int nk = kt + STAGES - 1;
            if (nk < KT) load_stage(nk, nk % STAGES);
            cp_async_commit();
        }
        const int stage = kt % STAGES;
        const uint32_t aB = sA + stage * A_STAGE_BYTES, bB = sB + stage * B_STAGE_BYTES;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            uint32_t af[4][4], bf[4][2];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = wm * 64 + i * 16 + (lane & 15);
                const int cc = ks * 2 + (lane >> 4);
                ldmatrix_x4(af[i][0], af[i][1], af[i][2], af[i][3], aB + swz(r, cc));
            }
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int r = wn * 32 + j * 16 + (lane & 7) + ((lane >> 4) << 3);
                const int cc = ks * 2 + ((lane >> 3) & 1);
                ldmatrix_x4(bf[2 * j][0], bf[2 * j][1], bf[2 * j + 1][0], bf[2 * j + 1][1], bB + swz(r, cc));
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) mma_16816(acc[i][j], af[i], bf[j][0], bf[j][1]);
        }
    }
    cp_async_wait<0>();

    // ---- epilogue ---------------------------------------------------------------------------
    const int gid = lane >> 2, tig = lane & 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int m = m0 + wm * 64 + i * 16 + gid + hrow * 8;
            if (m >= p.M) continue;
            const float* radd = p.rowadd ? p.rowadd + (size_t)(m / p.rows_per_batch) * p.ld_rowadd : nullptr;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int n = n0 + wn * 32 + j * 8 + tig * 2;
                if (n >= p.N) continue;
                float v0 = acc[i][j][hrow * 2 + 0], v1 = acc[i][j][hrow * 2 + 1];
                const bool has1 = (n + 1) < p.N;
                if (p.bias) {
                    v0 += p.bias[n];
                    if (has1) v1 += p.bias[n + 1];
                }
                if (radd) {
                    v0 += radd[n];
                    if (has1) v1 += radd[n + 1];
                }
                if (p.col_scale) {
                    v0 *= p.col_scale[n];
                    if (has1) v1 *= p.col_scale[n + 1];
                }
                if (p.act == 2 || p.act == 5) {  // GEGLU / SwiGLU: (a, gate) interleaved -> one output column n/2
                    float o = v0 * (p.act == 5 ? silu_f(v1) : gelu_erf_f(v1));
                    const int no = n >> 1;
                    if (p.residual) o += __half2float(p.residual[(size_t)m * p.ldr + no]);
                    if (p.out_f16)
                        ((__half*)p.out)[(size_t)m * p.ldo + no] = __float2half_rn(o);
                    else
                        ((float*)p.out)[(size_t)m * p.ldo + no] = o;
                    continue;
                }
                if (p.act != 0) {
                    v0 = act_f(v0, p.act);
                    v1 = act_f(v1, p.act);
                }
                if (p.residual) {
                    const __half* rp = p.residual + (size_t)m * p.ldr + n;
                    v0 += __half2float(rp[0]);
                    if (has1) v1 += __half2float(rp[1]);
                }
                if (p.out_f16) {
                    __half* op = (__half*)p.out + (size_t)m * p.ldo + n;
                    if (has1 && ((((size_t)m * p.ldo + n) & 1) == 0)) {
                        *reinterpret_cast<__half2*>(op) = __floats2half2_rn(v0, v1);
                    } else {
                        op[0] = __float2half_rn(v0);
                        if (has1) op[1] = __float2half_rn(v1);
                    }
                } else {
                    float* op = (float*)p.out + (size_t)m * p.ldo + n;
                    op[0] = v0;
                    if (has1) op[1] = v1;
                }
            }
        }
    }
}

int launch_gemm_mma(const anysd_gemm_params* q, cudaStream_t st) {
    GemmArgs a;
    a.A = (const __half*)q->A;
    a.W = (const __half*)q->W;
    a.bias = q->bias;
    a.rowadd = q->rowadd;
    a.residual = (const __half*)q->residual;
    a.out = q->out;
    a.M = q->M; a.N = q->N; a.K = q->K;
    a.lda = q->lda; a.ldw = q->ldw; a.ldo = q->ldo; a.ldr = q->ldr; a.ld_rowadd = q->ld_rowadd;
    a.rows_per_batch = q->rows_per_batch > 0 ? q->rows_per_batch : 1;
    a.act = q->act;
    a.out_f16 = q->out_dtype == ANYSD_F16;
    a.col_scale = q->col_scale;
    a.H = q->H; a.Wd = q->Wd; a.Cin = q->Cin; a.stride = q->stride; a.up = q->upsample;
    a.Ho = a.Wo = 0;
    if (q->conv) {
        const int Hl = q->H << q->upsample, Wl = q->Wd << q->upsample;
        a.Ho = (Hl + 2 - 3) / q->stride + 1;
        a.Wo = (Wl + 2 - 3) / q->stride + 1;
    }
    static bool attr_done[64][2];   // per device (function attributes are per-device)
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    dim3 grid(cdiv(q->N, BN), cdiv(q->M, BM));
    if (q->conv) {
        if (!attr_done[dev][1]) {
            cudaFuncSetAttribute(gemm_mma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
            attr_done[dev][1] = true;
        }
        gemm_mma_kernel<true><<<grid, GEMM_THREADS, GEMM_SMEM, st>>>(a);
    } else {
        if (!attr_done[dev][0]) {
            cudaFuncSetAttribute(gemm_mma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
            attr_done[dev][0] = true;
        }
        gemm_mma_kernel<false><<<grid, GEMM_THREADS, GEMM_SMEM, st>>>(a);
    }
    return check_launch(q->conv ? "conv3x3 (mma.sync)" : "gemm (mma.sync)");
}

}  // namespace anysd
