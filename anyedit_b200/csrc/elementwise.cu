// Layout conversion, embedding and sampler-update kernels (HBM/latency-bound, no tensor cores).
#include "common.cuh"

namespace anysd {

// ---- NCHW (f32|f16) -> NHWC fp16 channel slice --------------------------------------------
template <typename T, bool ACC>
__global__ void nchw_to_nhwc_kernel(const T* __restrict__ src, __half* __restrict__ dst, int C, int HW,
                                    int dstC, int c_off) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const T* s = src + (size_t)n * C * HW;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int c = c0 + i, hw = hw0 + threadIdx.x;
        if (c < C && hw < HW) tile[i][threadIdx.x] = (float)s[(size_t)c * HW + hw];
    }
    __syncthreads();
    __half* d = dst + (size_t)n * HW * dstC + c_off;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int hw = hw0 + i, c = c0 + threadIdx.x;
        if (c < C && hw < HW) {
            float v = tile[threadIdx.x][i];
            if (ACC) v += __half2float(d[(size_t)hw * dstC + c]);
            d[(size_t)hw * dstC + c] = __float2half_rn(v);
        }
    }
}

template <typename S, typename T>
__global__ void nhwc_to_nchw_kernel(const S* __restrict__ src, T* __restrict__ dst, int C, int HW, int src_ld) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const S* s = src + (size_t)n * HW * src_ld;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int hw = hw0 + i, c = c0 + threadIdx.x;
        if (c < C && hw < HW) tile[i][threadIdx.x] = (float)s[(size_t)hw * src_ld + c];
    }
    __syncthreads();
    T* d = dst + (size_t)n * C * HW;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int c = c0 + i, hw = hw0 + threadIdx.x;
        if (c < C && hw < HW) d[(size_t)c * HW + hw] = (T)tile[threadIdx.x][i];
    }
}

__global__ void concat_kernel(const uint4* __restrict__ a, int va, const uint4* __restrict__ b, int vb,
                              uint4* __restrict__ dst, long long total) {
    const int vt = va + vb;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        long long r = i / vt;
        int c = (int)(i - r * vt);
        dst[i] = (c < va) ? a[r * va + c] : b[r * vb + (c - va)];
    }
}

// decoded image (NCHW fp32 in [-1, 1]) -> NHWC uint8, as diffusers post-processes it: round(clamp(x / 2 + 1/2, 0, 1) * 255),
// each step rounded to fp32 (no FMA) and the last one half to even, like numpy's round
__global__ void image_to_u8_kernel(const float* __restrict__ src, unsigned char* __restrict__ dst, int C, int HW, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long px = i / C;
        const int c = (int)(i - px * C);
        const long long img = px / HW;
        const int hw = (int)(px - img * HW);
        float t = __fadd_rn(__fmul_rn(src[(img * C + c) * HW + hw], 0.5f), 0.5f);
        t = fminf(fmaxf(t, 0.f), 1.f);
        dst[i] = (unsigned char)rintf(__fmul_rn(t, 255.f));
    }
}

__global__ void cast_kernel(const float* __restrict__ src, __half* __restrict__ dst, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        dst[i] = __float2half_rn(src[i]);
}

// ---- timestep embedding (util.py:154-174) --------------------------------------------------
__global__ void timestep_embedding_kernel(const void* __restrict__ t, int t_dtype, __half* __restrict__ out, int N,
                                          int dim, float neg_log_period) {
    const int half_dim = dim / 2;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * dim) return;
    const int n = idx / dim, j = idx - n * dim;
    float tv = (t_dtype == ANYSD_I64) ? (float)((const long long*)t)[n] : ((const float*)t)[n];
    float v = 0.f;
    if (j < 2 * half_dim) {
        int f = (j < half_dim) ? j : j - half_dim;
        // same operation order as the reference: exp((-ln P * f) / half), all fp32
        float freq = expf(__fdiv_rn(__fmul_rn(neg_log_period, (float)f), (float)half_dim));
        float arg = __fmul_rn(tv, freq);
        v = (j < half_dim) ? cosf(arg) : sinf(arg);
    }
    out[idx] = __float2half_rn(v);
}

__global__ void emb_finalize_kernel(const float* __restrict__ emb_lin, const float* __restrict__ table,
                                    const long long* __restrict__ idx, int table_rows, float* __restrict__ emb_out,
                                    __half* __restrict__ silu_out, int N, int D) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * D) return;
    const int n = i / D, j = i - n * D;
    float v = emb_lin[i];
    if (table != nullptr && idx != nullptr) {
        long long r = idx[n];
        if (r >= 0 && r < table_rows) v += table[r * D + j];
    }
    if (emb_out) emb_out[i] = v;
    if (silu_out) silu_out[i] = __float2half_rn(v / (1.0f + expf(-v)));
}

// ---- CFG combine + DDIM update (ddim.py:211-212, 228-250) -------------------------------------
__global__ void cfg_ddim_kernel(const float4* __restrict__ x, const float4* __restrict__ eps,
                                const float4* __restrict__ noise, const float* __restrict__ coef, float scale, int cfg, int vparam,
                                float4* __restrict__ x_prev, float4* __restrict__ pred_x0, long long n4_total,
                                long long n4_half) {
    const float c_somat = coef[0], c_sqrt_at = coef[1], c_sqrt_aprev = coef[2], c_dir = coef[3], c_sigma = coef[4];
    // v-parameterisation (ddim.py:214-218, 224-226; ddpm.py predict_eps_from_z_and_v / predict_start_from_z_and_v):
    // coef[5] = sqrt(acp[t]), coef[6] = sqrt(1 - acp[t]) of the DDPM timestep t the model was called with
    const float c_sacp = vparam ? coef[5] : 0.f, c_s1m = vparam ? coef[6] : 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4_total;
         i += (long long)gridDim.x * blockDim.x) {
        float4 xv = x[i];
        float4 eu = eps[i], ec = cfg ? eps[i + n4_half] : eu;
        float4 nz = (noise != nullptr) ? noise[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 p0, o;
        // explicit _rn intrinsics: no FMA contraction, so the update is bit-identical to the
        // reference's separate fp32 mul / add / div tensor ops given the same eps.
#define ANYSD_DDIM_LANE(f)                                                                          \
        {                                                                                               \
            float e = cfg ? __fadd_rn(eu.f, __fmul_rn(scale, __fsub_rn(ec.f, eu.f))) : eu.f;            \
            float p;                                                                                    \
            if (vparam) {                                                                               \
                const float v = e;                                                                      \
                e = __fadd_rn(__fmul_rn(c_sacp, v), __fmul_rn(c_s1m, xv.f));                            \
                p = __fsub_rn(__fmul_rn(c_sacp, xv.f), __fmul_rn(c_s1m, v));                            \
            } else {                                                                                    \
                p = __fdiv_rn(__fsub_rn(xv.f, __fmul_rn(c_somat, e)), c_sqrt_at);                       \
            }                                                                                           \
            float r = __fadd_rn(__fmul_rn(c_sqrt_aprev, p), __fmul_rn(c_dir, e));                       \
            if (noise != nullptr) r = __fadd_rn(r, __fmul_rn(c_sigma, nz.f));                           \
            p0.f = p;                                                                                   \
            o.f = r;                                                                                    \
        }
        ANYSD_DDIM_LANE(x) ANYSD_DDIM_LANE(y) ANYSD_DDIM_LANE(z) ANYSD_DDIM_LANE(w)
#undef ANYSD_DDIM_LANE
        x_prev[i] = o;
        if (pred_x0 != nullptr) pred_x0[i] = p0;
    }
}

// ---- InstructPix2Pix three-way guidance + DDIM update (tools/global_tool.py:166-177) ----------------------------
// eps = [text ; image ; uncond] thirds:  e = e_unc + s_txt (e_txt - e_img) + s_img (e_img - e_unc), then the same
// update as above; same evaluation order and _rn intrinsics as the reference's fp32 tensor expression.
__global__ void cfg3_ddim_kernel(const float4* __restrict__ x, const float4* __restrict__ eps, const float4* __restrict__ noise,
                                 const float* __restrict__ coef, float s_txt, float s_img, float4* __restrict__ x_prev,
                                 float4* __restrict__ pred_x0, long long n4) {
    const float c_somat = coef[0], c_sqrt_at = coef[1], c_sqrt_aprev = coef[2], c_dir = coef[3], c_sigma = coef[4];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 xv = x[i], et = eps[i], ei = eps[i + n4], eu = eps[i + 2 * n4];
        const float4 nz = (noise != nullptr) ? noise[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 p0, o;
#define ANYSD_DDIM3_LANE(f)                                                                                       \
        {                                                                                                             \
            float e = __fadd_rn(__fadd_rn(eu.f, __fmul_rn(s_txt, __fsub_rn(et.f, ei.f))), __fmul_rn(s_img, __fsub_rn(ei.f, eu.f))); \
            float p = __fdiv_rn(__fsub_rn(xv.f, __fmul_rn(c_somat, e)), c_sqrt_at);                                   \
            float r = __fadd_rn(__fmul_rn(c_sqrt_aprev, p), __fmul_rn(c_dir, e));                                     \
            if (noise != nullptr) r = __fadd_rn(r, __fmul_rn(c_sigma, nz.f));                                         \
            p0.f = p;                                                                                                 \
            o.f = r;                                                                                                  \
        }
        ANYSD_DDIM3_LANE(x) ANYSD_DDIM3_LANE(y) ANYSD_DDIM3_LANE(z) ANYSD_DDIM3_LANE(w)
#undef ANYSD_DDIM3_LANE
        x_prev[i] = o;
        if (pred_x0 != nullptr) pred_x0[i] = p0;
    }
}

// ---- PLMS step (ldm/models/diffusion/plms.py:178-244): CFG combine + linear-multistep eps + DDIM update ----------
// coef[10] = {sqrt(1-a_t), sqrt(a_t), sqrt(a_prev), sqrt(1-a_prev), c0, c1, c2, c3, den, push}:
//   e' = (((c0 e - c1 o1) + c2 o2) - c3 o3) / den       the reference's left-to-right evaluation of
//        (3e - o1)/2, (23e - 16 o1 + 5 o2)/12, (55e - 59 o1 + 37 o2 - 9 o3)/24   (plms.py:229-238)
//        [c = (1,0,0,0)/1: e' = e (first half of the pseudo improved Euler step, :226-228);  (1,-1,0,0)/2: (e + o1)/2]
//   pred_x0 = (x - sqrt(1-a_t) e') / sqrt(a_t);  x_prev = sqrt(a_prev) pred_x0 + sqrt(1-a_prev) e'   (:205-225, sigma = 0)
//   push != 0: the history (o1, o2, o3) <- (e, o1, o2)   (old_eps.append / pop, :170-172)
// _rn intrinsics (no FMA contraction): bit-identical to the reference's fp32 tensor expressions given the same eps.
__global__ void cfg_plms_kernel(const float4* __restrict__ x, const float4* __restrict__ eps, const float* __restrict__ coef, float scale,
                                int cfg, float4* __restrict__ hist, float4* __restrict__ x_prev, float4* __restrict__ pred_x0,
                                long long n4) {
    const float c_somat = coef[0], c_sqrt_at = coef[1], c_sqrt_aprev = coef[2], c_dir = coef[3];
    const float c0 = coef[4], c1 = coef[5], c2 = coef[6], c3 = coef[7], den = coef[8];
    const bool push = coef[9] != 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 xv = x[i], eu = eps[i], ec = cfg ? eps[i + n4] : eu;
        const float4 o1 = hist[i], o2 = hist[i + n4], o3 = hist[i + 2 * n4];
        float4 e4, p0, o;
#define ANYSD_PLMS_LANE(f)                                                                                                    \
        {                                                                                                                         \
            const float e = cfg ? __fadd_rn(eu.f, __fmul_rn(scale, __fsub_rn(ec.f, eu.f))) : eu.f;                                \
            float ep = __fsub_rn(__fmul_rn(c0, e), __fmul_rn(c1, o1.f));                                                          \
            ep = __fsub_rn(__fadd_rn(ep, __fmul_rn(c2, o2.f)), __fmul_rn(c3, o3.f));                                              \
            ep = __fdiv_rn(ep, den);                                                                                              \
            const float p = __fdiv_rn(__fsub_rn(xv.f, __fmul_rn(c_somat, ep)), c_sqrt_at);                                        \
            e4.f = e;                                                                                                             \
            p0.f = p;                                                                                                             \
            o.f = __fadd_rn(__fmul_rn(c_sqrt_aprev, p), __fmul_rn(c_dir, ep));                                                    \
        }
        ANYSD_PLMS_LANE(x) ANYSD_PLMS_LANE(y) ANYSD_PLMS_LANE(z) ANYSD_PLMS_LANE(w)
#undef ANYSD_PLMS_LANE
        x_prev[i] = o;
        if (pred_x0 != nullptr) pred_x0[i] = p0;
        if (push) {
            hist[i + 2 * n4] = o2;
            hist[i + n4] = o1;
            hist[i] = e4;
        }
    }
}

// ---- DPM-Solver++(2M) step (ldm/models/diffusion/dpm_solver/dpm_solver.py:352-365, 469-513, 723-778) ------------------
// coef[6] = {sigma_s, alpha_s, sigma_t/sigma_s, c, 0.5 c, 1/r0}  (s = the time of this model call, t = the next grid point):
//   m     = (x - sigma_s e) / alpha_s                                   data prediction at s
//   x_t   = ((sigma_t/sigma_s) x - c m) - (0.5 c) ((1/r0) (m - m_prev))      c = alpha_t (exp(-h) - 1)
//           [first-order steps pass c = alpha_t expm1(-h) and 0.5 c = 0: the update of :469-513]
//   m_prev <- m
__global__ void cfg_dpmpp_kernel(const float4* __restrict__ x, const float4* __restrict__ eps, const float* __restrict__ coef, float scale,
                                 int cfg, float4* __restrict__ m_prev, float4* __restrict__ x_next, float4* __restrict__ x0_out,
                                 long long n4) {
    const float sig = coef[0], alp = coef[1], ratio = coef[2], c = coef[3], half_c = coef[4], inv_r0 = coef[5];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 xv = x[i], eu = eps[i], ec = cfg ? eps[i + n4] : eu, mp = m_prev[i];
        float4 m4, o;
#define ANYSD_DPMPP_LANE(f)                                                                                                   \
        {                                                                                                                         \
            const float e = cfg ? __fadd_rn(eu.f, __fmul_rn(scale, __fsub_rn(ec.f, eu.f))) : eu.f;                                \
            const float m = __fdiv_rn(__fsub_rn(xv.f, __fmul_rn(sig, e)), alp);                                                   \
            const float d1 = __fmul_rn(inv_r0, __fsub_rn(m, mp.f));                                                               \
            m4.f = m;                                                                                                             \
            o.f = __fsub_rn(__fsub_rn(__fmul_rn(ratio, xv.f), __fmul_rn(c, m)), __fmul_rn(half_c, d1));                           \
        }
        ANYSD_DPMPP_LANE(x) ANYSD_DPMPP_LANE(y) ANYSD_DPMPP_LANE(z) ANYSD_DPMPP_LANE(w)
#undef ANYSD_DPMPP_LANE
        x_next[i] = o;
        m_prev[i] = m4;
        if (x0_out != nullptr) x0_out[i] = m4;
    }
}

// ---- task router gate (AnySD restatement, oracle/anysd_oracle.py): -------------------------------
// gate[b, l, :] = softmax_e(W[l, e, :] . table[idx[b], :] + bias[l, e]); one CTA per (layer, sample),
// one warp per expert logit: 16-byte weight loads, warp-shuffle dot-product reduction, fp32 softmax.
__global__ void router_gate_kernel(const float* __restrict__ table, const long long* __restrict__ idx, int table_rows,
                                   const __half* __restrict__ W, const float* __restrict__ bias,
                                   float* __restrict__ gate, int L, int E, int D) {
    extern __shared__ float s_logit[];
    const int l = blockIdx.x, b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    long long r = idx[b];
    if (r < 0 || r >= table_rows) r = 0;
    const float* te = table + r * D;
    for (int e = warp; e < E; e += nw) {
        const __half* w = W + ((size_t)l * E + e) * D;
        float acc = 0.f;
        for (int k = lane * 8; k < D; k += 32 * 8) {
            uint4 u = __ldg(reinterpret_cast<const uint4*>(w + k));
            float f[8];
            unpack8(u, f);
            const float4 t0 = __ldg(reinterpret_cast<const float4*>(te + k));
            const float4 t1 = __ldg(reinterpret_cast<const float4*>(te + k + 4));
            acc += f[0] * t0.x + f[1] * t0.y + f[2] * t0.z + f[3] * t0.w + f[4] * t1.x + f[5] * t1.y + f[6] * t1.z +
                   f[7] * t1.w;
        }
        acc = warp_sum(acc);
        if (lane == 0) s_logit[e] = acc + bias[l * E + e];
    }
    __syncthreads();
    if (warp == 0) {
        float m = -INFINITY;
        for (int e = lane; e < E; e += 32) m = fmaxf(m, s_logit[e]);
        m = warp_max(m);
        float sum = 0.f;
        for (int e = lane; e < E; e += 32) sum += expf(s_logit[e] - m);
        sum = warp_sum(sum);
        for (int e = lane; e < E; e += 32) gate[((size_t)b * L + l) * E + e] = expf(s_logit[e] - m) / sum;
    }
}

}  // namespace anysd

using namespace anysd;

extern "C" {

int anysd_nchw_to_nhwc_f16(const void* src, int src_dtype, void* dst, int N, int C, int H, int W, int dst_C,
                           int dst_c_off, anysd_stream_t stream) {
    ANYSD_REQUIRE(src && dst, ANYSD_EINVAL, "nchw_to_nhwc: null pointer");
    ANYSD_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && dst_c_off >= 0 && dst_c_off + C <= dst_C, ANYSD_EINVAL,
                  "nchw_to_nhwc: bad shape N=%d C=%d H=%d W=%d dstC=%d off=%d", N, C, H, W, dst_C, dst_c_off);
    ANYSD_REQUIRE(src_dtype == ANYSD_F32 || src_dtype == ANYSD_F16, ANYSD_EINVAL, "nchw_to_nhwc: bad dtype");
    const int HW = H * W;
    dim3 grid(cdiv(HW, 32), cdiv(C, 32), N), block(32, 8);
    if (src_dtype == ANYSD_F32)
        nchw_to_nhwc_kernel<float, false><<<grid, block, 0, (cudaStream_t)stream>>>((const float*)src, (__half*)dst, C, HW,
                                                                                   dst_C, dst_c_off);
    else
        nchw_to_nhwc_kernel<__half, false><<<grid, block, 0, (cudaStream_t)stream>>>((const __half*)src, (__half*)dst, C, HW,
                                                                                    dst_C, dst_c_off);
    return check_launch("nchw_to_nhwc");
}

int anysd_add_nchw_into_nhwc_f16(const void* src, int src_dtype, void* dst, int N, int C, int H, int W,
                                 anysd_stream_t stream) {
    ANYSD_REQUIRE(src && dst && N > 0 && C > 0 && H > 0 && W > 0, ANYSD_EINVAL, "add_nchw_into_nhwc: bad args");
    ANYSD_REQUIRE(src_dtype == ANYSD_F32 || src_dtype == ANYSD_F16, ANYSD_EINVAL, "add_nchw_into_nhwc: bad dtype");
    const int HW = H * W;
    dim3 grid(cdiv(HW, 32), cdiv(C, 32), N), block(32, 8);
    if (src_dtype == ANYSD_F32)
        nchw_to_nhwc_kernel<float, true><<<grid, block, 0, (cudaStream_t)stream>>>((const float*)src, (__half*)dst, C, HW, C, 0);
    else
        nchw_to_nhwc_kernel<__half, true><<<grid, block, 0, (cudaStream_t)stream>>>((const __half*)src, (__half*)dst, C, HW, C, 0);
    return check_launch("add_nchw_into_nhwc");
}

int anysd_nhwc_to_nchw(const void* src, int src_dtype, int src_C, void* dst, int dst_dtype, int N, int C, int H, int W,
                       anysd_stream_t stream) {
    ANYSD_REQUIRE(src && dst, ANYSD_EINVAL, "nhwc_to_nchw: null pointer");
    ANYSD_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && src_C >= C, ANYSD_EINVAL, "nhwc_to_nchw: bad shape");
    ANYSD_REQUIRE((dst_dtype == ANYSD_F32 || dst_dtype == ANYSD_F16) && (src_dtype == ANYSD_F32 || src_dtype == ANYSD_F16),
                  ANYSD_EINVAL, "nhwc_to_nchw: bad dtype");
    const int HW = H * W;
    dim3 grid(cdiv(HW, 32), cdiv(C, 32), N), block(32, 8);
    cudaStream_t st = (cudaStream_t)stream;
    if (src_dtype == ANYSD_F16 && dst_dtype == ANYSD_F32)
        nhwc_to_nchw_kernel<__half, float><<<grid, block, 0, st>>>((const __half*)src, (float*)dst, C, HW, src_C);
    else if (src_dtype == ANYSD_F16)
        nhwc_to_nchw_kernel<__half, __half><<<grid, block, 0, st>>>((const __half*)src, (__half*)dst, C, HW, src_C);
    else if (dst_dtype == ANYSD_F32)
        nhwc_to_nchw_kernel<float, float><<<grid, block, 0, st>>>((const float*)src, (float*)dst, C, HW, src_C);
    else
        nhwc_to_nchw_kernel<float, __half><<<grid, block, 0, st>>>((const float*)src, (__half*)dst, C, HW, src_C);
    return check_launch("nhwc_to_nchw");
}

int anysd_concat_channels_f16(const void* a, int Ca, const void* b, int Cb, void* dst, long long rows,
                              anysd_stream_t stream) {
    ANYSD_REQUIRE(a && b && dst && rows > 0, ANYSD_EINVAL, "concat: null pointer / rows");
    ANYSD_REQUIRE(Ca > 0 && Cb > 0 && Ca % 8 == 0 && Cb % 8 == 0, ANYSD_EINVAL,
                  "concat: channel counts must be positive multiples of 8 (got %d, %d)", Ca, Cb);
    long long total = rows * ((Ca + Cb) / 8);
    int grid = (int)((total + 255) / 256);
    if (grid > sm_count() * 16) grid = sm_count() * 16;
    concat_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint4*)a, Ca / 8, (const uint4*)b, Cb / 8,
                                                          (uint4*)dst, total);
    return check_launch("concat");
}

int anysd_cast_f32_to_f16(const float* src, void* dst, long long n, anysd_stream_t stream) {
    ANYSD_REQUIRE(src && dst && n > 0, ANYSD_EINVAL, "cast: bad args");
    int grid = (int)((n + 255) / 256);
    if (grid > sm_count() * 16) grid = sm_count() * 16;
    cast_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, (__half*)dst, n);
    return check_launch("cast");
}

int anysd_image_to_u8(const float* src, void* dst, int N, int C, int H, int W, anysd_stream_t stream) {
    ANYSD_REQUIRE(src && dst && N > 0 && C > 0 && H > 0 && W > 0, ANYSD_EINVAL, "image_to_u8: bad args");
    const long long n = (long long)N * C * H * W;
    int grid = (int)((n + 255) / 256);
    if (grid > sm_count() * 16) grid = sm_count() * 16;
    image_to_u8_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, (unsigned char*)dst, C, H * W, n);
    return check_launch("image_to_u8");
}

int anysd_timestep_embedding_f16(const void* t, int t_dtype, void* out, int N, int dim, float max_period,
                                 anysd_stream_t stream) {
    ANYSD_REQUIRE(t && out && N > 0 && dim > 1, ANYSD_EINVAL, "timestep_embedding: bad args");
    ANYSD_REQUIRE(t_dtype == ANYSD_I64 || t_dtype == ANYSD_F32, ANYSD_EINVAL, "timestep_embedding: bad dtype");
    const float neg_log = -(float)log((double)max_period);
    timestep_embedding_kernel<<<cdiv((long long)N * dim, 256), 256, 0, (cudaStream_t)stream>>>(
        t, t_dtype, (__half*)out, N, dim, neg_log);
    return check_launch("timestep_embedding");
}

int anysd_emb_finalize(const float* emb_lin, const float* table, const long long* idx, int table_rows,
                       float* emb_out, void* silu_out, int N, int D, anysd_stream_t stream) {
    ANYSD_REQUIRE(emb_lin && N > 0 && D > 0, ANYSD_EINVAL, "emb_finalize: bad args");
    ANYSD_REQUIRE((table == nullptr) == (idx == nullptr), ANYSD_EINVAL,
                  "emb_finalize: table and idx must be given together");
    emb_finalize_kernel<<<cdiv((long long)N * D, 256), 256, 0, (cudaStream_t)stream>>>(
        emb_lin, table, idx, table_rows, emb_out, (__half*)silu_out, N, D);
    return check_launch("emb_finalize");
}

int anysd_cfg_ddim_step_f32(const float* x, const float* eps, const float* noise, const float* coef,
                            float guidance_scale, int cfg, int v_param, float* x_prev, float* pred_x0, long long n_per_batch,
                            int B, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && eps && coef && x_prev && B > 0 && n_per_batch > 0, ANYSD_EINVAL, "cfg_ddim_step: bad args");
    long long total = n_per_batch * B;
    ANYSD_REQUIRE(total % 4 == 0, ANYSD_EINVAL, "cfg_ddim_step: B*C*H*W must be a multiple of 4");
    long long n4 = total / 4;
    int grid = (int)((n4 + 255) / 256);
    if (grid > sm_count() * 8) grid = sm_count() * 8;
    cfg_ddim_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const float4*)x, (const float4*)eps,
                                                            (const float4*)noise, coef, guidance_scale, cfg, v_param,
                                                            (float4*)x_prev, (float4*)pred_x0, n4, n4);
    return check_launch("cfg_ddim_step");
}

int anysd_cfg3_ddim_step_f32(const float* x, const float* eps, const float* noise, const float* coef, float text_scale,
                             float image_scale, float* x_prev, float* pred_x0, long long n_per_batch, int B, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && eps && coef && x_prev && B > 0 && n_per_batch > 0, ANYSD_EINVAL, "cfg3_ddim_step: bad args");
    long long total = n_per_batch * B;
    ANYSD_REQUIRE(total % 4 == 0, ANYSD_EINVAL, "cfg3_ddim_step: B*C*H*W must be a multiple of 4");
    long long n4 = total / 4;
    int grid = (int)((n4 + 255) / 256);
    if (grid > sm_count() * 8) grid = sm_count() * 8;
    cfg3_ddim_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const float4*)x, (const float4*)eps, (const float4*)noise, coef, text_scale,
                                                            image_scale, (float4*)x_prev, (float4*)pred_x0, n4);
    return check_launch("cfg3_ddim_step");
}

int anysd_cfg_plms_step_f32(const float* x, const float* eps, const float* coef, float guidance_scale, int cfg, float* hist,
                            float* x_prev, float* pred_x0, long long n_per_batch, int B, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && eps && coef && hist && x_prev && B > 0 && n_per_batch > 0, ANYSD_EINVAL, "cfg_plms_step: bad args");
    long long total = n_per_batch * B;
    ANYSD_REQUIRE(total % 4 == 0, ANYSD_EINVAL, "cfg_plms_step: B*C*H*W must be a multiple of 4");
    long long n4 = total / 4;
    int grid = (int)((n4 + 255) / 256);
    if (grid > sm_count() * 8) grid = sm_count() * 8;
    cfg_plms_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const float4*)x, (const float4*)eps, coef, guidance_scale, cfg, (float4*)hist,
                                                            (float4*)x_prev, (float4*)pred_x0, n4);
    return check_launch("cfg_plms_step");
}

int anysd_cfg_dpmpp_step_f32(const float* x, const float* eps, const float* coef, float guidance_scale, int cfg, float* m_prev,
                             float* x_next, float* x0_out, long long n_per_batch, int B, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && eps && coef && m_prev && x_next && B > 0 && n_per_batch > 0, ANYSD_EINVAL, "cfg_dpmpp_step: bad args");
    long long total = n_per_batch * B;
    ANYSD_REQUIRE(total % 4 == 0, ANYSD_EINVAL, "cfg_dpmpp_step: B*C*H*W must be a multiple of 4");
    long long n4 = total / 4;
    int grid = (int)((n4 + 255) / 256);
    if (grid > sm_count() * 8) grid = sm_count() * 8;
    cfg_dpmpp_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const float4*)x, (const float4*)eps, coef, guidance_scale, cfg, (float4*)m_prev,
                                                             (float4*)x_next, (float4*)x0_out, n4);
    return check_launch("cfg_dpmpp_step");
}

int anysd_router_gate_f32(const float* table, const long long* idx, int table_rows, const void* W, const float* bias,
                          float* gate, int B, int L, int E, int D, anysd_stream_t stream) {
    ANYSD_REQUIRE(table && idx && W && bias && gate, ANYSD_EINVAL, "router_gate: null pointer");
    ANYSD_REQUIRE(B > 0 && L > 0 && E > 0 && E <= 1024 && D > 0 && D % 8 == 0 && B <= 65535, ANYSD_EINVAL,
                  "router_gate: bad sizes B=%d L=%d E=%d D=%d (D must be a multiple of 8)", B, L, E, D);
    int warps = E < 8 ? E : 8;
    router_gate_kernel<<<dim3(L, B), warps * 32, E * sizeof(float), (cudaStream_t)stream>>>(
        table, idx, table_rows, (const __half*)W, bias, gate, L, E, D);
    return check_launch("router_gate");
}
}
