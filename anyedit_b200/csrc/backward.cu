// Backward / training-step kernels (SURVEY.md a24; train.py:629-710).  First correct generation: simple, HBM- or
// latency-bound elementwise and reduction kernels; every contraction of the backward pass reuses anysd_gemm_f16 with
// transposed / rotated weight packs (host side), attention has its own file (attention_bwd.cu).
// Activation gradients are fp16 (the caller scales the loss), statistics and parameter gradients fp32.
#include <cooperative_groups.h>
#include <math.h>

#include "common.cuh"

namespace anysd {

__device__ __forceinline__ float sigmoid_f(float v) { return 1.0f / (1.0f + __expf(-v)); }
__device__ __forceinline__ float silu_grad_f(float z) {                 // d/dz z*sigmoid(z)
    const float s = sigmoid_f(z);
    return s * (1.0f + z * (1.0f - s));
}

// ---- GEGLU (attention.py:49-56), pre = interleaved (a_j, gate_j) ------------------------------------------------
__global__ void geglu_fwd_kernel(const uint4* __restrict__ pre, uint4* __restrict__ out, long long nvec) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        float f0[8], f1[8], o[8];
        unpack8(__ldg(pre + 2 * i), f0);
        unpack8(__ldg(pre + 2 * i + 1), f1);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            o[j] = f0[2 * j] * gelu_erf_f(f0[2 * j + 1]);
            o[4 + j] = f1[2 * j] * gelu_erf_f(f1[2 * j + 1]);
        }
        out[i] = pack8(o);
    }
}
__device__ __forceinline__ void geglu_grad(float a, float g, float dy, float& da, float& dg) {
    const float cdf = 0.5f * (1.0f + erff(g * 0.70710678118654752440f));
    const float pdf = 0.39894228040143267794f * __expf(-0.5f * g * g);
    da = dy * g * cdf;
    dg = dy * a * (cdf + g * pdf);
}
__global__ void geglu_bwd_kernel(const uint4* __restrict__ pre, const uint4* __restrict__ dout, uint4* __restrict__ dpre,
                                 long long nvec) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        float f0[8], f1[8], dy[8], d0[8], d1[8];
        unpack8(__ldg(pre + 2 * i), f0);
        unpack8(__ldg(pre + 2 * i + 1), f1);
        unpack8(__ldg(dout + i), dy);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            geglu_grad(f0[2 * j], f0[2 * j + 1], dy[j], d0[2 * j], d0[2 * j + 1]);
            geglu_grad(f1[2 * j], f1[2 * j + 1], dy[4 + j], d1[2 * j], d1[2 * j + 1]);
        }
        dpre[2 * i] = pack8(d0);
        dpre[2 * i + 1] = pack8(d1);
    }
}

__global__ void silu_bwd_f32_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        dx[i] = dy[i] * silu_grad_f(x[i]);
}

// ---- GroupNorm(+SiLU) backward ---------------------------------------------------------------------------------
// y = [silu](z), z = xhat * gamma + beta, xhat = (x - mean) * rstd over the group's HW x cpg elements:
//   dz = dy * silu'(z);  w = dz * gamma;  dx = rstd * (w - mean(w) - xhat * mean(w * xhat))
// One thread-block CLUSTER per (image, span of `gpc` whole groups that is also a whole number of 16-byte channel vectors); the
// cluster's CS CTAs split the HW rows, each with VC = gpc*cpg/8 vector columns x RL row lanes.  Four passes over the slab
// (mean; centred squares; the two sums; dx), the slab stays in L2.  Per-channel partials are folded over the row lanes in smem, then per
// group, then over the cluster through distributed shared memory in rank order (deterministic).  One CTA per slab would leave
// the 64x64 level at 128 CTAs with one 16-byte load in flight per thread.
constexpr int GNB_THREADS = 256;
__global__ void __launch_bounds__(GNB_THREADS) gn_bwd_kernel(const __half* __restrict__ x1, int C1, const __half* __restrict__ x2, int C2,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             const __half* __restrict__ dy, __half* __restrict__ dx, int HW, int cpg,
                                                             int gpc, float eps, int fuse_silu, int CS) {
    extern __shared__ float gsm[];                 // [2][RL][VC*8] partials | per group 4 floats | per group 2 cluster partials
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    const int crank = CS > 1 ? (int)cluster.block_rank() : 0;
    const int n = blockIdx.y;
    const int C = C1 + C2;
    const int VC = gpc * cpg / 8, CW = VC * 8;     // channel vectors / channels of this CTA
    const int c_base = (blockIdx.x / CS) * CW;
    const int rows_per = (HW + CS - 1) / CS;
    const int row_lo = crank * rows_per, row_hi = min(HW, row_lo + rows_per);
    const int RL = GNB_THREADS / VC;
    const int vl = threadIdx.x % VC, rl = threadIdx.x / VC;
    const bool active = rl < RL;
    float* part = gsm;                             // [2][RL][CW]
    float* grp = gsm + 2 * RL * CW;                // [gpc][4]: mean, rstd, mean(w), mean(w*xhat)
    float* cpart = grp + 4 * gpc;                  // [gpc][2]: this CTA's raw sums, read by the whole cluster
    const int c0 = c_base + vl * 8;                // first channel of this thread's vector (a vector never straddles x1|x2: C1 % 8 == 0)
    const bool first = c0 < C1;
    const __half* xb = first ? x1 + (size_t)n * HW * C1 + c0 : x2 + (size_t)n * HW * C2 + (c0 - C1);
    const int xs = first ? C1 : C2;
    const __half* dyb = dy + (size_t)n * HW * C + c0;
    __half* dxb = dx + (size_t)n * HW * C + c0;
    const float inv_cnt = 1.0f / ((float)HW * cpg);

    auto fold = [&](const float* a8, const float* b8, int slot_a, int slot_b) {
        // per-thread 8-channel partials -> per-group means into grp[g][slot_a / slot_b]
        __syncthreads();
        if (active) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                part[(0 * RL + rl) * CW + vl * 8 + j] = a8[j];
                part[(1 * RL + rl) * CW + vl * 8 + j] = b8[j];
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * CW; i += GNB_THREADS) {
            const int which = i / CW, c = i - which * CW;
            float t = 0.f;
            for (int r = 0; r < RL; ++r) t += part[(which * RL + r) * CW + c];
            part[(which * RL) * CW + c] = t;
        }
        __syncthreads();
        if (threadIdx.x < gpc) {
            float ta = 0.f, tb = 0.f;
            for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c) {
                ta += part[c];
                tb += part[RL * CW + c];
            }
            if (CS > 1) {
                cpart[threadIdx.x * 2] = ta;
                cpart[threadIdx.x * 2 + 1] = tb;
            } else {
                grp[threadIdx.x * 4 + slot_a] = ta * inv_cnt;
                grp[threadIdx.x * 4 + slot_b] = tb * inv_cnt;
            }
        }
        if (CS > 1) {
            cluster.sync();                        // every CTA's raw sums are in its own shared memory
            if (threadIdx.x < gpc) {
                float ta = 0.f, tb = 0.f;
                for (int rk = 0; rk < CS; ++rk) {  // rank order: the same sum in every CTA, whatever finishes first
                    const float* rp = cluster.map_shared_rank(cpart, rk);
                    ta += rp[threadIdx.x * 2];
                    tb += rp[threadIdx.x * 2 + 1];
                }
                grp[threadIdx.x * 4 + slot_a] = ta * inv_cnt;
                grp[threadIdx.x * 4 + slot_b] = tb * inv_cnt;
            }
            cluster.sync();                        // nobody overwrites its partials while a neighbour still reads them
        } else {
            __syncthreads();
        }
    };

    float a8[8], b8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a8[j] = b8[j] = 0.f;
    if (active)
#pragma unroll 4
        for (int r = row_lo + rl; r < row_hi; r += RL) {
            float f[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(xb + (size_t)r * xs)), f);
#pragma unroll
            for (int j = 0; j < 8; ++j) a8[j] += f[j];
        }
    fold(a8, b8, 0, 1);                            // slot 0: mean (b8 is zero; slot 1 is rewritten below)
    float mean8[8], rstd8[8], g8[8], be8[8];
    if (active) {
#pragma unroll
        for (int j = 0; j < 8; ++j) mean8[j] = grp[((vl * 8 + j) / cpg) * 4];
    }
    // Two-pass variance from centred squares: E[x^2] - mean^2 in fp32 loses about kappa = E[x^2] / var ulps, which a group with
    // a DC offset of 64 sigma (kappa = 4096) turns into a visible error in rstd and hence in dx.
#pragma unroll
    for (int j = 0; j < 8; ++j) a8[j] = 0.f;
    if (active)
#pragma unroll 4
        for (int r = row_lo + rl; r < row_hi; r += RL) {
            float f[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(xb + (size_t)r * xs)), f);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float d = f[j] - mean8[j];
                a8[j] = fmaf(d, d, a8[j]);
            }
        }
    fold(a8, b8, 1, 2);                            // slot 1: variance (slot 2 is rewritten by the next fold)
    if (threadIdx.x < gpc) grp[threadIdx.x * 4 + 1] = rsqrtf(grp[threadIdx.x * 4 + 1] + eps);
    __syncthreads();
    if (active) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int gl = (vl * 8 + j) / cpg;
            rstd8[j] = grp[gl * 4 + 1];
            g8[j] = gamma[c0 + j];
            be8[j] = beta[c0 + j];
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) a8[j] = b8[j] = 0.f;
    if (active)
#pragma unroll 4
        for (int r = row_lo + rl; r < row_hi; r += RL) {
            float f[8], d[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(xb + (size_t)r * xs)), f);
            unpack8(__ldg(reinterpret_cast<const uint4*>(dyb + (size_t)r * C)), d);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float xh = (f[j] - mean8[j]) * rstd8[j];
                float dd = d[j];
                if (fuse_silu) dd *= silu_grad_f(xh * g8[j] + be8[j]);
                const float w = dd * g8[j];
                a8[j] += w;
                b8[j] += w * xh;
            }
        }
    fold(a8, b8, 2, 3);
    if (active) {
        float mw8[8], mwx8[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int gl = (vl * 8 + j) / cpg;
            mw8[j] = grp[gl * 4 + 2];
            mwx8[j] = grp[gl * 4 + 3];
        }
#pragma unroll 4
        for (int r = row_lo + rl; r < row_hi; r += RL) {
            float f[8], d[8], o[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(xb + (size_t)r * xs)), f);
            unpack8(__ldg(reinterpret_cast<const uint4*>(dyb + (size_t)r * C)), d);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float xh = (f[j] - mean8[j]) * rstd8[j];
                float dd = d[j];
                if (fuse_silu) dd *= silu_grad_f(xh * g8[j] + be8[j]);
                o[j] = rstd8[j] * (dd * g8[j] - mw8[j] - xh * mwx8[j]);
            }
            *reinterpret_cast<uint4*>(dxb + (size_t)r * C) = pack8(o);
        }
    }
}

// ---- LayerNorm backward: one warp per token row ----------------------------------------------------------------
__global__ void __launch_bounds__(256) ln_bwd_kernel(const uint4* __restrict__ x, const float* __restrict__ gamma,
                                                     const uint4* __restrict__ dy, uint4* __restrict__ dx, long long M, int CV,
                                                     float eps) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= M) return;
    const int lane = threadIdx.x & 31;
    const uint4* xr = x + row * CV;
    const uint4* dr = dy + row * CV;
    const float inv_c = 1.0f / (CV * 8);
    float s = 0.f;
    for (int v = lane; v < CV; v += 32) {
        float f[8];
        unpack8(__ldg(xr + v), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += f[j];
    }
    const float mean = warp_sum(s) * inv_c;
    float q = 0.f;
    for (int v = lane; v < CV; v += 32) {
        float f[8];
        unpack8(__ldg(xr + v), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) q += (f[j] - mean) * (f[j] - mean);
    }
    const float rstd = rsqrtf(warp_sum(q) * inv_c + eps);
    float a = 0.f, b = 0.f;
    for (int v = lane; v < CV; v += 32) {
        float f[8], d[8];
        unpack8(__ldg(xr + v), f);
        unpack8(__ldg(dr + v), d);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float w = d[j] * gamma[v * 8 + j];
            a += w;
            b += w * (f[j] - mean) * rstd;
        }
    }
    const float mw = warp_sum(a) * inv_c, mwx = warp_sum(b) * inv_c;
    for (int v = lane; v < CV; v += 32) {
        float f[8], d[8], o[8];
        unpack8(__ldg(xr + v), f);
        unpack8(__ldg(dr + v), d);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float xh = (f[j] - mean) * rstd;
            o[j] = rstd * (d[j] * gamma[v * 8 + j] - mw - xh * mwx);
        }
        dx[row * CV + v] = pack8(o);
    }
}

// ---- per-image column sums: x [N, rows, C] fp16 -> out [N, ld_out] fp32 (time-embedding row add backward) ---------
__global__ void __launch_bounds__(256) colsum_kernel(const uint4* __restrict__ x, float* __restrict__ out, int rows, int CV, int ld_out,
                                                     int accumulate) {
    __shared__ float sm[32][8 * 8 + 1];
    const int n = blockIdx.y;
    const int cvl = threadIdx.x & 7, rl = threadIdx.x >> 3;       // 8 vector columns x 32 row lanes
    const int cv = blockIdx.x * 8 + cvl;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (cv < CV) {
        for (int r = rl; r < rows; r += 32) {
            float f[8];
            unpack8(__ldg(x + ((size_t)n * rows + r) * CV + cv), f);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] += f[j];
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sm[rl][cvl * 8 + j] = acc[j];
    __syncthreads();
    if (threadIdx.x < 64) {
        float t = 0.f;
        for (int r = 0; r < 32; ++r) t += sm[r][threadIdx.x];
        const int c = blockIdx.x * 64 + threadIdx.x;
        if (c < CV * 8) {
            float* o = out + (size_t)n * ld_out + c;
            *o = accumulate ? *o + t : t;
        }
    }
}

__global__ void add_f16_kernel(uint4* __restrict__ y, const uint4* __restrict__ x, long long nvec) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        float a[8], b[8];
        unpack8(y[i], a);
        unpack8(__ldg(x + i), b);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] += b[j];
        y[i] = pack8(a);
    }
}

__global__ void split_kernel(const uint4* __restrict__ src, uint4* __restrict__ a, int ca, uint4* __restrict__ b, int cb, long long total) {
    const int cv = ca + cb;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / cv;
        const int c = (int)(i - row * cv);
        const uint4 v = __ldg(src + i);
        if (c < ca) a[row * ca + c] = v;
        else b[row * cb + (c - ca)] = v;
    }
}

// dst [N, 2H, 2W, C]: dst[2y, 2x] = src[y, x], zero elsewhere (backward of a stride-2 conv = conv over this)
__global__ void zero_insert2x_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int H, int W, int CV, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % CV);
        long long t = i / CV;
        const int x = (int)(t % (2 * W));
        t /= 2 * W;
        const int y = (int)(t % (2 * H));
        const long long n = t / (2 * H);
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (!(x & 1) && !(y & 1)) v = __ldg(src + ((n * H + (y >> 1)) * W + (x >> 1)) * CV + c);
        dst[i] = v;
    }
}
// dst [N, H, W, C] = sum of the 2x2 block of src [N, 2H, 2W, C] (backward of nearest x2)
__global__ void sumpool2x_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int H, int W, int CV, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % CV);
        long long t = i / CV;
        const int x = (int)(t % W);
        t /= W;
        const int y = (int)(t % H);
        const long long n = t / H;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                float f[8];
                unpack8(__ldg(src + ((n * 2 * H + 2 * y + dy) * (2 * W) + 2 * x + dx) * CV + c), f);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += f[j];
            }
        dst[i] = pack8(acc);
    }
}

// ---- loss (train.py:696) ----------------------------------------------------------------------------------------
// pred, target fp32 NCHW [N, C, HW]; loss += mean((pred - target)^2); dpred NHWC fp16 [N, HW, Cpad] =
// grad_scale * 2 (pred - target) / numel, zero in the padding channels.  Two-stage deterministic sum: partial[blk].
__global__ void __launch_bounds__(256) mse_kernel(const float* __restrict__ pred, const float* __restrict__ target, int N, int C, int HW,
                                                  int Cpad, float grad_scale, const float* __restrict__ scale_dev, __half* __restrict__ dpred,
                                                  float* __restrict__ partial) {
    const long long numel = (long long)N * C * HW;
    const float k = grad_scale * (scale_dev ? *scale_dev : 1.0f) * 2.0f / (float)numel;
    float acc = 0.f;
    const long long pix = (long long)N * HW;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < pix; i += (long long)gridDim.x * blockDim.x) {
        const long long n = i / HW, hw = i - n * HW;
        for (int c = 0; c < Cpad; ++c) {
            float d = 0.f;
            if (c < C) {
                const long long idx = (n * C + c) * HW + hw;
                d = pred[idx] - target[idx];
                acc += d * d;
            }
            dpred[i * Cpad + c] = __float2half_rn(k * d);
        }
    }
    __shared__ float red[8];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += red[w];
        partial[blockIdx.x] = t / (float)numel;
    }
}
__global__ void sum_partials_kernel(const float* __restrict__ partial, int n, float* __restrict__ out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < n; ++i) t += (double)partial[i];
        *out = (float)t;
    }
}

// noisy = sqrt(acp[t]) x0 + sqrt(1 - acp[t]) noise (train.py:641; ddpm.py:356-359), fp32 NCHW, tables on the device
__global__ void q_sample_kernel(const float* __restrict__ x0, const float* __restrict__ noise, const long long* __restrict__ t,
                                const float* __restrict__ sqrt_acp, const float* __restrict__ sqrt_1m_acp, float* __restrict__ out,
                                long long n_per, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / n_per;
        const long long tt = t[b];
        out[i] = sqrt_acp[tt] * x0[i] + sqrt_1m_acp[tt] * noise[i];
    }
}

// torch.optim.AdamW single-tensor step (train.py:486-492): grad is multiplied by grad_scale (1 / loss scale) first
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             long long n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2_sqrt,
                             float grad_scale) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float gr = g[i] * grad_scale;
        float w = p[i] * (1.0f - lr * wd);
        const float mi = b1 * m[i] + (1.0f - b1) * gr;
        const float vi = b2 * v[i] + (1.0f - b2) * gr * gr;
        m[i] = mi;
        v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        w -= (lr / bc1) * mi / denom;
        p[i] = w;
    }
}

// ---- mixed-precision step control on the device (the GradScaler semantics accelerate gives train.py:694-709) ------------
// scaler[4] = {loss scale, growth tracker, optimizer steps taken, found_inf}.  No host synchronisation anywhere:
//   grad_check   found_inf = 1 if any gradient element (after the all-reduce) is inf / nan
//   adamw_scaled torch.optim.AdamW over one flat fp32 buffer; skipped when found_inf; step number = steps taken + 1;
//                gradients are divided by (loss scale x world) on the fly
//   scale_update found_inf ? (scale *= backoff, tracker = 0) : (steps += 1, ++tracker == interval -> scale *= growth); found_inf = 0
__global__ void grad_check_kernel(const float4* __restrict__ g, long long n4, const float* __restrict__ tail, int ntail,
                                  float* __restrict__ scaler) {
    bool bad = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = g[i];
        const uint32_t a = __float_as_uint(v.x), b = __float_as_uint(v.y), c = __float_as_uint(v.z), d = __float_as_uint(v.w);
        bad |= ((a & 0x7f800000u) == 0x7f800000u) | ((b & 0x7f800000u) == 0x7f800000u) | ((c & 0x7f800000u) == 0x7f800000u) |
               ((d & 0x7f800000u) == 0x7f800000u);
    }
    if (blockIdx.x == 0 && (int)threadIdx.x < ntail) bad |= (__float_as_uint(tail[threadIdx.x]) & 0x7f800000u) == 0x7f800000u;
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) scaler[3] = 1.0f;      // benign race: every writer stores 1
}

__global__ void adamw_scaled_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                    long long n, float lr, float b1, float b2, float eps, float wd, float inv_world,
                                    const float* __restrict__ scaler) {
    if (scaler[3] != 0.0f) return;                       // overflow somewhere in this step's gradients: skip it (GradScaler.step)
    const float step = scaler[2] + 1.0f;
    const float bc1 = 1.0f - powf(b1, step), bc2_sqrt = sqrtf(1.0f - powf(b2, step));
    const float grad_scale = inv_world / scaler[0];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float gr = g[i] * grad_scale;
        float w = p[i] * (1.0f - lr * wd);
        const float mi = b1 * m[i] + (1.0f - b1) * gr;
        const float vi = b2 * v[i] + (1.0f - b2) * gr * gr;
        m[i] = mi;
        v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        w -= (lr / bc1) * mi / denom;
        p[i] = w;
    }
}

__global__ void loss_scale_update_kernel(float* __restrict__ scaler, float growth, float backoff, int interval) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (scaler[3] != 0.0f) {
        scaler[0] *= backoff;
        scaler[1] = 0.0f;
    } else {
        scaler[2] += 1.0f;
        scaler[1] += 1.0f;
        if (interval > 0 && scaler[1] >= (float)interval) {
            scaler[0] *= growth;
            scaler[1] = 0.0f;
        }
    }
    scaler[3] = 0.0f;
}

// ---- small-M weight gradient: out[ka, kb] (+)= alpha * sum_m A[m, col(ka)] * B[m, kb] -----------------------------
// A [M, lda] fp16 with optional head padding (logical column ka lives at (ka / head_d) * head_stride + ka % head_d),
// B [M, ldb] fp16, out fp32 [Ka, ldo].  32 x 32 output tile per CTA, 16 x 16 threads, 2 x 2 outputs each.
__global__ void __launch_bounds__(256) gemm_tn_kernel(const __half* __restrict__ A, int lda, int head_d, int head_stride,
                                                      int group_c, int group_stride, const __half* __restrict__ B, int ldb,
                                                      float* __restrict__ out, int ldo, int M, int Ka, int Kb, float alpha,
                                                      int accumulate) {
    __shared__ float sA[32][33], sB[32][33];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int a0 = blockIdx.y * 32, b0 = blockIdx.x * 32;
    float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    for (int m0 = 0; m0 < M; m0 += 32) {
        for (int i = threadIdx.x; i < 32 * 32; i += 256) {
            const int mm = i >> 5, cc = i & 31;
            const int m = m0 + mm;
            float va = 0.f, vb = 0.f;
            if (m < M) {
                const int ka = a0 + cc;
                if (ka < Ka) {
                    int base = 0, c = ka;
                    if (group_c > 0) {
                        base = (ka / group_c) * group_stride;
                        c = ka % group_c;
                    }
                    const int col = base + (head_d > 0 ? (c / head_d) * head_stride + c % head_d : c);
                    va = __half2float(A[(size_t)m * lda + col]);
                }
                const int kb = b0 + cc;
                if (kb < Kb) vb = __half2float(B[(size_t)m * ldb + kb]);
            }
            sA[mm][cc] = va;
            sB[mm][cc] = vb;
        }
        __syncthreads();
#pragma unroll 8
        for (int mm = 0; mm < 32; ++mm) {
            const float x0 = sA[mm][ty * 2], x1 = sA[mm][ty * 2 + 1];
            const float y0 = sB[mm][tx * 2], y1 = sB[mm][tx * 2 + 1];
            acc[0][0] += x0 * y0; acc[0][1] += x0 * y1;
            acc[1][0] += x1 * y0; acc[1][1] += x1 * y1;
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int ka = a0 + ty * 2 + i, kb = b0 + tx * 2 + j;
            if (ka < Ka && kb < Kb) {
                float* o = out + (size_t)ka * ldo + kb;
                *o = (accumulate ? *o : 0.f) + alpha * acc[i][j];
            }
        }
}

// ---- gather + transpose: out[ka, m] = A[m, col(ka)] (column mapping as in gemm_tn), zero for m >= M ------------------
// Turns the small-M weight gradient dW = A^T B into two K-major operands for anysd_gemm_f16 (K = M rows).
__global__ void __launch_bounds__(256) gather_transpose_kernel(const __half* __restrict__ A, int lda, int head_d, int head_stride,
                                                               int group_c, int group_stride, __half* __restrict__ out, int ldo,
                                                               int M, int Ka) {
    __shared__ __half tile[32][34];
    const int k0 = blockIdx.y * 32, m0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 32 x 8
    for (int r = ty; r < 32; r += 8) {                               // r: row of A (m), tx: logical column
        const int m = m0 + r, ka = k0 + tx;
        __half v = __float2half(0.f);
        if (m < M && ka < Ka) {
            int base = 0, c = ka;
            if (group_c > 0) {
                base = (ka / group_c) * group_stride;
                c = ka % group_c;
            }
            const int col = base + (head_d > 0 ? (c / head_d) * head_stride + c % head_d : c);
            v = A[(size_t)m * lda + col];
        }
        tile[r][tx] = v;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {                               // r: logical column (row of out), tx: m
        const int ka = k0 + r, m = m0 + tx;
        if (ka < Ka && m < ldo) out[(size_t)ka * ldo + m] = tile[tx][r];
    }
}

// ---- router backward (restated spec, oracle/anysd_oracle.py): g = softmax(W te + b) per (sample, layer) -----------
// dlogit = g * (dg - sum_e g dg);  dW[l] += dlogit^T te;  db[l] += sum_n dlogit;  dte[n] += sum_l dlogit W[l]
// grid = L, block = 256.  gates / dgates [N, L, E] fp32; te [N, D] fp32 (gathered task embeddings); W [L, E, D] fp16.
__global__ void __launch_bounds__(256) router_bwd_kernel(const float* __restrict__ gates, const float* __restrict__ dgates,
                                                         const float* __restrict__ te, const __half* __restrict__ W, int N, int L, int E,
                                                         int D, float alpha, float* __restrict__ dW, float* __restrict__ db,
                                                         float* __restrict__ dte) {
    extern __shared__ float dl[];                 // [N, E]
    const int l = blockIdx.x;
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
        const float* g = gates + ((size_t)n * L + l) * E;
        const float* dg = dgates + ((size_t)n * L + l) * E;
        float dot = 0.f;
        for (int e = 0; e < E; ++e) dot += g[e] * dg[e];
        for (int e = 0; e < E; ++e) dl[n * E + e] = alpha * g[e] * (dg[e] - dot);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < E * D; i += blockDim.x) {
        const int e = i / D, d = i - e * D;
        float t = 0.f;
        for (int n = 0; n < N; ++n) t += dl[n * E + e] * te[(size_t)n * D + d];
        dW[((size_t)l * E + e) * D + d] += t;
    }
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
        float t = 0.f;
        for (int n = 0; n < N; ++n) t += dl[n * E + e];
        db[(size_t)l * E + e] += t;
    }
    for (int i = threadIdx.x; i < N * D; i += blockDim.x) {
        const int n = i / D, d = i - n * D;
        float t = 0.f;
        for (int e = 0; e < E; ++e) t += dl[n * E + e] * __half2float(W[((size_t)l * E + e) * D + d]);
        atomicAdd(dte + (size_t)n * D + d, t);
    }
}

// table_grad[idx[n]] += alpha * src[n]   (task-embedding gather backward)
__global__ void scatter_add_rows_kernel(const float* __restrict__ src, const long long* __restrict__ idx, int rows, int D, int table_rows,
                                        float alpha, float* __restrict__ table_grad) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)rows * D; i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i / D), d = (int)(i - (long long)n * D);
        const long long r = idx[n];
        if (r >= 0 && r < table_rows) atomicAdd(table_grad + r * D + d, alpha * src[i]);
    }
}

static int grid_for(long long n, int block = 256, int per_sm = 8) {
    long long g = (n + block - 1) / block;
    const long long cap = (long long)sm_count() * per_sm;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace anysd

using namespace anysd;

extern "C" {

int anysd_geglu_f16(const void* pre, void* out, long long M, int inner, anysd_stream_t stream) {
    ANYSD_REQUIRE(pre && out && M > 0 && inner > 0 && inner % 8 == 0, ANYSD_EINVAL, "geglu: bad args (inner %% 8 == 0)");
    const long long nvec = M * inner / 8;
    geglu_fwd_kernel<<<grid_for(nvec), 256, 0, (cudaStream_t)stream>>>((const uint4*)pre, (uint4*)out, nvec);
    return check_launch("geglu");
}

int anysd_geglu_bwd_f16(const void* pre, const void* d_out, void* d_pre, long long M, int inner, anysd_stream_t stream) {
    ANYSD_REQUIRE(pre && d_out && d_pre && M > 0 && inner > 0 && inner % 8 == 0, ANYSD_EINVAL, "geglu_bwd: bad args");
    const long long nvec = M * inner / 8;
    geglu_bwd_kernel<<<grid_for(nvec), 256, 0, (cudaStream_t)stream>>>((const uint4*)pre, (const uint4*)d_out, (uint4*)d_pre, nvec);
    return check_launch("geglu_bwd");
}

int anysd_silu_bwd_f32(const float* x, const float* dy, float* dx, long long n, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && dy && dx && n > 0, ANYSD_EINVAL, "silu_bwd: bad args");
    silu_bwd_f32_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, dy, dx, n);
    return check_launch("silu_bwd");
}

int anysd_groupnorm_bwd_nhwc_f16(const void* x1, int C1, const void* x2, int C2, const float* gamma, const float* beta,
                                 const void* dy, void* dx, int N, int HW, int G, float eps, int fuse_silu,
                                 anysd_stream_t stream) {
    ANYSD_REQUIRE(x1 && gamma && beta && dy && dx, ANYSD_EINVAL, "groupnorm_bwd: null pointer");
    if (x2 == nullptr) C2 = 0;
    const int C = C1 + C2;
    ANYSD_REQUIRE(N > 0 && HW > 0 && G > 0 && C1 > 0 && C2 >= 0 && C % G == 0 && N <= 65535, ANYSD_EINVAL, "groupnorm_bwd: bad shape");
    ANYSD_REQUIRE(C1 % 8 == 0 && C2 % 8 == 0, ANYSD_EINVAL, "groupnorm_bwd: channel counts must be multiples of 8");
    const int cpg = C / G;
    int gpc = 1;                                   // groups per CTA: smallest span that is a whole number of 8-channel vectors
    while ((gpc * cpg) % 8 != 0) ++gpc;
    ANYSD_REQUIRE(G % gpc == 0 && gpc * cpg / 8 <= GNB_THREADS, ANYSD_EUNSUPPORTED,
                  "groupnorm_bwd: C=%d, G=%d does not tile into 16-byte channel vectors", C, G);
    const int VC = gpc * cpg / 8, RL = GNB_THREADS / VC;
    const size_t smem = ((size_t)2 * RL * VC * 8 + 6 * gpc) * sizeof(float);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(gn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        ANYSD_REQUIRE(e == cudaSuccess, ANYSD_ECUDA, "groupnorm_bwd: smem opt-in failed: %s", cudaGetErrorString(e));
    }
    // CTAs per slab (cluster along x): enough rows per CTA to keep the RL row lanes busy
    static const char* cs_env = getenv("ANYSD_GNBWD_CLUSTER");
    // clusters only for the large maps: on the small ones the two cluster barriers per fold cost more than the parallelism buys
    // (chosen on the project's earlier GPU, not re-measured on the H100; ANYSD_GNBWD_CLUSTER overrides)
    int CS = HW >= 2048 ? 8 : 1;
    if (cs_env) CS = atoi(cs_env) >= 1 ? atoi(cs_env) : 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((G / gpc) * CS, N);
    cfg.blockDim = dim3(GNB_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CS;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t le = cudaLaunchKernelEx(&cfg, gn_bwd_kernel, (const __half*)x1, C1, (const __half*)x2, C2, gamma, beta, (const __half*)dy,
                                        (__half*)dx, HW, cpg, gpc, eps, fuse_silu, CS);
    ANYSD_REQUIRE(le == cudaSuccess, ANYSD_ECUDA, "groupnorm_bwd: launch failed: %s", cudaGetErrorString(le));
    return check_launch("groupnorm_bwd");
}

int anysd_layernorm_bwd_f16(const void* x, const float* gamma, const void* dy, void* dx, long long M, int C, float eps,
                            anysd_stream_t stream) {
    ANYSD_REQUIRE(x && gamma && dy && dx && M > 0 && C > 0 && C % 8 == 0, ANYSD_EINVAL, "layernorm_bwd: bad args (C %% 8 == 0)");
    ln_bwd_kernel<<<cdiv(M, 8), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, gamma, (const uint4*)dy, (uint4*)dx, M, C / 8, eps);
    return check_launch("layernorm_bwd");
}

int anysd_colsum_f16(const void* x, float* out, int N, int rows, int C, int ld_out, int accumulate, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && out && N > 0 && rows > 0 && C > 0 && C % 8 == 0 && ld_out >= C && N <= 65535, ANYSD_EINVAL, "colsum: bad args");
    colsum_kernel<<<dim3(cdiv(C, 64), N), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, out, rows, C / 8, ld_out, accumulate);
    return check_launch("colsum");
}

int anysd_add_f16(void* y, const void* x, long long n, anysd_stream_t stream) {
    ANYSD_REQUIRE(y && x && n > 0 && n % 8 == 0, ANYSD_EINVAL, "add: bad args (n %% 8 == 0)");
    add_f16_kernel<<<grid_for(n / 8), 256, 0, (cudaStream_t)stream>>>((uint4*)y, (const uint4*)x, n / 8);
    return check_launch("add");
}

int anysd_split_channels_f16(const void* src, void* a, int Ca, void* b, int Cb, long long rows, anysd_stream_t stream) {
    ANYSD_REQUIRE(src && a && b && rows > 0 && Ca > 0 && Cb > 0 && Ca % 8 == 0 && Cb % 8 == 0, ANYSD_EINVAL, "split: bad args");
    const long long total = rows * ((Ca + Cb) / 8);
    split_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)src, (uint4*)a, Ca / 8, (uint4*)b, Cb / 8, total);
    return check_launch("split");
}

int anysd_zero_insert2x_f16(const void* src, void* dst, int N, int H, int W, int C, anysd_stream_t stream) {
    ANYSD_REQUIRE(src && dst && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, ANYSD_EINVAL, "zero_insert2x: bad args");
    const long long total = (long long)N * 2 * H * 2 * W * (C / 8);
    zero_insert2x_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)src, (uint4*)dst, H, W, C / 8, total);
    return check_launch("zero_insert2x");
}

int anysd_sumpool2x_f16(const void* src, void* dst, int N, int H, int W, int C, anysd_stream_t stream) {
    ANYSD_REQUIRE(src && dst && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, ANYSD_EINVAL, "sumpool2x: bad args");
    const long long total = (long long)N * H * W * (C / 8);
    sumpool2x_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)src, (uint4*)dst, H, W, C / 8, total);
    return check_launch("sumpool2x");
}

size_t anysd_mse_workspace_bytes(void) { return (size_t)1024 * sizeof(float); }

int anysd_mse_loss_f32(const float* pred, const float* target, int N, int C, int HW, int Cpad, float grad_scale,
                       const float* grad_scale_dev, void* d_pred, float* loss, void* workspace, size_t workspace_bytes,
                       anysd_stream_t stream) {
    ANYSD_REQUIRE(pred && target && d_pred && loss && workspace, ANYSD_EINVAL, "mse_loss: null pointer");
    ANYSD_REQUIRE(N > 0 && C > 0 && HW > 0 && Cpad >= C && workspace_bytes >= anysd_mse_workspace_bytes(), ANYSD_EINVAL, "mse_loss: bad args");
    int grid = grid_for((long long)N * HW, 256, 4);
    if (grid > 1024) grid = 1024;
    mse_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(pred, target, N, C, HW, Cpad, grad_scale, grad_scale_dev, (__half*)d_pred,
                                                       (float*)workspace);
    int rc = check_launch("mse_loss");
    if (rc) return rc;
    sum_partials_kernel<<<1, 32, 0, (cudaStream_t)stream>>>((const float*)workspace, grid, loss);
    return check_launch("mse_loss (sum)");
}

int anysd_q_sample_f32(const float* x0, const float* noise, const long long* t, const float* sqrt_acp, const float* sqrt_1m_acp,
                       float* out, int B, long long n_per, anysd_stream_t stream) {
    ANYSD_REQUIRE(x0 && noise && t && sqrt_acp && sqrt_1m_acp && out && B > 0 && n_per > 0, ANYSD_EINVAL, "q_sample: bad args");
    const long long total = (long long)B * n_per;
    q_sample_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(x0, noise, t, sqrt_acp, sqrt_1m_acp, out, n_per, total);
    return check_launch("q_sample");
}

int anysd_adamw_f32(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n, float lr, float beta1,
                    float beta2, float eps, float weight_decay, int step, float grad_scale, anysd_stream_t stream) {
    ANYSD_REQUIRE(param && grad && exp_avg && exp_avg_sq && n > 0 && step >= 1, ANYSD_EINVAL, "adamw: bad args (step counts from 1)");
    const float bc1 = 1.0f - powf(beta1, (float)step);
    const float bc2s = sqrtf(1.0f - powf(beta2, (float)step));
    adamw_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps,
                                                              weight_decay, bc1, bc2s, grad_scale);
    return check_launch("adamw");
}

int anysd_grad_check_f32(const float* grad, long long n, float* scaler, anysd_stream_t stream) {
    ANYSD_REQUIRE(grad && scaler && n > 0, ANYSD_EINVAL, "grad_check: bad args");
    ANYSD_REQUIRE(((uintptr_t)grad % 16) == 0, ANYSD_EINVAL, "grad_check: the gradient buffer must be 16-byte aligned");
    const long long n4 = n / 4;
    grad_check_kernel<<<grid_for(n4 > 0 ? n4 : 1), 256, 0, (cudaStream_t)stream>>>((const float4*)grad, n4, grad + 4 * n4, (int)(n - 4 * n4), scaler);
    return check_launch("grad_check");
}

int anysd_adamw_scaled_f32(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n, float lr, float beta1,
                           float beta2, float eps, float weight_decay, float inv_world, const float* scaler, anysd_stream_t stream) {
    ANYSD_REQUIRE(param && grad && exp_avg && exp_avg_sq && scaler && n > 0 && inv_world > 0.f, ANYSD_EINVAL, "adamw_scaled: bad args");
    adamw_scaled_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps,
                                                                     weight_decay, inv_world, scaler);
    return check_launch("adamw_scaled");
}

int anysd_loss_scale_update_f32(float* scaler, float growth, float backoff, int interval, anysd_stream_t stream) {
    ANYSD_REQUIRE(scaler && growth >= 1.f && backoff > 0.f && backoff <= 1.f, ANYSD_EINVAL, "loss_scale_update: bad args");
    loss_scale_update_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(scaler, growth, backoff, interval);
    return check_launch("loss_scale_update");
}

int anysd_gemm_tn_f32(const void* A, int lda, int head_d, int head_stride, int group_c, int group_stride, const void* B, int ldb,
                      float* out, int ldo, int M, int Ka, int Kb, float alpha, int accumulate, anysd_stream_t stream) {
    ANYSD_REQUIRE(A && B && out && M > 0 && Ka > 0 && Kb > 0 && lda > 0 && ldb >= Kb && ldo >= Kb, ANYSD_EINVAL, "gemm_tn: bad args");
    ANYSD_REQUIRE(head_d == 0 || (head_d > 0 && head_stride >= head_d), ANYSD_EINVAL, "gemm_tn: bad head mapping");
    ANYSD_REQUIRE(group_c >= 0 && (group_c == 0 || group_stride > 0), ANYSD_EINVAL, "gemm_tn: bad group mapping");
    gemm_tn_kernel<<<dim3(cdiv(Kb, 32), cdiv(Ka, 32)), 256, 0, (cudaStream_t)stream>>>((const __half*)A, lda, head_d, head_stride, group_c,
                                                                                     group_stride, (const __half*)B, ldb, out, ldo, M, Ka,
                                                                                     Kb, alpha, accumulate);
    return check_launch("gemm_tn");
}

int anysd_gather_transpose_f16(const void* A, int lda, int head_d, int head_stride, int group_c, int group_stride, void* out, int ldo,
                               int M, int Ka, anysd_stream_t stream) {
    ANYSD_REQUIRE(A && out && M > 0 && Ka > 0 && lda > 0 && ldo >= M, ANYSD_EINVAL, "gather_transpose: bad args");
    ANYSD_REQUIRE(head_d == 0 || (head_d > 0 && head_stride >= head_d), ANYSD_EINVAL, "gather_transpose: bad head mapping");
    ANYSD_REQUIRE(group_c >= 0 && (group_c == 0 || group_stride > 0), ANYSD_EINVAL, "gather_transpose: bad group mapping");
    gather_transpose_kernel<<<dim3(cdiv(ldo, 32), cdiv(Ka, 32)), 256, 0, (cudaStream_t)stream>>>((const __half*)A, lda, head_d, head_stride,
                                                                                              group_c, group_stride, (__half*)out, ldo, M, Ka);
    return check_launch("gather_transpose");
}

int anysd_router_bwd_f32(const float* gates, const float* d_gates, const float* te, const void* W, int N, int L, int E, int D,
                         float alpha, float* dW, float* db, float* d_te, anysd_stream_t stream) {
    ANYSD_REQUIRE(gates && d_gates && te && W && dW && db && d_te, ANYSD_EINVAL, "router_bwd: null pointer");
    ANYSD_REQUIRE(N > 0 && L > 0 && E > 0 && D > 0 && (size_t)N * E * sizeof(float) <= 48 * 1024, ANYSD_EINVAL, "router_bwd: bad sizes");
    router_bwd_kernel<<<L, 256, (size_t)N * E * sizeof(float), (cudaStream_t)stream>>>(gates, d_gates, te, (const __half*)W, N, L, E, D,
                                                                                     alpha, dW, db, d_te);
    return check_launch("router_bwd");
}

int anysd_scatter_add_rows_f32(const float* src, const long long* idx, int rows, int D, int table_rows, float alpha, float* table_grad,
                               anysd_stream_t stream) {
    ANYSD_REQUIRE(src && idx && table_grad && rows > 0 && D > 0 && table_rows > 0, ANYSD_EINVAL, "scatter_add_rows: bad args");
    scatter_add_rows_kernel<<<grid_for((long long)rows * D), 256, 0, (cudaStream_t)stream>>>(src, idx, rows, D, table_rows, alpha, table_grad);
    return check_launch("scatter_add_rows");
}
}
