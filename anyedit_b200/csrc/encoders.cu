// Condition-encoder helpers (SURVEY.md 8f rank 2): everything else of the CLIP towers / Resampler runs on the UNet's kernels
// (LayerNorm, wgmma contractions with fused bias / GELU / QuickGELU / residual, wgmma attention).
//   embed_tokens        CLIPTextEmbeddings (transformers modeling_clip.py): token_embedding[ids] + position_embedding[pos]
//   attention_small     softmax(q k^T scale [+ causal mask]) v for short sequences: the CLIP text tower's causal 77-token
//                       self-attention (the wgmma attention kernel has no mask path; 77 x 77 x 64 per head is latency-sized)
#include "common.cuh"

namespace anysd {

__global__ void embed_tokens_kernel(const long long* __restrict__ ids, const __half* __restrict__ tok, const __half* __restrict__ pos,
                                    __half* __restrict__ out, int n, int D, int vocab) {
    const int row = blockIdx.x;                        // b * n + i
    const int i = row % n;
    long long id = ids[row];
    if (id < 0) id = 0;
    if (id >= vocab) id = vocab - 1;
    const __half2* t2 = reinterpret_cast<const __half2*>(tok + (size_t)id * D);
    const __half2* p2 = reinterpret_cast<const __half2*>(pos + (size_t)i * D);
    __half2* o2 = reinterpret_cast<__half2*>(out + (size_t)row * D);
    for (int c = threadIdx.x; c < D / 2; c += blockDim.x) {
        const float2 a = __half22float2(t2[c]), b = __half22float2(p2[c]);
        o2[c] = __floats2half2_rn(a.x + b.x, a.y + b.y);
    }
}

// one CTA per (head, batch): K and V of the head staged in shared memory (row pitch d + 2 halves: conflict-free column
// walks), one warp per query row: lane j owns keys j, j + 32, ... (<= 8 of them: n_kv <= 256), fp32 softmax, then every
// lane owns output dims lane, lane + 32, ...
constexpr int AS_MAX_KV = 256;
__global__ void __launch_bounds__(128) attention_small_kernel(const __half* __restrict__ q, const __half* __restrict__ k,
                                                              const __half* __restrict__ v, __half* __restrict__ out, int n_q, int n_kv,
                                                              int d, int ld_q, int ld_k, int ld_v, int ld_o, float scale, int causal) {
    extern __shared__ __half as_smem[];
    const int h = blockIdx.x, b = blockIdx.y;
    const int pitch = d + 2;
    __half* sk = as_smem;
    __half* sv = sk + (size_t)n_kv * pitch;
    float* sp = reinterpret_cast<float*>(sv + (size_t)n_kv * pitch);        // [4 warps][n_kv] probabilities
    float* sq = sp + 4 * n_kv;                                              // [4 warps][d] the warp's query row
    for (int i = threadIdx.x; i < n_kv * d; i += blockDim.x) {
        const int r = i / d, c = i - r * d;
        sk[r * pitch + c] = k[((size_t)b * n_kv + r) * ld_k + h * d + c];
        sv[r * pitch + c] = v[((size_t)b * n_kv + r) * ld_v + h * d + c];
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* pw = sp + warp * n_kv;
    float* qw = sq + warp * d;
    for (int i = warp; i < n_q; i += 4) {
        for (int c = lane; c < d; c += 32) qw[c] = __half2float(q[((size_t)b * n_q + i) * ld_q + h * d + c]) * scale;
        __syncwarp();
        float s[AS_MAX_KV / 32];
        float m = -INFINITY;
#pragma unroll
        for (int t = 0; t < AS_MAX_KV / 32; ++t) {
            const int j = lane + 32 * t;
            float acc = -INFINITY;
            if (j < n_kv && !(causal && j > i)) {
                acc = 0.f;
                for (int c = 0; c < d; ++c) acc = fmaf(qw[c], __half2float(sk[j * pitch + c]), acc);
            }
            s[t] = acc;
            m = fmaxf(m, acc);
        }
        m = warp_max(m);
        float l = 0.f;
#pragma unroll
        for (int t = 0; t < AS_MAX_KV / 32; ++t) {
            const int j = lane + 32 * t;
            const float p = (j < n_kv && s[t] > -INFINITY) ? __expf(s[t] - m) : 0.f;
            if (j < n_kv) pw[j] = p;
            l += p;
        }
        l = warp_sum(l);
        __syncwarp();
        const float inv = 1.0f / l;
        for (int c = lane; c < d; c += 32) {
            float acc = 0.f;
            for (int j = 0; j < n_kv; ++j) acc = fmaf(pw[j], __half2float(sv[j * pitch + c]), acc);
            out[((size_t)b * n_q + i) * ld_o + h * d + c] = __float2half_rn(acc * inv);
        }
        __syncwarp();
    }
}

}  // namespace anysd

using namespace anysd;

extern "C" {

int anysd_embed_tokens_f16(const long long* ids, const void* tok_table, const void* pos_table, void* out, int B, int n, int D, int vocab,
                           anysd_stream_t stream) {
    ANYSD_REQUIRE(ids && tok_table && pos_table && out && B > 0 && n > 0 && D > 0 && D % 2 == 0 && vocab > 0, ANYSD_EINVAL,
                  "embed_tokens: bad args");
    embed_tokens_kernel<<<B * n, 128, 0, (cudaStream_t)stream>>>(ids, (const __half*)tok_table, (const __half*)pos_table, (__half*)out, n, D,
                                                                 vocab);
    return check_launch("embed_tokens");
}

int anysd_attention_small_f16(const void* q, const void* k, const void* v, void* out, int B, int heads, int n_q, int n_kv, int d, int ld_q,
                              int ld_k, int ld_v, int ld_o, float scale, int causal, anysd_stream_t stream) {
    ANYSD_REQUIRE(q && k && v && out && B > 0 && heads > 0 && n_q > 0 && n_kv > 0 && d > 0, ANYSD_EINVAL, "attention_small: bad args");
    ANYSD_REQUIRE(n_kv <= AS_MAX_KV, ANYSD_EUNSUPPORTED, "attention_small: at most %d keys (got %d); long sequences use anysd_attention_f16",
                  AS_MAX_KV, n_kv);
    ANYSD_REQUIRE(!causal || n_q == n_kv, ANYSD_EINVAL, "attention_small: the causal mask needs n_q == n_kv");
    const size_t smem = (size_t)2 * n_kv * (d + 2) * sizeof(__half) + (size_t)4 * (n_kv + d) * sizeof(float);
    static int set_for[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (smem > 48 * 1024 && set_for[dev] < (int)smem) {
        cudaError_t e = cudaFuncSetAttribute(attention_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        ANYSD_REQUIRE(e == cudaSuccess, ANYSD_ECUDA, "attention_small: smem opt-in failed: %s", cudaGetErrorString(e));
        set_for[dev] = (int)smem;
    }
    attention_small_kernel<<<dim3(heads, B), 128, smem, (cudaStream_t)stream>>>((const __half*)q, (const __half*)k, (const __half*)v,
                                                                              (__half*)out, n_q, n_kv, d, ld_q, ld_k, ld_v, ld_o, scale, causal);
    return check_launch("attention_small");
}
}
