// Dense-prediction helpers of the Depth Anything V2 DPT head (depth_anything_v2/dpt.py, util/blocks.py) and of the UniFormer +
// UPerNet segmentor (uniformer/mmseg: backbones/uniformer.py, decode_heads/uper_head.py, psp_head.py); the convolutions and
// projections of both run on anysd_gemm_f16.
//   resize_bilinear      F.interpolate(mode="bilinear") with align_corners True or False at any (H, W) -> (Ho, Wo), NHWC fp16
//                        (C % 8 == 0, 16-byte vectors) with an optional fp16 addend of the output's shape folded in before the one
//                        rounding and an output row stride (a channel slice of a concat buffer); and a single-channel fp32 form
//                        (infer_image's align-corners resize to the raw image size)
//   relu                 y = max(x, 0) as a copy: ResidualConvUnit needs x (its residual) and relu(x) (its conv input)
//   depth_to_space       ConvTranspose2d(kernel = stride = r) as one contraction: [B*gh*gw, (ky, kx, co)] -> [B, r gh, r gw, co]
//   space_to_depth       its inverse with cropping: Conv2d(kernel = stride = r) as one contraction of [B*Ho*Wo, (ky, kx, c)] rows;
//                        also straight from a uint8 image
//   dwconv               depthwise Conv2d(k = 3 | 5, pad k / 2) with bias and an optional residual, NHWC fp16
//   adaptive_avg_pool    nn.AdaptiveAvgPool2d with PyTorch's bins, NHWC fp16
//   seg_labels           mmseg's two half-pixel resizes of the logits (to the network input, then to the original image) and
//                        the argmax over classes, per original pixel, without the two fp32 logit volumes; optional palette
//   hed_input            the HED edge network's (other_modules/HED/__init__.py) first 3x3 conv input as K = 32 im2col rows
//   max_pool2            F.max_pool2d(2, 2) on NHWC fp16, bit-exact
//   hed_edges            HEDdetector's post-processing: cv2's INTER_LINEAR resize of the five side maps, the mean, the fp64
//                        sigmoid and the inversion to uint8, per output pixel
#include "common.cuh"

namespace anysd {

// Source taps of output index o along one axis, as ATen computes them in fp32 (area_pixel_compute_scale /
// area_pixel_compute_source_index, UpSampleBilinear2d.cu): align_corners=True: src = o * (in - 1) / (out - 1);
// align_corners=False (half-pixel): src = max(in / out * (o + 0.5) - 0.5, 0).  The upper neighbour is clamped to the edge.
struct Tap {
    int i0, i1;
    float l0, l1;
};
__device__ __forceinline__ Tap bl_tap(int o, float scale, int in, bool align_corners) {
    float src = align_corners ? scale * (float)o : scale * ((float)o + 0.5f) - 0.5f;
    if (src < 0.0f) src = 0.0f;
    Tap t;
    t.i0 = (int)src;
    if (t.i0 > in - 1) t.i0 = in - 1;
    t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
    t.l1 = src - (float)t.i0;
    t.l0 = 1.0f - t.l1;
    return t;
}
static inline float bl_scale(int in, int out, bool align_corners) {
    if (!align_corners) return (float)in / (float)out;
    return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.0f;
}

// y rows are ldy_v vectors apart (a channel slice of a wider buffer); the addend is dense [N, Ho, Wo, C] and may be y itself
__global__ void resize_bilinear_f16_kernel(const uint4* __restrict__ x, const uint4* add, uint4* y, int H, int W, int Ho, int Wo,
                                           int CV, long long ldy_v, float sh, float sw, bool ac, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(i % CV);
        long long r = i / CV;
        const int ox = (int)(r % Wo);
        r /= Wo;
        const int oy = (int)(r % Ho);
        const long long n = r / Ho;
        const Tap ty = bl_tap(oy, sh, H, ac), tx = bl_tap(ox, sw, W, ac);
        const uint4* img = x + n * H * W * CV + cv;
        float a[8], b[8], c[8], d[8], o[8];
        unpack8(img[((long long)ty.i0 * W + tx.i0) * CV], a);
        unpack8(img[((long long)ty.i0 * W + tx.i1) * CV], b);
        unpack8(img[((long long)ty.i1 * W + tx.i0) * CV], c);
        unpack8(img[((long long)ty.i1 * W + tx.i1) * CV], d);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = ty.l0 * (tx.l0 * a[j] + tx.l1 * b[j]) + ty.l1 * (tx.l0 * c[j] + tx.l1 * d[j]);
        if (add != nullptr) {
            float e[8];
            unpack8(add[i], e);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] += e[j];
        }
        y[((n * Ho + oy) * Wo + ox) * ldy_v + cv] = pack8(o);
    }
}

__global__ void resize_bilinear_ac_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, int Ho, int Wo, float sh,
                                              float sw, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % Wo);
        const long long r = i / Wo;
        const int oy = (int)(r % Ho);
        const long long n = r / Ho;
        const Tap ty = bl_tap(oy, sh, H, true), tx = bl_tap(ox, sw, W, true);
        const float* img = x + n * H * W;
        y[i] = ty.l0 * (tx.l0 * img[ty.i0 * W + tx.i0] + tx.l1 * img[ty.i0 * W + tx.i1]) +
               ty.l1 * (tx.l0 * img[ty.i1 * W + tx.i0] + tx.l1 * img[ty.i1 * W + tx.i1]);
    }
}

__global__ void relu_f16_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long long nvec) {
    // per fp16 lane: sign bit set -> +0, else x unchanged (exact; -0 and negative infinities become +0)
    auto relu2 = [](uint32_t w) { return w & ~(((w >> 15) & 0x00010001u) * 0xFFFFu); };
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        const uint4 u = x[i];
        y[i] = make_uint4(relu2(u.x), relu2(u.y), relu2(u.z), relu2(u.w));
    }
}

// out[b, y r + ky, x r + kx, c] = g[(b gh + y) gw + x, (ky r + kx) C + c], 8 channels per thread
__global__ void depth_to_space_f16_kernel(const uint4* __restrict__ g, uint4* __restrict__ out, int gh, int gw, int r, int CV,
                                          long long total) {
    const int Wo = gw * r, Ho = gh * r;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(i % CV);
        long long t = i / CV;
        const int X = (int)(t % Wo);
        t /= Wo;
        const int Y = (int)(t % Ho);
        const long long b = t / Ho;
        const int y = Y / r, ky = Y - y * r, x = X / r, kx = X - x * r;
        out[i] = g[((b * gh + y) * gw + x) * ((long long)r * r * CV) + (ky * r + kx) * CV + cv];
    }
}

// g[(b Ho + y) Wo + x, (ky r + kx) C + c] = in[b, y r + ky, x r + kx, c] for y < Ho = H / r, x < Wo = W / r (the remainder rows and
// columns are cropped, as Conv2d(kernel = stride = r) floors); 8 channels per thread
__global__ void space_to_depth_f16_kernel(const uint4* __restrict__ in, uint4* __restrict__ g, int H, int W, int Ho, int Wo, int r,
                                          int CV, long long total) {
    const int rrCV = r * r * CV;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int col = (int)(i % rrCV);
        const long long row = i / rrCV;
        const int x = (int)(row % Wo);
        const long long t = row / Wo;
        const int y = (int)(t % Ho);
        const long long b = t / Ho;
        const int tap = col / CV, cv = col - tap * CV, ky = tap / r, kx = tap - ky * r;
        g[i] = in[((b * H + (long long)y * r + ky) * W + (long long)x * r + kx) * CV + cv];
    }
}

// the same from a uint8 HWC image with C channels (values exact in fp16), one output element per thread
__global__ void space_to_depth_u8_kernel(const uint8_t* __restrict__ in, __half* __restrict__ g, int H, int W, int Ho, int Wo, int r,
                                         int C, long long total) {
    const int rrC = r * r * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int col = (int)(i % rrC);
        const long long row = i / rrC;
        const int x = (int)(row % Wo);
        const long long t = row / Wo;
        const int y = (int)(t % Ho);
        const long long b = t / Ho;
        const int tap = col / C, c = col - tap * C, ky = tap / r, kx = tap - ky * r;
        g[i] = __int2half_rn((int)in[((b * H + (long long)y * r + ky) * W + (long long)x * r + kx) * C + c]);
    }
}

// Depthwise KxK conv, zero padding K / 2, stride 1: y = sum_taps w[tap, c] x[.., c] + bias[c] (+ residual), accumulated in fp32 in
// tap order (ky, kx) and rounded once.  w fp32 [K*K, C]; 8 channels of one pixel per thread.
template <int K>
__global__ void dwconv_f16_kernel(const uint4* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                  const uint4* __restrict__ res, uint4* __restrict__ y, int H, int W, int CV, long long total) {
    constexpr int P = K / 2;
    const int C = CV * 8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(i % CV);
        long long r = i / CV;
        const int ox = (int)(r % W);
        r /= W;
        const int oy = (int)(r % H);
        const long long n = r / H;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
            const int iy = oy + ky - P;
            if (iy < 0 || iy >= H) continue;
#pragma unroll
            for (int kx = 0; kx < K; ++kx) {
                const int ix = ox + kx - P;
                if (ix < 0 || ix >= W) continue;
                float v[8];
                unpack8(x[((n * H + iy) * W + ix) * CV + cv], v);
                const float4* wt = reinterpret_cast<const float4*>(w + (ky * K + kx) * C + cv * 8);
                const float4 w0 = wt[0], w1 = wt[1];
                acc[0] = fmaf(w0.x, v[0], acc[0]);
                acc[1] = fmaf(w0.y, v[1], acc[1]);
                acc[2] = fmaf(w0.z, v[2], acc[2]);
                acc[3] = fmaf(w0.w, v[3], acc[3]);
                acc[4] = fmaf(w1.x, v[4], acc[4]);
                acc[5] = fmaf(w1.y, v[5], acc[5]);
                acc[6] = fmaf(w1.z, v[6], acc[6]);
                acc[7] = fmaf(w1.w, v[7], acc[7]);
            }
        }
        const float4* bt = reinterpret_cast<const float4*>(bias + cv * 8);
        const float4 b0 = bt[0], b1 = bt[1];
        acc[0] += b0.x; acc[1] += b0.y; acc[2] += b0.z; acc[3] += b0.w;
        acc[4] += b1.x; acc[5] += b1.y; acc[6] += b1.z; acc[7] += b1.w;
        if (res != nullptr) {
            float e[8];
            unpack8(res[i], e);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] += e[j];
        }
        y[i] = pack8(acc);
    }
}

// nn.AdaptiveAvgPool2d((Ho, Wo)): cell (oy, ox) averages rows [floor(oy H / Ho), ceil((oy + 1) H / Ho)) and the same for columns
// (ATen's start_index / end_index; bins overlap when H is not a multiple of Ho, and when H < Ho).  fp32 sum, one rounding.
__global__ void adaptive_avg_pool_f16_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int H, int W, int Ho, int Wo, int CV,
                                             long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(i % CV);
        long long r = i / CV;
        const int ox = (int)(r % Wo);
        r /= Wo;
        const int oy = (int)(r % Ho);
        const long long n = r / Ho;
        const int y0 = (int)(((long long)oy * H) / Ho), y1 = (int)(((long long)(oy + 1) * H + Ho - 1) / Ho);
        const int x0 = (int)(((long long)ox * W) / Wo), x1 = (int)(((long long)(ox + 1) * W + Wo - 1) / Wo);
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
        for (int iy = y0; iy < y1; ++iy)
            for (int ix = x0; ix < x1; ++ix) {
                float v[8];
                unpack8(x[((n * H + iy) * W + ix) * CV + cv], v);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += v[j];
            }
        const float cnt = (float)((y1 - y0) * (x1 - x0));
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] /= cnt;
        y[i] = pack8(acc);
    }
}

// One half-pixel bilinear value from four fp32 samples, in ATen's expression order (upsample_bilinear2d_out_frame).
__device__ __forceinline__ float bl_mix(const Tap& ty, const Tap& tx, float a, float b, float c, float d) {
    return ty.l0 * (tx.l0 * a + tx.l1 * b) + ty.l1 * (tx.l0 * c + tx.l1 * d);
}

// Labels of mmseg's whole-image test (EncoderDecoder.encode_decode + whole_inference + simple_test): the logits [N, h, w, ldl]
// (fp32, classes in the first `classes` columns, ldl % 4 == 0) are resized half-pixel to the network input (Hm, Wm), that map
// half-pixel to the original image (Ho, Wo), and the label is the first class of largest value (softmax is monotonic).  Every
// intermediate value is recomputed in fp32 exactly as the first resize would store it, so neither fp32 volume exists.  Four
// classes per float4; one output pixel per thread.  palette (uint8 [classes, 3]) or NULL: rgb[pixel] = palette[label].
__global__ void seg_labels_kernel(const float* __restrict__ logits, int h, int w, int ldl, int classes, int Hm, int Wm, int Ho, int Wo,
                                  float s1h, float s1w, float s2h, float s2w, long long* __restrict__ labels,
                                  const uint8_t* __restrict__ palette, uint8_t* __restrict__ rgb, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % Wo);
        const long long r = i / Wo;
        const int oy = (int)(r % Ho);
        const long long n = r / Ho;
        const Tap t2y = bl_tap(oy, s2h, Hm, false), t2x = bl_tap(ox, s2w, Wm, false);
        // taps of the two intermediate rows and columns into the logits
        const Tap ty0 = bl_tap(t2y.i0, s1h, h, false), ty1 = bl_tap(t2y.i1, s1h, h, false);
        const Tap tx0 = bl_tap(t2x.i0, s1w, w, false), tx1 = bl_tap(t2x.i1, s1w, w, false);
        const float* img = logits + n * h * w * (long long)ldl;
        const float4* p[4][4];      // [intermediate (row, col) pair][source tap]
        const Tap* tys[2] = {&ty0, &ty1};
        const Tap* txs[2] = {&tx0, &tx1};
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b) {
                const Tap &ty = *tys[a], &tx = *txs[b];
                p[a * 2 + b][0] = reinterpret_cast<const float4*>(img + ((long long)ty.i0 * w + tx.i0) * ldl);
                p[a * 2 + b][1] = reinterpret_cast<const float4*>(img + ((long long)ty.i0 * w + tx.i1) * ldl);
                p[a * 2 + b][2] = reinterpret_cast<const float4*>(img + ((long long)ty.i1 * w + tx.i0) * ldl);
                p[a * 2 + b][3] = reinterpret_cast<const float4*>(img + ((long long)ty.i1 * w + tx.i1) * ldl);
            }
        float best = -INFINITY;
        int label = 0;
        for (int q = 0; q * 4 < classes; ++q) {
            float m[4][4];      // [intermediate pair][class in the quad]
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const Tap &ty = *tys[k >> 1], &tx = *txs[k & 1];
                const float4 a = __ldg(p[k][0] + q), b = __ldg(p[k][1] + q), c = __ldg(p[k][2] + q), d = __ldg(p[k][3] + q);
                m[k][0] = bl_mix(ty, tx, a.x, b.x, c.x, d.x);
                m[k][1] = bl_mix(ty, tx, a.y, b.y, c.y, d.y);
                m[k][2] = bl_mix(ty, tx, a.z, b.z, c.z, d.z);
                m[k][3] = bl_mix(ty, tx, a.w, b.w, c.w, d.w);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int cls = q * 4 + j;
                const float v = bl_mix(t2y, t2x, m[0][j], m[1][j], m[2][j], m[3][j]);
                if (cls < classes && v > best) {
                    best = v;
                    label = cls;
                }
            }
        }
        labels[i] = label;
        if (rgb != nullptr) {
            rgb[i * 3 + 0] = palette[label * 3 + 0];
            rgb[i * 3 + 1] = palette[label * 3 + 1];
            rgb[i * 3 + 2] = palette[label * 3 + 2];
        }
    }
}

// HED's first conv as one K = 32 contraction: the im2col row of pixel (n, y, x) of a uint8 HWC image (3 channels in the image's
// order), column (ky 3 + kx) 3 + c = fp16(s (img[n, y + ky - 1, x + kx - 1, c] - norm[c])) computed in fp32, zero outside the image
// (the reference pads h = x - norm, after the subtraction) and in columns 27..31.  One pixel (four 16-byte vectors) per thread.
__global__ void hed_input_kernel(const uint8_t* __restrict__ img, const float* __restrict__ norm, uint4* __restrict__ cols, int H, int W,
                                 float s, long long total) {
    const float m[3] = {norm[0], norm[1], norm[2]};
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W);
        const long long r = i / W;
        const int y = (int)(r % H);
        const long long n = r / H;
        __align__(16) __half v[32];
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = y + ky - 1;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = x + kx - 1;
                const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
                const uint8_t* p = img + ((n * H + iy) * W + ix) * 3;
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    v[(ky * 3 + kx) * 3 + c] = in ? __float2half_rn(((float)p[c] - m[c]) * s) : __float2half_rn(0.0f);
            }
        }
#pragma unroll
        for (int j = 27; j < 32; ++j) v[j] = __float2half_rn(0.0f);
        const uint4* src = reinterpret_cast<const uint4*>(v);
#pragma unroll
        for (int j = 0; j < 4; ++j) cols[i * 4 + j] = src[j];
    }
}

// F.max_pool2d(kernel 2, stride 2) (floor: a last odd row / column is dropped) on NHWC fp16, 8 channels per thread.  The window is
// scanned in ATen's order and a value replaces the running maximum when it is greater or NaN, so the result is one of the inputs,
// bit for bit as ATen picks it.
__device__ __forceinline__ uint32_t hmax2_first(uint32_t m, uint32_t v) {
    const __half2 a = *reinterpret_cast<const __half2*>(&m), b = *reinterpret_cast<const __half2*>(&v);
    const bool lo = __hgt(__low2half(b), __low2half(a)) || __hisnan(__low2half(b));
    const bool hi = __hgt(__high2half(b), __high2half(a)) || __hisnan(__high2half(b));
    return (lo ? (v & 0xFFFFu) : (m & 0xFFFFu)) | (hi ? (v & 0xFFFF0000u) : (m & 0xFFFF0000u));
}
__global__ void max_pool2_f16_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int H, int W, int Ho, int Wo, int CV,
                                     long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(i % CV);
        long long r = i / CV;
        const int ox = (int)(r % Wo);
        r /= Wo;
        const int oy = (int)(r % Ho);
        const long long n = r / Ho;
        const uint4* p = x + ((n * H + 2 * oy) * W + 2 * ox) * CV + cv;
        const long long row = (long long)W * CV;
        uint4 m = p[0];
        const uint4 t[3] = {p[CV], p[row], p[row + CV]};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            m.x = hmax2_first(m.x, t[k].x);
            m.y = hmax2_first(m.y, t[k].y);
            m.z = hmax2_first(m.z, t[k].z);
            m.w = hmax2_first(m.w, t[k].w);
        }
        y[i] = m;
    }
}

// HED's post-processing (the reference's HEDdetector.__call__) per output pixel: each of the five fp32 side maps resized to (H, W) as
// cv2.resize(INTER_LINEAR) does on float images (resize.cpp: scale = 1 / (out / in) and src = (dst + 0.5) scale - 0.5 in double,
// rounded to float, floored, clamped to the edge; weights (1 - f, f); the horizontal pass, then the vertical one, each product and
// sum rounded to fp32; a map of the output's size is copied), the mean in numpy's order (((((e0 + e1) + e2) + e3) + e4) / 5 in fp32,
// then 1 / (1 + exp(-m)) in fp64, times 255, clipped, truncated to uint8 and inverted (cv2.bitwise_not).  Map k: pixel (n, y, x) at
// p[k][((n h + y) w + x) ld].
struct HedMaps {
    const float* p[5];
    int h[5], w[5];
    double sh[5], sw[5];
};
struct CvTap {
    int i0, i1;
    float f;
};
__device__ __forceinline__ CvTap cv_tap(int d, double scale, int in) {
    float f = (float)__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5);
    int s = (int)floorf(f);
    f = __fsub_rn(f, (float)s);
    if (s < 0) f = 0.0f, s = 0;
    if (s >= in - 1) f = 0.0f, s = in - 1;
    return CvTap{s, s + 1 < in ? s + 1 : s, f};
}
__global__ void hed_edges_kernel(HedMaps m, int ld, int H, int W, uint8_t* __restrict__ out, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W);
        const long long r = i / W;
        const int y = (int)(r % H);
        const long long n = r / H;
        float sum = 0.0f;
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const int h = m.h[k], w = m.w[k];
            const float* img = m.p[k] + n * h * w * (long long)ld;
            float e;
            if (h == H && w == W) {
                e = img[((long long)y * w + x) * ld];
            } else {
                const CvTap ty = cv_tap(y, m.sh[k], h), tx = cv_tap(x, m.sw[k], w);
                const float a0 = __fsub_rn(1.0f, tx.f), b0 = __fsub_rn(1.0f, ty.f);
                const float* r0 = img + (long long)ty.i0 * w * ld;
                const float* r1 = img + (long long)ty.i1 * w * ld;
                const float h0 = __fadd_rn(__fmul_rn(r0[(long long)tx.i0 * ld], a0), __fmul_rn(r0[(long long)tx.i1 * ld], tx.f));
                const float h1 = __fadd_rn(__fmul_rn(r1[(long long)tx.i0 * ld], a0), __fmul_rn(r1[(long long)tx.i1 * ld], tx.f));
                e = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, ty.f));
            }
            sum = k == 0 ? e : __fadd_rn(sum, e);
        }
        const float mean = __fdiv_rn(sum, 5.0f);
        double v = __dmul_rn(__ddiv_rn(1.0, __dadd_rn(1.0, exp(-(double)mean))), 255.0);
        v = v < 0.0 ? 0.0 : (v > 255.0 ? 255.0 : v);
        out[i] = (uint8_t)(255 - (int)v);
    }
}

static int dp_grid(long long n, int block = 256, int per_sm = 8) {
    long long g = (n + block - 1) / block;
    const long long cap = (long long)sm_count() * per_sm;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace anysd

using namespace anysd;

extern "C" {

int anysd_resize_bilinear_f16(const void* x, const void* addend, void* y, int N, int H, int W, int C, int Ho, int Wo, int ldy,
                              int align_corners, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && y, ANYSD_EINVAL, "resize_bilinear: null pointer");
    ANYSD_REQUIRE(N > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 8 == 0, ANYSD_EINVAL,
                  "resize_bilinear: bad dims N=%d %dx%d -> %dx%d C=%d (C must be a multiple of 8)", N, H, W, Ho, Wo, C);
    ANYSD_REQUIRE(ldy >= C && ldy % 8 == 0, ANYSD_EINVAL, "resize_bilinear: ldy=%d must be a multiple of 8 and >= C=%d", ldy, C);
    ANYSD_REQUIRE(align_corners == 0 || align_corners == 1, ANYSD_EINVAL, "resize_bilinear: align_corners must be 0 or 1");
    ANYSD_REQUIRE((uintptr_t)x % 16 == 0 && (uintptr_t)y % 16 == 0 && (uintptr_t)addend % 16 == 0, ANYSD_EINVAL,
                  "resize_bilinear: x, y and addend must be 16-byte aligned");
    const bool ac = align_corners != 0;
    const long long total = (long long)N * Ho * Wo * (C / 8);
    resize_bilinear_f16_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>(
        (const uint4*)x, (const uint4*)addend, (uint4*)y, H, W, Ho, Wo, C / 8, ldy / 8, bl_scale(H, Ho, ac), bl_scale(W, Wo, ac), ac,
        total);
    return check_launch("resize_bilinear_f16");
}

int anysd_resize_bilinear_ac_f32(const float* x, float* y, int N, int H, int W, int Ho, int Wo, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && y, ANYSD_EINVAL, "resize_bilinear_f32: null pointer");
    ANYSD_REQUIRE(N > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, ANYSD_EINVAL, "resize_bilinear_f32: bad dims N=%d %dx%d -> %dx%d", N, H,
                  W, Ho, Wo);
    const long long total = (long long)N * Ho * Wo;
    resize_bilinear_ac_f32_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>(x, y, H, W, Ho, Wo, bl_scale(H, Ho, true), bl_scale(W, Wo, true),
                                                                                     total);
    return check_launch("resize_bilinear_f32");
}

int anysd_relu_f16(const void* x, void* y, long long n, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && y && n > 0 && n % 8 == 0, ANYSD_EINVAL, "relu: bad args (n %% 8 == 0)");
    ANYSD_REQUIRE((uintptr_t)x % 16 == 0 && (uintptr_t)y % 16 == 0, ANYSD_EINVAL, "relu: x and y must be 16-byte aligned");
    relu_f16_kernel<<<dp_grid(n / 8), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, (uint4*)y, n / 8);
    return check_launch("relu");
}

int anysd_depth_to_space_f16(const void* g, void* out, int B, int gh, int gw, int r, int C, anysd_stream_t stream) {
    ANYSD_REQUIRE(g && out, ANYSD_EINVAL, "depth_to_space: null pointer");
    ANYSD_REQUIRE(B > 0 && gh > 0 && gw > 0 && r > 0 && C > 0 && C % 8 == 0, ANYSD_EINVAL,
                  "depth_to_space: bad dims B=%d %dx%d r=%d C=%d (C must be a multiple of 8)", B, gh, gw, r, C);
    ANYSD_REQUIRE((uintptr_t)g % 16 == 0 && (uintptr_t)out % 16 == 0, ANYSD_EINVAL, "depth_to_space: pointers must be 16-byte aligned");
    const long long total = (long long)B * gh * r * gw * r * (C / 8);
    depth_to_space_f16_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)g, (uint4*)out, gh, gw, r, C / 8, total);
    return check_launch("depth_to_space");
}

int anysd_space_to_depth_f16(const void* in, void* g, int B, int H, int W, int C, int r, anysd_stream_t stream) {
    ANYSD_REQUIRE(in && g, ANYSD_EINVAL, "space_to_depth: null pointer");
    ANYSD_REQUIRE(B > 0 && r > 0 && H >= r && W >= r && C > 0 && C % 8 == 0, ANYSD_EINVAL,
                  "space_to_depth: bad dims B=%d %dx%d r=%d C=%d (C must be a multiple of 8, H and W >= r)", B, H, W, r, C);
    ANYSD_REQUIRE((uintptr_t)in % 16 == 0 && (uintptr_t)g % 16 == 0, ANYSD_EINVAL, "space_to_depth: pointers must be 16-byte aligned");
    const int Ho = H / r, Wo = W / r;
    const long long total = (long long)B * Ho * Wo * r * r * (C / 8);
    space_to_depth_f16_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)in, (uint4*)g, H, W, Ho, Wo, r, C / 8,
                                                                                  total);
    return check_launch("space_to_depth");
}

int anysd_space_to_depth_u8(const void* in, void* g, int B, int H, int W, int C, int r, anysd_stream_t stream) {
    ANYSD_REQUIRE(in && g, ANYSD_EINVAL, "space_to_depth_u8: null pointer");
    ANYSD_REQUIRE(B > 0 && r > 0 && H >= r && W >= r && C > 0, ANYSD_EINVAL, "space_to_depth_u8: bad dims B=%d %dx%d r=%d C=%d", B, H,
                  W, r, C);
    ANYSD_REQUIRE((uintptr_t)g % 2 == 0, ANYSD_EINVAL, "space_to_depth_u8: g must be 2-byte aligned");
    const int Ho = H / r, Wo = W / r;
    const long long total = (long long)B * Ho * Wo * r * r * C;
    space_to_depth_u8_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>((const uint8_t*)in, (__half*)g, H, W, Ho, Wo, r, C,
                                                                                 total);
    return check_launch("space_to_depth_u8");
}

int anysd_dwconv_f16(const void* x, const float* w, const float* bias, const void* residual, void* y, int N, int H, int W, int C,
                     int k, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && w && bias && y, ANYSD_EINVAL, "dwconv: null pointer");
    ANYSD_REQUIRE(k == 3 || k == 5, ANYSD_EINVAL, "dwconv: kernel size %d (3 or 5)", k);
    ANYSD_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, ANYSD_EINVAL,
                  "dwconv: bad dims N=%d %dx%d C=%d (C must be a multiple of 8)", N, H, W, C);
    ANYSD_REQUIRE((uintptr_t)x % 16 == 0 && (uintptr_t)y % 16 == 0 && (uintptr_t)residual % 16 == 0 && (uintptr_t)w % 16 == 0 &&
                      (uintptr_t)bias % 16 == 0,
                  ANYSD_EINVAL, "dwconv: pointers must be 16-byte aligned");
    ANYSD_REQUIRE(x != y, ANYSD_EINVAL, "dwconv: y must not alias x (neighbouring pixels are read)");
    const long long total = (long long)N * H * W * (C / 8);
    if (k == 3)
        dwconv_f16_kernel<3><<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, w, bias, (const uint4*)residual,
                                                                                (uint4*)y, H, W, C / 8, total);
    else
        dwconv_f16_kernel<5><<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, w, bias, (const uint4*)residual,
                                                                                (uint4*)y, H, W, C / 8, total);
    return check_launch("dwconv");
}

int anysd_adaptive_avg_pool_f16(const void* x, void* y, int N, int H, int W, int C, int Ho, int Wo, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && y, ANYSD_EINVAL, "adaptive_avg_pool: null pointer");
    ANYSD_REQUIRE(N > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 8 == 0, ANYSD_EINVAL,
                  "adaptive_avg_pool: bad dims N=%d %dx%d -> %dx%d C=%d (C must be a multiple of 8)", N, H, W, Ho, Wo, C);
    ANYSD_REQUIRE((uintptr_t)x % 16 == 0 && (uintptr_t)y % 16 == 0, ANYSD_EINVAL, "adaptive_avg_pool: pointers must be 16-byte aligned");
    const long long total = (long long)N * Ho * Wo * (C / 8);
    adaptive_avg_pool_f16_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, (uint4*)y, H, W, Ho, Wo, C / 8,
                                                                                     total);
    return check_launch("adaptive_avg_pool");
}

int anysd_seg_labels_f32(const float* logits, int N, int h, int w, int ldl, int classes, int Hm, int Wm, int Ho, int Wo,
                         long long* labels, const void* palette, void* rgb, anysd_stream_t stream) {
    ANYSD_REQUIRE(logits && labels, ANYSD_EINVAL, "seg_labels: null pointer");
    ANYSD_REQUIRE(N > 0 && h > 0 && w > 0 && Hm > 0 && Wm > 0 && Ho > 0 && Wo > 0, ANYSD_EINVAL,
                  "seg_labels: bad dims N=%d %dx%d -> %dx%d -> %dx%d", N, h, w, Hm, Wm, Ho, Wo);
    ANYSD_REQUIRE(classes > 0 && ldl >= classes && ldl % 4 == 0, ANYSD_EINVAL,
                  "seg_labels: classes=%d, ldl=%d (a multiple of 4, >= classes)", classes, ldl);
    ANYSD_REQUIRE((palette == nullptr) == (rgb == nullptr), ANYSD_EINVAL, "seg_labels: palette and rgb go together");
    ANYSD_REQUIRE((uintptr_t)logits % 16 == 0 && (uintptr_t)labels % 8 == 0, ANYSD_EINVAL, "seg_labels: misaligned pointers");
    const long long total = (long long)N * Ho * Wo;
    seg_labels_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>(
        logits, h, w, ldl, classes, Hm, Wm, Ho, Wo, bl_scale(h, Hm, false), bl_scale(w, Wm, false), bl_scale(Hm, Ho, false),
        bl_scale(Wm, Wo, false), labels, (const uint8_t*)palette, (uint8_t*)rgb, total);
    return check_launch("seg_labels");
}

int anysd_hed_input_u8(const void* img, const float* norm, void* cols, int B, int H, int W, float scale, anysd_stream_t stream) {
    ANYSD_REQUIRE(img && norm && cols, ANYSD_EINVAL, "hed_input: null pointer");
    ANYSD_REQUIRE(B > 0 && H > 0 && W > 0, ANYSD_EINVAL, "hed_input: bad dims B=%d %dx%d", B, H, W);
    ANYSD_REQUIRE((uintptr_t)cols % 16 == 0, ANYSD_EINVAL, "hed_input: cols must be 16-byte aligned");
    const long long total = (long long)B * H * W;
    hed_input_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>((const uint8_t*)img, norm, (uint4*)cols, H, W, scale, total);
    return check_launch("hed_input");
}

int anysd_max_pool2_f16(const void* x, void* y, int N, int H, int W, int C, anysd_stream_t stream) {
    ANYSD_REQUIRE(x && y, ANYSD_EINVAL, "max_pool2: null pointer");
    ANYSD_REQUIRE(N > 0 && H >= 2 && W >= 2 && C > 0 && C % 8 == 0, ANYSD_EINVAL,
                  "max_pool2: bad dims N=%d %dx%d C=%d (H, W >= 2; C must be a multiple of 8)", N, H, W, C);
    ANYSD_REQUIRE((uintptr_t)x % 16 == 0 && (uintptr_t)y % 16 == 0, ANYSD_EINVAL, "max_pool2: pointers must be 16-byte aligned");
    const int Ho = H / 2, Wo = W / 2;
    const long long total = (long long)N * Ho * Wo * (C / 8);
    max_pool2_f16_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, (uint4*)y, H, W, Ho, Wo, C / 8, total);
    return check_launch("max_pool2");
}

int anysd_hed_edges_u8(const float* const* maps, const int* sizes, int ld, int N, int H, int W, void* out, anysd_stream_t stream) {
    ANYSD_REQUIRE(maps && sizes && out, ANYSD_EINVAL, "hed_edges: null pointer");
    ANYSD_REQUIRE(N > 0 && H > 0 && W > 0 && ld > 0, ANYSD_EINVAL, "hed_edges: bad dims N=%d %dx%d ld=%d", N, H, W, ld);
    HedMaps m;
    for (int k = 0; k < 5; ++k) {
        m.p[k] = maps[k];
        m.h[k] = sizes[2 * k];
        m.w[k] = sizes[2 * k + 1];
        ANYSD_REQUIRE(m.p[k] && m.h[k] > 0 && m.w[k] > 0, ANYSD_EINVAL, "hed_edges: side map %d is null or empty (%dx%d)", k, m.h[k],
                      m.w[k]);
        ANYSD_REQUIRE((uintptr_t)m.p[k] % 4 == 0, ANYSD_EINVAL, "hed_edges: side map %d must be 4-byte aligned", k);
        // cv2 resize.cpp: inv_scale = (double)dsize / ssize, scale = 1. / inv_scale
        m.sh[k] = 1.0 / ((double)H / m.h[k]);
        m.sw[k] = 1.0 / ((double)W / m.w[k]);
    }
    const long long total = (long long)N * H * W;
    hed_edges_kernel<<<dp_grid(total), 256, 0, (cudaStream_t)stream>>>(m, ld, H, W, (uint8_t*)out, total);
    return check_launch("hed_edges");
}

}  // extern "C"
