// AnyDoor's pair preparation and crop-back (visual_reference_tool.py process_pairs / crop_back, tools/tool.py sobel), equal to
// the reference's OpenCV and numpy arithmetic (oracle/anydoor_oracle.py states every formula; DESIGN.md §10.8).
//   anydoor_bbox      one CTA per mask: pixel count, first / last row and column, and the largest value (the host refuses > 1)
//   anydoor_ref       the masked reference crop, expanded and padded to a square (never materialised: a source pixel is read
//                     through the per-pair geometry) -> 224 x 224 uint8 image, mask * 255, and ref = float32(x / 255 in double)
//   anydoor_hf_up     224 -> 256: the image (uint8 linear) and the mask / 255 (float64 linear) > 0.5
//   anydoor_hf_core   9 x 9 erode of the mask (= two 5 x 5 erodes, border ignored), 3 x 3 Sobel x / y with BORDER_REFLECT_101,
//                     convertScaleAbs, addWeighted(0.5, 0.5), channel max * mask, < 50 -> 0, uint8(s / 255 * img)
//   anydoor_hf_down   256 -> 224
//   anydoor_collage   per 512 x 512 output pixel: the target crop and the collage (the high-frequency map resized to the box
//                     and pasted) padded to a square with 0, resized; the mask channel is INTER_NEAREST of 1 in the box and in the
//                     padding band; jpg / hint = x / 127.5 - 1 in fp32
//   anydoor_crop_back the decoded image * 127.5 + 127.5 (two fp32 roundings), clipped, first row dropped, float32 linear resize
//                     to the padded crop, un-padded and pasted with a 5-pixel margin (truncated to uint8); elsewhere tar_image
// The host keeps only the integer box geometry (one int32 row of ANYDOOR_P per pair).  No FMA anywhere: every float product and
// sum is written with an _rn intrinsic, so the rounding is the reference's.
#include "common.cuh"

namespace anysd {

namespace {

enum {  // the per-pair geometry row (anydoor.py PairGeometry.row)
    P_RY0, P_RX0, P_RH, P_RW, P_ROY, P_ROX, P_RS,                     // ref crop origin / size, square -> crop offset, square side
    P_CY1, P_CX1, P_HC, P_WC, P_BY1, P_BX1, P_BH, P_BW, P_QY, P_QX, P_S2,  // target crop, box in it, square pad offset, side
    P_COUNT
};
static_assert(P_COUNT == ANYDOOR_P, "geometry row");

constexpr int REF = 224, HF = 256, OUT = 512, MARGIN = 5, THRESH = 50;

struct Tap {
    int i0, i1;
    float w0, w1;
};

// One axis of cv2.resize(INTER_LINEAR): f = float((d + 0.5) * (1 / (out / in)) - 0.5) in double, s = floor(f), f -= s.  Along x
// (clamp) an index outside [0, in - 1] is clamped with its fraction zeroed; along y only the two rows are clamped.
__device__ __forceinline__ Tap axis_tap(int d, int n_in, int n_out, bool clamp) {
    const double scale = __drcp_rn(__ddiv_rn((double)n_out, (double)n_in));
    float f = __double2float_rn(__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5));
    int s = (int)floorf(f);
    f = __fsub_rn(f, (float)s);
    if (clamp && (s < 0 || s >= n_in - 1)) {
        f = 0.0f;
        s = s < 0 ? 0 : n_in - 1;
    }
    Tap t;
    t.i0 = min(max(s, 0), n_in - 1);
    t.i1 = min(max(s + 1, 0), n_in - 1);
    t.w0 = __fsub_rn(1.0f, f);
    t.w1 = f;
    return t;
}

__device__ __forceinline__ int q11(float w) { return __float2int_rn(__fmul_rn(w, 2048.0f)); }

// uint8 INTER_LINEAR at output (oy, ox) of an (ih, iw) -> (oh, ow) resize, pixel values from fetch(y, x).
template <class Fetch>
__device__ __forceinline__ int resize_u8_at(int oy, int ox, int ih, int iw, int oh, int ow, Fetch fetch) {
    const Tap tx = axis_tap(ox, iw, ow, true), ty = axis_tap(oy, ih, oh, false);
    const int a0 = q11(tx.w0), a1 = q11(tx.w1), b0 = q11(ty.w0), b1 = q11(ty.w1);
    const int s0 = fetch(ty.i0, tx.i0) * a0 + fetch(ty.i0, tx.i1) * a1;
    const int s1 = fetch(ty.i1, tx.i0) * a0 + fetch(ty.i1, tx.i1) * a1;
    return ((((s0 >> 4) * b0) >> 16) + (((s1 >> 4) * b1) >> 16) + 2) >> 2;
}

__device__ __forceinline__ float norm127(int v) { return __fsub_rn(__fdiv_rn((float)v, 127.5f), 1.0f); }

// ---- generic exact uint8 resize ----------------------------------------------------------------------------------------
__global__ void resize_u8_kernel(const uint8_t* __restrict__ src, int ih, int iw, int C, uint8_t* __restrict__ dst, int oh, int ow) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= oh * ow) return;
    const int b = blockIdx.y, oy = p / ow, ox = p % ow;
    const uint8_t* s = src + (size_t)b * ih * iw * C;
    for (int c = 0; c < C; ++c)
        dst[((size_t)b * oh * ow + p) * C + c] =
            (uint8_t)resize_u8_at(oy, ox, ih, iw, oh, ow, [&](int y, int x) { return (int)s[((size_t)y * iw + x) * C + c]; });
}

// ---- bounding box of each mask -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) anydoor_bbox_kernel(const uint8_t* __restrict__ masks, int H, int W, int* __restrict__ out) {
    const uint8_t* m = masks + (size_t)blockIdx.x * H * W;
    int cnt = 0, y0 = H, y1 = -1, x0 = W, x1 = -1, mx = 0;
    for (int i = threadIdx.x; i < H * W; i += blockDim.x) {
        const int v = m[i];
        if (v) {
            const int y = i / W, x = i % W;
            cnt += v;
            y0 = min(y0, y), y1 = max(y1, y), x0 = min(x0, x), x1 = max(x1, x);
            mx = max(mx, v);
        }
    }
    __shared__ int red[6][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int o = 16; o > 0; o >>= 1) {
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        y0 = min(y0, __shfl_xor_sync(0xffffffffu, y0, o));
        y1 = max(y1, __shfl_xor_sync(0xffffffffu, y1, o));
        x0 = min(x0, __shfl_xor_sync(0xffffffffu, x0, o));
        x1 = max(x1, __shfl_xor_sync(0xffffffffu, x1, o));
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if (lane == 0) red[0][warp] = cnt, red[1][warp] = y0, red[2][warp] = y1, red[3][warp] = x0, red[4][warp] = x1, red[5][warp] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < nw; ++w) {
            cnt += red[0][w];
            y0 = min(y0, red[1][w]), y1 = max(y1, red[2][w]), x0 = min(x0, red[3][w]), x1 = max(x1, red[4][w]);
            mx = max(mx, red[5][w]);
        }
        int* o = out + blockIdx.x * 6;
        o[0] = cnt, o[1] = y0, o[2] = y1, o[3] = x0, o[4] = x1, o[5] = mx;
    }
}

// ---- reference branch ----------------------------------------------------------------------------------------------------
__global__ void anydoor_ref_kernel(const uint8_t* __restrict__ img, const uint8_t* __restrict__ mask, int H, int W,
                                   const int* __restrict__ geom, uint8_t* __restrict__ ref_u8, uint8_t* __restrict__ mask_u8,
                                   float* __restrict__ ref_f32) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= REF * REF) return;
    const int b = blockIdx.y, oy = p / REF, ox = p % REF;
    const int* g = geom + b * ANYDOOR_P;
    const uint8_t* im = img + (size_t)b * H * W * 3;
    const uint8_t* mk = mask + (size_t)b * H * W;
    const int S = g[P_RS];
    // square (y, x) -> the crop pixel, or -1 in the expansion and the square padding
    auto at = [&](int y, int x) -> long long {
        const int cy = y - g[P_ROY], cx = x - g[P_ROX];
        if (cy < 0 || cy >= g[P_RH] || cx < 0 || cx >= g[P_RW]) return -1;
        return (long long)(g[P_RY0] + cy) * W + (g[P_RX0] + cx);
    };
    const size_t o = (size_t)b * REF * REF + p;
    for (int c = 0; c < 3; ++c) {
        const int v = resize_u8_at(oy, ox, S, S, REF, REF, [&](int y, int x) {
            const long long i = at(y, x);
            return (i < 0 || !mk[i]) ? 255 : (int)im[i * 3 + c];
        });
        ref_u8[o * 3 + c] = (uint8_t)v;
        ref_f32[o * 3 + c] = __double2float_rn(__ddiv_rn((double)v, 255.0));
    }
    mask_u8[o] = (uint8_t)resize_u8_at(oy, ox, S, S, REF, REF, [&](int y, int x) {
        const long long i = at(y, x);
        return (i >= 0 && mk[i]) ? 255 : 0;
    });
}

// ---- sobel ---------------------------------------------------------------------------------------------------------------
__global__ void anydoor_hf_up_kernel(const uint8_t* __restrict__ ref_u8, const uint8_t* __restrict__ mask_u8,
                                     uint8_t* __restrict__ img256, uint8_t* __restrict__ m256) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HF * HF) return;
    const int b = blockIdx.y, oy = p / HF, ox = p % HF;
    const uint8_t* s = ref_u8 + (size_t)b * REF * REF * 3;
    const size_t o = (size_t)b * HF * HF + p;
    for (int c = 0; c < 3; ++c)
        img256[o * 3 + c] =
            (uint8_t)resize_u8_at(oy, ox, REF, REF, HF, HF, [&](int y, int x) { return (int)s[(y * REF + x) * 3 + c]; });
    // the float64 resize of mask / 255 (weights float32, products and sums in double), then > 0.5
    const uint8_t* m = mask_u8 + (size_t)b * REF * REF;
    const Tap tx = axis_tap(ox, REF, HF, true), ty = axis_tap(oy, REF, HF, false);
    auto v = [&](int y, int x) { return __ddiv_rn((double)m[y * REF + x], 255.0); };
    auto row = [&](int y) { return __dadd_rn(__dmul_rn(v(y, tx.i0), (double)tx.w0), __dmul_rn(v(y, tx.i1), (double)tx.w1)); };
    const double r = __dadd_rn(__dmul_rn(row(ty.i0), (double)ty.w0), __dmul_rn(row(ty.i1), (double)ty.w1));
    m256[o] = r > 0.5 ? 1 : 0;
}

__device__ __forceinline__ int reflect101(int v, int n) { return v < 0 ? -v : (v >= n ? 2 * n - 2 - v : v); }

__global__ void anydoor_hf_core_kernel(const uint8_t* __restrict__ img256, const uint8_t* __restrict__ m256,
                                       uint8_t* __restrict__ hf256) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HF * HF) return;
    const int b = blockIdx.y, y = p / HF, x = p % HF;
    const uint8_t* m = m256 + (size_t)b * HF * HF;
    const uint8_t* im = img256 + (size_t)b * HF * HF * 3;
    int keep = 1;
    for (int dy = -4; dy <= 4 && keep; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= HF) continue;
        for (int dx = -4; dx <= 4; ++dx) {
            const int xx = x + dx;
            if (xx >= 0 && xx < HF && !m[yy * HF + xx]) {
                keep = 0;
                break;
            }
        }
    }
    const int ym = reflect101(y - 1, HF), yp = reflect101(y + 1, HF), xm = reflect101(x - 1, HF), xp = reflect101(x + 1, HF);
    int s = 0;
    for (int c = 0; c < 3; ++c) {
        auto P = [&](int yy, int xx) { return (int)im[(yy * HF + xx) * 3 + c]; };
        const int gx = (P(ym, xp) - P(ym, xm)) + 2 * (P(y, xp) - P(y, xm)) + (P(yp, xp) - P(yp, xm));
        const int gy = (P(yp, xm) - P(ym, xm)) + 2 * (P(yp, x) - P(ym, x)) + (P(yp, xp) - P(ym, xp));
        const int ax = min(abs(gx), 255), ay = min(abs(gy), 255);
        s = max(s, __float2int_rn(__fmul_rn((float)(ax + ay), 0.5f)));      // addWeighted: rint((a + b) / 2), half to even
    }
    s *= keep;
    if (s < THRESH) s = 0;
    const float w = __fdiv_rn((float)s, 255.0f);
    const size_t o = ((size_t)b * HF * HF + p) * 3;
    for (int c = 0; c < 3; ++c) hf256[o + c] = (uint8_t)(int)__fmul_rn(w, (float)im[p * 3 + c]);
}

__global__ void anydoor_hf_down_kernel(const uint8_t* __restrict__ hf256, uint8_t* __restrict__ hf224) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= REF * REF) return;
    const int b = blockIdx.y, oy = p / REF, ox = p % REF;
    const uint8_t* s = hf256 + (size_t)b * HF * HF * 3;
    for (int c = 0; c < 3; ++c)
        hf224[((size_t)b * REF * REF + p) * 3 + c] =
            (uint8_t)resize_u8_at(oy, ox, HF, HF, REF, REF, [&](int y, int x) { return (int)s[(y * HF + x) * 3 + c]; });
}

// ---- target branch -------------------------------------------------------------------------------------------------------
__global__ void anydoor_collage_kernel(const uint8_t* __restrict__ tar, int H, int W, const uint8_t* __restrict__ hf224,
                                       const int* __restrict__ geom, float* __restrict__ jpg, float* __restrict__ hint) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= OUT * OUT) return;
    const int b = blockIdx.y, oy = p / OUT, ox = p % OUT;
    const int* g = geom + b * ANYDOOR_P;
    const uint8_t* t = tar + (size_t)b * H * W * 3;
    const uint8_t* hf = hf224 + (size_t)b * REF * REF * 3;
    const int S2 = g[P_S2], Hc = g[P_HC], Wc = g[P_WC], by1 = g[P_BY1], bx1 = g[P_BX1], bh = g[P_BH], bw = g[P_BW];
    const size_t o = (size_t)b * OUT * OUT + p;
    for (int c = 0; c < 3; ++c) {
        auto target = [&](int y, int x) {
            const int ty = y - g[P_QY], tx = x - g[P_QX];
            if (ty < 0 || ty >= Hc || tx < 0 || tx >= Wc) return -1;
            return ty * Wc + tx;
        };
        const int vt = resize_u8_at(oy, ox, S2, S2, OUT, OUT, [&](int y, int x) {
            const int i = target(y, x);
            return i < 0 ? 0 : (int)t[((size_t)(g[P_CY1] + i / Wc) * W + g[P_CX1] + i % Wc) * 3 + c];
        });
        const int vc = resize_u8_at(oy, ox, S2, S2, OUT, OUT, [&](int y, int x) {
            const int i = target(y, x);
            if (i < 0) return 0;
            const int ty = i / Wc - by1, tx = i % Wc - bx1;
            if (ty >= 0 && ty < bh && tx >= 0 && tx < bw)          // the high-frequency map resized to the box
                return resize_u8_at(ty, tx, REF, REF, bh, bw, [&](int yy, int xx) { return (int)hf[(yy * REF + xx) * 3 + c]; });
            return (int)t[((size_t)(g[P_CY1] + i / Wc) * W + g[P_CX1] + i % Wc) * 3 + c];
        });
        jpg[o * 3 + c] = norm127(vt);
        hint[o * 4 + c] = norm127(vc);
    }
    // INTER_NEAREST of the mask: 1 in the box, 0 elsewhere in the crop, 255 (-1.0 cast to uint8) in the padding band; then > 0.5
    const double inv = __drcp_rn(__ddiv_rn((double)OUT, (double)S2));
    const int sy = min((int)floor(__dmul_rn((double)oy, inv)), S2 - 1), sx = min((int)floor(__dmul_rn((double)ox, inv)), S2 - 1);
    const int ty = sy - g[P_QY], tx = sx - g[P_QX];
    const bool crop = ty >= 0 && ty < Hc && tx >= 0 && tx < Wc;
    const bool box = ty >= by1 && ty < by1 + bh && tx >= bx1 && tx < bx1 + bw;
    hint[o * 4 + 3] = (!crop || box) ? 1.0f : 0.0f;
}

// ---- crop back -----------------------------------------------------------------------------------------------------------
// decoded != 0: src is the decoder's fp32 [3, 512, 512] per pair; else the reference's pred, fp32 [511, 512, 3] already scaled,
// clipped and cut (crop_back's own argument).
__global__ void anydoor_crop_back_kernel(const float* __restrict__ src_, int decoded, const uint8_t* __restrict__ tar, int H, int W,
                                         const int* __restrict__ geom, uint8_t* __restrict__ out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= H * W) return;
    const int b = blockIdx.y, y = p / W, x = p % W;
    const int* g = geom + b * ANYDOOR_P;
    const size_t o = ((size_t)b * H * W + p) * 3;
    const int ly = y - g[P_CY1], lx = x - g[P_CX1];
    if (ly < MARGIN || ly >= g[P_HC] - MARGIN || lx < MARGIN || lx >= g[P_WC] - MARGIN) {
        for (int c = 0; c < 3; ++c) out[o + c] = tar[o + c];
        return;
    }
    const int S2 = g[P_S2], IH = OUT - 1, IW = OUT;               // the source is rows 1 .. 511 of the decoded image
    const Tap tx = axis_tap(lx + g[P_QX], IW, S2, true), ty = axis_tap(ly + g[P_QY], IH, S2, false);
    const float* d = src_ + (size_t)b * 3 * (decoded ? OUT : IH) * IW;
    for (int c = 0; c < 3; ++c) {
        auto src = [&](int yy, int xx) {
            if (!decoded) return d[((size_t)yy * IW + xx) * 3 + c];
            const float v = __fadd_rn(__fmul_rn(d[((size_t)c * OUT + yy + 1) * OUT + xx], 127.5f), 127.5f);
            return fminf(fmaxf(v, 0.0f), 255.0f);
        };
        auto row = [&](int yy) { return __fadd_rn(__fmul_rn(src(yy, tx.i0), tx.w0), __fmul_rn(src(yy, tx.i1), tx.w1)); };
        const float v = __fadd_rn(__fmul_rn(row(ty.i0), ty.w0), __fmul_rn(row(ty.i1), ty.w1));
        out[o + c] = (uint8_t)(int)v;                               // float -> uint8 assignment truncates
    }
}

dim3 grid2(int n, int B) { return dim3((n + 255) / 256, B); }

}  // namespace

}  // namespace anysd

using namespace anysd;

extern "C" {

int anysd_resize_linear_u8(const void* src, int B, int H, int W, int C, void* dst, int OH, int OW, anysd_stream_t stream) {
    ANYSD_REQUIRE(src && dst, ANYSD_EINVAL, "resize_linear_u8: null pointer");
    ANYSD_REQUIRE(B > 0 && B <= 65535 && H > 0 && W > 0 && C > 0 && OH > 0 && OW > 0, ANYSD_EINVAL,
                  "resize_linear_u8: bad dims B=%d %dx%dx%d -> %dx%d", B, H, W, C, OH, OW);
    ANYSD_REQUIRE((long long)H * W * C < (1LL << 31) && (long long)OH * OW * C < (1LL << 31), ANYSD_EINVAL,
                  "resize_linear_u8: image too large");
    resize_u8_kernel<<<grid2(OH * OW, B), 256, 0, (cudaStream_t)stream>>>((const uint8_t*)src, H, W, C, (uint8_t*)dst, OH, OW);
    return check_launch("resize_linear_u8");
}

int anysd_anydoor_bbox_u8(const void* masks, int B, int H, int W, void* out, anysd_stream_t stream) {
    ANYSD_REQUIRE(masks && out, ANYSD_EINVAL, "anydoor_bbox: null pointer");
    ANYSD_REQUIRE(B > 0 && H > 0 && W > 0 && (long long)H * W < (1LL << 23), ANYSD_EINVAL, "anydoor_bbox: bad dims B=%d %dx%d", B, H,
                  W);
    anydoor_bbox_kernel<<<B, 1024, 0, (cudaStream_t)stream>>>((const uint8_t*)masks, H, W, (int*)out);
    return check_launch("anydoor_bbox");
}

int anysd_anydoor_sobel(const void* ref_u8, const void* mask_u8, int B, void* img256, void* m256, void* hf256, void* hf224,
                        anysd_stream_t stream) {
    ANYSD_REQUIRE(ref_u8 && mask_u8 && img256 && m256 && hf256 && hf224, ANYSD_EINVAL, "anydoor_sobel: null pointer");
    ANYSD_REQUIRE(B > 0 && B <= 65535, ANYSD_EINVAL, "anydoor_sobel: bad batch %d", B);
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    anydoor_hf_up_kernel<<<grid2(HF * HF, B), 256, 0, st>>>((const uint8_t*)ref_u8, (const uint8_t*)mask_u8, (uint8_t*)img256,
                                                             (uint8_t*)m256);
    if ((rc = check_launch("anydoor_hf_up"))) return rc;
    anydoor_hf_core_kernel<<<grid2(HF * HF, B), 256, 0, st>>>((const uint8_t*)img256, (const uint8_t*)m256, (uint8_t*)hf256);
    if ((rc = check_launch("anydoor_hf_core"))) return rc;
    anydoor_hf_down_kernel<<<grid2(REF * REF, B), 256, 0, st>>>((const uint8_t*)hf256, (uint8_t*)hf224);
    return check_launch("anydoor_hf_down");
}

int anysd_anydoor_prepare(const void* ref_img, const void* ref_mask, int RH, int RW, const void* tar_img, int TH, int TW, int B, const void* geom,
                          void* ref_u8, void* mask_u8, void* img256, void* m256, void* hf256, void* hf224, void* ref_f32, void* jpg,
                          void* hint, anysd_stream_t stream) {
    ANYSD_REQUIRE(ref_img && ref_mask && tar_img && geom && ref_u8 && mask_u8 && img256 && m256 && hf256 && hf224 && ref_f32 && jpg &&
                      hint,
                  ANYSD_EINVAL, "anydoor_prepare: null pointer");
    ANYSD_REQUIRE(B > 0 && B <= 65535 && RH > 0 && RW > 0 && TH > 0 && TW > 0 && (long long)RH * RW * 3 < (1LL << 31) &&
                      (long long)TH * TW * 3 < (1LL << 31),
                  ANYSD_EINVAL, "anydoor_prepare: bad dims B=%d ref %dx%d tar %dx%d", B, RH, RW, TH, TW);
    cudaStream_t st = (cudaStream_t)stream;
    const int* g = (const int*)geom;
    int rc;
    anydoor_ref_kernel<<<grid2(REF * REF, B), 256, 0, st>>>((const uint8_t*)ref_img, (const uint8_t*)ref_mask, RH, RW, g,
                                                             (uint8_t*)ref_u8, (uint8_t*)mask_u8, (float*)ref_f32);
    if ((rc = check_launch("anydoor_ref"))) return rc;
    if ((rc = anysd_anydoor_sobel(ref_u8, mask_u8, B, img256, m256, hf256, hf224, stream))) return rc;
    anydoor_collage_kernel<<<grid2(OUT * OUT, B), 256, 0, st>>>((const uint8_t*)tar_img, TH, TW, (const uint8_t*)hf224, g, (float*)jpg,
                                                                 (float*)hint);
    return check_launch("anydoor_collage");
}

int anysd_anydoor_crop_back(const void* src, int decoded, const void* tar_img, int B, int H, int W, const void* geom, void* out,
                            anysd_stream_t stream) {
    ANYSD_REQUIRE(src && tar_img && geom && out, ANYSD_EINVAL, "anydoor_crop_back: null pointer");
    ANYSD_REQUIRE(B > 0 && B <= 65535 && H > 0 && W > 0 && (long long)H * W * 3 < (1LL << 31), ANYSD_EINVAL,
                  "anydoor_crop_back: bad dims B=%d %dx%d", B, H, W);
    anydoor_crop_back_kernel<<<grid2(H * W, B), 256, 0, (cudaStream_t)stream>>>((const float*)src, decoded, (const uint8_t*)tar_img, H, W,
                                                                                 (const int*)geom, (uint8_t*)out);
    return check_launch("anydoor_crop_back");
}

}  // extern "C"
