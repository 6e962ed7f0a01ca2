// AnyEdit's Canny sketch annotator (visual_condition_tool.py img2sketch: cvtColor(BGR2GRAY), GaussianBlur((3, 3), 0),
// Canny(low, high), bitwise_not), equal to OpenCV on every pixel.  All of it is integer arithmetic (DESIGN.md §10.7).
//   sketch_tile      per 32 x 32 output tile: the BGR image with a 3-pixel halo -> grey -> blur -> Sobel magnitude -> non-maximum
//                    suppression -> class (0 none, 1 weak, 2 strong, written to out), then union-find of the tile's candidates
//                    in shared memory; writes each candidate's tile-local root as its global label, -1 elsewhere, and clears
//                    the pixel's flag
//   sketch_merge     for every tile-border pixel, the union with its candidate neighbours in the tiles above, left and
//                    up-right, on the global labels (atomic-min union with path compression)
//   sketch_flag      every candidate's label is compressed to its root; a strong pixel flags its root
//   sketch_out       out = 255 - 255 (candidate && flagged[label]), the bitwise_not folded in
// Four launches per batch, whatever the image holds; a label is a pixel index in the batch, and always <= its own pixel's.
#include "common.cuh"

namespace anysd {

namespace {

constexpr int TW = 32, TH = 32, THREADS = 256;
constexpr int GW = TW + 6, GH = TH + 6;          // grey: the tile with a 3-pixel halo
constexpr int BW = TW + 4, BH = TH + 4;          // blur: 2-pixel halo
constexpr int MW = TW + 2, MH = TH + 2;          // magnitude: 1-pixel halo

__device__ __forceinline__ int clampi(int v, int n) { return v < 0 ? 0 : (v >= n ? n - 1 : v); }

// BORDER_REFLECT_101 for the positions -1 and n (the only ones the blur reads); further out any pixel of the image will do.
// An axis of length 1 reflects onto itself.
__device__ __forceinline__ int reflect101(int v, int n) {
    if (v < 0) v = -v;
    if (v >= n) v = 2 * n - 2 - v;
    return clampi(v, n);
}

struct TileSmem {
    uint8_t g[GH][GW];
    uint8_t b[BH][BW];
    int16_t m[MH][MW];
    int lab[TH * TW];
};

// Sobel dx, dy at blur position (by, bx); the blur array already holds the replicated border.
__device__ __forceinline__ void sobel3(const TileSmem& s, int by, int bx, int& dx, int& dy) {
    const int a0 = s.b[by - 1][bx - 1], a1 = s.b[by - 1][bx], a2 = s.b[by - 1][bx + 1];
    const int c0 = s.b[by][bx - 1], c2 = s.b[by][bx + 1];
    const int e0 = s.b[by + 1][bx - 1], e1 = s.b[by + 1][bx], e2 = s.b[by + 1][bx + 1];
    dx = (a2 - a0) + 2 * (c2 - c0) + (e2 - e0);
    dy = (e0 - a0) + 2 * (e1 - a1) + (e2 - a2);
}

__device__ __forceinline__ int find_smem(volatile int* lab, int x) {
    int p = lab[x];
    while (p != x) {
        x = p;
        p = lab[x];
    }
    return x;
}

// Union by atomic minimum: the larger root is pointed at the smaller one; a lost race (the root was linked meanwhile) retries
// from the new parent.  Labels only decrease, and always point to a lower index, so every find ends.
__device__ __forceinline__ void unite_smem(int* lab, int a, int b) {
    volatile int* v = lab;
    while (true) {
        a = find_smem(v, a);
        b = find_smem(v, b);
        if (a == b) return;
        if (a > b) {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicMin(&lab[b], a);
        if (old == b) return;
        b = old;
    }
}

// The same on the global labels, with path compression: a pixel's label is lowered to the root its find reached, which is an
// ancestor in the same set, so compression never links two sets and never raises a label.
__device__ __forceinline__ int find_global(int* L, int x) {
    volatile int* v = L;
    const int x0 = x;
    int p = v[x];
    while (p != x) {
        x = p;
        p = v[x];
    }
    if (x != x0) atomicMin(&L[x0], x);
    return x;
}

__device__ __forceinline__ void unite_global(int* L, int a, int b) {
    while (true) {
        a = find_global(L, a);
        b = find_global(L, b);
        if (a == b) return;
        if (a > b) {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicMin(&L[b], a);
        if (old == b) return;
        b = old;
    }
}

__global__ void __launch_bounds__(THREADS) sketch_tile_kernel(const uint8_t* __restrict__ img, int H, int W, int low, int high,
                                                               uint8_t* __restrict__ cls, int* __restrict__ labels,
                                                               uint8_t* __restrict__ flags) {
    __shared__ TileSmem s;
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    const long long base = (long long)blockIdx.z * H * W;
    const uint8_t* im = img + base * 3;

    // grey of the tile and a 3-pixel halo: BORDER_REFLECT_101 positions for the blur's reads outside the image
    for (int i = tid; i < GH * GW; i += THREADS) {
        const int ly = i / GW, lx = i - ly * GW;
        const int y = reflect101(y0 - 3 + ly, H), x = reflect101(x0 - 3 + lx, W);
        const uint8_t* p = im + ((long long)y * W + x) * 3;
        s.g[ly][lx] = (uint8_t)(((int)p[0] * 3735 + (int)p[1] * 19235 + (int)p[2] * 9798 + (1 << 14)) >> 15);
    }
    __syncthreads();
    // blur with a 2-pixel halo; a position outside the image holds the blur of the nearest image pixel (Sobel's
    // BORDER_REPLICATE), whose 3 x 3 grey window lies inside the grey halo
    for (int i = tid; i < BH * BW; i += THREADS) {
        const int ly = i / BW, lx = i - ly * BW;
        const int gy = clampi(y0 - 2 + ly, H) - (y0 - 3), gx = clampi(x0 - 2 + lx, W) - (x0 - 3);
        int v = 0;
#pragma unroll
        for (int r = -1; r <= 1; ++r) {
            const int h = s.g[gy + r][gx - 1] + 2 * s.g[gy + r][gx] + s.g[gy + r][gx + 1];
            v += (r == 0 ? 2 : 1) * h;
        }
        s.b[ly][lx] = (uint8_t)((v + 8) >> 4);
    }
    __syncthreads();
    // L1 magnitude with a 1-pixel halo; 0 outside the image (non-maximum suppression's border)
    for (int i = tid; i < MH * MW; i += THREADS) {
        const int ly = i / MW, lx = i - ly * MW;
        const int y = y0 - 1 + ly, x = x0 - 1 + lx;
        int m = 0;
        if (y >= 0 && y < H && x >= 0 && x < W) {
            int dx, dy;
            sobel3(s, ly + 1, lx + 1, dx, dy);
            m = abs(dx) + abs(dy);
        }
        s.m[ly][lx] = (int16_t)m;
    }
    __syncthreads();

    // non-maximum suppression and the class of each tile pixel; four rows per thread
    const int tx = tid % TW, ty = tid / TW;
    uint8_t c[TH * TW / THREADS];
#pragma unroll
    for (int k = 0; k < TH * TW / THREADS; ++k) {
        const int ly = ty + k * (THREADS / TW), y = y0 + ly, x = x0 + tx;
        c[k] = 0;
        if (y < H && x < W) {
            int dx, dy;
            sobel3(s, ly + 2, tx + 2, dx, dy);
            const int my = ly + 1, mx = tx + 1;
            const int m = s.m[my][mx];
            if (m > low) {
                const int xs = abs(dx), ys = abs(dy), t = xs * 13573;
                bool keep;
                if ((ys << 15) < t) {
                    keep = m > s.m[my][mx - 1] && m >= s.m[my][mx + 1];
                } else if ((ys << 15) > t + (xs << 16)) {
                    keep = m > s.m[my - 1][mx] && m >= s.m[my + 1][mx];
                } else {
                    const int sg = (dx ^ dy) < 0 ? -1 : 1;
                    keep = m > s.m[my - 1][mx - sg] && m > s.m[my + 1][mx + sg];
                }
                if (keep) c[k] = m > high ? 2 : 1;
            }
        }
        s.lab[ly * TW + tx] = c[k] ? ly * TW + tx : -1;
    }
    __syncthreads();
    // union-find of the tile's candidates: each unites with its candidate neighbours left, up-left, up and up-right
#pragma unroll
    for (int k = 0; k < TH * TW / THREADS; ++k) {
        if (!c[k]) continue;
        const int ly = ty + k * (THREADS / TW), i = ly * TW + tx;
        if (tx > 0 && s.lab[i - 1] >= 0) unite_smem(s.lab, i, i - 1);
        if (ly > 0) {
            if (tx > 0 && s.lab[i - TW - 1] >= 0) unite_smem(s.lab, i, i - TW - 1);
            if (s.lab[i - TW] >= 0) unite_smem(s.lab, i, i - TW);
            if (tx < TW - 1 && s.lab[i - TW + 1] >= 0) unite_smem(s.lab, i, i - TW + 1);
        }
    }
    __syncthreads();
    // the tile-local root is the component's first pixel in tile order, which is also its lowest index in the image
#pragma unroll
    for (int k = 0; k < TH * TW / THREADS; ++k) {
        const int ly = ty + k * (THREADS / TW), y = y0 + ly, x = x0 + tx;
        if (y >= H || x >= W) continue;
        const long long p = base + (long long)y * W + x;
        int lab = -1;
        if (c[k]) {
            const int r = find_smem(s.lab, ly * TW + tx);
            lab = (int)(base + (long long)(y0 + r / TW) * W + x0 + r % TW);
        }
        cls[p] = c[k];
        labels[p] = lab;
        flags[p] = 0;
    }
}

// One CTA per tile, one thread per tile-border pixel: the top row (its up-left, up and up-right neighbours, and left for the
// corner), the left column below the top row (left and up-left) and the right column below the top row (up-right).  Every
// 8-neighbour pair that straddles two tiles is a backward (left, up-left, up, up-right) pair of exactly one of these pixels.
constexpr int BORDER = TW + 2 * (TH - 1), MERGE_THREADS = 96;

__global__ void __launch_bounds__(MERGE_THREADS) sketch_merge_kernel(int H, int W, int* __restrict__ labels) {
    const int j = threadIdx.x;
    if (j >= BORDER) return;
    int y = blockIdx.y * TH, x = blockIdx.x * TW;
    bool top = false, left = false, right = false;
    if (j < TW) {
        x += j;
        top = true;
        left = j == 0;
    } else if (j < TW + TH - 1) {
        y += j - TW + 1;
        left = true;
    } else {
        y += j - (TW + TH - 1) + 1;
        x += TW - 1;
        right = true;
    }
    if (y >= H || x >= W) return;
    const long long base = (long long)blockIdx.z * H * W;
    const int p = (int)(base + (long long)y * W + x);
    if (labels[p] < 0) return;
    auto try_unite = [&](int yy, int xx) {
        if (yy < 0 || xx < 0 || xx >= W) return;
        const int q = (int)(base + (long long)yy * W + xx);
        if (labels[q] >= 0) unite_global(labels, p, q);
    };
    if (left) try_unite(y, x - 1);
    if (top || left) try_unite(y - 1, x - 1);
    if (top) try_unite(y - 1, x);
    if (top || right) try_unite(y - 1, x + 1);
}

__global__ void __launch_bounds__(256) sketch_flag_kernel(const uint8_t* __restrict__ cls, int* labels, uint8_t* flags,
                                                          long long total) {
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
        const uint8_t c = cls[p];
        if (!c) continue;
        // no union runs any more, so every label is final up to compression: plain loads and a plain store of the root
        int x = labels[p], q = labels[x];
        while (q != x) {
            x = q;
            q = labels[x];
        }
        labels[p] = x;
        if (c == 2) flags[x] = 1;
    }
}

__global__ void __launch_bounds__(256) sketch_out_kernel(uint8_t* cls_out, const int* __restrict__ labels,
                                                         const uint8_t* __restrict__ flags, long long total) {
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x)
        cls_out[p] = (cls_out[p] && flags[labels[p]]) ? 0 : 255;
}

int grid_1d(long long total) {
    const long long want = (total + 255) / 256, cap = (long long)sm_count() * 16;
    return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}

}  // namespace

}  // namespace anysd

using namespace anysd;

extern "C" {

size_t anysd_sketch_workspace_bytes(int B, int H, int W) {
    if (B <= 0 || H <= 0 || W <= 0) return 0;
    const size_t n = (size_t)B * H * W;
    return n * sizeof(int) + n;                  // int32 labels, then uint8 root flags
}

int anysd_sketch_u8(const void* img, int B, int H, int W, int low, int high, void* workspace, void* out, anysd_stream_t stream) {
    ANYSD_REQUIRE(img && workspace && out, ANYSD_EINVAL, "sketch: null pointer");
    ANYSD_REQUIRE(B > 0 && H > 0 && W > 0, ANYSD_EINVAL, "sketch: bad dims B=%d %dx%d", B, H, W);
    ANYSD_REQUIRE((long long)B * H * W <= 0x7fffffffLL, ANYSD_EINVAL,
                  "sketch: %d x %d x %d pixels overflow a 32-bit label", B, H, W);
    ANYSD_REQUIRE(low >= 0 && low <= high, ANYSD_EINVAL, "sketch: thresholds must satisfy 0 <= low <= high (got %d, %d)", low,
                  high);
    ANYSD_REQUIRE((uintptr_t)workspace % 4 == 0, ANYSD_EINVAL, "sketch: workspace must be 4-byte aligned");
    ANYSD_REQUIRE(B <= 65535, ANYSD_EINVAL, "sketch: batch %d exceeds the grid's z extent", B);
    const long long total = (long long)B * H * W;
    int* labels = (int*)workspace;
    uint8_t* flags = (uint8_t*)workspace + total * sizeof(int);
    uint8_t* o = (uint8_t*)out;
    cudaStream_t st = (cudaStream_t)stream;
    const int tx = (W + TW - 1) / TW, ty = (H + TH - 1) / TH;
    sketch_tile_kernel<<<dim3(tx, ty, B), THREADS, 0, st>>>((const uint8_t*)img, H, W, low, high, o, labels, flags);
    int rc = check_launch("sketch tile");
    if (rc) return rc;
    sketch_merge_kernel<<<dim3(tx, ty, B), MERGE_THREADS, 0, st>>>(H, W, labels);
    if ((rc = check_launch("sketch merge"))) return rc;
    sketch_flag_kernel<<<grid_1d(total), 256, 0, st>>>(o, labels, flags, total);
    if ((rc = check_launch("sketch flag"))) return rc;
    sketch_out_kernel<<<grid_1d(total), 256, 0, st>>>(o, labels, flags, total);
    return check_launch("sketch out");
}

}  // extern "C"
