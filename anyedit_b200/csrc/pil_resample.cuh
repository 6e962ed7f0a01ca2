// Host-side plans of Pillow's 8-bit resampling (Pillow src/libImaging/Resample.c precompute_coeffs / normalize_coeffs_8bpc,
// Geometry.c affine_fixed), shared by the CLIP preprocess (postfilter.cu) and the whole-image resize (inpaint.cu).
// A plan of one axis is, per output position, the entry (first source index, count, c_0 .. c_{k-1}) of stride 2 + k with
// coefficients in Pillow's 22-bit fixed point; a kernel sums (1 << 21) + sum_k src[first + k] c_k and clips (s >> 22) to a byte.
#pragma once

#include <math.h>

#include <vector>

namespace anysd {

constexpr int PIL_PREC = 22;

enum PilFilter { PIL_NEAREST = 0, PIL_BICUBIC = 3, PIL_LANCZOS = 1 };

// Pillow's bicubic filter, a = -0.5, support 2
inline double pil_bicubic(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0;
    if (x < 2.0) return (((x - 5.0) * x + 8.0) * x - 4.0) * a;
    return 0.0;
}

inline double pil_sinc(double x) {
    if (x == 0.0) return 1.0;
    x = x * M_PI;
    return sin(x) / x;
}

// Pillow's truncated sinc, support 3
inline double pil_lanczos(double x) {
    if (-3.0 <= x && x < 3.0) return pil_sinc(x) * pil_sinc(x / 3);
    return 0.0;
}

// One axis in -> out of a convolution filter, for output positions [first, first + n); returns the entry's k (dst = NULL: only
// the size).  A pass whose size does not change is the identity (Pillow skips it; one coefficient of 1 << 22 reproduces the skip
// exactly).  ``gain`` multiplies that identity coefficient.
inline int pil_axis_coeffs(PilFilter filter, int in, int out, int first, int n, std::vector<int>* dst, int gain = 1) {
    if (in == out) {
        if (dst)
            for (int i = 0; i < n; ++i) dst->insert(dst->end(), {first + i, 1, gain << PIL_PREC});
        return 1;
    }
    double (*fn)(double) = filter == PIL_LANCZOS ? pil_lanczos : pil_bicubic;
    const double filter_support = filter == PIL_LANCZOS ? 3.0 : 2.0;
    const double scale = (double)in / (double)out;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = filter_support * filterscale;
    const int ksize = (int)ceil(support) * 2 + 1;
    if (!dst) return ksize;
    std::vector<double> k(ksize);
    for (int i = 0; i < n; ++i) {
        const int xx = first + i;
        const double center = (xx + 0.5) * scale;
        const double ss = 1.0 / filterscale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in) xmax = in;
        xmax -= xmin;
        double ww = 0.0;
        for (int x = 0; x < xmax; ++x) {
            const double w = fn((x + xmin - center + 0.5) * ss);
            k[x] = w;
            ww += w;
        }
        dst->push_back(xmin);
        dst->push_back(xmax);
        for (int x = 0; x < ksize; ++x) {
            double w = x < xmax ? k[x] : 0.0;
            if (x < xmax && ww != 0.0) w /= ww;
            dst->push_back(w < 0 ? (int)(-0.5 + w * (1 << PIL_PREC)) : (int)(0.5 + w * (1 << PIL_PREC)));
        }
    }
    return ksize;
}

// Pillow's NEAREST resize of a full axis (Image.resize with NEAREST, which Pillow forces for mode "1"; Geometry.c
// ImagingScaleAffine): the source position starts at in / out * 0.5 and adds in / out per output pixel in double, index = (int)
// position.  Entries of one coefficient ``gain << 22``; an unchanged size is a copy, which this also gives.
inline void pil_axis_nearest(int in, int out, std::vector<int>* dst, int gain = 1) {
    const double a = (double)in / out;
    double pos = a * 0.5;
    for (int x = 0; x < out; ++x, pos += a) {
        int s = (int)pos;
        if (s > in - 1) s = in - 1;  // never taken: the position stays below in; kept in bounds all the same
        dst->insert(dst->end(), {s, 1, gain << PIL_PREC});
    }
}

}  // namespace anysd
