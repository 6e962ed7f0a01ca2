// anysd_gemm_f16: argument validation and kernel selection for every dense contraction on the path.
#include "common.cuh"

#include <stdlib.h>
#include <string.h>

namespace anysd {
int launch_gemm_mma(const anysd_gemm_params* q, cudaStream_t st);
int launch_gemm_wg(const anysd_gemm_params* q, cudaStream_t st);
bool wg_supported(const anysd_gemm_params* q);
int wg_stats_slabs(const anysd_gemm_params* q);
size_t wg_splitk_bytes(const anysd_gemm_params* q);
}

using namespace anysd;

extern "C" int anysd_gemm_f16(const anysd_gemm_params* p, anysd_stream_t stream) {
    ANYSD_REQUIRE(p != nullptr, ANYSD_EINVAL, "gemm: null params");
    ANYSD_REQUIRE(p->A && p->W && p->out, ANYSD_EINVAL, "gemm: null A/W/out");
    ANYSD_REQUIRE(p->M > 0 && p->N > 0 && p->K > 0, ANYSD_EINVAL, "gemm: bad M=%d N=%d K=%d", p->M, p->N, p->K);
    ANYSD_REQUIRE(p->K % 8 == 0 && p->ldw % 8 == 0 && p->ldw >= p->K, ANYSD_EINVAL,
                  "gemm: K=%d and ldw=%d must be multiples of 8 with ldw >= K", p->K, p->ldw);
    ANYSD_REQUIRE(((uintptr_t)p->A % 16) == 0 && ((uintptr_t)p->W % 16) == 0, ANYSD_EINVAL,
                  "gemm: A and W must be 16-byte aligned");
    ANYSD_REQUIRE(p->act >= 0 && p->act <= 6, ANYSD_EINVAL, "gemm: bad act %d", p->act);
    ANYSD_REQUIRE(p->out_dtype == ANYSD_F16 || p->out_dtype == ANYSD_F32, ANYSD_EINVAL, "gemm: bad out dtype");
    const bool glu = p->act == 2 || p->act == 5;
    const int n_out = glu ? p->N / 2 : p->N;
    ANYSD_REQUIRE(!glu || p->N % 2 == 0, ANYSD_EINVAL, "gemm: GEGLU / SwiGLU needs an even N");
    ANYSD_REQUIRE(p->act != 5 || !p->conv, ANYSD_EUNSUPPORTED, "gemm: SwiGLU (act 5) is for dense contractions only");
    ANYSD_REQUIRE(!p->col_scale || (p->act == 0 && !p->conv && !p->stats && !p->row_stats && !p->ln_stats), ANYSD_EUNSUPPORTED,
                  "gemm: col_scale needs act = 0, a dense contraction and no GroupNorm / row / LayerNorm statistics (act=%d conv=%d)",
                  p->act, p->conv);
    ANYSD_REQUIRE(p->ldo >= n_out, ANYSD_EINVAL, "gemm: ldo=%d < %d output columns", p->ldo, n_out);
    ANYSD_REQUIRE(!p->residual || p->ldr >= n_out, ANYSD_EINVAL, "gemm: ldr too small");
    ANYSD_REQUIRE(!p->rowadd || (p->rows_per_batch > 0 && p->ld_rowadd >= p->N), ANYSD_EINVAL,
                  "gemm: rowadd needs rows_per_batch > 0 and ld_rowadd >= N");
    if (p->conv) {
        ANYSD_REQUIRE(p->conv == 1, ANYSD_EINVAL, "gemm: conv must be 0 or 1 (3x3, pad 1)");
        ANYSD_REQUIRE(p->Nimg > 0 && p->H > 0 && p->Wd > 0 && p->Cin > 0 && p->Cin % 8 == 0, ANYSD_EINVAL,
                      "conv3x3: bad image dims N=%d H=%d W=%d Cin=%d (Cin must be a multiple of 8)", p->Nimg, p->H,
                      p->Wd, p->Cin);
        ANYSD_REQUIRE(p->stride == 1 || p->stride == 2, ANYSD_EINVAL, "conv3x3: stride must be 1 or 2");
        ANYSD_REQUIRE(p->upsample == 0 || p->upsample == 1, ANYSD_EINVAL, "conv3x3: upsample must be 0 or 1");
        ANYSD_REQUIRE(p->K == 9 * p->Cin, ANYSD_EINVAL, "conv3x3: K=%d != 9*Cin=%d", p->K, 9 * p->Cin);
        ANYSD_REQUIRE(p->conv_pad == 0 || (p->conv_pad == 1 && p->stride == 2 && !p->upsample), ANYSD_EINVAL,
                      "conv3x3: conv_pad must be 0, or 1 with stride 2 (right/bottom padding of the first-stage Downsample)");
        const int Hl = p->H << p->upsample, Wl = p->Wd << p->upsample;
        const int Ho = p->conv_pad ? (Hl - 2) / 2 + 1 : (Hl - 1) / p->stride + 1;
        const int Wo = p->conv_pad ? (Wl - 2) / 2 + 1 : (Wl - 1) / p->stride + 1;
        ANYSD_REQUIRE((long long)p->Nimg * Ho * Wo == p->M, ANYSD_EINVAL, "conv3x3: M=%d != N*Ho*Wo=%lld", p->M,
                      (long long)p->Nimg * Ho * Wo);
    } else {
        ANYSD_REQUIRE(p->lda % 8 == 0 && p->lda >= p->K, ANYSD_EINVAL, "gemm: lda=%d must be a multiple of 8 and >= K",
                      p->lda);
    }
    // Kernel selection.  The persistent wgmma/TMA kernel (gemm_wgmma.cu) takes every contraction whose layout constraints
    // hold: all nn.Linear / 1x1 convs and every 3x3 conv with Cin % 64 == 0 (stride 1|2, upsample through the workspace),
    // fp16 or fp32 output.  mma.sync covers what is left (Cin % 64 != 0 convs, N % 8 != 0).
    // ANYSD_GEMM=mma is a test/debug switch used to cross-check the two kernels against each other.
    static const char* force = getenv("ANYSD_GEMM");
    const bool allow_wg = !force || !strcmp(force, "wgmma");
    if (allow_wg && wg_supported(p)) return launch_gemm_wg(p, (cudaStream_t)stream);
    ANYSD_REQUIRE(p->row_stats == nullptr && p->ln_stats == nullptr, ANYSD_EUNSUPPORTED,
                  "gemm: LayerNorm fold / row statistics need the persistent wgmma path");
    ANYSD_REQUIRE(p->stats == nullptr, ANYSD_EUNSUPPORTED, "gemm: output statistics need the persistent wgmma path");
    ANYSD_REQUIRE(!(p->conv && p->conv_pad), ANYSD_EUNSUPPORTED,
                  "conv3x3 with right/bottom padding needs the persistent wgmma path (Cin %% 64 == 0)");
    return launch_gemm_mma(p, (cudaStream_t)stream);
}

extern "C" int anysd_gemm_stats_slabs(const anysd_gemm_params* p) {
    if (p == nullptr || !p->A || !p->W || !p->out) return 0;
    static const char* force = getenv("ANYSD_GEMM");
    if (force && strcmp(force, "wgmma")) return 0;
    if (p->conv && (p->Cin <= 0 || p->K != 9 * p->Cin)) return 0;
    return wg_supported(p) ? wg_stats_slabs(p) : 0;
}

extern "C" size_t anysd_gemm_splitk_workspace_bytes(const anysd_gemm_params* p) {
    if (p == nullptr || !p->A || !p->W || !p->out) return 0;
    static const char* force = getenv("ANYSD_GEMM");
    if (force && strcmp(force, "wgmma")) return 0;
    if (p->conv && (p->Cin <= 0 || p->K != 9 * p->Cin)) return 0;
    return wg_supported(p) ? wg_splitk_bytes(p) : 0;
}
