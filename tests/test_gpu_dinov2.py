"""AnyDoor's reference-image encoder on the GPU (``encoders.FrozenDinoV2Encoder``, DINOv2 ViT-g/14 + projector) and the two
contraction epilogues it adds:

* SwiGLU (act 5) and the per-column output scale (``col_scale``, LayerScale) element by element against a float64 reference,
  at every tile width (ANYSD_GEMM_BN, one child process each: the switch is read once per process) and on the mma.sync
  kernel (ANYSD_GEMM=mma), bit-identical across widths; every combination ``col_scale`` does not serve is refused with
  ANYSD_EUNSUPPORTED on both kernels;
* the tiny encoder against transformers' ``Dinov2Model`` golden, the real width (D 1536, 24 heads, 4 layers) against the fp32
  CPU oracle, the full 40-layer model (determinism, batch independence, the all-zero unconditional image);
* ``ControlDenoiser.get_learned_conditioning`` and a ControlNet DDIM run fed by the encoder.

Bound per output element (same terms as tests/test_gpu_contraction.py, from the fp16-rounded operands):
    pre = acc + bias (+ rowadd),  e_pre = C_ACC 2^-24 (K (|A| |W|^T) + |bias| + |rowadd|)
    col_scale:  |s| e_pre + C_ACC 2^-24 |s pre|                          (the product rounds once)
    SwiGLU:     |silu(g)| e_a + (|a| + e_a) (1.13 e_g + 2^-21 (1 + |g|))  (1.13: the steepest slope of SiLU; libm-grade expf)
    + C_ACC 2^-24 (|y| + |residual|) with a residual, + 2^-11 |y| + 2^-25 for fp16 outputs.
"""
import ctypes as C
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
G = os.path.join(os.path.dirname(__file__), "golden")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
WIDTHS = (64, 128, 192, 256)
U, C_ACC, SLOPE = 2.0 ** -24, 4, 1.13
FWD_TOL = 4e-3
COL0 = 8


# ---- epilogue cases ---------------------------------------------------------------------------------------------------
def _case(name, M, N, K, act=0, cs=False, res=False, rowadd=False, rpb=0, f32=False):
    return dict(name=name, M=M, N=N, K=K, act=act, cs=cs, res=res, rowadd=rowadd, rpb=rpb, f32=f32)


# M = 1000: a ragged last row tile; N = 448: a partial last column tile at every width; K = 392 = 6 x 64 + 8: a K tail.
# M = 514 = 257 x 2: two 224-pixel images; the DINOv2 w12 / w3 / attention projection shapes.
CASES = {c["name"]: c for c in [
    _case("swiglu_f16", 1000, 448, 392, act=5),
    _case("swiglu_rowadd_res_f16", 1000, 448, 392, act=5, res=True, rowadd=True, rpb=200),
    _case("swiglu_f32", 1000, 448, 392, act=5, f32=True),
    _case("swiglu_k8_res", 300, 320, 8, act=5, res=True),
    _case("ls_res_f16", 1000, 448, 392, cs=True, res=True),
    _case("ls_rowadd_res_f16", 1000, 448, 392, cs=True, res=True, rowadd=True, rpb=200),
    _case("ls_f32", 1000, 448, 392, cs=True, f32=True),
    _case("dinov2_w12", 514, 8192, 1536, act=5),
    _case("dinov2_w3_ls2", 514, 1536, 4096, cs=True, res=True),
    _case("dinov2_proj_ls1", 514, 1536, 1536, cs=True, res=True),
]}


def _n_out(c):
    return c["N"] // 2 if c["act"] == 5 else c["N"]


def _inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    M, N, K = c["M"], c["N"], c["K"]
    T = {"A": rn(M, K).half(), "W": (rn(N, K) * 1.5 * K ** -0.5).half(), "bias": 0.1 * rn(N)}
    if c["cs"]:
        T["cs"] = 0.3 + 1.2 * torch.rand(N, generator=g)
    if c["rowadd"]:
        T["rowadd"] = rn(-(-M // c["rpb"]), N + 16)
    if c["res"]:
        T["res"] = rn(M, _n_out(c) + 16).half()
    return T


def _run(ops, names, inputs):
    out = {}
    for n in names:
        c, T = CASES[n], {k: v.cuda() for k, v in inputs[n].items()}
        dt = torch.float32 if c["f32"] else torch.float16
        buf = torch.full((c["M"], COL0 + _n_out(c) + 16), float("nan"), dtype=dt, device="cuda")
        ops.gemm(T["A"], T["W"], buf[:, COL0:COL0 + _n_out(c)], bias=T["bias"], act=c["act"], col_scale=T.get("cs"),
                 rowadd=T["rowadd"][:, COL0:COL0 + c["N"]] if c["rowadd"] else None, rows_per_batch=c["rpb"],
                 residual=T["res"][:, COL0:COL0 + _n_out(c)] if c["res"] else None)
        torch.cuda.synchronize()
        out[n] = buf.cpu()
    return out


def _probe_col_scale():
    """Return code of anysd_gemm_f16 for every combination col_scale does not serve, and for SwiGLU on a conv (0 for a
    plain col_scale contraction)."""
    from anyedit_b200 import _lib
    lib = _lib.load()
    M, N, K = 128, 128, 64
    A, W = torch.randn(M, K, device="cuda").half(), torch.randn(N, K, device="cuda").half()
    img = torch.randn(1, 8, 16, 64, device="cuda").half()
    Wc = torch.randn(N, 9 * 64, device="cuda").half()
    out = torch.empty(M, N, dtype=torch.float16, device="cuda")
    s, bias = torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
    f32buf = torch.zeros(1 << 16, device="cuda")

    def params(**kw):
        p = _lib.GemmParams()
        p.A, p.W, p.out, p.col_scale = A.data_ptr(), W.data_ptr(), out.data_ptr(), s.data_ptr()
        p.M, p.N, p.K, p.lda, p.ldw, p.ldo, p.out_dtype = M, N, K, K, K, N, _lib.F16
        for k, v in kw.items():
            setattr(p, k, v)
        return p
    variants = {"plain": params()}
    for act in (1, 2, 3, 4, 5):
        variants[f"act{act}"] = params(act=act)
    conv = dict(A=img.data_ptr(), W=Wc.data_ptr(), K=9 * 64, ldw=9 * 64, conv=1, Nimg=1, H=8, Wd=16, Cin=64, stride=1)
    variants["conv"] = params(**conv)
    variants["swiglu_conv"] = params(**conv, act=5, col_scale=None)           # SwiGLU is dense only, with or without a scale
    variants["stats"] = params(stats=f32buf.data_ptr(), stats_images=2, rows_per_batch=64)
    variants["row_stats"] = params(row_stats=f32buf.data_ptr())
    variants["ln_stats"] = params(ln_stats=f32buf.data_ptr(), ln_colsum=f32buf.data_ptr(), bias=bias.data_ptr(), ln_eps=1e-5)
    rc = {k: int(lib.anysd_gemm_f16(C.byref(p), None)) for k, p in variants.items()}
    torch.cuda.synchronize()
    return rc


def _reference(c, T):
    A, W = T["A"].double(), T["W"].double()
    acc, P = A @ W.t(), A.abs() @ W.abs().t()
    bias = T["bias"].double()
    pre, mag = acc + bias, bias.abs().expand_as(acc)
    if c["rowadd"]:
        ra = T["rowadd"].double()[:, COL0:COL0 + c["N"]][torch.arange(c["M"]) // c["rpb"]]
        pre, mag = pre + ra, mag + ra.abs()
    e = C_ACC * U * (c["K"] * P + mag)
    if c["cs"]:
        s = T["cs"].double()
        y = pre * s
        e = s.abs() * e + C_ACC * U * y.abs()
    elif c["act"] == 5:                               # interleaved (a, gate) columns -> a * silu(gate)
        a, gt, ea, eg = pre[:, 0::2], pre[:, 1::2], e[:, 0::2], e[:, 1::2]
        sg = gt * torch.sigmoid(gt)
        y = a * sg
        e = sg.abs() * ea + (a.abs() + ea) * (SLOPE * eg + 2.0 ** -21 * (1.0 + gt.abs()))
    else:
        y = pre
    if c["res"]:
        r = T["res"].double()[:, COL0:COL0 + _n_out(c)]
        y = y + r
        e = e + C_ACC * U * (y.abs() + r.abs())
    return y, e


def _check(c, ref, buf, label):
    y, e = ref
    n_out = _n_out(c)
    assert buf[:, :COL0].isnan().all() and buf[:, COL0 + n_out:].isnan().all(), f"{label} {c['name']}: wrote outside its window"
    out = buf[:, COL0:COL0 + n_out].double()
    bound = e if c["f32"] else e + 2.0 ** -11 * (y.abs() + e) + 2.0 ** -25
    ratio = (out - y).abs() / bound
    worst = float(ratio.max())
    assert worst <= 1.0, f"{label} {c['name']}: worst err/bound {worst:.3g} ({int((ratio > 1).sum())} elements, {int(out.isnan().sum())} NaN)"
    return worst


@pytest.fixture(scope="module")
def cuda_ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from anyedit_b200 import ops
    assert tuple(ops.device_info())[1:] == (9, 0), "sm_90a kernels need a Hopper GPU (H100)"
    return ops


@pytest.fixture(scope="module")
def epi(cuda_ops, tmp_path_factory):
    inputs = {n: _inputs(c, 300 + i) for i, (n, c) in enumerate(CASES.items())}
    d = tmp_path_factory.mktemp("dinov2_epilogues")
    torch.save(inputs, d / "inputs.pt")
    refs = {n: _reference(CASES[n], inputs[n]) for n in CASES}
    return SimpleNamespace(inputs=inputs, dir=d, refs=refs, natural=_run(cuda_ops, list(CASES), inputs))


def _child(epi, tag, env):
    out = epi.dir / f"out_{tag}.pt"
    e = {k: v for k, v in os.environ.items() if not k.startswith("ANYSD_GEMM")}
    e.update(env)
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), os.path.abspath(__file__), "--worker",
           str(epi.dir / "inputs.pt"), str(out)]
    r = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"worker {tag} failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    return torch.load(out)


def test_epilogues_natural_width(epi):
    for n, c in CASES.items():
        print(f"natural {n:22s} worst err/bound {_check(c, epi.refs[n], epi.natural[n], 'natural'):.3f}")


@pytest.mark.parametrize("bn", WIDTHS)
def test_epilogues_forced_width_bit_identical(epi, bn):
    got = _child(epi, f"bn{bn}", {"ANYSD_GEMM_BN": str(bn)})
    for n, c in CASES.items():
        w = _check(c, epi.refs[n], got[n], f"BN={bn}")
        same = torch.equal(got[n].view(torch.int32 if c["f32"] else torch.int16), epi.natural[n].view(torch.int32 if c["f32"] else torch.int16))
        print(f"BN={bn:3d} {n:22s} worst err/bound {w:.3f} bit-identical to natural: {same}")
        assert same, f"BN={bn} {n}: not bit-identical to the natural width"


def test_epilogues_mma_and_refusals(epi):
    got = _child(epi, "mma", {"ANYSD_GEMM": "mma"})
    for n, c in CASES.items():
        print(f"mma     {n:22s} worst err/bound {_check(c, epi.refs[n], got[n], 'mma'):.3f}")
    from anyedit_b200 import _lib
    for label, rc in (("wgmma", _probe_col_scale()), ("mma", got["__probe__"])):
        assert rc.pop("plain") == 0, f"{label}: a plain col_scale contraction was refused"
        bad = {k: v for k, v in rc.items() if v != _lib.EUNSUPPORTED}
        assert not bad, f"{label}: col_scale combinations not refused with ANYSD_EUNSUPPORTED: {bad}"


# ---- the encoder --------------------------------------------------------------------------------------------------------
def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.fixture(scope="module")
def tiny(cuda_ops):
    """FrozenDinoV2Encoder at the golden's tiny configuration with its weights (transformers names through the key map)."""
    from anyedit_b200.encoders import FrozenDinoV2Encoder, dinov2_from_transformers
    from oracle import dinov2_oracle as O, weights
    g = np.load(os.path.join(G, "dinov2_tiny.npz"))
    meta = json.load(open(os.path.join(G, "dinov2_tiny_keys.json")))
    seed, pseed, iseed = meta["seeds"]
    hf = O.seeded_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, seed)
    proj = weights.make_state_dict({k: tuple(v) for k, v in meta["projector_keys"].items()}, pseed)
    assert weights.checksum({**hf, **proj}) == pytest.approx(float(g["wsum"]), rel=1e-12)
    enc = FrozenDinoV2Encoder(config=dict(meta["config"], projection_dim=meta["projection_dim"], interpolate_offset=0.0))
    enc.load_state_dict({**{"model." + k: v for k, v in dinov2_from_transformers(hf).items()}, **proj}, strict=True)
    return enc.cuda(), g, iseed


def test_tiny_encoder_vs_transformers(tiny):
    from oracle import dinov2_oracle as O
    enc, g, iseed = tiny
    for i, (H, W) in enumerate(O.TINY_SIZES):
        out = enc(O.tiny_images((H, W), iseed + i).cuda())
        e = rel(out, g[f"out_{H}x{W}"])
        print(f"[dinov2 tiny {H}x{W}, {(H // 14) * (W // 14) + 1} tokens] rel-L2 vs transformers {e:.2e}")
        assert out.dtype == torch.float32 and tuple(out.shape) == g[f"out_{H}x{W}"].shape and e < FWD_TOL


def test_real_width_vs_oracle(cuda_ops):
    """D = 1536, 24 heads of 64, SwiGLU hidden 4096, 224 x 224 -> 257 tokens, 4 layers, hub interpolation (offset 0.1)."""
    from anyedit_b200.encoders import FrozenDinoV2Encoder
    from oracle import dinov2_oracle as O
    enc = FrozenDinoV2Encoder(config={"num_hidden_layers": 4})
    sd = O.seeded_state_dict({k: tuple(v.shape) for k, v in enc.state_dict().items()}, 23)
    enc.load_state_dict(sd, strict=True)
    x = torch.rand(2, 3, 224, 224, generator=torch.Generator().manual_seed(24))
    out = enc.cuda()(x.cuda())
    ref = O.encoder(sd, x, 24, offset=0.1)
    e = rel(out, ref)
    print(f"[dinov2 real width, 4 layers, B=2] rel-L2 vs fp32 oracle {e:.2e}")
    assert tuple(out.shape) == (2, 257, 1024) and e < FWD_TOL


def test_full_vitg14_determinism_and_batch_independence(cuda_ops):
    from anyedit_b200.encoders import FrozenDinoV2Encoder
    torch.manual_seed(0)
    with torch.device("cuda"):
        enc = FrozenDinoV2Encoder()
    assert len(enc.model.blocks) == 40 and sum(p.numel() for p in enc.model.parameters()) > 1.1e9
    x = torch.rand(2, 3, 224, 224, generator=torch.Generator().manual_seed(25)).cuda()
    a = enc(x)
    assert a.dtype == torch.float32 and tuple(a.shape) == (2, 257, 1024) and bool(a.isfinite().all())
    assert torch.equal(enc([x[:1], x[1:]]), a), "two calls differ"
    for i in range(2):
        assert torch.equal(enc(x[i:i + 1])[0], a[i]), f"image {i}: batch 1 != batch 2"
    z = enc(torch.zeros(2, 3, 224, 224, device="cuda"))           # AnyDoor's unconditional context
    assert bool(z.isfinite().all()) and torch.equal(z[0], z[1])


def test_control_denoiser_conditioning(tiny):
    """get_learned_conditioning runs the encoder; its context drives a ControlNet DDIM run exactly like the same tensor."""
    from anyedit_b200.cldm import ControlDenoiser, ControlledUnetModel, ControlNet
    from anyedit_b200.ddim import DDIMSampler
    from oracle import dinov2_oracle as O, weights
    enc, _, iseed = tiny
    g = np.load(os.path.join(G, "cldm_tiny.npz"))
    meta = json.load(open(os.path.join(G, "cldm_tiny_keys.json")))
    cn, un = ControlNet(**meta["control_config"]), ControlledUnetModel(**meta["unet_config"])
    cn.load_state_dict(weights.make_state_dict({k: tuple(v) for k, v in meta["control_keys"].items()}, int(g["cseed"])))
    un.load_state_dict(weights.make_state_dict({k: tuple(v) for k, v in meta["unet_keys"].items()}, int(g["useed"])))
    den = ControlDenoiser(un, cn, cond_stage_model=enc).cuda()
    img = O.tiny_images(O.TINY_SIZES[0], iseed).cuda()
    ctx = den.get_learned_conditioning(img)
    assert torch.equal(ctx, enc(img)) and ctx.shape[-1] == 64
    unc = den.get_learned_conditioning(torch.zeros_like(img))
    hint = torch.from_numpy(g["hint"]).cuda()
    x_T = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(26)).cuda()
    runs = []
    for c, u in ((ctx, unc), (ctx.clone(), unc.clone())):
        o, _ = DDIMSampler(den, use_cuda_graph=False).sample(5, 2, (4, 16, 16), {"c_concat": [hint], "c_crossattn": [c]}, verbose=False,
                                                             x_T=x_T, eta=0.0, unconditional_guidance_scale=4.0,
                                                             unconditional_conditioning={"c_concat": [hint], "c_crossattn": [u]})
        runs.append(o)
    assert bool(runs[0].isfinite().all()) and torch.equal(runs[0], runs[1])


def _worker(argv):
    from anyedit_b200 import ops
    inputs = torch.load(argv[0])
    res = _run(ops, list(CASES), inputs)
    res["__probe__"] = _probe_col_scale()
    torch.save(res, argv[1])
    return 0


if __name__ == "__main__" and sys.argv[1:2] == ["--worker"]:
    sys.exit(_worker(sys.argv[2:]))
