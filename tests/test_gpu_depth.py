"""Depth Anything V2 on the GPU (``depth.DepthAnythingV2``) and the kernels it adds:

* the ReLU epilogue (act 6) of anysd_gemm_f16, dense and 3x3 conv, fp16 and fp32 output, with bias and residual, element by
  element against a float64 bound at every wgmma tile width (ANYSD_GEMM_BN, one child process each: the switch is read once per
  process) and on the mma.sync kernel (ANYSD_GEMM=mma); bit-identical across widths; refused where SiLU is refused;
* the align-corners bilinear resize against float64 ``F.interpolate`` on the five head sizes and a non-square map, with and
  without the addend, and its fp32 single-channel form; ``relu`` and ``depth_to_space`` bit for bit; the transposed conv
  (contraction + depth_to_space) against float64 ``conv_transpose2d``;
* the tiny model against the reference's golden (depth maps, intermediate tokens, ``infer_image``) and the SwiGLU backbone of
  ``FrozenDinoV2Encoder`` against the hub class; vitl at its real width (4 blocks, full head) against the fp32 oracle at
  518 x 518 and 518 x 784; the full 24-block vitl for determinism, batch independence and the state-dict round trip.

Bound per output element (terms of tests/test_gpu_contraction.py): pre = acc + bias, e = 4 2^-24 (K (|A| |W|^T) + |bias|);
ReLU is 1-Lipschitz, so relu(pre) keeps e; + 4 2^-24 (|y| + |residual|) with a residual, + 2^-11 |y| + 2^-25 for fp16 outputs.
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
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
G = os.path.join(os.path.dirname(__file__), "golden")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
WIDTHS = (64, 128, 192, 256)
U, C_ACC = 2.0 ** -24, 4
COL0 = 8
# rel-L2 tolerances of the model tests (measured values in DESIGN.md §10.4)
TINY_TOL, TOK_TOL, SWIGLU_TOL, REAL_TOL = 4e-3, 3e-3, 3e-3, 3e-3


# ---- the ReLU epilogue ------------------------------------------------------------------------------------------------
def _case(name, M=0, N=0, K=0, res=False, f32=False, conv=None):
    if conv:
        M, K = conv[0] * conv[1] * conv[2], 9 * conv[3]
    return dict(name=name, M=M, N=N, K=K, res=res, f32=f32, conv=conv)


# dense: M = 1000 ragged, N = 448 a partial last column tile at every width, K = 392 a K tail; conv: (images, H, W, Cin) --
# Cin 64 / 256 take the wgmma kernel, Cin 32 the mma.sync kernel; N = 32 is the head's output_conv2[0]
CASES = {c["name"]: c for c in [
    _case("dense_f16", 1000, 448, 392),
    _case("dense_res_f16", 1000, 448, 392, res=True),
    _case("dense_f32", 1000, 448, 392, f32=True),
    _case("dense_res_f32", 1000, 448, 392, res=True, f32=True),
    _case("dense_k8_res", 300, 320, 8, res=True),
    _case("dense_n8_f32", 2000, 8, 32, f32=True),
    _case("conv64_res_f16", N=128, res=True, conv=(2, 12, 20, 64)),
    _case("conv64_f32", N=128, f32=True, conv=(2, 12, 20, 64)),
    _case("conv256_n32_f16", N=32, conv=(1, 19, 28, 256)),
    _case("conv32_res_f16", N=64, res=True, conv=(3, 9, 11, 32)),
]}


def _inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    T = {"A": rn(*c["conv"]).half() if c["conv"] else rn(c["M"], c["K"]).half()}
    T["W"] = (rn(c["N"], c["K"]) * 1.5 * c["K"] ** -0.5).half()
    T["bias"] = 0.1 * rn(c["N"])
    if c["res"]:
        T["res"] = rn(c["M"], c["N"] + 16).half()
    return T


def _run(ops, inputs):
    out = {}
    for n, c in CASES.items():
        T = {k: v.cuda() for k, v in inputs[n].items()}
        dt = torch.float32 if c["f32"] else torch.float16
        buf = torch.full((c["M"], COL0 + c["N"] + 16), float("nan"), dtype=dt, device="cuda")
        res = T["res"][:, COL0:COL0 + c["N"]] if c["res"] else None
        (ops.conv3x3 if c["conv"] else ops.gemm)(T["A"], T["W"], buf[:, COL0:COL0 + c["N"]], bias=T["bias"], act=6, residual=res)
        torch.cuda.synchronize()
        out[n] = buf.cpu()
    return out


def _probe_refusals():
    """Return codes of anysd_gemm_f16 for ReLU with the LayerNorm fold, row statistics and col_scale (refused like SiLU's
    combinations), plus a plain ReLU contraction (0)."""
    from anyedit_b200 import _lib
    lib = _lib.load()
    M, N, K = 128, 128, 64
    A, W = torch.randn(M, K, device="cuda").half(), torch.randn(N, K, device="cuda").half()
    out = torch.empty(M, N, dtype=torch.float16, device="cuda")
    s, bias = torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
    f32buf = torch.zeros(1 << 16, device="cuda")

    def params(**kw):
        p = _lib.GemmParams()
        p.A, p.W, p.out, p.act = A.data_ptr(), W.data_ptr(), out.data_ptr(), 6
        p.M, p.N, p.K, p.lda, p.ldw, p.ldo, p.out_dtype = M, N, K, K, K, N, _lib.F16
        for k, v in kw.items():
            setattr(p, k, v)
        return p
    variants = {"plain": params(), "col_scale": params(col_scale=s.data_ptr()), "row_stats": params(row_stats=f32buf.data_ptr()),
                "ln_stats": params(ln_stats=f32buf.data_ptr(), ln_colsum=f32buf.data_ptr(), bias=bias.data_ptr(), ln_eps=1e-5),
                "act7": params(act=7)}
    rc = {k: int(lib.anysd_gemm_f16(C.byref(p), None)) for k, p in variants.items()}
    torch.cuda.synchronize()
    return rc


def _reference(c, T):
    W = T["W"].double()
    if c["conv"]:
        n, H, Wd, ci = c["conv"]
        x = T["A"].double().permute(0, 3, 1, 2)
        w = W.view(c["N"], 3, 3, ci).permute(0, 3, 1, 2)
        acc = F.conv2d(x, w, padding=1).permute(0, 2, 3, 1).reshape(-1, c["N"])
        P = F.conv2d(x.abs(), w.abs(), padding=1).permute(0, 2, 3, 1).reshape(-1, c["N"])
    else:
        A = T["A"].double()
        acc, P = A @ W.t(), A.abs() @ W.abs().t()
    bias = T["bias"].double()
    pre = acc + bias
    e = C_ACC * U * (c["K"] * P + bias.abs())
    y = pre.clamp_min(0)
    if c["res"]:
        r = T["res"].double()[:, COL0:COL0 + c["N"]]
        y = y + r
        e = e + C_ACC * U * (y.abs() + r.abs())
    return y, e


def _check(c, ref, buf, label):
    y, e = ref
    assert buf[:, :COL0].isnan().all() and buf[:, COL0 + c["N"]:].isnan().all(), f"{label} {c['name']}: wrote outside its window"
    out = buf[:, COL0:COL0 + c["N"]].double()
    bound = e if c["f32"] else e + 2.0 ** -11 * (y.abs() + e) + 2.0 ** -25
    ratio = (out - y).abs() / bound
    worst = float(ratio.max())
    assert worst <= 1.0, f"{label} {c['name']}: worst err/bound {worst:.3g} ({int((ratio > 1).sum())} elements, {int(out.isnan().sum())} NaN)"
    if not c["res"]:
        assert float((out == 0).double().mean()) > 0.3, f"{label} {c['name']}: the ReLU clamped too few outputs"
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
    inputs = {n: _inputs(c, 400 + i) for i, (n, c) in enumerate(CASES.items())}
    d = tmp_path_factory.mktemp("relu_epilogue")
    torch.save(inputs, d / "inputs.pt")
    refs = {n: _reference(CASES[n], inputs[n]) for n in CASES}
    return SimpleNamespace(inputs=inputs, dir=d, refs=refs, natural=_run(cuda_ops, inputs))


def _child(epi, tag, env):
    out = epi.dir / f"out_{tag}.pt"
    e = {k: v for k, v in os.environ.items() if not k.startswith("ANYSD_GEMM")}
    e.update(env)
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), os.path.abspath(__file__), "--worker",
           str(epi.dir / "inputs.pt"), str(out)]
    r = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"worker {tag} failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    return torch.load(out)


def test_relu_epilogue_natural_width(epi):
    for n, c in CASES.items():
        print(f"natural {n:18s} worst err/bound {_check(c, epi.refs[n], epi.natural[n], 'natural'):.3f}")


@pytest.mark.parametrize("bn", WIDTHS)
def test_relu_epilogue_forced_width_bit_identical(epi, bn):
    got = _child(epi, f"bn{bn}", {"ANYSD_GEMM_BN": str(bn)})
    for n, c in CASES.items():
        w = _check(c, epi.refs[n], got[n], f"BN={bn}")
        iv = torch.int32 if c["f32"] else torch.int16
        same = torch.equal(got[n].view(iv), epi.natural[n].view(iv))
        print(f"BN={bn:3d} {n:18s} worst err/bound {w:.3f} bit-identical to natural: {same}")
        assert same, f"BN={bn} {n}: not bit-identical to the natural width"


def test_relu_epilogue_mma_and_refusals(epi):
    from anyedit_b200 import _lib
    got = _child(epi, "mma", {"ANYSD_GEMM": "mma"})
    for n, c in CASES.items():
        print(f"mma     {n:18s} worst err/bound {_check(c, epi.refs[n], got[n], 'mma'):.3f}")
    for label, rc in (("wgmma", _probe_refusals()), ("mma", got["__probe__"])):
        assert rc.pop("plain") == 0, f"{label}: a plain ReLU contraction was refused"
        assert rc.pop("act7") == _lib.EINVAL, f"{label}: act 7 accepted"
        bad = {k: v for k, v in rc.items() if v != _lib.EUNSUPPORTED}
        assert not bad, f"{label}: ReLU combinations not refused with ANYSD_EUNSUPPORTED: {bad}"


# ---- resize, relu copy, depth-to-space ----------------------------------------------------------------------------------
RESIZES = [(19, 19, 37, 37, 256), (37, 37, 74, 74, 256), (74, 74, 148, 148, 256), (148, 148, 296, 296, 256),
           (296, 296, 518, 518, 64), (37, 56, 74, 112, 256)]


def _resize_bound(x, ref, H, W, fp16):
    """fp32 source coordinates (rounding of the scale and of o * scale: <= 2 ulp of the coordinate on each axis, a weight error
    of at most 2^-22 max(H, W)) and fp32 sums of four products, then one fp16 rounding."""
    m = float(x.abs().max())
    b = (4 * 2.0 ** -22 * max(H, W) + 16 * U) * m
    return b + (2.0 ** -11 * ref.abs() + 2.0 ** -25 if fp16 else 4 * U * ref.abs())


@pytest.mark.parametrize("H,W,Ho,Wo,Cc", RESIZES)
def test_resize_bilinear_vs_fp64(cuda_ops, H, W, Ho, Wo, Cc):
    g = torch.Generator().manual_seed(H * 1000 + W)
    x = torch.randn(1, H, W, Cc, generator=g).half()
    add = torch.randn(1, Ho, Wo, Cc, generator=g).half()
    ref = F.interpolate(x.double().permute(0, 3, 1, 2), (Ho, Wo), mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    for addend in (None, add):
        y = torch.empty(1, Ho, Wo, Cc, dtype=torch.float16, device="cuda")
        cuda_ops.resize_bilinear(x.cuda(), y, addend=addend.cuda() if addend is not None else None)
        want = ref + (addend.double() if addend is not None else 0)
        r = ((y.cpu().double() - want).abs() / _resize_bound(x, want, H, W, True)).max()
        print(f"resize {H}x{W}->{Ho}x{Wo} C={Cc} addend={addend is not None}: worst err/bound {float(r):.3f}")
        assert float(r) <= 1.0
    x32 = torch.randn(3, H, W, generator=g)
    y32 = torch.empty(3, Ho, Wo, device="cuda")
    cuda_ops.resize_bilinear(x32.cuda(), y32)
    ref32 = F.interpolate(x32.double()[:, None], (Ho, Wo), mode="bilinear", align_corners=True)[:, 0]
    assert float(((y32.cpu().double() - ref32).abs() / _resize_bound(x32, ref32, H, W, False)).max()) <= 1.0


def test_resize_fp32_to_raw_size(cuda_ops):
    """infer_image's resize: any size, down or up, including a one-pixel side."""
    x = torch.randn(1, 518, 784, generator=torch.Generator().manual_seed(5))
    for (h, w) in ((480, 640), (1080, 1920), (1, 7), (333, 1)):
        y = torch.empty(1, h, w, device="cuda")
        cuda_ops.resize_bilinear(x.cuda(), y)
        ref = F.interpolate(x.double()[:, None], (h, w), mode="bilinear", align_corners=True)[:, 0]
        assert float(((y.cpu().double() - ref).abs() / _resize_bound(x, ref, 518, 784, False)).max()) <= 1.0, (h, w)


def test_relu_copy_and_depth_to_space_bit_exact(cuda_ops):
    g = torch.Generator().manual_seed(6)
    x = torch.randn(3, 37, 37, 256, generator=g).half()
    x.view(-1)[:4] = torch.tensor([float("-inf"), float("inf"), -0.0, 0.0]).half()
    y = torch.empty_like(x, device="cuda")
    cuda_ops.relu(x.cuda(), y)
    assert torch.equal(y.cpu(), torch.relu(x)) and not bool(y.cpu().signbit().any())
    for r, C_ in ((4, 64), (2, 512)):
        gt = torch.randn(2 * 7 * 13, r * r * C_, generator=g).half()
        out = torch.empty(2, 7 * r, 13 * r, C_, dtype=torch.float16, device="cuda")
        cuda_ops.depth_to_space(gt.cuda(), out, r)
        want = gt.view(2, 7, 13, r, r, C_).permute(0, 1, 3, 2, 4, 5).reshape(2, 7 * r, 13 * r, C_)
        assert torch.equal(out.cpu(), want), r


def test_transposed_conv_vs_fp64(cuda_ops):
    """ConvTranspose2d(k = stride = r): contraction with the packed weight and repeated bias, then depth_to_space."""
    from anyedit_b200.depth import _pack_deconv
    from anyedit_b200.unet import _Param
    g = torch.Generator().manual_seed(7)
    for r, ci in ((4, 256), (2, 512)):
        p = _Param((ci, ci, r, r), kind="conv")
        with torch.no_grad():
            p.weight.copy_(torch.randn(ci, ci, r, r, generator=g) * ci ** -0.5)
            p.bias.copy_(0.1 * torch.randn(ci, generator=g))
        w, b, rr = _pack_deconv(p, "cuda")
        x = torch.randn(1, 37, 37, ci, generator=g).half()
        gmat = torch.empty(37 * 37, r * r * ci, dtype=torch.float16, device="cuda")
        cuda_ops.gemm(x.cuda().view(-1, ci), w, gmat, bias=b)
        out = torch.empty(1, 37 * r, 37 * r, ci, dtype=torch.float16, device="cuda")
        cuda_ops.depth_to_space(gmat, out, rr)
        wd = p.weight.detach().half().double()
        ref = F.conv_transpose2d(x.double().permute(0, 3, 1, 2), wd, p.bias.detach().double(), stride=r).permute(0, 2, 3, 1)
        P = F.conv_transpose2d(x.double().abs().permute(0, 3, 1, 2), wd.abs(), stride=r).permute(0, 2, 3, 1)
        e = C_ACC * U * (ci * P + p.bias.detach().double().abs()) + 2.0 ** -11 * ref.abs() + 2.0 ** -25
        worst = float(((out.cpu().double() - ref).abs() / e).max())
        print(f"conv_transpose2d r={r} C={ci}: worst err/bound {worst:.3f}")
        assert worst <= 1.0


# ---- the model ------------------------------------------------------------------------------------------------------------
def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.fixture(scope="module")
def tiny(cuda_ops):
    from anyedit_b200.depth import DepthAnythingV2
    from oracle import depth_oracle as O, weights
    g = np.load(os.path.join(G, "depth_anything_tiny.npz"))
    meta = json.load(open(os.path.join(G, "depth_anything_tiny_keys.json")))
    sd = O.seeded_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, meta["seeds"][0])
    assert weights.checksum(sd) == pytest.approx(float(g["wsum"]), rel=1e-12)
    m = DepthAnythingV2(encoder="vits", **O.TINY_HEAD, config=O.TINY_BACKBONE, layer_idx=O.TINY_LAYERS)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), g, meta


def test_tiny_depth_vs_reference(tiny):
    from oracle import depth_oracle as O
    m, g, meta = tiny
    for i, size in enumerate(O.TINY_SIZES):
        out = m(O.tiny_images(size, meta["seeds"][1] + i).cuda())
        want = g["depth_%dx%d" % size]
        e = rel(out, want)
        print(f"[depth tiny {size}] rel-L2 vs reference {e:.2e}; positive {float((out > 0).float().mean()):.3f}")
        assert out.dtype == torch.float32 and tuple(out.shape) == want.shape and e < TINY_TOL
        assert float((out > 0).float().mean()) > 0.5
    x = O.tiny_images(O.TINY_SIZES[0], meta["seeds"][1])[:1].cuda()
    feats = m.pretrained.get_intermediate_layers(x, O.TINY_LAYERS, return_class_token=True)
    patches, B, gh, gw = m.pretrained.intermediate_patches(x, O.TINY_LAYERS)
    for i, ((t, c), p) in enumerate(zip(feats, patches)):
        e = max(rel(t, g[f"tok{i}"]), rel(c, g[f"cls{i}"]))
        print(f"[depth tiny] block {O.TINY_LAYERS[i]} normed tokens rel-L2 {e:.2e}")
        assert e < TOK_TOL and torch.equal(p.view(1, gh * gw, -1).float(), t)
    assert len(m.pretrained.get_intermediate_layers(x, 2)) == 2


def test_tiny_infer_image(tiny):
    pytest.importorskip("cv2")
    from oracle import depth_oracle as O
    m, g, meta = tiny
    d = m.infer_image(O.raw_image(meta["seeds"][3]), 126)
    e = rel(d, g["infer_depth"])
    print(f"[depth tiny infer_image] rel-L2 vs reference {e:.2e}")
    assert isinstance(d, np.ndarray) and d.shape == (60, 90) and e < TINY_TOL


def test_swiglu_backbone_vs_hub(cuda_ops):
    """encoders.Dinov2Model with the SwiGLU MLP (FrozenDinoV2Encoder's backbone) against the hub class itself, offset 0.1."""
    from anyedit_b200.encoders import Dinov2Model
    from oracle import depth_oracle as O, dinov2_oracle
    g = np.load(os.path.join(G, "depth_anything_tiny.npz"))
    meta = json.load(open(os.path.join(G, "depth_anything_tiny_keys.json")))
    m = Dinov2Model(O.TINY_SWIGLU, interpolate_offset=0.1)
    m.load_state_dict(dinov2_oracle.seeded_state_dict({k: tuple(v) for k, v in meta["swiglu_keys"].items()}, meta["seeds"][2]), strict=True)
    f = m.cuda().forward_features(O.tiny_images(O.TINY_SIZES[1], meta["seeds"][2], B=1).cuda())
    e = rel(torch.cat([f["x_norm_clstoken"][:, None], f["x_norm_patchtokens"]], 1), g["swiglu_x_norm"])
    print(f"[dinov2 SwiGLU backbone, 7 x 13 patches] rel-L2 vs hub {e:.2e}")
    assert e < SWIGLU_TOL


@pytest.mark.parametrize("H,W", [(518, 518), (518, 784)])
def test_vitl_real_width_vs_oracle(cuda_ops, H, W):
    """D 1024, 16 heads, 4 GELU blocks read at [0, 1, 2, 3], the full-width head (features 256, out_channels 256/512/1024/1024)."""
    from anyedit_b200.depth import DepthAnythingV2
    from oracle import depth_oracle as O
    m = DepthAnythingV2(encoder="vitl", config={"num_hidden_layers": 4}, layer_idx=[0, 1, 2, 3])
    sd = O.seeded_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, 31)
    m.load_state_dict(sd, strict=True)
    x = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(32))
    out = m.cuda()(x.cuda())
    with torch.no_grad():
        ref = O.depth(sd, x, [0, 1, 2, 3], 16)
    e = rel(out, ref)
    print(f"[depth vitl real width, 4 blocks, {H}x{W}] rel-L2 vs fp32 oracle {e:.2e}; positive {float((ref > 0).float().mean()):.3f}")
    assert tuple(out.shape) == (1, H, W) and e < REAL_TOL


def test_full_vitl_determinism_batch_independence_round_trip(cuda_ops):
    from anyedit_b200.depth import DepthAnythingV2
    torch.manual_seed(0)
    m = DepthAnythingV2(encoder="vitl", features=256, out_channels=[256, 512, 1024, 1024])
    assert len(m.pretrained.blocks) == 24 and len(m.state_dict()) == 407
    m = m.cuda().eval()
    x = torch.randn(3, 3, 518, 518, generator=torch.Generator().manual_seed(33)).cuda()
    a = m(x)
    assert a.dtype == torch.float32 and tuple(a.shape) == (3, 518, 518) and bool(a.isfinite().all())
    assert torch.equal(m(x), a), "two calls differ"
    for i in range(3):
        assert torch.equal(m(x[i:i + 1])[0], a[i]), f"image {i}: batch 1 != batch 3"
    m2 = DepthAnythingV2(encoder="vitl")
    m2.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()}, strict=True)
    assert torch.equal(m2.cuda()(x[:1])[0], a[0]), "state dict round trip changed the output"


def _worker(argv):
    from anyedit_b200 import ops
    inputs = torch.load(argv[0])
    res = _run(ops, inputs)
    res["__probe__"] = _probe_refusals()
    torch.save(res, argv[1])
    return 0


if __name__ == "__main__" and sys.argv[1:2] == ["--worker"]:
    sys.exit(_worker(sys.argv[2:]))
