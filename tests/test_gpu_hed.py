"""The HED scribble annotator on the GPU (``hed.ControlNetHED_Apache2`` / ``hed.HEDdetector``) and the kernels it adds:

* the 2x2 max-pool bit for bit against ``F.max_pool2d`` on odd sizes; the input kernel bit for bit against a torch construction of
  its taps, and the first conv (one K = 32 contraction on them) against float64 within the element bound; the edge kernel against
  the reference's cv2 / numpy post-processing on the same fp32 side maps;
* the real-width network against the reference's golden (three small sizes) and against the fp32 oracle on the GPU at 480 x 640
  and 512 x 512 with TF32 off; activations beyond fp16's range but inside 65504 / S; determinism, batch independence, the
  strict state-dict round trip, the launch count and the detector's file and batched paths.

Element bound (terms of tests/test_gpu_segment.py): fp32 sums of n products carry <= n 2^-24 of the sum of magnitudes; one fp16
rounding adds 2^-11 |y| + 2^-25.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
G = os.path.join(os.path.dirname(__file__), "golden")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
U = 2.0 ** -24
# about 3x the values measured on the H100 (DESIGN.md §10.6): worst side map 2.2e-3 (golden) and 2.7e-3 (real sizes); 1.2 % and
# 2.8 % of uint8 pixels differ, by at most 1
GOLD_SIDE_TOL, REAL_SIDE_TOL = 6.5e-3, 8e-3        # side-map rel-L2
GOLD_SAME, REAL_SAME = 0.965, 0.915                # fraction of identical uint8 pixels
MAX_DELTA = 2                                      # largest |uint8 difference|
SIZES = [(48, 64), (61, 93), (17, 200), (480, 640), (512, 512)]


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def cuda_ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from anyedit_b200 import ops
    assert tuple(ops.device_info())[1:] == (9, 0), "sm_90a kernels need a Hopper GPU (H100)"
    return ops


def nchw(t):
    return t.permute(0, 3, 1, 2)


def side_sizes(H, W):
    out = [(H, W)]
    for _ in range(4):
        H, W = H // 2, W // 2
        out.append((H, W))
    return out


def compare_u8(got, want, name):
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    same = float((d == 0).mean())
    print(f"{name}: {same:.5f} of uint8 pixels identical, max |delta| {int(d.max())}")
    return same, int(d.max())


# ---- kernels -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cc", [64, 128, 256, 512])
@pytest.mark.parametrize("B,H,W", [(2, 13, 17), (3, 7, 9), (2, 2, 3)])
def test_max_pool_bit_exact(cuda_ops, B, H, W, Cc):
    x = torch.randn(B, H, W, Cc, generator=torch.Generator().manual_seed(H * W + Cc)).half().cuda()
    x[0, 0, 0, :8] = 0.0
    x[0, 0, 1, :8] = -0.0                              # ties of +0 / -0 keep the first in window order, as ATen does
    y = torch.empty(B, H // 2, W // 2, Cc, dtype=torch.float16, device="cuda")
    cuda_ops.max_pool2(x, y)
    want = F.max_pool2d(nchw(x), 2, 2).permute(0, 2, 3, 1)
    assert torch.equal(y.view(torch.int16), want.contiguous().view(torch.int16))


def _model(seed=111, **gains):
    from anyedit_b200.hed import ControlNetHED_Apache2
    from oracle import hed_oracle as O
    sd = O.seeded_state_dict(seed, **gains)
    m = ControlNetHED_Apache2()
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


def test_input_kernel_and_first_conv(cuda_ops):
    from anyedit_b200.hed import S
    from oracle import hed_oracle as O
    m, sd = _model()
    B, H, W = 2, 19, 23
    img = torch.from_numpy(O.images((H, W), 7, B=B)).cuda()
    P = m._packed()
    cols = torch.empty(B * H * W, 32, dtype=torch.float16, device="cuda")
    cuda_ops.hed_input(img, P["norm"], cols, S)
    h = F.pad(((nchw(img).float() - sd["norm"].cuda()) * S), (1, 1, 1, 1))        # zero padding after the subtraction
    taps = torch.stack([h[:, :, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)], 1)   # [B, tap, c, H, W]
    want = torch.zeros(B * H * W, 32, dtype=torch.float16, device="cuda")
    want[:, :27] = taps.permute(0, 3, 4, 1, 2).reshape(B * H * W, 27).half()
    assert torch.equal(cols.view(torch.int16), want.view(torch.int16))

    w, b = P["blocks"][0]["convs"][0]
    y = torch.empty(B * H * W, 64, dtype=torch.float16, device="cuda")
    cuda_ops.gemm(cols, w, y, bias=b, act=6)
    a, wd, bd = cols.double(), w.double(), b.double()
    ref = (a @ wd.t() + bd).clamp_min(0)
    bound = 34 * U * (a.abs() @ wd.abs().t() + bd.abs()) + 2.0 ** -11 * ref.abs() + 2.0 ** -25
    q = float(((y.double() - ref).abs() / bound).max())
    print(f"first conv (K = 32) worst err/bound {q:.3f}")
    assert q <= 1.0


@pytest.mark.parametrize("H,W", SIZES)
def test_edges_vs_cv2(cuda_ops, H, W):
    """The edge kernel against the reference's cv2.resize / np.mean / float64 sigmoid on the same fp32 side maps: identical uint8
    wherever the host's 255 sigmoid(mean) is more than 1e-4 from an integer, |delta| <= 1 elsewhere (cv2 may round its resize
    differently in the last bits)."""
    from oracle import hed_oracle as O
    g = torch.Generator().manual_seed(H * 1000 + W)
    B = 2
    maps = [torch.randn(B, h, w, generator=g) * 2.0 + 0.5 * k - 1.0 for k, (h, w) in enumerate(side_sizes(H, W))]
    v = O.post_sigmoid([t[:, None] for t in maps], H, W)
    want = O.edge_map([t[:, None] for t in maps], H, W)
    # contiguous maps (ld 1) and one column of [B, h, w, 8] buffers (ld 8, as the model passes them)
    wide = [torch.zeros(*t.shape, 8) for t in maps]
    for t, w8 in zip(maps, wide):
        w8[..., 0] = t
    for name, dev_maps in (("ld 1", [t.cuda() for t in maps]), ("ld 8", [w8.cuda()[..., 0] for w8 in wide])):
        out = torch.empty(B, H, W, dtype=torch.uint8, device="cuda")
        cuda_ops.hed_edges(dev_maps, out)
        got = out.cpu().numpy()
        clear = np.abs(v - np.round(v)) > 1e-4
        d = np.abs(got.astype(np.int32) - want.astype(np.int32))
        print(f"edges {H}x{W} {name}: {float((d == 0).mean()):.6f} identical, {float(clear.mean()):.4f} of pixels clear of an "
              f"integer, max |delta| {int(d.max())}")
        assert bool((d[clear] == 0).all()) and int(d.max()) <= 1


# ---- model -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(G, "hed_golden.npz")), json.load(open(os.path.join(G, "hed_keys.json")))


def test_model_vs_reference_golden(cuda_ops, gold, tmp_path):
    from anyedit_b200.hed import HEDdetector
    g, meta = gold
    from oracle import hed_oracle as O
    path = os.path.join(tmp_path, "ControlNetHED.pth")
    torch.save(O.seeded_state_dict(meta["seeds"][0]), path)
    det = HEDdetector(path)
    import cv2
    for H, W in meta["sizes"]:
        s = f"{H}x{W}"
        img = g[f"img{s}"]
        sides = det.netNetwork(torch.from_numpy(img)[None].cuda())
        for k, e in enumerate(sides):
            err = rel(e[0, 0], g[f"side{s}_{k}"])
            print(f"[hed golden] {s} side {k} {tuple(e.shape)} rel-L2 vs reference {err:.2e}")
            assert tuple(e.shape[2:]) == g[f"side{s}_{k}"].shape and err <= GOLD_SIDE_TOL
        edge = det.detect(img[None])[0]
        same, dmax = compare_u8(edge, g[f"edge{s}"], f"[hed golden] {s} edge map vs reference")
        assert same >= GOLD_SAME and dmax <= MAX_DELTA
        src, dst = os.path.join(tmp_path, f"{s}.png"), os.path.join(tmp_path, f"{s}_edge.png")
        cv2.imwrite(src, img)
        det(src, dst)
        assert np.array_equal(cv2.imread(dst, cv2.IMREAD_UNCHANGED), edge), "__call__ and detect disagree"
        assert torch.equal(det.detect(torch.from_numpy(img)[None].cuda()).cpu(), torch.from_numpy(edge)[None])


def _oracle_on_gpu(sd, img):
    """The fp32 oracle on this GPU with TF32 off (restored after)."""
    from oracle import hed_oracle as O
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return O.side_maps({k: v.cuda() for k, v in sd.items()}, img)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags


@pytest.mark.parametrize("H,W", [(480, 640), (512, 512)])
def test_real_size_vs_fp32_oracle(cuda_ops, H, W):
    from oracle import hed_oracle as O
    m, sd = _model(seed=112)
    img = torch.from_numpy(O.images((H, W), 113)).cuda()
    want = _oracle_on_gpu(sd, img)
    got = m(img)
    errs = [rel(a, b) for a, b in zip(got, want)]
    print(f"[hed real] {H}x{W} side-map rel-L2 vs fp32 oracle: " + ", ".join(f"{e:.2e}" for e in errs))
    same, dmax = compare_u8(m.edge_map(img).cpu().numpy(), O.edge_map(want, H, W), f"[hed real] {H}x{W} edge map vs fp32 oracle")
    assert max(errs) <= REAL_SIDE_TOL and same >= REAL_SAME and dmax <= MAX_DELTA


def test_range_beyond_fp16(cuda_ops):
    """Inflated conv gains: the fp32 activations exceed 65504 but stay below 65504 / S, and the side maps stay finite and match."""
    from anyedit_b200.hed import S
    from oracle import hed_oracle as O
    m, sd = _model(seed=114, conv_gain=2 * 2 ** 0.5)
    img = torch.from_numpy(O.images((64, 96), 115)).cuda()
    sdc = {k: v.cuda() for k, v in sd.items()}
    h, peak = nchw(img).float() - sdc["norm"], 0.0
    for b, (_, _, n) in enumerate(O.BLOCKS, 1):
        h = F.max_pool2d(h, 2) if b > 1 else h
        for i in range(n):
            h = F.relu(F.conv2d(h, sdc[f"block{b}.convs.{i}.weight"], sdc[f"block{b}.convs.{i}.bias"], padding=1))
            peak = max(peak, float(h.max()))
    print(f"[hed range] peak fp32 activation {peak:.3e} (fp16 max 65504, 65504 / S = {65504 / S:.3e})")
    assert 65504 < peak < 65504 / S / 4
    want = _oracle_on_gpu(sd, img)
    got = m(img)
    errs = [rel(a, b) for a, b in zip(got, want)]
    print("[hed range] side-map rel-L2 vs fp32 oracle: " + ", ".join(f"{e:.2e}" for e in errs))
    assert all(bool(t.isfinite().all()) for t in got) and max(errs) <= REAL_SIDE_TOL


def test_determinism_batch_independence_round_trip(cuda_ops):
    from anyedit_b200 import ops
    from anyedit_b200.hed import ControlNetHED_Apache2
    m, _ = _model(seed=116)
    g = torch.Generator().manual_seed(117)
    x = torch.randint(0, 256, (3, 130, 161, 3), generator=g, dtype=torch.uint8).cuda()
    sides = [t.clone() for t in m(x)]
    n0 = ops.launch_count
    e = m.edge_map(x)
    assert ops.launch_count - n0 == 24, f"{ops.launch_count - n0} launches for one batch (24 planned)"
    assert all(torch.equal(a, b) for a, b in zip(m(x), sides)) and torch.equal(m.edge_map(x), e), "two calls differ"
    for i in range(3):
        assert all(torch.equal(a[0], b[i]) for a, b in zip(m(x[i:i + 1]), sides)), f"image {i}: batch 1 != batch 3"
        assert torch.equal(m.edge_map(x[i:i + 1])[0], e[i])
    m2 = ControlNetHED_Apache2()
    m2.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()}, strict=True)
    assert torch.equal(m2.cuda().edge_map(x), e), "state dict round trip changed the output"
