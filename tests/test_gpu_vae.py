"""First stage on the GPU (SURVEY.md 8f rank 1): ``anyedit_b200.autoencoder.AutoencoderKL`` against golden outputs of the
reference's own Encoder / Decoder (tests/golden/make_golden_vae.py), plus the three pieces it adds to the C ABI: the conv
kernel's right/bottom padding mode, the row softmax of the wide single-head attention, the posterior sampling kernel."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), "golden")
FWD_TOL = 4e-3            # fp16 operands / fp32 accumulate vs the fp32 reference, relative L2


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _build(name):
    from anyedit_b200.autoencoder import AutoencoderKL
    from oracle import weights
    g = np.load(os.path.join(G, f"{name}.npz"))
    meta = json.load(open(os.path.join(G, f"{name}_keys.json")))
    net = AutoencoderKL(meta["config"], embed_dim=4)
    sd = weights.make_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, int(g["seed"]))
    assert weights.checksum(sd) == pytest.approx(float(g["wsum"]), rel=1e-12)
    net.load_state_dict(sd, strict=True)
    return net.cuda(), g


def test_conv_right_bottom_padding_vs_torch():
    """F.pad(x, (0,1,0,1)) + conv3x3 stride 2 pad 0 (model.py:83-85), even and odd sizes."""
    from anyedit_b200 import ops
    from anyedit_b200.unet import _pack_conv3
    gen = torch.Generator().manual_seed(3)
    for (N, H, W, C, Co) in ((2, 16, 12, 64, 64), (1, 9, 7, 128, 64), (3, 32, 32, 64, 128)):
        x, w, b = torch.randn(N, C, H, W, generator=gen), torch.randn(Co, C, 3, 3, generator=gen) * 0.05, torch.randn(Co, generator=gen)
        ref = F.conv2d(F.pad(x.half().float(), (0, 1, 0, 1)), w.half().float(), b, stride=2)
        xin = x.permute(0, 2, 3, 1).contiguous().half().cuda()
        out = torch.empty(N, ref.shape[2], ref.shape[3], Co, dtype=torch.float16, device="cuda")
        ops.conv3x3(xin, _pack_conv3(w, "cuda"), out.view(-1, Co), bias=b.cuda(), stride=2, pad_rb=True)
        e = rel(out.permute(0, 3, 1, 2), ref)
        assert e < 1e-3, (N, H, W, e)


def test_softmax_rows_and_posterior_kernels():
    from anyedit_b200 import ops
    gen = torch.Generator().manual_seed(4)
    S = torch.randn(70, 200, generator=gen) * 6
    P = torch.empty(70, 200, dtype=torch.float16, device="cuda")
    ops.softmax_rows(S.cuda(), P, 0.37)
    assert rel(P, torch.softmax(S * 0.37, -1)) < 1e-3
    mom, noise = torch.randn(2, 8, 5, 6, generator=gen) * 3, torch.randn(2, 4, 5, 6, generator=gen)
    mom[0, 5, 0, 0], mom[1, 6, 1, 1] = 50.0, -80.0                       # exercise the clamp
    mean, logvar = mom.chunk(2, 1)
    logvar = logvar.clamp(-30.0, 20.0)
    sample, lv = torch.empty(2, 4, 5, 6, device="cuda"), torch.empty(2, 4, 5, 6, device="cuda")
    ops.gaussian_posterior(mom.cuda(), noise.cuda(), sample, lv, scale=0.18215)
    assert torch.equal(lv.cpu(), logvar)
    assert torch.allclose(sample.cpu(), 0.18215 * (mean + torch.exp(0.5 * logvar) * noise), rtol=2e-6, atol=1e-6)


@pytest.mark.parametrize("name", ["vae_mid", "vae_tiny"])
def test_autoencoder_vs_reference_golden(name):
    """encode -> moments and decode -> image against the reference Encoder / Decoder (+ the 1x1 quant convs): vae_mid has
    the SD ladder at half width (64..512 channels, C = 512 mid attention on the two-contraction path, C = 128 attention on
    the wgmma attention kernel, the right/bottom-padded Downsample); vae_tiny (32..128 channels) runs the decoder on
    the kernels' fallback tiles."""
    net, g = _build(name)
    img = net.decode(torch.from_numpy(g["z"]).cuda())
    e_img = rel(img, torch.from_numpy(g["img"]))
    print(f"[{name}] decode rel-L2 vs reference = {e_img:.3e}")
    assert tuple(img.shape) == g["img"].shape and e_img < FWD_TOL, e_img
    if name == "vae_tiny":
        return                                           # its 32-channel Downsample is below the 64-channel conv block
    post = net.encode(torch.from_numpy(g["x"]).cuda())
    e_mom = rel(post.parameters, torch.from_numpy(g["moments"]))
    print(f"[{name}] encode moments rel-L2 vs reference = {e_mom:.3e}")
    assert tuple(post.parameters.shape) == g["moments"].shape and e_mom < FWD_TOL, e_mom
    mean, logvar = torch.from_numpy(g["moments"]).chunk(2, 1)
    assert rel(post.mode(), mean) < FWD_TOL
    noise = torch.randn(mean.shape, generator=torch.Generator().manual_seed(1))
    z = post.sample(noise.cuda())
    assert rel(z, mean + torch.exp(0.5 * logvar.clamp(-30, 20)) * noise) < 2 * FWD_TOL
    # the LatentDiffusion-side helpers (ddpm.py): scale_factor folded into the kernels
    from anyedit_b200.diffusion import LatentDenoiser
    from anyedit_b200.unet import UNetModel
    tiny = json.load(open(os.path.join(G, "tiny_a_keys.json")))["config"]
    ld = LatentDenoiser(UNetModel(**tiny), "hybrid", first_stage_model=net, scale_factor=0.18215).cuda()
    zs = ld.get_first_stage_encoding(ld.encode_first_stage(torch.from_numpy(g["x"]).cuda()), noise.cuda())
    assert torch.allclose(zs, 0.18215 * z, rtol=1e-5, atol=1e-6)
    dec = ld.decode_first_stage(torch.from_numpy(g["z"]).cuda() * 0.18215)
    assert rel(dec, torch.from_numpy(g["img"])) < FWD_TOL
