#!/usr/bin/env python
"""Times AnyEdit's post-filter scores on the GPU (DESIGN.md §10.10): the preprocess kernel alone for B = 64 pairs of 640 x 480
originals and 512 x 512 edits (CLIP-H's 64 edited images, ViT-B/32's 128 images), and ``score_pairs`` in pairs/s at B = 1, 8,
64 with seeded real-width weights (ViT-H/14 + its 1024-wide text tower, ViT-B/32).  When ``transformers`` is importable, the
reference-style arm: one pair at a time, an fp32 eager ``transformers.CLIPModel`` and an fp16 ViT-B/32 on the same GPU (the
processors' CPU time included, as utils.py runs them).  CUDA events; the card's name and power limit are read in the same run.
Usage: python tests/diag_postfilter.py [--out results/diag_postfilter.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(HERE, "golden"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from anyedit_b200 import ops
    from anyedit_b200.encoders import CLIPModel
    from anyedit_b200.postfilter import pixel_lut, score_pairs
    from oracle import weights
    import make_golden_postfilter as mg
    torch.set_grad_enabled(False)
    dev = torch.device("cuda")
    res = {"card": card()}
    rng = np.random.default_rng(0)
    B = 64
    orig = [torch.from_numpy(rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)).to(dev) for _ in range(B)]
    edit = [torch.from_numpy(rng.integers(0, 256, (512, 512, 3), dtype=np.uint8)).to(dev) for _ in range(B)]
    lut_h, lut_b = pixel_lut("floor", dev), pixel_lut("round", dev)
    res["preprocess_h_64_ms"] = timed(lambda: ops.clip_preprocess(edit, lut_h, 14, "floor"), 50)
    res["preprocess_b32_128_ms"] = timed(lambda: ops.clip_preprocess(orig + edit, lut_b, 32, "round"), 50)
    tab, R, sm = ops.clip_preprocess_plan([tuple(t.shape[:2]) for t in orig + edit], "round", 32)
    res["preprocess_plan_b32_128"] = {"rows_per_cta": R, "smem_bytes": sm, "table_ints": tab.numel()}
    print(res, flush=True)

    def model(name):
        cfg, seed = mg.CONFIGS[name]
        m = CLIPModel(cfg)
        shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        sd = weights.make_state_dict(shapes, seed)
        sd["logit_scale"] = torch.tensor(mg.LOGIT_SCALE)
        m.load_state_dict(sd, strict=False)
        return m.cuda(), sd

    m_h, sd_h = model("real_h")
    m_b, sd_b = model("real_b32")
    ids_h = mg.token_ids(mg.CONFIGS["real_h"][0], 5, [12] * B)
    ids_in, ids_out = mg.token_ids(mg.CONFIGS["real_b32"][0], 6, [9] * B), mg.token_ids(mg.CONFIGS["real_b32"][0], 7, [15] * B)
    # score_pairs needs equal shapes per pair (the L1 distance): both images cut to 480 x 512
    o_c, e_c = [o[:, :512].contiguous() for o in orig], [e[:480].contiguous() for e in edit]
    for b in (1, 8, 64):
        ms = timed(lambda: score_pairs(m_h, m_b, o_c[:b], e_c[:b], ids_in[:b], ids_h[:b], output_ids_b32=ids_out[:b]),
                   5 if b == 64 else 10, warm=2)
        res[f"score_pairs_B{b}_pairs_per_s"] = b / (ms / 1e3)
        print(b, res[f"score_pairs_B{b}_pairs_per_s"], flush=True)
    try:
        import transformers
        from PIL import Image
        from transformers import CLIPConfig, CLIPImageProcessorPil
        from transformers import CLIPModel as HFCLIP
        ref_h = HFCLIP(CLIPConfig(**mg.CONFIGS["real_h"][0])).eval()
        ref_h.load_state_dict(sd_h, strict=False)
        ref_h = ref_h.to(dev)
        ref_b = HFCLIP(CLIPConfig(**mg.CONFIGS["real_b32"][0])).eval()
        ref_b.load_state_dict(sd_b, strict=False)
        ref_b = ref_b.half().to(dev)
        proc = mg.processors()
        n = 8
        pil_o = [o.cpu().numpy() for o in o_c[:n]]
        pil_e = [e.cpu().numpy() for e in e_c[:n]]

        def ref_pair(i):
            px = proc[0]([pil_e[i]]).to(dev)
            ref_h(input_ids=ids_h[i:i + 1].to(dev), pixel_values=px).logits_per_image.item()
            pa, pb = proc[1]([pil_o[i]]).to(dev).half(), proc[1]([pil_e[i]]).to(dev).half()
            fa, fb = ref_b.get_image_features(pixel_values=pa), ref_b.get_image_features(pixel_values=pb)
            ta = ref_b.get_text_features(input_ids=ids_in[i:i + 1].to(dev))
            tb = ref_b.get_text_features(input_ids=ids_out[i:i + 1].to(dev))
            fa, fb, ta, tb = (getattr(t, "pooler_output", t) for t in (fa, fb, ta, tb))
            torch.nn.functional.cosine_similarity(fb - fa, tb - ta).item()
            a, b = pil_o[i], pil_e[i]
            np.sum(np.abs(a - b)) / a.size / 255

        ref_pair(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            ref_pair(i)
        torch.cuda.synchronize()
        res["reference_style_pairs_per_s"] = n / (time.perf_counter() - t0)
        res["transformers"] = transformers.__version__
    except ImportError:
        res["reference_style_pairs_per_s"] = "not measured (transformers not importable)"
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
