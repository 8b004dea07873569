"""Whole-step timing of the BASELINE.md B2 comparator (tools/gpu_reference.py) next to this repo's path, same GPU, same process.
Run on a GPU:  python tools/time_reference.py [--scenes 2] [--steps 5]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointcept_b200 import synth  # noqa: E402
from pointcept_b200.ptv3 import PTv3Segmentor, ptv3_base_config  # noqa: E402
from tools import gpu_reference  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    dev = "cuda"
    hb = synth.make_batch(a.scenes, seed=100)
    d = {k: torch.from_numpy(v).to(dev) for k, v in hb.items()}
    d["offset_host"] = [int(v) for v in hb["offset"]]
    d["grid_max_host"] = [int(v) for v in hb["grid_coord"].max(0)]
    n = d["offset_host"][-1]
    res = {}
    for name in ("reference_gpu", "ours"):
        torch.manual_seed(0)
        model = PTv3Segmentor(num_classes=20, backbone_out_channels=64, spatial_reorder=(name == "ours"), **ptv3_base_config()).to(dev).train()
        opt = torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.05, fused=True)

        def step():
            opt.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = model(dict(d))
            out["loss"].backward()
            opt.step()
            return out["loss"]

        if name == "reference_gpu":
            with gpu_reference.reference_gpu_ops():
                res[name] = timed(step, a)
        else:
            res[name] = timed(step, a)
        del model, opt
        torch.cuda.empty_cache()
    out = {k: dict(ms_per_step=v[0], points_per_s=n / (v[0] * 1e-3), loss=v[1]) for k, v in res.items()}
    out["ratio_ours_over_reference"] = res["reference_gpu"][0] / res["ours"][0]
    out["points_per_step"] = n
    try:
        out["flash_attn"] = gpu_reference.stock_flash_attn()[1]
    except Exception as e:
        out["flash_attn"] = repr(e)
    print(json.dumps(out))


def timed(step, a):
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.steps, float(loss)


if __name__ == "__main__":
    main()
