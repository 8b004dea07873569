"""Kernel-time breakdown of one PT-v3m1 base training step (torch.profiler / CUPTI), run on a GPU."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointcept_b200 import synth  # noqa: E402
from pointcept_b200.ptv3 import PTv3Segmentor, ptv3_base_config  # noqa: E402

dev = "cuda"
torch.manual_seed(0)
model = PTv3Segmentor(num_classes=20, backbone_out_channels=64, **ptv3_base_config()).to(dev).train()
opt = torch.optim.AdamW(model.parameters(), lr=1e-4, fused=True)
hb = synth.make_batch(2, seed=100)
d = {k: torch.from_numpy(v).to(dev) for k, v in hb.items()}
d["offset_host"] = [int(v) for v in hb["offset"]]
d["grid_max_host"] = [int(v) for v in hb["grid_coord"].max(0)]


def step():
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = model(d)
    out["loss"].backward()
    opt.step()


for _ in range(3):
    step()
torch.cuda.synchronize()
from torch.profiler import ProfilerActivity, profile  # noqa: E402

with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    for _ in range(2):
        step()
    torch.cuda.synchronize()
ka = prof.key_averages()
rows = sorted([e for e in ka if e.device_time_total > 0 and e.device_type.name == "CUDA"], key=lambda e: -e.device_time_total)
tot = sum(e.device_time_total for e in rows)
print(f"total CUDA kernel time per step: {tot / 2 / 1000:.2f} ms over {sum(e.count for e in rows) // 2} kernels")
for e in rows[:45]:
    print(f"{e.device_time_total / 2 / 1000:9.3f} ms  {100 * e.device_time_total / tot:5.1f}%  n={e.count // 2:5d}  {e.key[:110]}")

# CPU side: where does the host time of a step go?
rows_cpu = sorted(ka, key=lambda e: -e.self_cpu_time_total)
tot_cpu = sum(e.self_cpu_time_total for e in ka)
print(f"\ntotal self CPU time per step (profiler overhead included): {tot_cpu / 2 / 1000:.1f} ms")
for e in rows_cpu[:40]:
    print(f"{e.self_cpu_time_total / 2 / 1000:9.3f} ms  n={e.count // 2:5d}  {e.key[:90]}")
import cProfile, pstats, io, time
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(3):
    step()
torch.cuda.synchronize()
print(f"\nwall per step (no profiler): {(time.perf_counter() - t0) / 3 * 1e3:.1f} ms")
pr = cProfile.Profile()
pr.enable()
for _ in range(2):
    step()
torch.cuda.synchronize()
pr.disable()
sio = io.StringIO()
pstats.Stats(pr, stream=sio).sort_stats("tottime").print_stats(35)
print(sio.getvalue()[:6000])
