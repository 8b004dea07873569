#!/usr/bin/env python
"""points/sec forward+backward of PT-v3m1 "base" (configs/scannet/semseg-pt-v3m1-0-base.py) on synthetic
ScanNet-scale scenes, sharded by whole scenes over N GPUs (DDP, NCCL gradient all-reduce only).

    python bench.py --gpus 1 --steps 20 --warmup 5
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference ...      # the CPU restatement of the reference path, host cores

One step = zero_grad + forward (bf16 autocast) + loss + backward (+ DDP all-reduce) + AdamW step on a batch of
`--scenes-per-gpu` scenes per rank (weak scaling; BASELINE config 4: batch 16 over 8 GPUs = 2 scenes / GPU).
Prints ONE JSON line on rank 0.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "points/sec fwd+bwd (PTv3-base, ScanNet-scale synth)"   # --workload spunet34 reports the same unit for SpUNet-34
UNIT = "points/s"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--scenes-per-gpu", type=int, default=2)
    ap.add_argument("--voxels", type=int, default=120_000, help="voxels per synthetic scene")
    ap.add_argument("--cpu-voxels", type=int, default=120_000, help="scene size of the bounded CPU sample (one scene)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--cpu-timeout", type=int, default=240)
    ap.add_argument("--workload", default="ptv3_base", choices=["ptv3_base", "spunet34"],
                    help="ptv3_base = the headline metric (BASELINE config 4 shape); spunet34 = BASELINE config 3 (supplementary)")
    ap.add_argument("--fused-linear", action="store_true", help="fused bias-gradient Linear (pays off for GPU-bound batches)")
    ap.add_argument("--no-reorder", action="store_true", help="keep level-0 points in input order (no z-order memory layout)")
    ap.add_argument("--kernel-impl", type=int, default=None, help="0 auto, 1 SIMT kernels, 2 tensor-core kernels")
    ap.add_argument("--no-supplementary", action="store_true", help="skip the short BASELINE config 3 / config 5 runs")
    ap.add_argument("--no-gpu-reference", action="store_true", help="skip the BASELINE.md B2 comparator (stock flash-attn + torch conv)")
    ap.add_argument("--gpu-reference-steps", type=int, default=5)
    ap.add_argument("--bucket-mb", type=int, default=100, help="DDP gradient bucket size")
    ap.add_argument("--no-static-graph", action="store_true", help="DDP without static_graph")
    ap.add_argument("--grad-exchange", default="flat", choices=["flat", "ddp"],
                    help="N > 1: pointcept_b200.reducer.FlatGradReducer (one hook, two collectives per step) or torch DDP")
    ap.add_argument("--side-priority", type=int, default=-1,
                    help="CUDA priority of the prefetch stream that prepares the next batch (-1 = high: its host reads are not queued "
                         "behind the training backlog; 0 = default priority)")
    ap.add_argument("--force-dist", action="store_true",
                    help="N = 1 only: initialise NCCL with world size 1 and run the gradient exchange anyway (measures its overhead)")
    ap.add_argument("--torch-profile", default=None, help="write a torch.profiler (CUPTI) per-kernel breakdown of two extra steps to this file")
    ap.add_argument("--torch-adamw", action="store_true", help="torch.optim.AdamW(fused=True) instead of pointcept_b200.optim.FusedAdamW")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write what the last timed step computed (rank 0) as DIR/<name>.npy: seg_logits, loss and a "
                         "fixed, seeded sample of the parameter gradients (float32, < 64 MB in all), to compare two builds output for output")
    return ap.parse_args()


def log(msg):
    print(f"[bench {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def host_cores():
    """usable host cores: affinity mask, further limited by a cgroup cpu quota if one is set"""
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            txt = open(path).read().split()
            if path.endswith("cpu.max"):
                if txt[0] != "max":
                    n = min(n, max(1, int(float(txt[0]) / float(txt[1]) + 0.5)))
            else:
                q = int(txt[0])
                if q > 0:
                    per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
                    n = min(n, max(1, int(q / per + 0.5)))
        except Exception:
            pass
    return max(1, n)


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(hbm=d["hbm_gbs"], tensor=d["bf16_tflops"], tensor_sustained=d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                    source="measured")
    return dict(hbm=3350.0, tensor=989.0, tensor_sustained=989.0, source="H100 SXM data sheet (dense bf16, 700 W), not measured")


# ---------------------------------------------------------------------------------------------------------
# clocks sampler (nvidia-smi, during the timed region)
# ---------------------------------------------------------------------------------------------------------
class ClockSampler:
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.lines, self.proc = [], None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100",
                                          "-i", str(index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return None
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                mx.append(float(f[1]))
            except ValueError:
                continue
            for nm, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        if not sm:
            return None
        return dict(sm_mhz=statistics.median(sm), sm_max_mhz=max(mx), reasons=sorted(reasons), samples=len(sm))


# ---------------------------------------------------------------------------------------------------------
# CPU arm: the oracle restatement of the reference path, all host threads, bounded sample
# ---------------------------------------------------------------------------------------------------------
def cpu_step_fn(voxels, seed=0):
    import numpy as np
    import torch
    from oracle import ptv3_cpu
    from pointcept_b200 import synth
    from pointcept_b200.ptv3 import PTv3Segmentor, ptv3_base_config

    cores = host_cores()
    torch.set_num_threads(cores)
    cfg = ptv3_base_config()
    torch.manual_seed(0)
    model = PTv3Segmentor(num_classes=20, backbone_out_channels=64, **cfg)   # parameters only; never executed on CPU
    sd = {k: v.detach().clone().requires_grad_(v.is_floating_point()) for k, v in model.state_dict().items()}
    bsd = {k[len("backbone."):]: v for k, v in sd.items() if k.startswith("backbone.")}
    batch = synth.make_batch(1, seed=seed, target_voxels=voxels)
    n = int(batch["offset"][-1])

    def step():
        for v in sd.values():
            v.grad = None
        feat = ptv3_cpu.forward(bsd, dict(grid_coord=batch["grid_coord"], feat=batch["feat"], offset=batch["offset"]), cfg, bn_training=True)
        logits = torch.nn.functional.linear(feat, sd["seg_head.weight"], sd["seg_head.bias"])
        loss = torch.nn.functional.cross_entropy(logits, torch.from_numpy(batch["segment"]))
        loss.backward()
        return float(loss.detach())

    return step, n, cores


def run_reference(args):
    """--impl reference: the reference's own CPU path (its serialization / padding / dense attention math as restated
    and pinned in oracle/, spconv restated) timed on the host cores.  Only rank 0 works."""
    if int(os.environ.get("RANK", "0")) != 0:
        return
    step, n, cores = cpu_step_fn(args.cpu_voxels)
    log(f"reference arm: {n} voxels on {cores} host cores")
    t0 = time.perf_counter()
    step()                                   # warm-up (also tells us how long a step takes)
    warm = time.perf_counter() - t0
    log(f"warm-up step {warm:.1f}s")
    steps = max(1, min(args.steps, 3, int(90.0 / max(warm, 1e-3))))   # keep the whole arm within a few minutes
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    dt = (time.perf_counter() - t0) / steps
    val = n / dt
    sample = f"1 scene x {n} voxels, PTv3-base fwd+bwd fp32, torch CPU, {steps} timed step(s)"
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": args.gpus, "steps": steps, "warmup": 1,
        "ms_per_step": dt * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
        "config": {"workload": "PT-v3m1 base (configs/scannet/semseg-pt-v3m1-0-base.py), bounded CPU sample", "sample": sample},
        "cpu_baseline": {"value": val, "unit": UNIT, "cores": cores, "kind": "port", "sample": sample},
        "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }))


# ---------------------------------------------------------------------------------------------------------
# GPU arm
# ---------------------------------------------------------------------------------------------------------
ATTAINABLE = {  # structural ceilings of the D = 16 attention kernels as a fraction of the tensor peak (DESIGN.md section 4)
    "attn_fwd": "exp pipe: 64 MMA-flop per ex2 at 16 ex2/clk/SM (132 SMs, 1.98 GHz) caps the forward near 0.27 of the dense bf16 tensor peak",
    "attn_bwd": "160 MMA-flop per score and two ex2 per score (dK/dV and dQ kernels each form P) at 16 ex2/clk/SM cap the backward "
                "near 0.34 of the dense bf16 tensor peak",
}


def build_model(workload, dev, args, in_channels=6, num_classes=20):
    import torch
    from pointcept_b200.ptv3 import PTv3Segmentor, ptv3_base_config
    if workload == "spunet34":
        from pointcept_b200.spunet import SpUNetBase

        class _SpUNetSeg(torch.nn.Module):
            """SpUNet-v1m1 stock widths (configs/scannet/semseg-spunet-v1m1-0-base.py:10-20) + CE loss"""

            def __init__(self):
                super().__init__()
                self.backbone = SpUNetBase(in_channels, num_classes)

            def prepare(self, d):
                return d

            def forward(self, d):
                logits = self.backbone(d)
                return dict(seg_logits=logits, loss=torch.nn.functional.cross_entropy(logits.float(), d["segment"]))

        return _SpUNetSeg().to(dev).train()
    cfg = dict(ptv3_base_config(), in_channels=in_channels)
    return PTv3Segmentor(num_classes=num_classes, backbone_out_channels=64, spatial_reorder=not args.no_reorder, **cfg).to(dev).train()


def measure(args, workload, scenes, voxels, steps, warmup, kind="indoor", want_profile=False, want_e2e=True, sample_clocks=False,
            reference_stack=False):
    """One workload on this rank's GPU (all ranks call it together): -> dict with value / ms / e2e / launches / clocks / profile."""
    import contextlib
    import torch
    import torch.distributed as dist
    from pointcept_b200 import _lib, synth

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device("cuda", local)
    torch.manual_seed(0)
    in_ch, n_cls = (4, 16) if kind == "lidar" else (6, 20)
    model = build_model(workload, dev, args, in_ch, n_cls)
    n_params = sum(p.numel() for p in model.parameters())
    net, reducer = model, None
    dist_on = world > 1 or (args.force_dist and dist.is_initialized())
    if dist_on and not reference_stack and args.grad_exchange == "flat":
        from pointcept_b200.reducer import FlatGradReducer     # the gradient all-reduce of engines/defaults.py:22-43, flat + overlapped
        reducer = FlatGradReducer(model.parameters())
    elif dist_on and not reference_stack:
        net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], broadcast_buffers=False, gradient_as_bucket_view=True,
                                                        bucket_cap_mb=args.bucket_mb, static_graph=not args.no_static_graph)
    if reference_stack or args.torch_adamw:
        opt = torch.optim.AdamW(net.parameters(), lr=1e-4, weight_decay=0.05, fused=True)
    else:
        from pointcept_b200.optim import FusedAdamW      # same update rule, one launch for all 486 tensors
        opt = FusedAdamW(net.parameters(), lr=1e-4, weight_decay=0.05)
    hb = synth.make_batch(scenes, seed=100 + rank, target_voxels=voxels, kind=kind, num_classes=n_cls)
    pinned = {k: torch.from_numpy(v).pin_memory() for k, v in hb.items()}
    offset_host = [int(v) for v in hb["offset"]]
    grid_max_host = [int(v) for v in hb["grid_coord"].max(0)]
    n_points = offset_host[-1]
    h2d_bytes = sum(t.numel() * t.element_size() for t in pinned.values())
    ctx = contextlib.nullcontext()
    if reference_stack:
        from tools import gpu_reference
        ctx = gpu_reference.reference_gpu_ops()

    def to_device():
        d = {k: t.to(dev, non_blocking=True) for k, t in pinned.items()}
        d["offset_host"], d["grid_max_host"] = offset_host, grid_max_host   # host metadata the collate already has
        return d

    last = {}

    def step(d):
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = net(d)
        if args.dump_outputs:
            last["out"] = out
        out["loss"].backward()
        if reducer is not None:
            reducer.finish()
        opt.step()
        return out["loss"]

    # Coordinate-only preparation (serialization, pooling index plans: the model's only host syncs) of the NEXT batch runs on
    # a side stream while the current batch trains, the way a data loader prefetches: its syncs then wait for the small
    # side-stream queue instead of the whole training backlog.  Work is done every step (nothing is cached across steps).
    side = torch.cuda.Stream(priority=args.side_priority)
    main = torch.cuda.current_stream()

    def prepare_async(make_inputs):
        with torch.cuda.stream(side):
            d = make_inputs()
            point = model.prepare(d)
            point["segment"] = d["segment"]
            ev = torch.cuda.Event()
            ev.record(side)
        if hasattr(point, "record_stream"):
            point.record_stream(main)
        else:
            for v in point.values():
                if isinstance(v, torch.Tensor) and v.is_cuda:
                    v.record_stream(main)
        return point, ev

    def run_steps(n, make_inputs, on_loss=None):
        nxt = prepare_async(make_inputs)
        for i in range(n):
            point, ev = nxt
            if i + 1 < n:
                nxt = prepare_async(make_inputs)
            main.wait_event(ev)
            loss = step(point)
            if on_loss is not None:
                on_loss(i, loss)

    def sync_all():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def allmax(x):
        t = torch.tensor([x], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    res = dict(points_per_gpu=n_points, params_M=round(n_params / 1e6, 2), h2d_bytes=h2d_bytes)
    with ctx:
        resident = to_device()
        torch.cuda.synchronize()
        resident_inputs = lambda: dict(resident)   # noqa: E731
        run_steps(max(warmup, 3), resident_inputs)
        sync_all()
        # ---- timed region 1: inputs resident in HBM, CUDA events, max over ranks ------------------------------
        L = _lib.lib()
        launches0 = L.b2pc_launch_count()
        sampler = ClockSampler(local) if (rank == 0 and sample_clocks) else None
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        sync_all()
        e0.record()
        run_steps(steps, resident_inputs)
        e1.record()
        sync_all()
        res["clocks"] = sampler.stop() if sampler else None
        res["launches"] = int(L.b2pc_launch_count() - launches0)
        ms_total = allmax(e0.elapsed_time(e1))
        pts = torch.tensor([float(n_points)], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(pts, op=dist.ReduceOp.SUM)
        total_points = float(pts.item())
        res.update(total_points=total_points, ms_per_step=ms_total / steps, value=total_points * steps / (ms_total * 1e-3))
        if args.dump_outputs and want_profile and rank == 0:
            dump_outputs(args.dump_outputs, last["out"], model)
        last.clear()
        # ---- roofline leg: the same steps, same (compiled) binding, with the library's own event pair around every hot entry
        # point (b2pc_profile_*); kept out of region 1 so that the event bookkeeping does not tax the headline number
        if want_profile:
            n_prof = min(steps, 3)
            p0, p1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            sync_all()
            L.b2pc_profile_enable(1)
            p0.record()
            run_steps(n_prof, resident_inputs)
            p1.record()
            sync_all()
            L.b2pc_profile_enable(0)
            res["profile"] = _lib.profile_collect()
            res["profile_ms_total"] = p0.elapsed_time(p1)
            res["profile_steps"] = n_prof
        if want_profile and args.torch_profile and rank == 0:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as tp:
                run_steps(2, resident_inputs)
                torch.cuda.synchronize()
            rows = sorted([e for e in tp.key_averages() if e.device_time_total > 0], key=lambda e: -e.device_time_total)
            tot = sum(e.device_time_total for e in rows)
            with open(args.torch_profile, "w") as f:
                f.write(f"# torch.profiler (CUPTI) device time of {workload} training steps, per step: {tot / 2e3:.2f} ms in "
                        f"{sum(e.count for e in rows) // 2} kernels / memsets / copies\n")
                own = sum(e.device_time_total for e in rows if "b2pc::" in e.key)
                f.write(f"# b2pc:: kernels {100 * own / tot:.1f} % of device time\n")
                for e in rows[:90]:
                    f.write(f"{e.device_time_total / 2e3:9.3f} ms {100 * e.device_time_total / tot:5.1f}%  n={e.count // 2:5d}  {e.key[:150]}\n")
        # ---- timed region 2: end to end through the public API with HOST buffers ---------------------------------
        if want_e2e:
            loss_pinned = torch.zeros(steps, dtype=torch.float32).pin_memory()
            sync_all()
            t0 = time.perf_counter()

            def read_loss(i, loss):                                    # device -> host read of the step's result
                loss_pinned[i:i + 1].copy_(loss.detach().float().reshape(1), non_blocking=True)

            run_steps(steps, to_device, read_loss)                     # host -> device copy of every step's inputs inside prepare_async
            torch.cuda.synchronize()
            dt = allmax(time.perf_counter() - t0)
            res["e2e_value"] = total_points * steps / dt
            res["loss_last"] = float(loss_pinned[-1])
    if reducer is not None:
        res["grad_exchange"] = dict(kind="flat", steps=reducer.stats["steps"], overlapped_steps=reducer.stats["early_steps"], late_steps=reducer.stats["late_steps"],
                                    early_bytes=4 * reducer.early_end, total_bytes=4 * reducer.flat.numel())
        reducer.remove()
    elif dist_on and not reference_stack:
        res["grad_exchange"] = dict(kind="ddp", bucket_mb=args.bucket_mb, static_graph=not args.no_static_graph)
    del net, model, opt, reducer
    torch.cuda.empty_cache()
    return res


def dump_outputs(out_dir, out, model, grad_sample=1 << 20):
    """What the last timed step computed: the segmentation logits and loss the forward returned and, of the parameter gradients
    (all of them together are larger than the 64 MB budget), the `grad_sample` entries of their concatenation in named_parameters()
    order at the sorted positions torch.randperm(n, generator=torch.Generator().manual_seed(0))[:grad_sample] picks.  The parameter
    update of that step is not included."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "seg_logits.npy"), out["seg_logits"].detach().float().cpu().numpy())
    np.save(os.path.join(out_dir, "loss.npy"), out["loss"].detach().float().cpu().numpy().reshape(1))
    grads = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).detach().float().reshape(-1) for _, p in model.named_parameters()])
    g = torch.Generator().manual_seed(0)
    idx = torch.randperm(grads.numel(), generator=g)[:grad_sample].sort().values
    np.save(os.path.join(out_dir, "grad_sample.npy"), grads[idx.to(grads.device)].cpu().numpy())


def rooflines(prof, prof_ms_total, pk):
    """per entry point: achieved algorithmic rate against the bound that applies (SURVEY.md 8(d)) -> (list, shares)"""
    out, shares = [], {}
    for name, r in prof.items():
        shares[name] = round(r["ms"] / prof_ms_total, 4)
        if r["ms"] <= 0:
            continue
        ent = dict(kernel=name, launches=r["calls"], avg_ms=r["ms"] / r["calls"], share_of_step=shares[name])
        if name.startswith("attn"):
            ach = r["flops"] / (r["ms"] * 1e-3) / 1e12
            ent.update(bound="tensor", achieved=ach, peak=pk["tensor_sustained"], unit="TFLOP/s", frac=ach / pk["tensor_sustained"],
                       peak_source=pk["source"] + " (sustained cuBLAS bf16)", ceiling=ATTAINABLE[name],
                       hbm_gbs=r["bytes"] / (r["ms"] * 1e-3) / 1e9)
        elif r["bytes"] > 0:
            ach = r["bytes"] / (r["ms"] * 1e-3) / 1e9
            ent.update(bound="hbm", achieved=ach, peak=pk["hbm"], unit="GB/s", frac=ach / pk["hbm"], peak_source=pk["source"] + " (copy)")
        else:
            continue
        out.append(ent)
    out.sort(key=lambda e: -e["share_of_step"])
    return out, shares


def measure_grid_sample(scenes, voxels, dev, pk, iters=20):
    """GPU voxelisation + collate (SURVEY 8(f).3) of `scenes` raw ScanNet-scale scenes (~2 raw points per 2 cm voxel): the
    transform in front of the hot path, timed alone with CUDA events; raw points/s and its HBM roofline fraction."""
    import numpy as np
    import torch
    from pointcept_b200 import datasets, synth
    hb = synth.make_batch(scenes, seed=7, target_voxels=voxels)
    rng = np.random.default_rng(7)
    grid, off = hb["grid_coord"], hb["offset"]
    raw, sizes, s = [], [], 0
    for e in off:
        g = grid[s:e]
        pick = rng.integers(0, len(g), 2 * len(g))
        raw.append(((g[pick] + rng.random((len(pick), 3))) * 0.02).astype(np.float32))
        sizes.append(len(pick))
        s = e
    coord = torch.from_numpy(np.concatenate(raw)).to(dev)
    feat = torch.randn(coord.shape[0], 6, device=dev)
    seg = torch.randint(0, 20, (coord.shape[0],), device=dev, dtype=torch.int32)
    batch = dict(coord=coord, feat=feat, segment=seg, offset=torch.tensor(np.cumsum(sizes)), index_valid_keys=["coord", "feat", "segment"])
    tr = datasets.GridSample(grid_size=0.02, hash_type="fnv", mode="train", return_grid_coord=True, seed=1)
    for _ in range(3):
        out = tr(dict(batch))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = tr(dict(batch))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    n = coord.shape[0]
    # algorithmic bytes per raw point: 2 x 12 B coord reads (extent, key), 24 B grid_coord + 8 B key out, 8 radix passes x 32 B
    # (sort.cuh), run heads / ids / inverse ~ 60 B; per voxel: pick + payload gather ~ (8 + 12 + 24 + 24 + 4) x 2 B
    bytes_alg = n * (24 + 32 + 8 * 32 + 60) + out["coord"].shape[0] * 144
    return dict(workload=f"GridSample(0.02, fnv, train) + collate of {scenes} raw scenes, {n} raw points -> {out['coord'].shape[0]} voxels",
                value=n / (ms * 1e-3), unit="raw points/s", ms=ms, bound="hbm", achieved=bytes_alg / (ms * 1e-3) / 1e9, peak=pk["hbm"],
                frac=bytes_alg / (ms * 1e-3) / 1e9 / pk["hbm"], note="includes one host read (voxel counts) per call")


def run_ours(args):
    import torch
    import torch.distributed as dist
    from pointcept_b200 import ops

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device -- the CUDA operators have no CPU fallback (use --impl reference for the CPU arm)")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1 or args.force_dist:
        os.environ.setdefault("NCCL_DEBUG", "WARN")
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29541")
        dist.init_process_group("nccl", device_id=dev, rank=rank, world_size=world)
    if args.kernel_impl is not None:
        ops.set_impl(args.kernel_impl)
    if args.fused_linear:
        from pointcept_b200.ptv3 import FusedLinear
        FusedLinear.use_fused_bias_grad = True

    log(f"rank {rank}: headline workload {args.workload}, {args.scenes_per_gpu} scenes/GPU")
    main = measure(args, args.workload, args.scenes_per_gpu, args.voxels, args.steps, args.warmup, want_profile=True, sample_clocks=True)
    log(f"rank {rank}: {main['ms_per_step']:.1f} ms/step")
    pk = peaks()
    roofs, shares = rooflines(main.get("profile", {}), main.get("profile_ms_total", 1.0), pk)

    # ---- supplementary, driver-visible lines for the other BASELINE configs (short runs; same contract: warm-up >= 3, events) ----
    supp = {}
    if not args.no_supplementary and world == 1:   # single-GPU lines (per-GPU shapes of configs 3 and 5); N > 1 runs measure scaling
        try:
            other = "spunet34" if args.workload == "ptv3_base" else "ptv3_base"
            r = measure(args, other, 8 if other == "spunet34" else 2, args.voxels, 10, 3, want_e2e=False)
            supp["config3_spunet34" if other == "spunet34" else "config4_ptv3_base"] = dict(
                workload=("SpUNet-v1m1 34 fwd+bwd+AdamW, 8 ScanNet-scale scenes per GPU (BASELINE config 3)" if other == "spunet34"
                          else "PT-v3m1 base, 2 scenes per GPU"),
                value=r["value"], unit=UNIT, ms_per_step=r["ms_per_step"], points_per_gpu=r["points_per_gpu"], steps=10, warmup=3)
            r = measure(args, "ptv3_base", 4, 300_000, 6, 3, kind="lidar", want_e2e=False)
            supp["config5_ptv3_lidar"] = dict(workload="PT-v3m1 base (in_channels 4) fwd+bwd+AdamW, 4 nuScenes-scale sweeps per GPU "
                                              "(BASELINE config 5 per-GPU shape)", value=r["value"], unit=UNIT, ms_per_step=r["ms_per_step"],
                                              points_per_gpu=r["points_per_gpu"], steps=6, warmup=3)
        except Exception as e:  # supplementary lines never take the headline down
            supp["error"] = repr(e)[:300]
        try:
            supp["grid_sample"] = measure_grid_sample(args.scenes_per_gpu, args.voxels, dev, pk)
        except Exception as e:
            supp["grid_sample"] = dict(error=repr(e)[:300])

    # ---- BASELINE.md B2: the reference's GPU stack on the same box (stock flash-attn + torch-native rulebook conv) -------------
    gref = None
    if not args.no_gpu_reference and world == 1:   # single-GPU comparator (the multi-GPU runs measure scaling, not the ratio)
        try:
            from tools import gpu_reference
            fa_ver = gpu_reference.stock_flash_attn()[1]
            r = measure(args, args.workload, args.scenes_per_gpu, args.voxels, args.gpu_reference_steps, 3, want_e2e=False,
                        reference_stack=True)
            gref = dict(value=r["value"], unit=UNIT, ms_per_step=r["ms_per_step"], steps=args.gpu_reference_steps, warmup=3,
                        what=gpu_reference.DESCRIPTION.format(fa=fa_ver), ratio_ours_over_reference=main["value"] / r["value"])
        except Exception as e:
            gref = dict(value=None, error=repr(e)[:300])

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    cpu = None
    if not args.no_cpu_baseline and world == 1:
        log("cpu_baseline: running the oracle port on the host cores (bounded subprocess)")
        try:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--impl", "reference", "--steps", "1", "--warmup", "1",
                                "--cpu-voxels", str(args.cpu_voxels)], capture_output=True, text=True, timeout=args.cpu_timeout,
                               env=dict(os.environ, RANK="0", WORLD_SIZE="1", CUDA_VISIBLE_DEVICES=""))
            js = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
            cpu = json.loads(js[-1])["cpu_baseline"] if js else dict(value=None, unit=UNIT, error=p.stderr[-300:])
        except subprocess.TimeoutExpired:
            cpu = dict(value=None, unit=UNIT, cores=host_cores(), kind="port",
                       sample=f"1 scene x {args.cpu_voxels} voxels", error=f"did not finish within {args.cpu_timeout}s")

    line = {
        "metric": METRIC, "value": main["value"], "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
        "ms_per_step": main["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "bf16", "data": "synthetic",
        "config": {"workload": ("PT-v3m1 base (configs/scannet/semseg-pt-v3m1-0-base.py) fwd+bwd+AdamW, BASELINE config 4 shape: "
                                if args.workload == "ptv3_base" else
                                "SpUNet-v1m1 34 (configs/scannet/semseg-spunet-v1m1-0-base.py) fwd+bwd+AdamW, BASELINE config 3 shape: ")
                               + f"{args.scenes_per_gpu} synthetic ScanNet-scale scenes per GPU",
                   "scenes_per_gpu": args.scenes_per_gpu, "points_per_gpu": main["points_per_gpu"], "global_points": int(main["total_points"]),
                   "params_M": main["params_M"], "patch_size": 1024, "orders": 4, "parallelism": f"dp{world}",
                   "grad_exchange": main.get("grad_exchange"),
                   "l2": "no explicit flush: one step streams several GB of activations, far beyond the 50 MB L2",
                   "kernel_impl": ops.get_impl(), "spatial_reorder": not args.no_reorder, "loss_last": main.get("loss_last"),
                   "binding": "compiled" if ops.binding() is not None else "ctypes"},
        "e2e": {"value": main.get("e2e_value"), "unit": UNIT, "h2d_bytes_per_step": main["h2d_bytes"], "d2h_bytes_per_step": 4},
        "gpu_launches": main["launches"],
        "clocks": main["clocks"],
        "roofline": roofs[0] if roofs else None,
        "rooflines": roofs,
        "kernel_time_share": shares,
        "cpu_baseline": cpu,
        "gpu_reference": gref,
        "supplementary": supp,
    }
    print(json.dumps(line))
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    a = parse()
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)
