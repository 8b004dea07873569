"""Per-shape timing of the sparse-conv kernels (run on a GPU): SIMT vs tensor-core kernels, achieved algorithmic GB/s."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointcept_b200 import ops, synth  # noqa: E402

DEV = "cuda"


def bench(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    b = synth.make_batch(2, seed=100)
    grid = b["grid_coord"]
    bid = np.repeat(np.arange(2), np.diff(b["offset"], prepend=0))
    levels = []
    g, bb = grid, bid
    for s in range(5):
        levels.append((g, bb))
        key = np.concatenate([bb[:, None], g >> 1], 1)
        u = np.unique(key, axis=0)
        bb, g = u[:, 0], u[:, 1:]
    cfgs = [(0, 32, 3), (0, 64, 3), (1, 64, 3), (2, 128, 3), (3, 256, 3), (0, 16, 5), (4, 512, 3)]
    impls = [int(x) for x in os.environ.get("IMPLS", "1,2").split(",")]
    if "ONLY" in os.environ:
        cfgs = [cfgs[int(i)] for i in os.environ["ONLY"].split(",")]
    for lvl, C, ks in cfgs:
        g, bb = levels[lvl]
        n = len(g)
        idx = torch.from_numpy(np.concatenate([bb[:, None], g], 1).astype(np.int32)).to(DEV)
        shape = (g.max(0) + 96).tolist()
        t_rb = bench(lambda: ops.rulebook_subm(idx, shape, ks), 5)
        pair = ops.rulebook_subm(idx, shape, ks)
        kv = pair.shape[0]
        valid = int((pair >= 0).sum())
        cout = 32 if ks == 5 else C
        feat = torch.randn(n, C, device=DEV).bfloat16().requires_grad_(True)
        w = (torch.randn(cout, kv, C, device=DEV) * 0.05).requires_grad_(True)
        dout = torch.randn(n, cout, device=DEV).bfloat16()
        line = f"N={n:7d} C={C:3d}->{cout:3d} kv={kv:3d} pairs/N={valid / n:5.1f} rulebook={t_rb:.3f}ms |"
        gath = valid * C * 2 + n * cout * 2 + pair.numel() * 4 + kv * C * cout * 2
        for impl in impls:
            ops.set_impl(impl)
            wb = w.detach().bfloat16().contiguous()
            tf = bench(lambda: ops._gather_gemm(feat.detach(), wb, None, pair, n, C, cout, kv, False, False))
            tb = bench(lambda: ops._gather_gemm(dout, wb, None, pair, n, cout, C, kv, True, True))
            out = ops.sparse_conv(feat, w, None, pair, pair, True)
            tall = bench(lambda: out.backward(dout, retain_graph=True))
            line += f" impl{impl}: fwd {tf:.3f}ms ({gath / tf / 1e6:.0f} GB/s) bwd_data {tb:.3f}ms dW {tall - tb:.3f}ms |"
        print(line, flush=True)
    ops.set_impl(0)


if __name__ == "__main__":
    main()
