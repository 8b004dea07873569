"""Host-side logic that needs no GPU: synthetic scenes, the reference-compatible module tree, the drop-in
import surface, and the N>1 sharding / reduction logic of bench.py under gloo (world_size 2)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from pointcept_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_synthetic_scene_is_seeded_and_calibrated():
    c1, g1 = synth.indoor_scene(3, target_voxels=20_000)
    c2, g2 = synth.indoor_scene(3, target_voxels=20_000)
    assert np.array_equal(g1, g2) and len(g1) == 20_000
    assert len(np.unique(g1, axis=0)) == len(g1)          # voxels are unique
    assert g1.min() == 0
    nb = synth.neighbour_stats(g1)
    assert 8.0 < nb < 14.0, nb                              # ~11 active 3^3 neighbours (SURVEY 8(d))
    b = synth.make_batch(3, seed=1, target_voxels=5000)
    assert b["offset"].tolist() == [5000, 10000, 15000] and b["feat"].shape == (15000, 6)


def test_dropin_modules_register_under_reference_import_names():
    import pointcept_b200
    pointcept_b200.install(flash_attn=True)
    import flash_attn
    import spconv.pytorch as spconv
    assert spconv.modules.is_spconv_module(spconv.SubMConv3d(4, 8, 3))
    assert not spconv.modules.is_spconv_module(torch.nn.Linear(2, 2))
    m = spconv.SparseConv3d(4, 8, kernel_size=2, stride=2, bias=False, indice_key="spconv1")
    assert tuple(m.weight.shape) == (8, 2, 2, 2, 4) and m.bias is None
    assert tuple(spconv.SubMConv3d(6, 32, kernel_size=5, padding=1, bias=False, indice_key="stem").weight.shape) == (32, 5, 5, 5, 6)
    assert callable(flash_attn.flash_attn_varlen_qkvpacked_func)
    x = spconv.SparseConvTensor(torch.zeros(3, 4), torch.zeros(3, 4, dtype=torch.int32), [8, 8, 8], 1)
    y = x.replace_feature(torch.ones(3, 2))
    assert y.indice_dict is x.indice_dict and y.features.shape == (3, 2)
    with pytest.raises(NotImplementedError):
        flash_attn.flash_attn_varlen_qkvpacked_func(torch.zeros(4, 3, 1, 16), torch.tensor([0, 4]), 4, dropout_p=0.1)
    for k in [k for k in sys.modules if k == "spconv" or k.startswith("spconv.") or k.startswith("flash_attn")]:
        del sys.modules[k]


def test_unmodified_reference_models_build_on_the_dropins_with_identical_state_dict(golden_dir):
    """The reference's own PT-v3m1 / SpUNet-v1m1 files, imported unmodified on top of our spconv / flash_attn modules
    (tests/golden/reference_dropin.npz, tools/gen_golden.py::gen_dropin_abi), produce the same parameter names and shapes as the
    mirrors (checkpoint ABI), and the reference's Point.sparsify() builds the same SparseConvTensor as the mirror's."""
    from pointcept_b200.ptv3 import PointTransformerV3, ptv3_base_config
    from pointcept_b200.spunet import SpUNetBase
    from pointcept_b200.structure import Point
    ref = json.loads(str(np.load(os.path.join(golden_dir, "reference_dropin.npz"))["json"]))
    a = [[k, list(v.shape)] for k, v in PointTransformerV3(**ptv3_base_config()).state_dict().items()]
    assert a == ref["ptv3_base"] and len(a) > 400
    a = [[k, list(v.shape)] for k, v in SpUNetBase(6, 20).state_dict().items()]
    assert a == ref["spunet_6_20"] and len(a) > 300
    import pointcept_b200
    pointcept_b200.install(flash_attn=True)
    import spconv.pytorch as spconv
    sp = ref["sparsify"]
    pt = Point(grid_coord=torch.tensor(sp["grid_coord"]), feat=torch.randn(len(sp["grid_coord"]), 6), offset=torch.tensor(sp["offset"]))
    pt.sparsify()
    x = pt.sparse_conv_feat
    assert isinstance(x, spconv.SparseConvTensor) and x.indices.dtype == torch.int32 and x.batch_size == sp["batch_size"]
    assert x.indices.tolist() == sp["indices"] and [int(v) for v in x.spatial_shape] == sp["spatial_shape"]
    assert spconv.modules.is_spconv_module(spconv.SubMConv3d(6, 8, 3, indice_key="k"))
    for k in [k for k in sys.modules if k.split(".")[0] in ("spconv", "flash_attn")]:
        del sys.modules[k]


def test_serialized_gather_backward_without_sort_matches_plain_indexing():
    """The structured backward of the [order] / [inverse] gathers of SerializedAttention (ptv3m1:188,216): pure torch, runs on CPU."""
    from oracle import padding as opad
    from pointcept_b200.ptv3 import _SerializedGather, _SerializedScatterBack
    torch.manual_seed(0)
    for offset, K in (([5, 17, 20], 4), ([3, 11], 4), ([1024, 2049, 3000], 1024), ([10], 16)):
        pad, unpad, _ = opad.padding_and_inverse(offset, K)
        n = offset[-1]
        order = torch.randperm(n)
        inverse = torch.empty_like(order)
        inverse[order] = torch.arange(n)
        pad, unpad = torch.from_numpy(pad), torch.from_numpy(unpad)
        order_pad, primary = order[pad], unpad[inverse]
        slots, op = [], 0
        for a, b in zip([0] + offset[:-1], offset):
            cnt = b - a
            npad = ((cnt + K - 1) // K * K) if cnt > K else cnt
            if npad != cnt:
                slots.append(torch.arange(op + npad - (K - cnt % K), op + npad))
            op += npad
        dup = torch.cat(slots) if slots else torch.zeros(0, dtype=torch.long)
        assert torch.equal(order_pad[primary], torch.arange(n))          # every point has one primary slot
        x = torch.randn(n, 3, requires_grad=True)
        x2 = x.detach().clone().requires_grad_(True)
        g = torch.randn(len(pad), 3)
        _SerializedGather.apply(x, order_pad, primary, dup, order_pad[dup]).backward(g)
        x2[order_pad].backward(g)
        assert torch.allclose(x.grad, x2.grad)
        y = torch.randn(len(pad), 3, requires_grad=True)
        y2 = y.detach().clone().requires_grad_(True)
        g2 = torch.randn(n, 3)
        _SerializedScatterBack.apply(y, primary).backward(g2)
        y2[primary].backward(g2)
        assert torch.allclose(y.grad, y2.grad)


def _gloo_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    # the reductions bench.py performs: total points (SUM) and step time (MAX over ranks)
    hb = synth.make_batch(2, seed=100 + rank, target_voxels=1500 + 100 * rank)
    pts = torch.tensor([float(hb["offset"][-1])], dtype=torch.float64)
    dist.all_reduce(pts, op=dist.ReduceOp.SUM)
    ms = torch.tensor([10.0 + 5 * rank], dtype=torch.float64)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    # DDP gradient averaging on a parameter set shaped like ours (plain nn.Parameters, all used every step)
    torch.manual_seed(0)
    lin = torch.nn.Linear(8, 4)
    ddp = torch.nn.parallel.DistributedDataParallel(lin, broadcast_buffers=False)
    x = torch.full((3, 8), float(rank + 1))
    ddp(x).sum().backward()
    if rank == 0:
        json.dump(dict(points=pts.item(), ms=ms.item(), grad=lin.weight.grad[0, 0].item()), open(out, "w"))
    dist.destroy_process_group()


def test_two_rank_gloo_sharding_and_reductions(tmp_path):
    import torch.multiprocessing as mp
    out = str(tmp_path / "r.json")
    mp.spawn(_gloo_worker, args=(2, 29611, out), nprocs=2, join=True)
    r = json.load(open(out))
    assert r["points"] == 2 * 1500 + 2 * 1600       # different scenes per rank, whole scenes only
    assert r["ms"] == 15.0                           # max over ranks
    assert abs(r["grad"] - 3 * (1 + 2) / 2) < 1e-6   # DDP averages gradients


def _cpu_pack(name, grads, offs, flat):
    """test-only packer (the product packs with one b2pc_multi_cast launch on the GPU)"""
    for g, o in zip(grads, offs):
        flat[o:o + g.numel()].copy_(g.reshape(-1))


def _reducer_worker(rank, world, port, out):
    import torch.distributed as dist
    from pointcept_b200.reducer import FlatGradReducer
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(rank)          # ranks start from DIFFERENT parameters: the reducer broadcasts rank 0's, like DDP
    net = torch.nn.Sequential(torch.nn.Linear(6, 16), torch.nn.GELU(), torch.nn.Linear(16, 16), torch.nn.LayerNorm(16),
                              torch.nn.Linear(16, 5, bias=False), torch.nn.Linear(5, 3))
    red = FlatGradReducer(net.parameters(), early_fraction=0.5, pack=_cpu_pack)
    import copy
    twin = copy.deepcopy(net)        # no reducer on it: the rank-local gradients the exchange must average
    ref = [p.detach().clone() for p in net.parameters()]
    gathered = [torch.zeros_like(ref[0]) for _ in range(world)]
    dist.all_gather(gathered, ref[0])
    same_start = all(torch.equal(g, gathered[0]) for g in gathered)
    worst, early = 0.0, []
    for step in range(5):
        set_none = step != 2
        if step == 4 and rank == 1:      # this rank's trigger never fires: it must still issue the same collectives (late), no hang
            red._trigger_handle.remove()
        for p in net.parameters():
            if set_none:
                p.grad = None
            elif p.grad is not None:
                p.grad.zero_()
        torch.manual_seed(100 * step + rank)
        x = torch.randn(7 + rank, 6)      # ranks hold different batches
        net(x).square().mean().backward()
        local = torch.autograd.grad(twin(x).square().mean(), list(twin.parameters()))
        red.finish()
        early.append(red.stats["early_steps"])
        for p, g in zip(net.parameters(), local):
            want = g.clone()
            dist.all_reduce(want)
            want /= world
            worst = max(worst, float((p.grad - want).abs().max()))
            assert p.grad.data_ptr() >= red.flat.data_ptr() and p.grad.data_ptr() < red.flat.data_ptr() + 4 * red.flat.numel()
    if rank == 0:
        json.dump(dict(worst=worst, early=early, same_start=same_start, n_early=red.n_early, order=red.order, stats=red.stats), open(out, "w"))
    else:
        assert red.stats == dict(steps=5, early_steps=3, late_steps=1)
    dist.destroy_process_group()


def test_flat_grad_reducer_two_ranks_gloo(tmp_path):
    """pointcept_b200/reducer.py (the a12 exchange): rank average of every gradient, arrival-order layout agreed across ranks,
    early group reduced from the autograd hook, both zero_grad flavours."""
    import torch.multiprocessing as mp
    out = str(tmp_path / "r.json")
    mp.spawn(_reducer_worker, args=(2, 29613, out), nprocs=2, join=True)
    r = json.load(open(out))
    assert r["same_start"]
    assert r["worst"] < 1e-6
    assert r["early"] == [0, 1, 2, 3, 4]              # first step lays the buffer out; every later step overlaps the early group
    assert r["stats"] == dict(steps=5, early_steps=4, late_steps=0)   # (rank 1 ran its last step late: asserted in the worker)
    assert 0 < r["n_early"] < 9
    assert r["order"][0] in (7, 8)                    # the last layer's gradients arrive first


def test_flat_grad_reducer_single_rank_edge_cases():
    """world size 1 (gloo, in-process): no early group when early_fraction = 0, loud errors for an unused parameter, hooks removed."""
    import torch.distributed as dist
    from pointcept_b200.reducer import FlatGradReducer
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29619")
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        torch.manual_seed(0)
        net = torch.nn.Sequential(torch.nn.Linear(4, 8), torch.nn.ReLU(), torch.nn.Linear(8, 2))
        red = FlatGradReducer(net.parameters(), early_fraction=0.0, pack=_cpu_pack)
        for _ in range(3):
            for p in net.parameters():
                p.grad = None
            x = torch.randn(5, 4)
            net(x).sum().backward()
            want = [p.grad.clone() for p in net.parameters()]
            red.finish()
            assert all(torch.equal(p.grad, w) for p, w in zip(net.parameters(), want))
        assert red.stats == dict(steps=3, early_steps=0, late_steps=0) and red.n_early == 0
        assert red.flat.numel() == sum((p.numel() + 3) // 4 * 4 for p in net.parameters())      # 16-byte aligned slices
        red.enabled = False            # gradient accumulation micro-steps: the reducer stays out of the way
        net(torch.randn(5, 4)).sum().backward()
        red.finish()
        assert red.stats["steps"] == 3
        red.remove()
        # a parameter that takes no part in the loss: refused on the first step, like DDP(find_unused_parameters=False)
        unused = torch.nn.Linear(3, 3)
        red2 = FlatGradReducer(list(net.parameters()) + list(unused.parameters()), pack=_cpu_pack)
        for p in net.parameters():
            p.grad = None
        net(torch.randn(5, 4)).sum().backward()
        with pytest.raises(RuntimeError, match="received no gradient"):
            red2.finish()
        red2.remove()
        with pytest.raises(RuntimeError, match="GPU only"):                 # the product packer has no CPU path
            red3 = FlatGradReducer(net.parameters())
            for p in net.parameters():
                p.grad = None
            net(torch.randn(5, 4)).sum().backward()
            red3.finish()
        red3.remove()
    finally:
        dist.destroy_process_group()


def test_bench_reference_arm_is_silent_on_other_ranks():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1"],
                       capture_output=True, text=True, timeout=120, env=env)
    assert p.returncode == 0 and p.stdout.strip() == ""


def test_bench_reference_arm_prints_one_json_line():
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1",
                        "--cpu-voxels", "2500"], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "points/s" and d["value"] > 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0


def test_non_flash_rpe_attention_branch_matches_reference_fixture(golden_dir):
    """SerializedAttention(enable_flash=False, enable_rpe=True) of the mirror (the reference's eager branch, ptv3m1:29-48,173-206)
    against the reference module itself (tests/golden/attention_rpe.npz, tools/gen_golden.py): output, input gradient and the
    gradient of the RPE table, loaded through the reference's state_dict.  Pure torch: runs on CPU."""
    from pointcept_b200.ptv3 import SerializedAttention
    from pointcept_b200.structure import Point
    g = np.load(os.path.join(golden_dir, "attention_rpe.npz"))
    attn = SerializedAttention(channels=32, num_heads=2, patch_size=64, enable_rpe=True, enable_flash=False, upcast_attention=True,
                               upcast_softmax=True, order_index=1)
    attn.load_state_dict({k[4:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd::")})
    feat = torch.from_numpy(g["feat"]).requires_grad_(True)
    offset = torch.from_numpy(g["offset"])
    pt = Point(offset=offset, offset_host=[int(v) for v in g["offset"]], grid_coord=torch.from_numpy(g["grid_coord"]), feat=feat,
               serialized_order=torch.from_numpy(g["order"]), serialized_inverse=torch.from_numpy(g["inverse"]),
               pad=torch.from_numpy(g["pad"]), unpad=torch.from_numpy(g["unpad"]), cu_seqlens_key=torch.from_numpy(g["cu"]))
    out = attn(pt).feat
    assert attn.patch_size == int(g["patch_size"]) == 48          # shrunk to the smallest scene
    out.backward(torch.from_numpy(g["dout"]))
    assert torch.allclose(out.detach(), torch.from_numpy(g["out"]), rtol=1e-5, atol=1e-6)
    assert torch.allclose(feat.grad, torch.from_numpy(g["dfeat"]), rtol=1e-4, atol=1e-6)
    assert torch.allclose(attn.rpe.rpe_table.grad, torch.from_numpy(g["d_rpe_table"]), rtol=1e-4, atol=1e-6)


def collate_inputs():
    """the seeded inputs of the collate_fn comparison (tools/gen_golden.py::gen_collate runs the reference on the same ones)"""
    g = torch.Generator().manual_seed(0)

    def sample(n, with_offset=True):
        d = dict(coord=torch.randn(n, 3, generator=g), grid_coord=torch.randint(0, 50, (n, 3), generator=g),
                 segment=torch.randint(0, 20, (n,), generator=g), name="scene%d" % n)
        if with_offset:
            d["offset"] = torch.tensor([n])
        return d

    batch = [sample(5), sample(9), sample(1)]
    tensors = [torch.randn(4, 2, generator=g), torch.randn(3, 2, generator=g)]
    return dict(batch=batch, tensors=tensors, no_offset=[sample(5, False), sample(2, False)])


def test_collate_fn_matches_the_reference_function(golden_dir):
    """pointcept_b200.datasets.collate_fn vs the reference's own collate_fn (pointcept/datasets/utils.py:19-73) on CPU tensors: dicts with
    per-sample offsets (what Collect emits), bare tensors, tuples of tensors (offset appended), lists of numbers, strings.  The
    reference's results are stored in tests/golden/collate_fn.pt (tools/gen_golden.py::gen_collate)."""
    from pointcept_b200 import datasets
    ref = torch.load(os.path.join(golden_dir, "collate_fn.pt"), weights_only=True)
    inp = collate_inputs()

    def same(a, b):
        if isinstance(a, torch.Tensor):
            assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a, b)
        elif isinstance(a, dict):
            assert a.keys() == b.keys()
            for k in a:
                same(a[k], b[k])
        elif isinstance(a, (list, tuple)):
            assert len(a) == len(b)
            for x, y in zip(a, b):
                same(x, y)
        else:
            assert a == b

    batch = inp["batch"]
    same(ref["batch"], datasets.collate_fn([dict(d) for d in batch]))
    # a fragment list: per-sample offsets that already hold several scenes (test-time fragments are collated twice, test.py:170-176)
    same(ref["two"], datasets.collate_fn([dict(d) for d in ref["two_in"]]))
    same(ref["tensors"], datasets.collate_fn(list(inp["tensors"])))
    # tuples of per-point tensors: the reference's Sequence branch (utils.py:35-40) appends to its samples, so it only serves
    # append-able non-list sequences; here tuples give the same result it describes: columns + cumulative int32 offset
    cols = datasets.collate_fn([(torch.ones(4, 3), torch.arange(4)), (torch.zeros(2, 3), torch.arange(2))])
    assert [tuple(c.shape) for c in cols] == [(6, 3), (6,), (2,)] and cols[2].tolist() == [4, 6] and cols[2].dtype == torch.int32
    same(ref["numbers"], datasets.collate_fn([[1, 2], [3]]))
    same(ref["strings"], datasets.collate_fn(["a", "b"]))
    # extension, documented: a dict without any offset key gets one from its coord lengths (the reference's datasets add it in Collect)
    out = datasets.collate_fn(inp["no_offset"])
    assert out["offset"].tolist() == [5, 7]
