"""Whole-path parity: PT-v3m1 on the CUDA operators vs (a) the UNMODIFIED reference model run on CPU
(tests/golden/ptv3_tiny.npz) and (b) the CPU oracle model on a fresh seeded input; SpUNet-v1m1 vs a dense
restatement built from oracle/spconv_ref.py."""
import os

import numpy as np
import pytest
import torch

from oracle import ptv3_cpu
from oracle import spunet_cpu
from oracle import fixture_dout, fixture_state_dict
from oracle import spconv_ref as osp
from pointcept_b200 import ops, synth
from pointcept_b200.ptv3 import PointTransformerV3
from pointcept_b200.spunet import SpUNetBase

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


def _tiny_model(sd):
    m = PointTransformerV3(**ptv3_cpu.TINY_CFG)
    m.load_state_dict(sd)
    for mod in m.modules():
        if hasattr(mod, "shuffle_orders"):
            mod.shuffle_orders = False
    return m.to(DEV).train()


@pytest.mark.parametrize("impl", [1, 0])
def test_ptv3_tiny_matches_reference_model(golden_dir, impl):
    g = np.load(os.path.join(golden_dir, "ptv3_tiny.npz"))
    sd = fixture_state_dict(g)
    model = _tiny_model(sd)
    data = dict(coord=torch.from_numpy(g["coord"]).to(DEV), grid_coord=torch.from_numpy(g["grid_coord"]).to(DEV),
                feat=torch.from_numpy(g["feat"]).to(DEV), offset=torch.from_numpy(g["offset"]).to(DEV))
    old = ops.get_impl()
    ops.set_impl(impl)
    try:
        out = model(data).feat
        out.backward(fixture_dout(g).to(DEV))
    finally:
        ops.set_impl(old)
    # fp32 everywhere except the attention core, which takes bf16 q/k/v and returns bf16 (reference :209,:215):
    # 2e-2 relative on the final activations after 10 blocks, 5e-2 on weight gradients.
    assert rel_l2(out.detach(), torch.from_numpy(g["out"])) < 2e-2
    grads = {k[6:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("grad::")}
    params = dict(model.named_parameters())
    for k, ref in grads.items():
        assert rel_l2(params[k].grad, ref) < 5e-2, k


def test_ptv3_tiny_vs_cpu_oracle_with_bf16_attention_emulated(golden_dir):
    """Same rounding points on both sides (bf16 at the attention boundary): tighter tolerance, fresh input."""
    g = np.load(os.path.join(golden_dir, "ptv3_tiny.npz"))
    sd = fixture_state_dict(g)
    model = _tiny_model(sd)
    b = synth.make_batch(3, seed=21, target_voxels=900)
    data = dict(coord=torch.from_numpy(b["coord"]).to(DEV), grid_coord=torch.from_numpy(b["grid_coord"]).to(DEV),
                feat=torch.from_numpy(b["feat"]).to(DEV), offset=torch.from_numpy(b["offset"]).to(DEV))
    out = model(data).feat
    ref = ptv3_cpu.forward(sd, dict(grid_coord=b["grid_coord"], feat=b["feat"], offset=b["offset"]), ptv3_cpu.TINY_CFG,
                           bn_training=True, attn_dtype=torch.bfloat16)
    assert rel_l2(out.detach(), ref.detach()) < 5e-3


def test_ptv3_tiny_backward_all_parameter_gradients_vs_cpu_oracle(golden_dir):
    """Backward at tight tolerance: every parameter gradient of the tiny PT-v3m1 against autograd through the CPU oracle with
    the same bf16 rounding points at the attention boundary (ptv3m1:209,215).  <= 1e-2 relative per parameter; a dropped
    borrowed-token gradient or a wrong offset flip in the conv backward shows up as O(1)."""
    g = np.load(os.path.join(golden_dir, "ptv3_tiny.npz"))
    sd = fixture_state_dict(g)
    model = _tiny_model(sd)
    b = synth.make_batch(3, seed=22, target_voxels=1100)     # 3 scenes: padded + borrowed patches at every level
    data = dict(coord=torch.from_numpy(b["coord"]).to(DEV), grid_coord=torch.from_numpy(b["grid_coord"]).to(DEV),
                feat=torch.from_numpy(b["feat"]).to(DEV), offset=torch.from_numpy(b["offset"]).to(DEV))
    torch.manual_seed(3)
    dout = torch.randn(len(b["feat"]), 32)
    out = model(data).feat
    out.backward(dout.to(DEV))
    sdr = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in sd.items()}
    ref = ptv3_cpu.forward(sdr, dict(grid_coord=b["grid_coord"], feat=b["feat"], offset=b["offset"]), ptv3_cpu.TINY_CFG,
                           bn_training=True, attn_dtype=torch.bfloat16)
    ref.backward(dout)
    assert rel_l2(out.detach(), ref.detach()) < 5e-3
    # Parameters whose gradient is zero in exact arithmetic (a bias in front of BatchNorm, the key bias of the attention: softmax
    # is shift invariant) hold pure rounding noise on both sides; they are checked for smallness instead of relative error.
    gmax = max(float(v.grad.norm()) for k, v in sdr.items() if v.grad is not None)
    worst, noise = {}, {}
    for k, p in model.named_parameters():
        assert p.grad is not None, k
        rn = float(sdr[k].grad.norm())
        if rn < 1e-5 * gmax:
            noise[k] = float(p.grad.norm()) / gmax
        else:
            worst[k] = rel_l2(p.grad, sdr[k].grad)
    print("largest relative gradient errors:", sorted(worst.items(), key=lambda kv: -kv[1])[:6])
    print("parameters with (numerically) zero reference gradient:", len(noise), "max |g|/gmax", max(noise.values()) if noise else 0.0)
    assert len(worst) > 100
    # the oracle rounds q/k/v and the attention output to bf16 like the operator, but not P and dS inside the kernel (8 mantissa
    # bits before the PV / dV / dK / dQ products): a few per cent on the gradients closest to the attention; 5e-2 per parameter
    bad = {k: v for k, v in worst.items() if v >= 5e-2}
    assert not bad, bad
    assert all(v < 1e-4 for v in noise.values()), noise


@pytest.mark.parametrize("amp", [torch.bfloat16, torch.float16])
def test_ptv3_tiny_autocast_runs_tensor_core_convs_and_matches_oracle(golden_dir, amp):
    """Autocast step (stock configs run fp16 AMP + GradScaler: configs/_base_/default_runtime.py:19, engines/train.py:203,351):
    features reach the sparse convs in half precision, so the tensor-core conv kernels are on the path (B2PC_IMPL=2 semantics are
    asserted through the launch counter of the tensor-core entry points)."""
    g = np.load(os.path.join(golden_dir, "ptv3_tiny.npz"))
    sd = fixture_state_dict(g)
    model = _tiny_model(sd)
    data = dict(coord=torch.from_numpy(g["coord"]).to(DEV), grid_coord=torch.from_numpy(g["grid_coord"]).to(DEV),
                feat=torch.from_numpy(g["feat"]).to(DEV), offset=torch.from_numpy(g["offset"]).to(DEV))
    opt = torch.optim.SGD(model.parameters(), lr=0.0)
    scaler = torch.amp.GradScaler("cuda", enabled=amp == torch.float16, init_scale=1024.0)
    old = ops.get_impl()
    ops.set_impl(2)          # tensor-core kernels or an error (the stem pads 6 -> 16 channels to get there)
    try:
        for attempt in range(8):     # GradScaler semantics (engines/train.py:351-360): a step whose scaled gradients overflow fp16
            opt.zero_grad(set_to_none=True)   # is skipped and the scale halves; the first step that fits is the one compared
            with torch.autocast("cuda", dtype=amp):
                out = model(dict(data)).feat
            loss = (out.float() * fixture_dout(g).to(DEV)).sum()
            scale_before = scaler.get_scale()
            scaler.scale(loss).backward()
            scaler.unscale_(opt)
            scaler.step(opt)
            scaler.update()
            if scaler.get_scale() >= scale_before:
                break
    finally:
        ops.set_impl(old)
    assert scaler.get_scale() >= scale_before, "every attempt overflowed"
    print("GradScaler settled at", scaler.get_scale(), "after", attempt + 1, "attempt(s)")
    # half-precision rounding at every Linear / conv boundary (8 / 11 mantissa bits) vs the reference model's fp32 run, 10 blocks
    # deep: 5e-2 on the output, 2e-1 on weight gradients for bf16; fp16 (the stock AMP dtype) 1e-2 / 5e-2
    e_out = rel_l2(out.detach().float(), torch.from_numpy(g["out"]))
    grads = {k[6:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("grad::")}
    params = dict(model.named_parameters())
    e_g = {k: rel_l2(params[k].grad, ref) for k, ref in grads.items()}
    print("autocast", amp, "out", e_out, "grads", e_g)
    assert all(torch.isfinite(params[k].grad).all() for k in grads)
    assert e_out < (5e-2 if amp == torch.bfloat16 else 1e-2)
    assert max(e_g.values()) < (2e-1 if amp == torch.bfloat16 else 5e-2), e_g


def test_spatial_reorder_is_permutation_equivalent(golden_dir):
    g = np.load(os.path.join(golden_dir, "ptv3_tiny.npz"))
    sd = fixture_state_dict(g)
    data = dict(coord=torch.from_numpy(g["coord"]).to(DEV), grid_coord=torch.from_numpy(g["grid_coord"]).to(DEV),
                feat=torch.from_numpy(g["feat"]).to(DEV), offset=torch.from_numpy(g["offset"]).to(DEV))
    outs = []
    for flag in (False, True):
        model = _tiny_model(sd)
        model.spatial_reorder = flag
        outs.append(model(dict(data)).feat.detach())
    # same math, different summation order inside BatchNorm statistics and bf16 attention tiles
    assert rel_l2(outs[1], outs[0]) < 5e-3


def test_ptv3_serialization_tables_bit_exact_through_the_model():
    from oracle import serialization as oser
    from pointcept_b200.structure import Point
    b = synth.make_batch(2, seed=5, target_voxels=30_000)
    p = Point(grid_coord=torch.from_numpy(b["grid_coord"]).to(DEV), offset=torch.from_numpy(b["offset"]).to(DEV),
              feat=torch.from_numpy(b["feat"]).to(DEV))
    p.serialization(order=list(oser.ORDERS), shuffle_orders=False)
    bid = np.repeat(np.arange(2), np.diff(b["offset"], prepend=0))
    code, order, inverse, depth = oser.serialize(b["grid_coord"], bid, oser.ORDERS)
    assert p.serialized_depth == depth
    assert np.array_equal(p.serialized_code.cpu().numpy(), code)
    assert np.array_equal(p.serialized_order.cpu().numpy(), order)
    assert np.array_equal(p.serialized_inverse.cpu().numpy(), inverse)


def test_spunet_forward_backward_vs_oracle_convs():
    """SpUNet-v1m1 (small widths) fp32: every sparse conv replaced, on the oracle side, by oracle/spconv_ref.py."""
    torch.manual_seed(0)
    model = SpUNetBase(6, 13, base_channels=16, channels=(16, 32, 48, 64, 64, 48, 32, 32), layers=(1, 1, 1, 1, 1, 1, 1, 1)).to(DEV).train()
    b = synth.make_batch(2, seed=8, target_voxels=4000)
    data = dict(grid_coord=torch.from_numpy(b["grid_coord"]).to(DEV), feat=torch.from_numpy(b["feat"]).to(DEV),
                offset=torch.from_numpy(b["offset"]).to(DEV))
    out = model(data)
    assert out.shape == (len(b["feat"]), 13)
    out.square().mean().backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters())
    # oracle replay of the same network on CPU
    ref = spunet_cpu.forward({k: v.detach().cpu() for k, v in model.state_dict().items()}, b, model)
    assert rel_l2(out.detach(), ref) < 1e-3


# ---- BASELINE.json configs 3 and 5 at full scene size: size-independent properties -------------------------------------------
def test_spunet34_scannet_scale_forward_backward_properties():
    """config 3 shape (SpUNet-v1m1 stock widths) on 2 x 120k-voxel scenes under fp16 autocast (the reference's AMP dtype)."""
    torch.manual_seed(0)
    model = SpUNetBase(6, 20).to(DEV).train()
    b = synth.make_batch(2, seed=31)
    data = dict(grid_coord=torch.from_numpy(b["grid_coord"]).to(DEV), feat=torch.from_numpy(b["feat"]).to(DEV),
                offset=torch.from_numpy(b["offset"]).to(DEV))
    with torch.autocast("cuda", dtype=torch.float16):
        out = model(data)
    assert out.shape == (len(b["feat"]), 20) and torch.isfinite(out).all()
    torch.nn.functional.cross_entropy(out.float(), torch.from_numpy(b["segment"]).to(DEV)).backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters())
    # rulebook properties at this size: strided tables are mutually inverse, every input lands in exactly one output
    from pointcept_b200 import ops
    bid = np.repeat(np.arange(2), np.diff(b["offset"], prepend=0))
    idx = torch.from_numpy(np.concatenate([bid[:, None], b["grid_coord"]], 1).astype(np.int32)).to(DEV)
    shape = (b["grid_coord"].max(0) + 96).tolist()
    out_idx, oshape, pf, pb = ops.rulebook_strided(idx, shape, 2, 2)
    n, m = idx.shape[0], out_idx.shape[0]
    assert int((pb >= 0).sum()) == n and int((pf >= 0).sum()) == n
    k, i = torch.nonzero(pb >= 0, as_tuple=True)
    assert torch.equal(pf[k, pb[k, i].long()].long(), i)
    keys = ((out_idx[:, 0].long() * oshape[0] + out_idx[:, 1]) * oshape[1] + out_idx[:, 2]) * oshape[2] + out_idx[:, 3]
    assert bool((keys[1:] > keys[:-1]).all())                    # ascending, distinct
    assert torch.equal(out_idx[pb.max(0).values.long(), 1:], idx[:, 1:] >> 1)


def test_ptv3_nuscenes_scale_forward_backward_properties():
    """config 5 shape: PT-v3m1 base widths, in_channels 4, one ~300k-voxel LiDAR-like sweep (extent > 2^11 -> depth 12)."""
    from pointcept_b200.ptv3 import PTv3Segmentor, ptv3_base_config
    from pointcept_b200.structure import Point
    torch.manual_seed(0)
    b = synth.make_batch(1, seed=41, kind="lidar", num_classes=16)
    cfg = dict(ptv3_base_config(), in_channels=4)
    model = PTv3Segmentor(num_classes=16, backbone_out_channels=64, **cfg).to(DEV).train()
    data = {k: torch.from_numpy(v).to(DEV) for k, v in b.items()}
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = model(data)
    assert out["seg_logits"].shape == (len(b["feat"]), 16) and torch.isfinite(out["seg_logits"]).all()
    out["loss"].backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters())
    p = Point(grid_coord=data["grid_coord"], offset=data["offset"], feat=data["feat"])
    p.serialization(order=["z", "z-trans", "hilbert", "hilbert-trans"])
    assert p.serialized_depth == 12
    sorted_codes = torch.gather(p.serialized_code, 1, p.serialized_order)
    assert bool((sorted_codes[:, 1:] > sorted_codes[:, :-1]).all())          # strictly sorted: voxels are unique
    n = sorted_codes.shape[1]
    assert torch.equal(torch.gather(p.serialized_inverse, 1, p.serialized_order), torch.arange(n, device=DEV).expand(4, n))


def _both_bindings(fn):
    res = {}
    for name in ("ctypes", "compiled"):
        ops.set_binding(name)
        try:
            torch.manual_seed(0)
            res[name] = fn()
        finally:
            ops.set_binding("auto")
    return res["ctypes"], res["compiled"]


def test_compiled_binding_matches_ctypes_binding(golden_dir):
    """The pybind/C++ autograd binding and the ctypes/Python binding drive the same C ABI.  Deterministic operators must agree
    exactly; operators that reduce with fp32 red.add (attention dQ, offset-split conv) and the whole model agree to the run-to-run
    noise of those reductions under bf16 (measured 6e-3 on the tiny model's output between two runs of the SAME binding)."""
    from pointcept_b200 import _lib
    from pointcept_b200.ptv3 import _SerializedGather
    if _lib.torch_binding() is None:
        pytest.skip("compiled binding not built")
    n, c = 3000, 64

    def ln():
        x = torch.randn(n, c, device=DEV, requires_grad=True)
        w = torch.randn(c, device=DEV, requires_grad=True)
        b = torch.randn(c, device=DEV, requires_grad=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = ops.layer_norm(x, w, b, 1e-5, True)
        y.float().square().sum().backward()
        return y.detach(), x.grad, w.grad, b.grad

    def lin():
        x = torch.randn(n, c, device=DEV, requires_grad=True)
        w = torch.randn(96, c, device=DEV, requires_grad=True)
        b = torch.randn(96, device=DEV, requires_grad=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = ops.linear(x, w, b)
        y.float().square().sum().backward()
        return y.detach(), x.grad, w.grad, b.grad

    def pool():
        lens = torch.full((n // 4,), 4, device=DEV)
        start = torch.arange(0, n, 4, device=DEV)
        order = torch.randperm(n, device=DEV)
        x = torch.randn(n, c, device=DEV).bfloat16().requires_grad_(True)
        y = ops.segment_max(x, order, start, lens)
        y.float().square().sum().backward()
        return y.detach(), x.grad

    for fn in (ln, lin, pool):
        a, b_ = _both_bindings(fn)
        for i, (u, v) in enumerate(zip(a, b_)):
            if fn is lin and i == 2:
                # weight gradient: the compiled node takes it from the GEMM in fp32, the ctypes node rounds it to bf16 like autocast
                assert rel_l2(v, u) < 4e-3
            else:
                assert torch.equal(u, v), fn.__name__

    def attn():
        qkv = torch.randn(2048 + 300, 3, 2, 16, device=DEV).bfloat16().requires_grad_(True)
        cu = torch.tensor([0, 1024, 2048, 2348], dtype=torch.int32, device=DEV)
        y = ops.patch_attention(qkv, cu, 1024, 0.25)
        y.float().square().sum().backward()
        return y.detach().float(), qkv.grad.float()

    a, b_ = _both_bindings(attn)
    assert torch.equal(a[0], b_[0]) and rel_l2(b_[1], a[1]) < 1e-2

    g = np.load(os.path.join(golden_dir, "ptv3_tiny.npz"))
    sd = fixture_state_dict(g)
    data = dict(coord=torch.from_numpy(g["coord"]).to(DEV), grid_coord=torch.from_numpy(g["grid_coord"]).to(DEV),
                feat=torch.from_numpy(g["feat"]).to(DEV), offset=torch.from_numpy(g["offset"]).to(DEV))

    def model():
        m = _tiny_model(sd)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = m(dict(data)).feat
        out.float().square().mean().backward()
        return out.detach().float(), m.embedding.stem.conv.weight.grad.clone()

    a, b_ = _both_bindings(model)
    assert rel_l2(b_[0], a[0]) < 3e-2 and rel_l2(b_[1], a[1]) < 1e-1


def test_drop_path_add_semantics():
    torch.manual_seed(0)
    n, c, p = 20000, 64, 0.3
    s = torch.randn(n, c, device=DEV)
    x = torch.randn(n, c, device=DEV).bfloat16().requires_grad_(True)
    out = ops.drop_path_add(s, x, p, True)
    delta = out - s
    dropped = (delta.abs().sum(1) == 0)
    kept = ~dropped
    assert abs(float(dropped.float().mean()) - p) < 0.02
    assert rel_l2(delta[kept], x.detach().float()[kept] / (1 - p)) < 1e-6
    out.sum().backward()
    assert torch.equal(x.grad[dropped].float(), torch.zeros_like(x.grad[dropped].float()))
    assert rel_l2(x.grad[kept].float(), torch.full_like(x.grad[kept].float(), 1 / (1 - p))) < 5e-3
    assert torch.equal(ops.drop_path_add(s, x.detach(), p, False), s + x.detach())


def test_flat_grad_reducer_nccl_packs_bit_exact_and_feeds_fused_adamw(golden_dir):
    """pointcept_b200/reducer.py on the GPU (NCCL, world size 1 inside this process: the average over one rank is the identity):
    the one-launch pack (b2pc_multi_cast, fp32 destination) copies every gradient bit-exactly into the arrival-order flat buffer,
    the early group is exchanged from the autograd hook, p.grad become slices of the buffer and FusedAdamW steps from them exactly
    as it does from the loose gradients.  The N > 1 protocol itself is covered under gloo (tests/test_host_logic.py)."""
    import torch.distributed as dist
    from pointcept_b200.optim import FusedAdamW
    from pointcept_b200.reducer import FlatGradReducer
    g = np.load(os.path.join(golden_dir, "ptv3_tiny.npz"))
    sd = fixture_state_dict(g)
    data = dict(coord=torch.from_numpy(g["coord"]).to(DEV), grid_coord=torch.from_numpy(g["grid_coord"]).to(DEV),
                feat=torch.from_numpy(g["feat"]).to(DEV), offset=torch.from_numpy(g["offset"]).to(DEV))
    dout = fixture_dout(g).to(DEV)
    own_pg = not dist.is_initialized()
    if own_pg:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29547")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", torch.cuda.current_device()))
    try:
        model = _tiny_model(sd)
        twin = _tiny_model(sd)                       # same parameters, takes the gradients loose
        red = FlatGradReducer(model.parameters(), early_fraction=0.5)
        opt, opt_twin = FusedAdamW(model.parameters(), lr=1e-3, weight_decay=0.05), FusedAdamW(twin.parameters(), lr=1e-3, weight_decay=0.05)
        for step in range(3):
            opt.zero_grad(set_to_none=True)
            (model(dict(data)).feat.float() * dout).sum().backward()
            loose = [p.grad for p in model.parameters()]          # the tensors autograd produced (kept alive here)
            red.finish()
            for p, gl in zip(model.parameters(), loose):
                assert p.grad.data_ptr() != gl.data_ptr() and torch.equal(p.grad, gl)     # bit-exact copy into the flat buffer
                assert red.flat.data_ptr() <= p.grad.data_ptr() < red.flat.data_ptr() + 4 * red.flat.numel()
            # the twin takes the same gradients loose: both optimizers must produce the same parameters, bit for bit
            for q, gl in zip(twin.parameters(), loose):
                q.grad = gl.clone()
            opt.step()
            opt_twin.step()
            for p, q in zip(model.parameters(), twin.parameters()):
                assert torch.equal(p, q)
        assert red.stats == dict(steps=3, early_steps=2, late_steps=0) and 0 < red.n_early < len(red.params)
        assert 0.5 * red.flat.numel() <= red.early_end < red.flat.numel()
        red.remove()
    finally:
        if own_pg:
            dist.destroy_process_group()
