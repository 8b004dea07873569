"""Parity of the CUDA path (through the C ABI) against the CPU oracle and the reference-generated fixtures.
Integer work is bit-exact; floating point tolerances are stated at each assert."""
import os

import numpy as np
import pytest
import torch

from oracle import attention as oattn
from oracle import padding as opad
from oracle import serialization as oser
from oracle import spconv_ref as osp
from pointcept_b200 import ops, synth

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


# ---- serialization ---------------------------------------------------------------------------------
def test_encode_bit_exact_vs_reference_fixtures(golden_dir):
    g = np.load(os.path.join(golden_dir, "serialization.npz"))
    for name in ("d3", "d9", "d10", "d12", "d16"):
        depth = int(g[f"{name}_depth"])
        code = ops.serialize_encode(torch.from_numpy(g[f"{name}_grid"]).to(DEV), torch.from_numpy(g[f"{name}_batch"]).to(DEV),
                                    depth, list(oser.ORDERS)).cpu().numpy()
        for i, order in enumerate(oser.ORDERS):
            assert np.array_equal(code[i], g[f"{name}_{order}"]), (name, order)


def test_encode_bit_exact_vs_oracle_random_and_subset_of_orders():
    rng = np.random.default_rng(0)
    for depth, n in ((1, 8), (7, 5000), (9, 120_000), (12, 300_000), (16, 70_001)):
        gc = rng.integers(0, 1 << depth, size=(n, 3)).astype(np.int32)
        b = np.sort(rng.integers(0, 32, size=n)).astype(np.int64)
        for orders in (list(oser.ORDERS), ["hilbert-trans", "z"]):
            code = ops.serialize_encode(torch.from_numpy(gc).to(DEV), torch.from_numpy(b).to(DEV), depth, orders).cpu().numpy()
            for i, o in enumerate(orders):
                assert np.array_equal(code[i], oser.encode(gc, b, depth, o)), (depth, o)
    # batch=None and empty input
    code = ops.serialize_encode(torch.from_numpy(gc).to(DEV), None, 16, ["z"]).cpu().numpy()
    assert np.array_equal(code[0], oser.encode(gc, None, 16, "z"))
    assert ops.serialize_encode(torch.zeros((0, 3), dtype=torch.int32, device=DEV), None, 4, ["z"]).shape == (1, 0)


def test_point_serialization_matches_reference_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "point_padding.npz"))
    depth = int(g["ser_depth"])
    code = ops.serialize_encode(torch.from_numpy(g["ser_grid"]).to(DEV), torch.from_numpy(g["ser_batch"]).to(DEV), depth, list(oser.ORDERS))
    order, inverse = ops.serialize_sort(code, 3 * depth + 2)
    assert np.array_equal(code.cpu().numpy(), g["ser_code"])
    assert np.array_equal(order.cpu().numpy(), g["ser_order"])
    assert np.array_equal(inverse.cpu().numpy(), g["ser_inverse"])


@pytest.mark.parametrize("n,k,bits", [(1, 1, 8), (2047, 2, 13), (2048, 4, 31), (2049, 4, 33), (120_000, 4, 31), (1_900_000, 4, 63)])
def test_radix_sort_stable_argsort(n, k, bits):
    gen = torch.Generator().manual_seed(n)
    hi = (1 << bits) - 1 if bits < 63 else (1 << 62)
    code = torch.randint(0, hi, (k, n), generator=gen, dtype=torch.int64)
    code[:, : n // 3] = code[:, n // 3: 2 * (n // 3)][:, : n // 3]  # force duplicates: stability matters
    order, inverse = ops.serialize_sort(code.to(DEV), bits)
    want = torch.sort(code, dim=1, stable=True).indices
    assert torch.equal(order.cpu(), want)
    ar = torch.arange(n).expand(k, n)
    assert torch.equal(torch.gather(inverse.cpu(), 1, want), ar)


def test_padding_tables(golden_dir):
    g = np.load(os.path.join(golden_dir, "point_padding.npz"))
    cases = [(g[f"pad_{c}_offset"].tolist(), int(g[f"pad_{c}_K"])) for c in "abcdefgh"]
    cases += [([120_000, 239_999, 240_000 + 1023, 400_000], 1024), ([7], 1024), ([1024], 1024), ([1025], 1024)]
    for offset, K in cases:
        pad, unpad, cu = ops.patch_padding(torch.tensor(offset, device=DEV), offset, K)
        wp, wu, wc = opad.padding_and_inverse(offset, K)
        assert np.array_equal(pad.cpu().numpy(), wp), (offset, K)
        assert np.array_equal(unpad.cpu().numpy(), wu), (offset, K)
        assert np.array_equal(cu.cpu().numpy(), wc), (offset, K)


# ---- rulebooks ----------------------------------------------------------------------------------------
def _voxels_16(p, seed, batch=1):
    rng = np.random.default_rng(seed)
    rows = []
    for b in range(batch):
        occ = np.argwhere(rng.random((16, 16, 16)) < p)
        rows.append(np.concatenate([np.full((len(occ), 1), b), occ], 1))
    idx = np.concatenate(rows).astype(np.int32)
    return idx[rng.permutation(len(idx))] if p < 1 else idx


@pytest.mark.parametrize("p,ksize,batch", [(0.3, 3, 1), (1.0, 3, 1), (0.3, 5, 2), (0.05, 3, 3), (0.3, 1, 1), (0.3, (3, 1, 5), 2)])
def test_subm_rulebook_bit_exact_16cube(p, ksize, batch):
    idx = _voxels_16(p, 5, batch)
    shape = [16 + 96] * 3 if p < 1 else [16, 16, 16]
    pair = ops.rulebook_subm(torch.from_numpy(idx).to(DEV), shape, ksize)
    assert np.array_equal(pair.cpu().numpy(), osp.subm_rulebook(idx, shape, ksize))


def test_subm_rulebook_scannet_scale_and_large_extent():
    b = synth.make_batch(2, seed=3)
    bid = np.repeat(np.arange(2), np.diff(b["offset"], prepend=0))
    idx = np.concatenate([bid[:, None], b["grid_coord"]], 1).astype(np.int32)
    shape = (b["grid_coord"].max(0) + 96).tolist()
    pair = ops.rulebook_subm(torch.from_numpy(idx).to(DEV), shape, 3).cpu().numpy()
    assert np.array_equal(pair, osp.subm_rulebook(idx, shape, 3))
    # symmetry property used by the backward pass: pair[k, j] = i  <=>  pair[KV-1-k, i] = j
    k, j = np.nonzero(pair >= 0)
    assert np.array_equal(pair[26 - k, pair[k, j]], j)
    # nuScenes-like extent: linearised keys exceed 32 bits
    c, g = synth.lidar_scene(1, target_voxels=60_000)
    idx = np.concatenate([np.full((len(g), 1), 31), g], 1).astype(np.int32)
    shape = (g.max(0) + 96).tolist()
    assert 32 * shape[0] * shape[1] * shape[2] > 2 ** 32
    assert np.array_equal(ops.rulebook_subm(torch.from_numpy(idx).to(DEV), shape, 3).cpu().numpy(), osp.subm_rulebook(idx, shape, 3))


@pytest.mark.parametrize("p,ksize,stride,padding", [(0.3, 2, 2, 0), (1.0, 2, 2, 0), (0.2, 3, 2, 1), (0.3, 3, 1, 1), (0.1, 2, 2, 0)])
def test_strided_rulebook_bit_exact(p, ksize, stride, padding):
    idx = _voxels_16(p, 9, 2)
    shape = [16, 16, 16]
    out_idx, out_shape, pf, pb = ops.rulebook_strided(torch.from_numpy(idx).to(DEV), shape, ksize, stride, padding)
    w_idx, w_shape, w_pf, w_pb = osp.strided_rulebook(idx, shape, ksize, stride, padding)
    assert out_shape == w_shape
    assert np.array_equal(out_idx.cpu().numpy(), w_idx)
    assert np.array_equal(pf.cpu().numpy(), w_pf)
    assert np.array_equal(pb.cpu().numpy(), w_pb)


# ---- sparse convolution arithmetic -------------------------------------------------------------------------
def _conv_case(idx, shape, cin, cout, ksize, dtype, seed, impl, bias=True, tol=1e-3):
    torch.manual_seed(seed)
    n = len(idx)
    kv = int(np.prod(ksize if isinstance(ksize, tuple) else (ksize,) * 3))
    pair_np = osp.subm_rulebook(idx, shape, ksize)
    feat = torch.randn(n, cin).to(dtype)
    w = (torch.randn(cout, kv, cin) * (1.0 / np.sqrt(cin * 11))).to(dtype)
    b = torch.randn(cout).to(dtype) if bias else None
    dout = torch.randn(n, cout).to(dtype)
    # oracle on identically rounded inputs, fp64 math
    f64 = feat.double().requires_grad_(True)
    w64 = w.double().requires_grad_(True)
    b64 = b.double().requires_grad_(True) if bias else None
    ref = osp.conv_apply(f64, w64, pair_np, b64)
    ref.backward(dout.double())
    pair = torch.from_numpy(pair_np).to(DEV)
    fg = feat.to(DEV).requires_grad_(True)
    wg = w.float().to(DEV).requires_grad_(True)     # fp32 master weight, as nn.Parameter under autocast
    bg = b.float().to(DEV).requires_grad_(True) if bias else None
    old = ops.get_impl()
    ops.set_impl(impl)
    try:
        out = ops.sparse_conv(fg, wg, bg, pair, pair, True)
        out.backward(dout.to(DEV))
    finally:
        ops.set_impl(old)
    # activations compared under identical output rounding (bf16 has an 1.1e-3 rms quantisation floor otherwise)
    assert rel_l2(out.detach().float(), ref.detach().to(dtype).float()) < tol, "forward"
    assert rel_l2(fg.grad.float(), f64.grad.to(dtype).float()) < tol, "dfeat"
    assert rel_l2(wg.grad, w64.grad) < tol, "dweight"
    if bias:
        assert rel_l2(bg.grad, b64.grad) < tol, "dbias"


@pytest.mark.parametrize("cin,cout,ksize", [(6, 32, 3), (32, 32, 3), (96, 96, 3), (6, 32, 5), (16, 48, 1)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_subm_conv_16cube_simt(cin, cout, ksize, dtype):
    """BASELINE config 1: SubMConv3d on one 16^3 scene, forward + backward vs the CPU oracle, <= 1e-3 rel."""
    idx = _voxels_16(0.3, 1)
    _conv_case(idx, [112, 112, 112], cin, cout, ksize, dtype, 0, impl=1)


def test_subm_conv_dense_cube_and_wide_channels_simt():
    idx = _voxels_16(1.0, 1)
    _conv_case(idx, [16, 16, 16], 32, 64, 3, torch.float16, 1, impl=1, bias=False)
    idx = _voxels_16(0.1, 2)
    _conv_case(idx, [112] * 3, 256, 256, 3, torch.bfloat16, 2, impl=1)
    _conv_case(idx, [112] * 3, 384, 256, 3, torch.float16, 3, impl=1, bias=False)


def test_strided_and_inverse_conv_vs_oracle():
    torch.manual_seed(0)
    idx = _voxels_16(0.3, 4, 2)
    shape = [16, 16, 16]
    out_idx, oshape, pf, pb = osp.strided_rulebook(idx, shape, 2, 2)
    n, m = len(idx), len(out_idx)
    for dtype in (torch.float32, torch.float16):
        feat = torch.randn(n, 32).to(dtype)
        w = (torch.randn(64, 8, 32) * 0.2).to(dtype)
        dout = torch.randn(m, 64).to(dtype)
        f64, w64 = feat.double().requires_grad_(True), w.double().requires_grad_(True)
        ref = osp.conv_apply(f64, w64, pf)
        ref.backward(dout.double())
        fg, wg = feat.to(DEV).requires_grad_(True), w.float().to(DEV).requires_grad_(True)
        out = ops.sparse_conv(fg, wg, None, torch.from_numpy(pf).to(DEV), torch.from_numpy(pb).to(DEV), False)
        out.backward(dout.to(DEV))
        assert rel_l2(out.detach().float(), ref.detach().to(dtype).float()) < 1e-3
        assert rel_l2(fg.grad.float(), f64.grad.to(dtype).float()) < 1e-3
        assert rel_l2(wg.grad, w64.grad) < 1e-3
        # inverse conv: M rows -> N rows through the same rulebook, roles swapped
        x = torch.randn(m, 64).to(dtype)
        wi = (torch.randn(48, 8, 64) * 0.2).to(dtype)
        di = torch.randn(n, 48).to(dtype)
        x64, wi64 = x.double().requires_grad_(True), wi.double().requires_grad_(True)
        refi = osp.inverse_conv_apply(x64, wi64, pb)
        refi.backward(di.double())
        xg, wig = x.to(DEV).requires_grad_(True), wi.float().to(DEV).requires_grad_(True)
        outi = ops.sparse_conv(xg, wig, None, torch.from_numpy(pb).to(DEV), torch.from_numpy(pf).to(DEV), False)
        outi.backward(di.to(DEV))
        assert rel_l2(outi.detach().float(), refi.detach().to(dtype).float()) < 1e-3
        assert rel_l2(xg.grad.float(), x64.grad.to(dtype).float()) < 1e-3
        assert rel_l2(wig.grad, wi64.grad) < 1e-3


# ---- patch attention ------------------------------------------------------------------------------------------
def _attn_case(lens, H, D, dtype, impl, seed=0, tol_out=2e-3, tol_grad=4e-3):
    torch.manual_seed(seed)
    T = sum(lens)
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32)
    qkv = (torch.randn(T, 3, H, D) * 1.5).to(dtype)
    dout = torch.randn(T, H, D).to(dtype)
    scale = D ** -0.5
    ref, ref_lse = oattn.varlen_attention(qkv, cu, scale, return_lse=True)
    ref_d = oattn.varlen_attention_grads(qkv, cu, dout, scale)
    q = qkv.to(DEV).requires_grad_(True)
    old = ops.get_impl()
    ops.set_impl(impl)
    try:
        out, lse = ops.patch_attention(q, cu.to(DEV), max(lens), scale, return_lse=True)
        out.backward(dout.to(DEV))
    finally:
        ops.set_impl(old)
    # fp16/bf16 outputs: compare under identical output rounding; P is rounded to the MMA operand type inside
    # the tensor-core kernel, hence 2e-3 / 4e-3 rather than 1e-3 for bf16.
    assert rel_l2(out.detach().float(), ref.to(dtype).float()) < tol_out, "out"
    assert float((lse.cpu() - ref_lse).abs().max()) < 2e-3, "lse"
    assert rel_l2(q.grad.float(), ref_d.to(dtype).float()) < tol_grad, "dqkv"


@pytest.mark.parametrize("lens,H", [([1024], 2), ([1024, 1024, 1024], 4), ([48, 48, 48], 2), ([700], 2), ([1024, 333, 1, 129, 128], 3),
                                    ([2048, 100], 1)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_patch_attention_simt_vs_oracle(lens, H, dtype):
    # bf16 gradients: delta = sum(dout*out) is taken from the saved bf16 output (the flash-attn contract), which alone
    # contributes ~2e-3 relative; fp16 keeps 1e-3.
    _attn_case(lens, H, 16, dtype, impl=1, tol_out=1e-3, tol_grad=1e-3 if dtype == torch.float16 else 4e-3)


def test_patch_attention_simt_other_head_dims():
    _attn_case([256, 100], 2, 32, torch.bfloat16, impl=1, tol_out=1e-3, tol_grad=4e-3)
    _attn_case([200], 1, 64, torch.float16, impl=1, tol_out=1e-3, tol_grad=1e-3)


def test_patch_attention_matches_reference_dense_branch_fixture(golden_dir):
    """fp32 activations of the reference's non-flash branch (SerializedAttention, ptv3m1:190-206), rounded to bf16
    at the op boundary exactly as its flash branch does (:209)."""
    g = np.load(os.path.join(golden_dir, "attention_dense.npz"))
    H, C = int(g["H"]), int(g["C"])
    order = torch.from_numpy(g["order"])[torch.from_numpy(g["pad"])]
    inverse = torch.from_numpy(g["unpad"])[torch.from_numpy(g["inverse"])]
    qkv = torch.from_numpy(g["qkv_full"])[order].reshape(-1, 3, H, C // H)
    out = ops.patch_attention(qkv.to(DEV).bfloat16(), torch.from_numpy(g["cu"]).to(DEV), int(g["K"]), float(g["scale"]))
    core = out.float().reshape(-1, C).cpu()[inverse]
    # bf16 inputs/outputs vs the reference's fp32 activations: 1e-2 rel (bf16 has 8 bits of mantissa)
    assert rel_l2(core, torch.from_numpy(g["core_out"])) < 1e-2


def test_patch_attention_against_flash_attn_if_present():
    """Where it is installed, flash-attn 2.8.3 (the package the reference pins, scripts/build_image.sh:73) is the GPU oracle."""
    fa = pytest.importorskip("flash_attn")
    if not hasattr(fa, "flash_attn_varlen_qkvpacked_func") or "b2pc" in getattr(fa, "__version__", ""):
        pytest.skip("stock flash_attn not importable")
    torch.manual_seed(0)
    lens = [1024] * 40 + [517]
    T, H, D = sum(lens), 4, 16
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
    qkv = torch.randn(T, 3, H, D, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    dout = torch.randn(T, H, D, device=DEV, dtype=torch.bfloat16)
    try:
        ref = fa.flash_attn_varlen_qkvpacked_func(qkv, cu, 1024, softmax_scale=0.25)
    except Exception as e:  # wheel without a kernel image for this GPU
        pytest.skip(f"flash_attn unusable here: {e}")
    ref.backward(dout)
    gref = qkv.grad.clone()
    qkv.grad = None
    out = ops.patch_attention(qkv, cu, 1024, 0.25)
    out.backward(dout)
    assert rel_l2(out.detach().float(), ref.detach().float()) < 4e-3
    assert rel_l2(qkv.grad.float(), gref.float()) < 8e-3


# ---- tensor-core kernels (impl=2): same oracles, plus A/B against the SIMT kernels at full size ---------------------------
@pytest.mark.parametrize("lens,H", [([1024], 2), ([1024, 1024, 1024], 4), ([48, 48, 48], 2), ([700], 2), ([1024, 333, 1, 129, 128], 3),
                                    ([2048, 100], 1)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_patch_attention_tcgen05_vs_oracle(lens, H, dtype):
    # P is rounded to the MMA operand type (bf16: 8 bits) before PV: 3e-3 on the output for bf16, 1e-3 for fp16
    _attn_case(lens, H, 16, dtype, impl=2, tol_out=3e-3 if dtype == torch.bfloat16 else 1e-3,
               tol_grad=6e-3 if dtype == torch.bfloat16 else 2e-3)


def test_tensor_core_attention_gradients_are_bitwise_reproducible():
    """Same inputs, same bits: the backward forms every gradient element in a fixed order (no atomics), so two calls agree exactly."""
    torch.manual_seed(0)
    lens = [1024] * 6 + [333]
    T, H = sum(lens), 2
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
    qkv = (torch.randn(T, 3, H, 16, device=DEV) * 1.5).bfloat16()
    dout = torch.randn(T, H, 16, device=DEV).bfloat16()
    grads = []
    old = ops.get_impl()
    ops.set_impl(2)
    try:
        for _ in range(2):
            q = qkv.clone().requires_grad_(True)
            ops.patch_attention(q, cu, 1024, 0.25).backward(dout)
            grads.append(q.grad)
    finally:
        ops.set_impl(old)
    assert torch.equal(grads[0], grads[1])


@pytest.mark.parametrize("cin,cout", [(32, 32), (64, 64), (96, 96), (128, 64), (16, 48), (256, 256), (384, 256), (512, 512)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_subm_conv_tcgen05_vs_oracle(cin, cout, dtype):
    idx = _voxels_16(0.3 if cin <= 128 else 0.08, 1)
    _conv_case(idx, [112, 112, 112], cin, cout, 3, dtype, 0, impl=2)


def test_subm_conv_tcgen05_large_kernel_volume():
    """5^3 stem geometry (125 offsets > one 32-offset rulebook chunk) on the tensor-core path."""
    _conv_case(_voxels_16(0.3, 2), [112] * 3, 16, 32, 5, torch.bfloat16, 4, impl=2, bias=False)
    _conv_case(_voxels_16(0.2, 3, 2), [112] * 3, 32, 48, 5, torch.float16, 5, impl=2)


def test_stem_conv_module_pads_odd_channel_counts():
    from pointcept_b200.spconv import pytorch as spconv
    torch.manual_seed(0)
    idx = _voxels_16(0.3, 6)
    n = len(idx)
    conv = spconv.SubMConv3d(6, 32, kernel_size=5, padding=1, bias=False, indice_key="stem").to(DEV)
    feat = torch.randn(n, 6, device=DEV)
    x = spconv.SparseConvTensor(feat, torch.from_numpy(idx).to(DEV), [112] * 3, 1)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = conv(x).features
    y.float().square().sum().backward()
    pair = osp.subm_rulebook(idx, [112] * 3, 5)
    w64 = conv.weight.detach().cpu().reshape(32, 125, 6).bfloat16().double().requires_grad_(True)
    ref = osp.conv_apply(feat.cpu().bfloat16().double(), w64, pair)
    assert rel_l2(y.detach().float(), ref.detach().bfloat16().float()) < 1e-3
    (ref.bfloat16().double().detach() * 0 + ref).square().sum().backward()
    assert rel_l2(conv.weight.grad.reshape(32, 125, 6), w64.grad) < 1e-2   # upstream gradient is 2*y in bf16 on the GPU side


def test_subm_conv_tcgen05_tile_edges():
    _conv_case(_voxels_16(1.0, 1), [16, 16, 16], 32, 64, 3, torch.float16, 1, impl=2, bias=False)   # dense cube, 32 full tiles
    _conv_case(_voxels_16(0.031, 3), [112] * 3, 64, 64, 3, torch.bfloat16, 2, impl=2)               # fewer rows than one tile
    _conv_case(_voxels_16(0.3, 5, 3), [112] * 3, 64, 32, (3, 1, 3), torch.float16, 3, impl=2)        # KV = 9, batch 3


def test_tcgen05_matches_simt_at_scannet_scale():
    torch.manual_seed(0)
    b = synth.make_batch(1, seed=4)
    n = len(b["grid_coord"])
    idx = torch.from_numpy(np.concatenate([np.zeros((n, 1)), b["grid_coord"]], 1).astype(np.int32)).to(DEV)
    pair = ops.rulebook_subm(idx, (b["grid_coord"].max(0) + 96).tolist(), 3)
    feat = torch.randn(n, 64, device=DEV).bfloat16().requires_grad_(True)
    w = (torch.randn(64, 27, 64, device=DEV) * 0.04).requires_grad_(True)
    bias = torch.randn(64, device=DEV).requires_grad_(True)
    dout = torch.randn(n, 64, device=DEV).bfloat16()
    res = {}
    for impl in (1, 2):
        ops.set_impl(impl)
        feat.grad = w.grad = bias.grad = None
        out = ops.sparse_conv(feat, w, bias, pair, pair, True)
        out.backward(dout)
        res[impl] = (out.detach().float(), feat.grad.float().clone(), w.grad.clone())
    ops.set_impl(0)
    for a, b_ in zip(res[1], res[2]):
        assert rel_l2(b_, a) < 2e-3


# ---- glue: fused LayerNorm ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [32, 64, 128, 256, 512])
@pytest.mark.parametrize("xdt,autocast", [(torch.float32, False), (torch.bfloat16, True), (torch.float32, True), (torch.float16, False)])
def test_fused_layer_norm_vs_torch(c, xdt, autocast):
    torch.manual_seed(c)
    n = 3001
    x = (torch.randn(n, c, device=DEV) * 2 + 0.5).to(xdt).requires_grad_(True)
    w = torch.randn(c, device=DEV).requires_grad_(True)
    b = torch.randn(c, device=DEV).requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        y = ops.layer_norm(x, w, b, 1e-5)
    dy = torch.randn_like(y)
    y.backward(dy)
    x64 = x.detach().double().requires_grad_(True)
    w64, b64 = w.detach().double().requires_grad_(True), b.detach().double().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(x64, (c,), w64, b64, 1e-5)
    ref.backward(dy.double())
    assert y.dtype == (torch.float32 if (autocast or xdt == torch.float32) else xdt)
    tol = 1e-5 if y.dtype == torch.float32 else 1e-3
    assert rel_l2(y.detach().float(), ref.detach().to(y.dtype).float()) < tol
    assert rel_l2(x.grad.float(), x64.grad.to(xdt).float()) < (1e-5 if xdt == torch.float32 else 1e-3)
    assert rel_l2(w.grad, w64.grad) < 1e-4 and rel_l2(b.grad, b64.grad) < 1e-4


# ---- serialized pooling / gathers (8(f).1) -------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_segment_max_and_unpool_add_vs_plain_torch(dtype):
    torch.manual_seed(0)
    n, c = 5000, 48
    lens = torch.randint(1, 9, (2000,))
    lens = lens[torch.cumsum(lens, 0) <= n]
    lens[-1] += n - int(lens.sum())
    m = len(lens)
    start = torch.cumsum(lens, 0) - lens
    order = torch.randperm(n)
    cluster = torch.empty(n, dtype=torch.long)
    cluster[order] = torch.repeat_interleave(torch.arange(m), lens)
    x = torch.randn(n, c).to(dtype)
    xg = x.to(DEV).requires_grad_(True)
    out = ops.segment_max(xg, order.to(DEV), start.to(DEV), lens.to(DEV))
    xr = x.float().requires_grad_(True)
    ref = torch.full((m, c), -float("inf")).scatter_reduce(0, cluster[:, None].expand(-1, c), xr, "amax", include_self=True)
    assert torch.equal(out.detach().float().cpu(), ref.detach())
    g = torch.randn(m, c).to(dtype)
    out.backward(g.to(DEV))
    # reference gradient: the (first) arg-max row of each cluster/channel receives the gradient
    xs = x.float()[order]
    seg = torch.repeat_interleave(torch.arange(m), lens)
    is_max = xs == ref.detach()[seg]
    first = torch.zeros_like(is_max)
    seen = torch.zeros(m, c, dtype=torch.bool)
    for r in range(n):
        first[r] = is_max[r] & ~seen[seg[r]]
        seen[seg[r]] |= is_max[r]
    want = torch.zeros(n, c)
    want[order] = first.float() * g.float()[seg]
    assert torch.equal(xg.grad.float().cpu(), want.to(dtype).float())
    # unpooling: parent + child[cluster]
    parent = torch.randn(n, c).to(dtype)
    child = torch.randn(m, c).to(dtype)
    pg, cg = parent.to(DEV).requires_grad_(True), child.to(DEV).requires_grad_(True)
    dy = torch.randn(n, c).to(dtype).to(DEV)
    ops.unpool_add(pg, cg, cluster.to(DEV), order.to(DEV), lens.to(DEV)).backward(dy)
    p2, c2 = parent.double().requires_grad_(True), child.double().requires_grad_(True)
    (p2 + c2[cluster]).backward(dy.double().cpu())
    assert rel_l2(pg.grad.float(), p2.grad) < 1e-6
    assert rel_l2(cg.grad.float(), c2.grad) < (1e-6 if dtype == torch.float32 else 5e-3)


@pytest.mark.parametrize("cin,cout", [(32, 96), (64, 64), (128, 512), (64, 20), (512, 1536)])
@pytest.mark.parametrize("autocast", [False, True])
def test_fused_linear_matches_torch_linear(cin, cout, autocast):
    torch.manual_seed(0)
    n = 4099
    x = torch.randn(n, cin, device=DEV, requires_grad=True)
    w = (torch.randn(cout, cin, device=DEV) * 0.1).requires_grad_(True)
    b = torch.randn(cout, device=DEV).requires_grad_(True)
    x2, w2, b2 = [t.detach().clone().requires_grad_(True) for t in (x, w, b)]
    dy = torch.randn(n, cout, device=DEV)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        y = ops.linear(x, w, b)
        y2 = torch.nn.functional.linear(x2, w2, b2)
    assert y.dtype == y2.dtype and torch.equal(y, y2)
    y.backward(dy.to(y.dtype))
    y2.backward(dy.to(y2.dtype))
    assert torch.equal(x.grad, x2.grad)
    if autocast:
        # the weight gradient leaves the GEMM in fp32 (half-precision operands, fp32 accumulate, no bf16 rounding of the result):
        # tighter against exact arithmetic than autocast's bf16 dW, and equal to it within one bf16 rounding
        want = dy.to(y.dtype).double().t() @ x.detach().to(y.dtype).double()
        assert w.grad.dtype == torch.float32 and rel_l2(w.grad, want) < 1e-5 and rel_l2(w2.grad, want) < 4e-3
    else:
        assert torch.equal(w.grad, w2.grad)
    # bias gradient: ours is an fp32 sum of the (bf16) upstream gradient, torch's is a bf16-accumulated reduction under autocast
    assert rel_l2(b.grad, dy.to(y.dtype).double().sum(0)) < 1e-5
    assert rel_l2(b.grad, b2.grad) < (1e-5 if not autocast else 1e-2)
