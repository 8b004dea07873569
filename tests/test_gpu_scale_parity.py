"""Parity at the sizes BASELINE.json names (one full ~120k-voxel ScanNet-scale scene), tensor-core kernels against the CPU
oracle (never against another kernel of this repo), plus direct tests of the compiled autograd nodes around the attention."""
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


_SCENE = {}


def _scene():
    if not _SCENE:
        b = synth.make_batch(1, seed=4)
        n = len(b["grid_coord"])
        idx = np.concatenate([np.zeros((n, 1)), b["grid_coord"]], 1).astype(np.int32)
        _SCENE.update(b=b, n=n, idx=idx, shape=(b["grid_coord"].max(0) + 96).tolist(), pairs={})
    return _SCENE


def _pair(ks):
    s = _scene()
    if ks not in s["pairs"]:
        s["pairs"][ks] = osp.subm_rulebook(s["idx"], s["shape"], ks)
    return s["pairs"][ks]


# ---- sparse convolution: tensor-core kernels vs the oracle on one full scene (SubM call sites of ptv3m1:278-284,499-506 and
# spunet:43-68,114-121; 128->96 is SpUNet's dec0 width) ------------------------------------------------------------------
@pytest.mark.parametrize("cin,cout,ks", [(32, 32, 3), (64, 64, 3), (16, 32, 5), (128, 96, 3)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_tcgen05_conv_vs_oracle_full_scene(cin, cout, ks, dtype):
    s = _scene()
    n = s["n"]
    assert n >= 100_000
    pair_np = _pair(ks)
    # the GPU rulebook is bit-exact against the oracle at this size
    pair = ops.rulebook_subm(torch.from_numpy(s["idx"]).to(DEV), s["shape"], ks)
    assert np.array_equal(pair.cpu().numpy(), pair_np)
    torch.manual_seed(cin * 1000 + cout)
    kv = pair_np.shape[0]
    pairs_per_row = float((pair_np >= 0).sum()) / n
    feat = torch.randn(n, cin).to(dtype)
    w = (torch.randn(cout, kv, cin) / np.sqrt(cin * pairs_per_row)).to(dtype)
    b = torch.randn(cout).to(dtype)
    dout = torch.randn(n, cout).to(dtype)
    f64, w64, b64 = feat.double().requires_grad_(True), w.double().requires_grad_(True), b.double().requires_grad_(True)
    ref = osp.conv_apply(f64, w64, pair_np, b64)
    ref.backward(dout.double())
    fg, wg, bg = feat.to(DEV).requires_grad_(True), w.float().to(DEV).requires_grad_(True), b.float().to(DEV).requires_grad_(True)
    old = ops.get_impl()
    ops.set_impl(2)     # tensor cores or error: a silent SIMT fallback cannot pass for the tensor-core path
    try:
        out = ops.sparse_conv(fg, wg, bg, pair, pair, True)
        out.backward(dout.to(DEV))
    finally:
        ops.set_impl(old)
    # identical output rounding on both sides; 1e-3 relative (north-star tolerance)
    assert rel_l2(out.detach().float(), ref.detach().to(dtype).float()) < 1e-3, "forward"
    assert rel_l2(fg.grad.float(), f64.grad.to(dtype).float()) < 1e-3, "dfeat"
    assert rel_l2(wg.grad, w64.grad) < 1e-3, "dweight"
    assert rel_l2(bg.grad, b64.grad) < 1e-3, "dbias"


def test_tcgen05_strided_and_inverse_conv_vs_oracle_full_scene():
    """SparseConv3d k2 s2 + paired SparseInverseConv3d (spunet:137-144,173-179) on one full scene, 32 -> 64 -> 32."""
    s = _scene()
    n = s["n"]
    out_idx, oshape, pf_np, pb_np = osp.strided_rulebook(s["idx"], s["shape"], 2, 2)
    g_idx, g_shape, pf, pb = ops.rulebook_strided(torch.from_numpy(s["idx"]).to(DEV), s["shape"], 2, 2)
    assert g_shape == oshape and np.array_equal(g_idx.cpu().numpy(), out_idx)
    assert np.array_equal(pf.cpu().numpy(), pf_np) and np.array_equal(pb.cpu().numpy(), pb_np)
    m = len(out_idx)
    torch.manual_seed(5)
    dtype = torch.bfloat16
    feat = torch.randn(n, 32).to(dtype)
    w = (torch.randn(64, 8, 32) * 0.1).to(dtype)
    dout = torch.randn(m, 64).to(dtype)
    f64, w64 = feat.double().requires_grad_(True), w.double().requires_grad_(True)
    ref = osp.conv_apply(f64, w64, pf_np)
    ref.backward(dout.double())
    old = ops.get_impl()
    ops.set_impl(2)
    try:
        fg, wg = feat.to(DEV).requires_grad_(True), w.float().to(DEV).requires_grad_(True)
        out = ops.sparse_conv(fg, wg, None, pf, pb, False)
        out.backward(dout.to(DEV))
        x = torch.randn(m, 64).to(dtype)
        wi = (torch.randn(32, 8, 64) * 0.1).to(dtype)
        di = torch.randn(n, 32).to(dtype)
        x64, wi64 = x.double().requires_grad_(True), wi.double().requires_grad_(True)
        refi = osp.inverse_conv_apply(x64, wi64, pb_np)
        refi.backward(di.double())
        xg, wig = x.to(DEV).requires_grad_(True), wi.float().to(DEV).requires_grad_(True)
        outi = ops.sparse_conv(xg, wig, None, pb, pf, False)
        outi.backward(di.to(DEV))
    finally:
        ops.set_impl(old)
    assert rel_l2(out.detach().float(), ref.detach().to(dtype).float()) < 1e-3
    assert rel_l2(fg.grad.float(), f64.grad.to(dtype).float()) < 1e-3
    assert rel_l2(wg.grad, w64.grad) < 1e-3
    assert rel_l2(outi.detach().float(), refi.detach().to(dtype).float()) < 1e-3
    assert rel_l2(xg.grad.float(), x64.grad.to(dtype).float()) < 1e-3
    assert rel_l2(wig.grad, wi64.grad) < 1e-3


# ---- BASELINE config 2: serialized attention over one full scene -----------------------------------------------------------
@pytest.mark.parametrize("K,H", [(1024, 2), (48, 2), (1024, 4)])
def test_serialized_attention_full_scene_vs_oracle(K, H):
    """encode -> sort -> padding tables -> patch attention over ~120k points (118 patches of 1024, or ~2500 of 48), every
    integer table bit-exact against the oracle and the attention output / gradients against its dense fp32 math
    (ptv3m1:114-222)."""
    s = _scene()
    b, n = s["b"], s["n"]
    depth = oser.serialization_depth(b["grid_coord"])
    bid = np.zeros(n, dtype=np.int64)
    code = ops.serialize_encode(torch.from_numpy(b["grid_coord"]).to(DEV), torch.from_numpy(bid).to(DEV), depth, ["hilbert"])
    order, inverse = ops.serialize_sort(code, 3 * depth + 1)
    wc, wo, wi, _ = oser.serialize(b["grid_coord"], bid, ["hilbert"], depth)
    assert np.array_equal(code.cpu().numpy(), wc) and np.array_equal(order.cpu().numpy(), wo) and np.array_equal(inverse.cpu().numpy(), wi)
    pad, unpad, cu = ops.patch_padding(torch.tensor([n], device=DEV), [n], K)
    wp, wu, wcu = opad.padding_and_inverse([n], K)
    assert np.array_equal(pad.cpu().numpy(), wp) and np.array_equal(unpad.cpu().numpy(), wu) and np.array_equal(cu.cpu().numpy(), wcu)
    torch.manual_seed(K + H)
    D = 16
    x = (torch.randn(n, 3, H, D) * 1.2).bfloat16()
    gather = torch.from_numpy(wo[0][wp])
    qkv = x[gather]
    dout = torch.randn(qkv.shape[0], H, D).bfloat16()
    cu_t = torch.from_numpy(wcu)
    ref, ref_lse = oattn.varlen_attention(qkv, cu_t, D ** -0.5, return_lse=True)
    ref_d = oattn.varlen_attention_grads(qkv, cu_t, dout, D ** -0.5)
    q = qkv.to(DEV).requires_grad_(True)
    old = ops.get_impl()
    ops.set_impl(2)
    try:
        out, lse = ops.patch_attention(q, cu, K, D ** -0.5, return_lse=True)
        out.backward(dout.to(DEV))
    finally:
        ops.set_impl(old)
    # bf16: P is rounded to 8 mantissa bits before PV inside the kernel (flash-attn does the same): 3e-3 / 6e-3
    assert rel_l2(out.detach().float(), ref.bfloat16().float()) < 3e-3
    assert float((lse.cpu() - ref_lse).abs().max()) < 2e-3
    assert rel_l2(q.grad.float(), ref_d.bfloat16().float()) < 6e-3


def test_attention_ignores_non_finite_rows_of_neighbouring_sequences():
    """A ragged last block reads rows of the NEXT sequence in the packed tensor (bulk tile loads); they must never leak, even
    when they hold Inf / NaN."""
    torch.manual_seed(0)
    H, D = 2, 16
    lens = [700, 300, 1024]
    T = sum(lens)
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32)
    qkv = torch.randn(T, 3, H, D).bfloat16()
    dout = torch.randn(T, H, D).bfloat16()
    ref = oattn.varlen_attention(qkv[:700], cu[:2], D ** -0.5)
    ref_d = oattn.varlen_attention_grads(qkv[:700], cu[:2], dout[:700], D ** -0.5)
    bad = qkv.clone()
    bad[700:1000] = float("nan")
    bad[700:1000, 1] = float("inf")
    bad_dout = dout.clone()
    bad_dout[700:1000] = float("nan")
    for impl in (2,):
        ops.set_impl(impl)
        try:
            q = bad.to(DEV).requires_grad_(True)
            out = ops.patch_attention(q, cu.to(DEV), 1024, D ** -0.5)
            out.backward(bad_dout.to(DEV))
        finally:
            ops.set_impl(0)
        assert torch.isfinite(out[:700]).all() and torch.isfinite(out[1000:]).all()
        assert rel_l2(out[:700].detach().float(), ref.bfloat16().float()) < 3e-3
        assert torch.isfinite(q.grad[:700]).all() and torch.isfinite(q.grad[1000:]).all()
        assert rel_l2(q.grad[:700].float(), ref_d.bfloat16().float()) < 6e-3


# ---- the autograd nodes around the attention (compiled binding and python twin) against plain indexing ---------------------
@pytest.mark.parametrize("binding", ["compiled", "ctypes"])
def test_serialized_gather_scatter_unpool_nodes_vs_plain_indexing(binding):
    from pointcept_b200 import _lib
    from pointcept_b200.ptv3 import serialized_gather, serialized_scatter_back
    if binding == "compiled" and _lib.torch_binding() is None:
        pytest.skip("compiled binding not built")
    ops.set_binding(binding)
    try:
        torch.manual_seed(1)
        K = 64
        offset = [150, 150 + 64, 150 + 64 + 333, 150 + 64 + 333 + 20]     # padded + borrowed, exact, padded, short
        n = offset[-1]
        pad, unpad, cu = opad.padding_and_inverse(offset, K)
        order = np.concatenate([np.random.default_rng(b).permutation(np.arange(a, e)) for b, (a, e) in
                                enumerate(zip([0] + offset[:-1], offset))])
        inverse = np.empty_like(order)
        inverse[order] = np.arange(n)
        order_pad = torch.from_numpy(order[pad]).to(DEV)
        primary = torch.from_numpy(unpad[inverse]).to(DEV)
        x = torch.randn(n, 3, 2, 16, device=DEV, dtype=torch.float64).reshape(n, -1)
        x1 = x.clone().requires_grad_(True)
        x2 = x.clone().requires_grad_(True)
        dy = torch.randn(len(pad), x.shape[1], device=DEV, dtype=torch.float64)
        y1 = serialized_gather(x1, order_pad, primary, offset, K)
        y2 = x2[order_pad]
        assert torch.equal(y1, y2)
        y1.backward(dy)
        y2.backward(dy)
        # borrowed rows receive two contributions: exact in fp64 up to the order of one addition
        assert torch.allclose(x1.grad, x2.grad, rtol=0, atol=1e-12)
        assert int((torch.bincount(order_pad, minlength=n) == 2).sum()) > 0      # the case really has borrowed rows
        # scatter back
        t1 = torch.randn(len(pad), 32, device=DEV, dtype=torch.float64).requires_grad_(True)
        t2 = t1.detach().clone().requires_grad_(True)
        dz = torch.randn(n, 32, device=DEV, dtype=torch.float64)
        z1 = serialized_scatter_back(t1, primary)
        z2 = t2[primary]
        assert torch.equal(z1, z2)
        z1.backward(dz)
        z2.backward(dz)
        assert torch.equal(t1.grad, t2.grad)
    finally:
        ops.set_binding("auto")
