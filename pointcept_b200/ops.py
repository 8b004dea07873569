"""torch-tensor front end of the C ABI (include/b2pc.h): allocation, stream plumbing and autograd.

Every function requires CUDA tensors and raises otherwise -- there is no CPU / eager fallback.
"""
import ctypes
import os

import torch

from . import _lib

ORDER_IDS = {"z": 0, "z-trans": 1, "hilbert": 2, "hilbert-trans": 3}
_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}

# 0 = auto (tensor-core kernels where supported), 1 = SIMT reference kernels, 2 = tensor-core kernels or error
_impl = int(os.environ.get("B2PC_IMPL", "0"))


def set_impl(v):
    global _impl
    _impl = int(v)


def get_impl():
    return _impl


# optional per-op CUDA-event timing (bench.py's roofline leg): name -> list of (start, end, meta)
_prof = None


def profile_start():
    global _prof
    _prof = {}


def profile_stop():
    global _prof
    p, _prof = _prof, None
    return p


class _timed:
    def __init__(self, name, meta):
        self.name, self.meta = name, meta

    def __enter__(self):
        if _prof is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *a):
        if _prof is not None:
            self.e1.record()
            _prof.setdefault(self.name, []).append((self.e0, self.e1, self.meta))


def binding():
    """compiled autograd binding (pointcept_b200/csrc/torch_binding.cpp) or None; never used while the per-op profiler runs"""
    if _prof is not None or _force_ctypes:
        return None
    return _lib.torch_binding()


_force_ctypes = False


def set_binding(name):
    """"ctypes" forces the Python/ctypes binding (the reference binding), anything else lets the compiled one be used if built."""
    global _force_ctypes
    _force_ctypes = name == "ctypes"


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts):
    cur = None
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError("pointcept_b200 operators run on CUDA tensors only (got a %s tensor); "
                               "there is no CPU fallback" % t.device.type)
        if cur is None:
            cur = torch.cuda.current_device()
        if t.device.index != cur:
            # the ctypes binding launches on the CURRENT device's stream; the compiled binding pins the tensor's device itself
            raise RuntimeError(f"ctypes binding: tensor on cuda:{t.device.index} but the current device is cuda:{cur}; wrap the call in "
                               "`with torch.cuda.device_of(tensor):` (or use the compiled binding, which guards the device itself)")


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _ws(nbytes, device):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


def _i3(v):
    v = (v, v, v) if isinstance(v, int) else tuple(int(x) for x in v)
    assert len(v) == 3
    return (ctypes.c_int * 3)(*v), v


# ------------------------------------------------------------------------------------------------
# serialization
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
def serialize_encode(grid_coord, batch, depth, orders):
    """codes [len(orders), N] int64; all orders in one kernel (serialization/default.py:9-24)."""
    _need_cuda(grid_coord, batch)
    gc = grid_coord if (grid_coord.dtype == torch.int32 and grid_coord.is_contiguous()) else grid_coord.int().contiguous()
    if batch is not None and (batch.dtype != torch.int64 or not batch.is_contiguous()):
        batch = batch.long().contiguous()
    n = gc.shape[0]
    ids = (ctypes.c_int * len(orders))(*[ORDER_IDS[o] for o in orders])
    code = torch.empty((len(orders), n), dtype=torch.int64, device=gc.device)
    if n == 0:
        return code
    L = _lib.lib()
    _lib.check(L.b2pc_serialize_encode(_p(gc), _p(batch), n, int(depth), ids, len(orders), _p(code), _stream()), "serialize_encode")
    return code


@torch.no_grad()
def serialize_sort(code, key_bits):
    """order, inverse [k, N] int64 for code [k, N] int64 (structure.py:93-100)."""
    _need_cuda(code)
    code = code.contiguous()
    k, n = code.shape
    order = torch.empty_like(code)
    inverse = torch.empty_like(code)
    if n == 0:
        return order, inverse
    L = _lib.lib()
    ws = _ws(L.b2pc_serialize_sort_workspace_bytes(n, k), code.device)
    _lib.check(L.b2pc_serialize_sort(_p(code), n, k, int(key_bits), _p(order), _p(inverse), _p(ws), ws.numel(), _stream()),
               "serialize_sort")
    return order, inverse


@torch.no_grad()
def patch_padding(offset, offset_host, patch_size):
    """pad, unpad, cu_seqlens as SerializedAttention.get_padding_and_inverse (ptv3m1:114-170).

    offset: device int64 [B]; offset_host: the same values on the host (list of ints)."""
    _need_cuda(offset)
    K = int(patch_size)
    counts = [b - a for a, b in zip([0] + list(offset_host[:-1]), offset_host)]
    padded = [((c + K - 1) // K * K) if c > K else c for c in counts]
    n, t_pad = int(offset_host[-1]), sum(padded)
    n_seq = sum(((c + K - 1) // K) if c > 0 else 0 for c in padded)
    dev = offset.device
    pad = torch.empty(t_pad, dtype=torch.int64, device=dev)
    unpad = torch.empty(n, dtype=torch.int64, device=dev)
    cu = torch.empty(n_seq + 1, dtype=torch.int32, device=dev)
    off = offset if offset.dtype == torch.int64 else offset.long()
    L = _lib.lib()
    _lib.check(L.b2pc_patch_padding(_p(off.contiguous()), len(offset_host), K, n, t_pad, n_seq, _p(pad), _p(unpad), _p(cu), _stream()),
               "patch_padding")
    return pad, unpad, cu


# ------------------------------------------------------------------------------------------------
# patch attention
# ------------------------------------------------------------------------------------------------
class PatchAttentionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, cu_seqlens, max_seqlen, scale):
        _need_cuda(qkv, cu_seqlens)
        if qkv.dtype not in (torch.float16, torch.bfloat16):
            raise RuntimeError("patch attention takes fp16 or bf16 qkv (flash-attn contract), got %s" % qkv.dtype)
        qkv = qkv.contiguous()
        T, three, H, D = qkv.shape
        assert three == 3
        cu = cu_seqlens if cu_seqlens.dtype == torch.int32 else cu_seqlens.int()
        cu = cu.contiguous()
        out = torch.empty((T, H, D), dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty((H, T), dtype=torch.float32, device=qkv.device)
        L = _lib.lib()
        with _timed("patch_attn_fwd", (cu, H, D)):
            _lib.check(L.b2pc_patch_attn_fwd(_p(qkv), _DTYPES[qkv.dtype], _p(cu), cu.numel() - 1, int(max_seqlen), T, H, D,
                                             float(scale), _p(out), _p(lse), _impl, _stream()), "patch_attn_fwd")
        ctx.save_for_backward(qkv, out, lse, cu)
        ctx.max_seqlen, ctx.scale = int(max_seqlen), float(scale)
        ctx.mark_non_differentiable(lse)
        return out, lse

    @staticmethod
    def backward(ctx, dout, _dlse):
        qkv, out, lse, cu = ctx.saved_tensors
        T, _, H, D = qkv.shape
        dout = dout.contiguous()
        dqkv = torch.empty_like(qkv)
        L = _lib.lib()
        ws = _ws(L.b2pc_patch_attn_bwd_workspace_bytes(T, H, D), qkv.device)
        with _timed("patch_attn_bwd", (cu, H, D)):
            _lib.check(L.b2pc_patch_attn_bwd(_p(dout), _p(qkv), _p(out), _p(lse), _DTYPES[qkv.dtype], _p(cu), cu.numel() - 1,
                                             ctx.max_seqlen, T, H, D, ctx.scale, _p(dqkv), _p(ws), ws.numel(), _impl, _stream()),
                       "patch_attn_bwd")
        return dqkv, None, None, None


def patch_attention(qkv, cu_seqlens, max_seqlen, scale=None, return_lse=False):
    if scale is None:
        scale = qkv.shape[-1] ** -0.5
    B = binding()
    if B is not None and not return_lse:
        return B.patch_attention(qkv, cu_seqlens, int(max_seqlen), float(scale), _impl)
    out, lse = PatchAttentionFn.apply(qkv, cu_seqlens, max_seqlen, scale)
    return (out, lse) if return_lse else out


# ------------------------------------------------------------------------------------------------
# rulebooks
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
def rulebook_subm(indices, spatial_shape, ksize, dilation=1):
    """pair [KV, N] int32 (input row or -1) for a submanifold convolution."""
    _need_cuda(indices)
    assert indices.dtype == torch.int32 and indices.dim() == 2 and indices.shape[1] == 4
    indices = indices.contiguous()
    n = indices.shape[0]
    shp, _ = _i3(list(spatial_shape))
    ks, kt = _i3(ksize)
    dl, _ = _i3(dilation)
    kv = kt[0] * kt[1] * kt[2]
    pair = torch.empty((kv, n), dtype=torch.int32, device=indices.device)
    if n == 0:
        return pair
    L = _lib.lib()
    ws = _ws(L.b2pc_rulebook_workspace_bytes(n, 1), indices.device)
    _lib.check(L.b2pc_rulebook_subm(_p(indices), n, shp, ks, dl, _p(pair), _p(ws), ws.numel(), _stream()), "rulebook_subm")
    return pair


@torch.no_grad()
def rulebook_strided(indices, spatial_shape, ksize, stride, padding=0, dilation=1):
    """-> out_indices [M,4] int32 (ascending (b,x,y,z)), out_shape, pair_fwd [KV,M], pair_bwd [KV,N].
    One host sync to learn M (as spconv does)."""
    _need_cuda(indices)
    assert indices.dtype == torch.int32 and indices.dim() == 2 and indices.shape[1] == 4
    indices = indices.contiguous()
    n = indices.shape[0]
    shp, shape_t = _i3(list(spatial_shape))
    ks, kt = _i3(ksize)
    st, stt = _i3(stride)
    pd, pdt = _i3(padding)
    dl, dlt = _i3(dilation)
    kv = kt[0] * kt[1] * kt[2]
    out_shape = [(shape_t[a] + 2 * pdt[a] - dlt[a] * (kt[a] - 1) - 1) // stt[a] + 1 for a in range(3)]
    L = _lib.lib()
    dev = indices.device
    if n == 0:
        z = torch.empty((kv, 0), dtype=torch.int32, device=dev)
        return torch.empty((0, 4), dtype=torch.int32, device=dev), out_shape, z, z.clone()
    ws = _ws(L.b2pc_rulebook_strided_workspace_bytes(n, ks, st, dl), dev)
    num = torch.zeros(2, dtype=torch.int64, device=dev)
    _lib.check(L.b2pc_rulebook_strided_begin(_p(indices), n, shp, ks, st, pd, dl, _p(num), _p(ws), ws.numel(), _stream()),
               "rulebook_strided_begin")
    m, bmax = (int(v) for v in num.tolist())        # the one host sync: output count (+ the batch bound of the sort keys)
    out_indices = torch.empty((m, 4), dtype=torch.int32, device=dev)
    pair_fwd = torch.empty((kv, m), dtype=torch.int32, device=dev)
    pair_bwd = torch.empty((kv, n), dtype=torch.int32, device=dev)
    _lib.check(L.b2pc_rulebook_strided_finish(_p(indices), n, shp, ks, st, pd, dl, m, bmax + 1, _p(out_indices), _p(pair_fwd), _p(pair_bwd),
                                              _p(ws), ws.numel(), _stream()), "rulebook_strided_finish")
    return out_indices, out_shape, pair_fwd, pair_bwd


# ------------------------------------------------------------------------------------------------
# sparse convolution arithmetic
# ------------------------------------------------------------------------------------------------
def _gather_gemm(feat, weight, bias, pair, n_out, c_in, c_out, kv, transpose_w, flip):
    out = torch.empty((n_out, c_out), dtype=feat.dtype, device=feat.device)
    L = _lib.lib()
    wsb = L.b2pc_spconv_gather_gemm_workspace_bytes(n_out, c_in, c_out, kv)
    ws = _ws(wsb, feat.device) if wsb else None
    with _timed("spconv_gather_gemm", (pair, c_in, c_out, feat.element_size())):
        _lib.check(L.b2pc_spconv_gather_gemm(_p(feat), _p(weight), _p(bias), _p(pair), pair.shape[1], feat.shape[0], n_out, c_in,
                                             c_out, kv, int(transpose_w), int(flip), _DTYPES[feat.dtype], _p(out), _p(ws), wsb, _impl,
                                             _stream()), "spconv_gather_gemm")
    return out


class SparseConvFn(torch.autograd.Function):
    """out = bias + sum_k feat[table_fwd[k]] @ weight[:, k, :].T

    feat [N_in, Cin] (fp32/fp16/bf16); weight [Cout, KV, Cin] fp32 master parameter (cast to feat's dtype
    inside, its gradient is produced in fp32); table_fwd [KV, N_out]; table_bwd [KV, N_in] is the rulebook
    of the opposite direction (SubM: the same table read with flipped offsets)."""

    @staticmethod
    def forward(ctx, feat, weight, bias, table_fwd, table_bwd, flip_bwd):
        _need_cuda(feat, weight, table_fwd)
        if feat.dtype not in _DTYPES:
            raise RuntimeError("sparse conv features must be fp32/fp16/bf16, got %s" % feat.dtype)
        feat = feat.contiguous()
        c_out, kv, c_in = weight.shape
        assert feat.shape[1] == c_in, (feat.shape, weight.shape)
        w = weight.detach().to(feat.dtype).contiguous()
        b = bias.detach().to(feat.dtype).contiguous() if bias is not None else None
        n_out = table_fwd.shape[1]
        out = _gather_gemm(feat, w, b, table_fwd, n_out, c_in, c_out, kv, False, False)
        ctx.save_for_backward(feat, w, table_fwd, table_bwd)
        ctx.flip_bwd = bool(flip_bwd)
        ctx.has_bias = bias is not None
        ctx.wdtype = weight.dtype
        return out

    @staticmethod
    def backward(ctx, dout):
        feat, w, table_fwd, table_bwd = ctx.saved_tensors
        c_out, kv, c_in = w.shape
        dout = dout.contiguous()
        if dout.dtype != feat.dtype:
            dout = dout.to(feat.dtype)
        dfeat = dweight = dbias = None
        if ctx.needs_input_grad[0]:
            dfeat = _gather_gemm(dout, w, None, table_bwd, feat.shape[0], c_out, c_in, kv, True, ctx.flip_bwd)
        if ctx.needs_input_grad[1]:
            dweight = torch.empty((c_out, kv, c_in), dtype=torch.float32, device=feat.device)
            L = _lib.lib()
            n_out = table_fwd.shape[1]
            ws = _ws(L.b2pc_spconv_bwd_weight_workspace_bytes(n_out, c_in, c_out, kv), feat.device)
            with _timed("spconv_bwd_weight", (table_fwd, c_in, c_out, feat.element_size())):
                _lib.check(L.b2pc_spconv_bwd_weight(_p(feat), _p(dout), _p(table_fwd), table_fwd.shape[1], feat.shape[0], n_out, c_in,
                                                    c_out, kv, _DTYPES[feat.dtype], _p(dweight), _p(ws), ws.numel(), _impl, _stream()),
                           "spconv_bwd_weight")
            if ctx.wdtype != torch.float32:
                dweight = dweight.to(ctx.wdtype)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            dbias = dout.float().sum(0)
        return dfeat, dweight, dbias, None, None, None


def sparse_conv(feat, weight, bias, table_fwd, table_bwd, flip_bwd, w16=None, b16=None):
    B = binding()
    if B is not None and feat.dtype in _DTYPES:
        return B.sparse_conv(feat, weight, bias, table_fwd, table_bwd, bool(flip_bwd), _impl, w16, b16)
    return SparseConvFn.apply(feat, weight, bias, table_fwd, table_bwd, flip_bwd)


# ------------------------------------------------------------------------------------------------
# glue: fused LayerNorm (fp32 statistics; output fp32 under autocast like torch's autocast policy)
# ------------------------------------------------------------------------------------------------
class LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps, out_dtype):
        _need_cuda(x, weight)
        x = x.contiguous()
        n, c = x.shape
        y = torch.empty((n, c), dtype=out_dtype, device=x.device)
        mean = torch.empty(n, dtype=torch.float32, device=x.device)
        rstd = torch.empty(n, dtype=torch.float32, device=x.device)
        w = weight.detach()
        if w.dtype != torch.float32 or not w.is_contiguous():
            w = w.float().contiguous()
        b = bias.detach() if bias is not None else None
        if b is not None and (b.dtype != torch.float32 or not b.is_contiguous()):
            b = b.float().contiguous()
        L = _lib.lib()
        _lib.check(L.b2pc_layer_norm_fwd(_p(x), _DTYPES[x.dtype], _p(w), _p(b), n, c, float(eps), _p(y), _DTYPES[out_dtype], _p(mean),
                                         _p(rstd), _stream()), "layer_norm_fwd")
        ctx.save_for_backward(x, w, mean, rstd)
        ctx.has_bias = bias is not None
        ctx.pdtype = weight.dtype
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, mean, rstd = ctx.saved_tensors
        n, c = x.shape
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        dg = torch.empty(c, dtype=torch.float32, device=x.device)
        db = torch.empty(c, dtype=torch.float32, device=x.device) if ctx.has_bias else None
        L = _lib.lib()
        ws = _ws(L.b2pc_layer_norm_bwd_workspace_bytes(n, c), x.device)
        _lib.check(L.b2pc_layer_norm_bwd(_p(dy), _DTYPES[dy.dtype], _p(x), _DTYPES[x.dtype], _p(w), _p(mean), _p(rstd), n, c, _p(dx),
                                         _p(dg), _p(db), _p(ws), ws.numel(), _stream()), "layer_norm_bwd")
        return dx, dg.to(ctx.pdtype), (db.to(ctx.pdtype) if db is not None else None), None, None


def layer_norm_supported(x, c):
    return x.is_cuda and x.dim() == 2 and x.dtype in _DTYPES and c in (32, 64, 128, 256, 512)


def layer_norm(x, weight, bias, eps=1e-5, emit_autocast_dtype=False):
    """nn.LayerNorm over the last dim of [N, C]; under autocast the result is fp32 (torch's autocast policy for layer_norm).

    emit_autocast_dtype: the only consumer is an autocast Linear, which would round this fp32 result to the autocast dtype
    as its first step -- emit that dtype directly (bit-identical values, one cast kernel and 2/3 of the bytes less)."""
    if torch.is_autocast_enabled():
        out_dtype = torch.get_autocast_dtype("cuda") if emit_autocast_dtype else torch.float32
    else:
        out_dtype = x.dtype
    B = binding()
    if B is not None:
        return B.layer_norm(x, weight, bias, float(eps), _DTYPES[out_dtype])
    return LayerNormFn.apply(x, weight, bias, eps, out_dtype)


# ------------------------------------------------------------------------------------------------
# serialized pooling / unpooling (clusters = runs of the order-0 sorted sequence)
# ------------------------------------------------------------------------------------------------
class SegmentMaxFn(torch.autograd.Function):
    """out[m] = max over rows order[start[m] : start[m]+len[m]] of x  -- the [indices] gather, segment_csr(max) and its
    backward in one kernel each (argmax saved)."""

    @staticmethod
    def forward(ctx, x, order, seg_start, seg_len):
        _need_cuda(x, order)
        x = x.contiguous()
        n, c = x.shape
        m = seg_start.shape[0]
        out = torch.empty((m, c), dtype=x.dtype, device=x.device)
        arg = torch.empty((m, c), dtype=torch.int32, device=x.device)
        L = _lib.lib()
        _lib.check(L.b2pc_segment_max_fwd(_p(x), _DTYPES[x.dtype], _p(order), _p(seg_start), _p(seg_len), m, c, _p(out), _p(arg),
                                          _stream()), "segment_max_fwd")
        ctx.save_for_backward(arg)
        ctx.n = n
        return out

    @staticmethod
    def backward(ctx, dout):
        (arg,) = ctx.saved_tensors
        m, c = arg.shape
        dout = dout.contiguous()
        dx = torch.empty((ctx.n, c), dtype=dout.dtype, device=dout.device)
        L = _lib.lib()
        _lib.check(L.b2pc_segment_max_bwd(_p(dout), _DTYPES[dout.dtype], _p(arg), m, c, ctx.n, _p(dx), _stream()), "segment_max_bwd")
        return dx, None, None, None


def segment_max(x, order, seg_start, seg_len):
    B = binding()
    if B is not None:
        return B.segment_max(x, order, seg_start, seg_len)
    return SegmentMaxFn.apply(x, order, seg_start, seg_len)


@torch.no_grad()
def pool_plan(code, order0, batch, grid_coord, pooling_depth, n_scene):
    """Index side of SerializedPooling (ptv3m1:371-398) on the device with one host read.
    -> dict(cluster [N], head_pos / head_indices / lengths [M], code [n_orders, M], batch [M], grid_coord [M,3], counts list[int])"""
    _need_cuda(code, order0, batch, grid_coord)
    code = code.contiguous()
    k, n = code.shape
    dev = code.device
    order0 = order0.contiguous()
    batch = batch if (batch.dtype == torch.int64 and batch.is_contiguous()) else batch.long().contiguous()
    gc = grid_coord if (grid_coord.dtype == torch.int32 and grid_coord.is_contiguous()) else grid_coord.int().contiguous()
    i64 = dict(dtype=torch.int64, device=dev)
    cluster, head_pos, head_idx, lengths = (torch.empty(n, **i64) for _ in range(4))
    code_out = torch.empty((k, n), **i64)
    batch_out = torch.empty(n, **i64)
    grid_out = torch.empty((n, 3), dtype=torch.int32, device=dev)
    meta = torch.empty(1 + n_scene, **i64)
    L = _lib.lib()
    ws = _ws(L.b2pc_pool_plan_workspace_bytes(n), dev)
    _lib.check(L.b2pc_pool_plan(_p(code), k, n, _p(order0), _p(batch), _p(gc), int(pooling_depth), int(n_scene), _p(cluster), _p(head_pos),
                                _p(head_idx), _p(lengths), _p(code_out), _p(batch_out), _p(grid_out), _p(meta), _p(ws), ws.numel(), _stream()),
               "pool_plan")
    mh = meta.tolist()              # the single host sync of this pooling stage
    m = int(mh[0])
    return dict(cluster=cluster, head_pos=head_pos[:m], head_indices=head_idx[:m], lengths=lengths[:m], code=code_out[:, :m].contiguous(),
                batch=batch_out[:m], grid_coord=grid_out[:m], counts=[int(v) for v in mh[1:]])


class UnpoolAddFn(torch.autograd.Function):
    """out = parent + child[cluster]  (SerializedUnpooling, ptv3m1:479); the gradient of child is a segment sum over the
    parent's sorted order instead of a sort-based index_put."""

    @staticmethod
    def forward(ctx, parent, child, cluster, order, seg_len):
        ctx.save_for_backward(order, seg_len)
        ctx.dtypes = (parent.dtype, child.dtype)
        return parent + child.index_select(0, cluster)

    @staticmethod
    def backward(ctx, dy):
        order, seg_len = ctx.saved_tensors
        dchild = torch.segment_reduce(dy.index_select(0, order), "sum", lengths=seg_len, axis=0, unsafe=True)
        return dy.to(ctx.dtypes[0]), dchild.to(ctx.dtypes[1]), None, None, None


def unpool_add(parent, child, cluster, order, seg_len):
    B = binding()
    if B is not None:
        return B.unpool_add(parent, child, cluster, order, seg_len)
    return UnpoolAddFn.apply(parent, child, cluster, order, seg_len)


# ------------------------------------------------------------------------------------------------
# glue: Linear with a fused bias-gradient reduction (point features are tall matrices: N >> C)
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
def colsum(x):
    """fp32 column sums of a [N, C] CUDA matrix."""
    _need_cuda(x)
    x = x.contiguous()
    n, c = x.shape
    out = torch.empty(c, dtype=torch.float32, device=x.device)
    L = _lib.lib()
    ws = _ws(L.b2pc_colsum_workspace_bytes(n, c), x.device)
    _lib.check(L.b2pc_colsum(_p(x), _DTYPES[x.dtype], n, c, _p(out), _p(ws), ws.numel(), _stream()), "colsum")
    return out


class LinearFn(torch.autograd.Function):
    """y = x @ W^T + b in the compute dtype (the autocast dtype under autocast), gradients as autocast produces them, except
    that the bias gradient is one fused fp32 column-sum kernel instead of a tall-matrix torch reduction."""

    @staticmethod
    def forward(ctx, x, weight, bias, cdtype):
        xc = x if x.dtype == cdtype else x.to(cdtype)
        wc = weight if weight.dtype == cdtype else weight.to(cdtype)
        bc = None if bias is None else (bias if bias.dtype == cdtype else bias.to(cdtype))
        with torch.autocast("cuda", enabled=False):
            y = torch.nn.functional.linear(xc, wc, bc)
        ctx.save_for_backward(xc, wc)
        ctx.meta = (x.dtype, weight.dtype, None if bias is None else bias.dtype)
        return y

    @staticmethod
    def backward(ctx, dy):
        xc, wc = ctx.saved_tensors
        xd, wd, bd = ctx.meta
        dy = dy.contiguous()
        dx = dw = db = None
        with torch.autocast("cuda", enabled=False):
            if ctx.needs_input_grad[0]:
                dx = dy @ wc
                if dx.dtype != xd:
                    dx = dx.to(xd)
            if ctx.needs_input_grad[1]:
                dw = dy.t() @ xc
                if dw.dtype != wd:
                    dw = dw.to(wd)
            if bd is not None and ctx.needs_input_grad[2]:
                db = colsum(dy)
                if db.dtype != bd:
                    db = db.to(bd)
        return dx, dw, db, None


def linear(x, weight, bias, w16=None, b16=None):
    """F.linear for 2-D CUDA inputs with the fused bias gradient; falls back to F.linear otherwise.
    w16 / b16: up-to-date half-precision shadows of weight / bias (HalfShadows); they spare the per-call cast kernels."""
    if x.is_cuda and x.dim() == 2 and weight.shape[0] % 4 == 0 and x.dtype in _DTYPES:
        cdtype = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled() else x.dtype
        B = binding()
        if B is not None:
            return B.linear(x, weight, bias, _DTYPES[cdtype], w16, b16)
        return LinearFn.apply(x, weight, bias, cdtype)
    return torch.nn.functional.linear(x, weight, bias)


def fused_residual(shortcut, x, u=None, keep=1.0, ln_a=None, ln_b=None, emit_half=False, x_bias=None):
    """csrc/fused.cuh through the compiled binding: r = shortcut + dropscale * [LN_a](x); optional half copy of r; optional
    y = LN_b(r) in x's dtype.  ln_a / ln_b: nn.LayerNorm modules or None.  Returns (r, r16 or None, y or None).
    x_bias: bias parameter of the Linear that produced x when that Linear was called with the bias detached -- its gradient
    (column sums of dx) is then produced by this node's backward instead of a separate reduction."""
    B = binding()
    assert B is not None, "fused_residual needs the compiled binding"
    outs = B.fused_residual(shortcut, x, u, float(keep),
                            None if ln_a is None else ln_a.weight, None if ln_a is None else ln_a.bias, 1e-5 if ln_a is None else ln_a.eps,
                            None if ln_b is None else ln_b.weight, None if ln_b is None else ln_b.bias, 1e-5 if ln_b is None else ln_b.eps,
                            bool(emit_half), x_bias)
    r = outs[0]
    r16 = outs[1] if emit_half else None
    y = outs[-1] if ln_b is not None else None
    return r, r16, y


def fused_residual_supported(x, c):
    return binding() is not None and x.is_cuda and x.dim() == 2 and x.dtype in _DTYPES and c in (32, 64, 128, 256, 512)


def gelu(x, x_bias=None):
    """exact (erf) GELU, one kernel per direction through the compiled binding; torch otherwise.
    x_bias: bias of the Linear that produced x when it entered that Linear detached: its gradient (column sums of the GELU
    backward's result) then comes out of the same kernel that computes that result."""
    B = binding()
    if B is not None and x.is_cuda and x.dtype in _DTYPES and x.numel() % 4 == 0:
        return B.gelu(x, x_bias)
    assert x_bias is None
    return torch.nn.functional.gelu(x)


def gelu_fused_ok(x):
    return binding() is not None and x.is_cuda and x.dim() == 2 and x.dtype in _DTYPES and x.shape[1] % 4 == 0


_param_epoch = 0


def bump_param_epoch():
    """Called by writers that modify parameters through raw pointers (optim.FusedAdamW): shadows handed out before are stale."""
    global _param_epoch
    _param_epoch += 1


class HalfShadows:
    """Half-precision shadows of the fp32 parameters that feed GEMM-shaped kernels (Linear and sparse-conv weights / biases).
    autocast re-casts every weight on every forward with one kernel each (~250 launches per PT-v3 step); here ONE launch
    (b2pc_multi_cast) refreshes all shadows whenever a parameter changed (optimizer step, load_state_dict), detected through the
    tensors' version counters.  Modules read ``_w16`` / ``_b16`` only while ``_w16_ver`` matches the parameter's version."""

    def __init__(self, model):
        self.model = model
        self._key = None
        self._ver = None
        self._plan = None
        self._mods = None

    def _modules(self):
        if self._mods is None:
            self._mods = [m for m in self.model.modules() if getattr(m, "_b2pc_half_shadow", False)]
        return self._mods

    @torch.no_grad()
    def sync(self, dtype):
        B = binding()
        if B is None:
            return
        mods = self._modules()
        params = []
        for m in mods:
            params.append(m.weight)
            if m.bias is not None:
                params.append(m.bias)
        if not params or not params[0].is_cuda or any(p.dtype != torch.float32 for p in params):
            return
        key = (dtype, params[0].device, tuple(p.data_ptr() for p in params))
        if key != self._key:
            total = sum((p.numel() + 7) // 8 * 8 for p in params)
            flat = torch.empty(total, dtype=dtype, device=params[0].device)
            shadows, off = [], 0
            for p in params:
                shadows.append(flat[off:off + p.numel()].view(p.shape))
                off += (p.numel() + 7) // 8 * 8
            i = 0
            for m in mods:
                m._w16 = shadows[i]
                i += 1
                if m.bias is not None:
                    m._b16 = shadows[i]
                    i += 1
                else:
                    m._b16 = None
            self._plan = B.make_cast_plan([p.detach() for p in params], shadows)
            self._key, self._ver = key, None
            self._flat = flat
        ver = (sum(p._version for p in params), _param_epoch)
        if ver != self._ver:
            B.run_cast_plan(self._plan[0], self._plan[1], self._plan[2], _DTYPES[dtype])
            self._ver = ver
            for m in mods:
                m._w16_ver = (m.weight._version, _param_epoch)
                m._b16_ver = (m.bias._version, _param_epoch) if m.bias is not None else None


def shadow_of(module, dtype):
    """(w16, b16) of a module managed by HalfShadows if they are current for `dtype`, else (None, None)."""
    w16 = getattr(module, "_w16", None)
    if w16 is None or w16.dtype != dtype or getattr(module, "_w16_ver", None) != (module.weight._version, _param_epoch):
        return None, None
    b16 = getattr(module, "_b16", None)
    if module.bias is not None and (b16 is None or getattr(module, "_b16_ver", None) != (module.bias._version, _param_epoch)):
        return None, None
    return w16, b16


def drop_path_add(shortcut, x, drop_prob, training):
    """shortcut + DropPath(x) (per-row stochastic depth, timm semantics with scale_by_keep) as one kernel when the compiled
    binding is present; plain torch ops otherwise."""
    if drop_prob == 0.0 or not training:
        return shortcut + x
    keep = 1.0 - drop_prob
    B = binding()
    if (B is not None and x.is_cuda and x.dim() == 2 and x.shape[1] % 4 == 0 and shortcut.shape == x.shape
            and x.dtype in _DTYPES and (shortcut.dtype == torch.float32 or shortcut.dtype == x.dtype)):
        return B.drop_path_add(shortcut, x, keep)
    mask = x.new_empty((x.shape[0], 1)).bernoulli_(keep)
    if keep > 0.0:
        mask.div_(keep)
    return shortcut + x * mask


# ------------------------------------------------------------------------------------------------
# GPU voxelisation / collate (SURVEY 8(f).3; pointcept/datasets/transform.py:840-958, datasets/utils.py:19-73)
# ------------------------------------------------------------------------------------------------
class GridSamplePlan:
    """Device-side result of b2pc_grid_sample_plan for a batch of raw scenes (see include/b2pc.h)."""
    __slots__ = ("coord", "offset", "offset_host", "grid_size", "math_f64", "grid_coord", "inverse", "sort_index", "vox_start",
                 "vox_count", "meta", "m", "new_offset_host", "count_max_host", "min_cell_host")

    def select(self, mode, arg):
        """idx [M] int64: one member of every voxel; mode "train" (arg = seed) or "test" (arg = fragment number)."""
        idx = torch.empty(self.m, dtype=torch.int64, device=self.coord.device)
        if self.m:
            _lib.check(_lib.lib().b2pc_grid_sample_select(_p(self.sort_index), _p(self.vox_start), _p(self.vox_count), _p(self.meta),
                                                          len(self.offset_host), self.m, 0 if mode == "train" else 1,
                                                          ctypes.c_uint64(int(arg) & 0xFFFFFFFFFFFFFFFF), _p(idx), _stream()), "grid_sample_select")
        return idx

    def displacement(self, idx, out_dtype=None):
        out_dtype = out_dtype or torch.float64      # numpy promotes `scaled - grid_coord(int64) - 0.5` to float64 in either mode
        out = torch.empty((idx.shape[0], 3), dtype=out_dtype, device=idx.device)
        g = (ctypes.c_double * 3)(*self.grid_size)
        if idx.shape[0]:
            _lib.check(_lib.lib().b2pc_grid_sample_displacement(_p(self.coord), _p(idx), _p(self.meta), len(self.offset_host), idx.shape[0], g,
                                                                int(self.math_f64), _p(out), int(out_dtype == torch.float64), _stream()),
                       "grid_sample_displacement")
        return out


@torch.no_grad()
def grid_sample_plan(coord, offset_host, grid_size, hash_type="fnv", math="float64"):
    """Voxelise B concatenated raw scenes in one pass.  coord [N,3] fp32 CUDA, offset_host: cumulative scene sizes (python ints),
    grid_size scalar or 3 values.  One host read (voxel counts) at the end -- the only synchronisation."""
    _need_cuda(coord)
    coord = coord if (coord.dtype == torch.float32 and coord.is_contiguous()) else coord.float().contiguous()
    offset_host = [int(x) for x in offset_host]
    n, nb = coord.shape[0], len(offset_host)
    sizes = [offset_host[0]] + [offset_host[i] - offset_host[i - 1] for i in range(1, nb)]
    if nb == 0 or offset_host[-1] != n or min(sizes) <= 0:
        raise ValueError("grid_sample_plan: offset must be the cumulative sizes of non-empty scenes and end at len(coord)")
    gs = [float(grid_size)] * 3 if not hasattr(grid_size, "__len__") else [float(x) for x in grid_size]
    assert len(gs) == 3 and hash_type in ("fnv", "ravel") and math in ("float64", "float32")
    dev = coord.device
    plan = GridSamplePlan()
    plan.coord, plan.offset_host, plan.grid_size, plan.math_f64 = coord, offset_host, gs, math == "float64"
    plan.offset = torch.tensor(offset_host, dtype=torch.int64).to(dev, non_blocking=True)
    plan.grid_coord = torch.empty((n, 3), dtype=torch.int64, device=dev)
    plan.inverse = torch.empty(n, dtype=torch.int64, device=dev)
    plan.sort_index = torch.empty(n, dtype=torch.int64, device=dev)
    plan.vox_start = torch.empty(n, dtype=torch.int64, device=dev)
    plan.vox_count = torch.empty(n, dtype=torch.int64, device=dev)
    plan.meta = torch.empty(1 + 5 * nb, dtype=torch.int64, device=dev)
    L = _lib.lib()
    row = max(sizes)
    ws = _ws(L.b2pc_grid_sample_workspace_bytes(n, nb, row), dev)
    g = (ctypes.c_double * 3)(*gs)
    _lib.check(L.b2pc_grid_sample_plan(_p(coord), _p(plan.offset), nb, n, row, g, 0 if hash_type == "fnv" else 1, int(plan.math_f64),
                                       _p(plan.grid_coord), _p(plan.inverse), _p(plan.sort_index), _p(plan.vox_start), _p(plan.vox_count),
                                       _p(plan.meta), _p(ws), ws.numel(), _stream()), "grid_sample_plan")
    meta = plan.meta.tolist()   # the one host read
    plan.m = meta[0]
    plan.new_offset_host = meta[1:1 + nb]
    plan.count_max_host = meta[1 + nb:1 + 2 * nb]
    plan.min_cell_host = [meta[1 + 2 * nb + 3 * b:1 + 2 * nb + 3 * b + 3] for b in range(nb)]
    plan.vox_start, plan.vox_count = plan.vox_start[:plan.m], plan.vox_count[:plan.m]
    return plan


@torch.no_grad()
def gather_rows(src, idx):
    """src[idx] for a row-major tensor of any dtype (index_operator, transform.py:24-40)."""
    _need_cuda(src, idx)
    src = src.contiguous()
    idx = idx if (idx.dtype == torch.int64 and idx.is_contiguous()) else idx.long().contiguous()
    out = torch.empty((idx.shape[0],) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    row_bytes = src.element_size() * (src[0].numel() if src.shape[0] else 1)
    if idx.shape[0] and row_bytes:
        _lib.check(_lib.lib().b2pc_gather_rows(_p(src), row_bytes, _p(idx), idx.shape[0], _p(out), _stream()), "gather_rows")
    return out


# ------------------------------------------------------------------------------------------------
# variants sharing the kernels (SURVEY 8(f).4): kNN query, fragment voting, PointROPE
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
def knn_query(nsample, xyz, offset, new_xyz=None, new_offset=None):
    """pointops.knn_query (libs/pointops/functions/query.py:7-26): -> idx [m,nsample] int32 (-1 placeholder), dist [m,nsample]."""
    if new_xyz is None or new_offset is None:
        new_xyz, new_offset = xyz, offset
    _need_cuda(xyz, new_xyz, offset, new_offset)
    assert xyz.is_contiguous() and new_xyz.is_contiguous() and xyz.dtype == torch.float32 and new_xyz.dtype == torch.float32
    offset, new_offset = offset.int().contiguous(), new_offset.int().contiguous()
    m = new_xyz.shape[0]
    idx = torch.empty((m, nsample), dtype=torch.int32, device=xyz.device)
    dist2 = torch.empty((m, nsample), dtype=torch.float32, device=xyz.device)
    _lib.check(_lib.lib().b2pc_knn_query(_p(xyz), _p(offset), _p(new_xyz), _p(new_offset), offset.shape[0], m, int(nsample), _p(idx), _p(dist2),
                                         _stream()), "knn_query")
    return idx, torch.sqrt(dist2)


@torch.no_grad()
def vote_accumulate(pred, index, logits):
    """pred[index] += softmax(logits, -1) in place (pointcept/engines/test.py:193-203); pred fp32 [N, C]."""
    _need_cuda(pred, index, logits)
    assert pred.dtype == torch.float32 and pred.is_contiguous() and logits.shape[1] == pred.shape[1]
    logits = logits.contiguous()
    index = index if (index.dtype == torch.int64 and index.is_contiguous()) else index.long().contiguous()
    _lib.check(_lib.lib().b2pc_vote_accumulate(_p(logits), _DTYPES[logits.dtype], _p(index), logits.shape[0], logits.shape[1], _p(pred), _stream()),
               "vote_accumulate")
    return pred


def _point_rope_(tokens, pos, n_tokens, token_stride, n_heads, head_dim, base, fwd):
    _lib.check(_lib.lib().b2pc_point_rope(_p(tokens), _DTYPES[tokens.dtype], _p(pos), n_tokens, token_stride, n_heads, head_dim, float(base),
                                          float(fwd), _stream()), "point_rope")


def pointrope_(tokens, positions, base, fwd):
    """The ``pointrope.pointrope(tokens, positions, base, F0)`` entry point (libs/pointrope/pointrope.cpp): tokens [B,N,H,D] rotated IN
    PLACE, positions [B,N,3] int64."""
    _need_cuda(tokens, positions)
    assert tokens.dim() == 4 and tokens.is_contiguous(), "tokens are not contiguous"
    b, n, h, d = tokens.shape
    assert positions.is_contiguous() and tuple(positions.shape) == (b, n, 3), "bad pos.shape"
    assert d % 6 == 0, "token dim must be multiple of 6"
    positions = positions if positions.dtype == torch.int64 else positions.long()
    _point_rope_(tokens, positions, b * n, h * d, h, d, base, fwd)
    return tokens


class _RopeQKV(torch.autograd.Function):
    """LitePT's q/k rotation (litept_v1.py:231-250) fused on the packed tensor: qkv [T,3,H,D] -> same layout with q and k rotated;
    replaces two float casts, four transposes, two rope launches, a stack and a cast.  Backward = rotation by the negative angle."""

    @staticmethod
    def forward(ctx, qkv, pos, base, f0):
        out = qkv.clone()
        t, _, h, d = out.shape
        _point_rope_(out, pos, t, 3 * h * d, 2 * h, d, base, f0)
        ctx.save_for_backward(pos)
        ctx.base, ctx.f0 = base, f0
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.clone().contiguous()
        t, _, h, d = g.shape
        _point_rope_(g, ctx.saved_tensors[0], t, 3 * h * d, 2 * h, d, ctx.base, -ctx.f0)
        return g, None, None, None


def rope_qkv(qkv, pos, base=100.0, f0=1.0):
    _need_cuda(qkv, pos)
    assert qkv.dim() == 4 and qkv.shape[1] == 3 and qkv.is_contiguous() and qkv.shape[3] % 6 == 0
    pos = pos.reshape(-1, 3)
    pos = pos if (pos.dtype == torch.int64 and pos.is_contiguous()) else pos.long().contiguous()
    assert pos.shape[0] == qkv.shape[0]
    return _RopeQKV.apply(qkv, pos, float(base), float(f0))


# ------------------------------------------------------------------------------------------------
# fused cross-entropy (pointcept/models/losses/misc.py:13-40)
# ------------------------------------------------------------------------------------------------
class _CrossEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, ignore_index):
        _need_cuda(logits, target)
        logits = logits.contiguous()
        target = target if (target.dtype == torch.int64 and target.is_contiguous()) else target.long().contiguous()
        n, c = logits.shape
        L = _lib.lib()
        lse = torch.empty(n, dtype=torch.float32, device=logits.device)
        loss_count = torch.empty(2, dtype=torch.float32, device=logits.device)
        ws = _ws(L.b2pc_cross_entropy_workspace_bytes(n), logits.device)
        _lib.check(L.b2pc_cross_entropy_fwd(_p(logits), _DTYPES[logits.dtype], _p(target), n, c, int(ignore_index), _p(lse), _p(loss_count), _p(ws),
                                            ws.numel(), _stream()), "cross_entropy_fwd")
        ctx.save_for_backward(logits, target, lse, loss_count)
        ctx.ignore_index = int(ignore_index)
        return loss_count[0]

    @staticmethod
    def backward(ctx, g):
        logits, target, lse, loss_count = ctx.saved_tensors
        n, c = logits.shape
        g = g.detach().float().reshape(1).contiguous()
        d = torch.empty_like(logits)
        _lib.check(_lib.lib().b2pc_cross_entropy_bwd(_p(logits), _DTYPES[logits.dtype], _p(target), _p(lse), _p(g), _p(loss_count), n, c,
                                                     ctx.ignore_index, _p(d), _stream()), "cross_entropy_bwd")
        return d, None, None


def cross_entropy(logits, target, ignore_index=-1):
    """nn.functional.cross_entropy(logits, target, ignore_index=...) with reduction="mean" -> scalar fp32 loss."""
    assert logits.dim() == 2 and target.dim() == 1 and target.shape[0] == logits.shape[0] and logits.shape[0] > 0
    return _CrossEntropy.apply(logits, target, ignore_index)
