"""BASELINE.md B2 comparator: the reference's GPU path for the same PT-v3m1 / SpUNet step on the same GPU.

What the reference runs on a GPU is third-party: flash-attn 2.8.3 (when installed; the FA2 mma.sync
kernels) and spconv (NOT installable offline: `pip install spconv-cu124 / -cu126` finds no matching distribution).  This module re-wires the mirror models
of this repo onto that stack:
  * attention   -> stock ``flash_attn.flash_attn_varlen_qkvpacked_func`` (the exact call of ptv3m1:208-214)
  * sparse conv -> torch-native rulebook convolution, per kernel offset gather -> ``mm`` -> ``index_add_`` (spconv's "Native"
                   algorithm expressed with library ops), explicit backward with the same three ops
  * glue        -> stock torch: nn.LayerNorm, nn.Linear, advanced indexing for the [order] / [inverse] gathers (ptv3m1:188,216),
                   ``torch.segment_reduce`` for the pooling (torch_scatter is not in the image), plain DropPath
Index-side work (serialization, padding tables, rulebooks) stays on this repo's kernels in BOTH arms -- the reference would use
spconv's hash tables and torch.argsort there -- which only makes this comparator faster than the real reference, never slower.
Nothing here is on the product path; only bench.py's ``gpu_reference`` leg and tools/ import it.
"""
import contextlib

import torch

from pointcept_b200 import ops
from pointcept_b200 import ptv3 as _ptv3


def _pair_lists(pair):
    """dense table [KV, N_out] -> per-offset (in_rows, out_rows) index tensors; two host syncs per rulebook (spconv's native
    path copies its per-offset pair counts to the host as well)."""
    cache = getattr(pair, "_b2_ref_lists", None)
    if cache is not None:
        return cache
    valid = pair >= 0
    counts = valid.sum(1).tolist()
    kj = torch.nonzero(valid)
    out_rows = kj[:, 1].split(counts)
    in_rows = pair[valid].long().split(counts)
    lists = [(i, o) if c else None for c, i, o in zip(counts, in_rows, out_rows)]
    try:
        pair._b2_ref_lists = lists
    except Exception:
        pass
    return lists


class _NativeConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, weight, bias, table_fwd):
        lists = _pair_lists(table_fwd)
        w = weight.to(feat.dtype)
        n_out = table_fwd.shape[1]
        out = feat.new_zeros((n_out, w.shape[0])) if bias is None else bias.to(feat.dtype).expand(n_out, -1).contiguous()
        for k, l in enumerate(lists):
            if l is not None:
                out.index_add_(0, l[1], feat.index_select(0, l[0]) @ w[:, k, :].t())
        ctx.save_for_backward(feat, w)
        ctx.lists, ctx.has_bias, ctx.wdtype = lists, bias is not None, weight.dtype
        return out

    @staticmethod
    def backward(ctx, dout):
        feat, w = ctx.saved_tensors
        dout = dout.to(feat.dtype)
        dfeat = torch.zeros_like(feat)
        dw = torch.zeros(w.shape, dtype=torch.float32, device=w.device)
        for k, l in enumerate(ctx.lists):
            if l is not None:
                g = dout.index_select(0, l[1])
                dfeat.index_add_(0, l[0], g @ w[:, k, :])
                dw[:, k, :] = (g.t() @ feat.index_select(0, l[0])).float()
        db = dout.float().sum(0) if ctx.has_bias else None
        return dfeat, dw.to(ctx.wdtype), db, None


def native_sparse_conv(feat, weight, bias, table_fwd, table_bwd, flip_bwd, w16=None, b16=None):
    return _NativeConvFn.apply(feat, weight, bias, table_fwd)


def _segment_max(x, order, seg_start, seg_len):
    return torch.segment_reduce(x.index_select(0, order), "max", lengths=seg_len, axis=0, unsafe=True)


def _drop_path_add(shortcut, x, drop_prob, training):
    if drop_prob == 0.0 or not training:
        return shortcut + x
    keep = 1.0 - drop_prob
    mask = x.new_empty((x.shape[0], 1)).bernoulli_(keep).div_(keep)
    return shortcut + x * mask


def stock_flash_attn():
    import flash_attn
    if "b2pc" in getattr(flash_attn, "__version__", ""):
        raise RuntimeError("the name flash_attn resolves to this repo's drop-in, not the stock package")
    return flash_attn.flash_attn_varlen_qkvpacked_func, flash_attn.__version__


@contextlib.contextmanager
def reference_gpu_ops():
    """Inside this context the mirror models run on the stock library stack described in the module docstring."""
    fa, _ = stock_flash_attn()

    def fa_call(qkv, cu_seqlens, max_seqlen, dropout_p=0.0, softmax_scale=None, **kw):
        return fa(qkv, cu_seqlens, max_seqlen, dropout_p=dropout_p, softmax_scale=softmax_scale)

    saved = dict(sparse_conv=ops.sparse_conv, layer_norm_supported=ops.layer_norm_supported, segment_max=ops.segment_max,
                 unpool_add=ops.unpool_add, drop_path_add=ops.drop_path_add, binding=ops.binding)
    saved_ptv3 = dict(fa=_ptv3.flash_attn_varlen_qkvpacked_func, g=_ptv3.serialized_gather, s=_ptv3.serialized_scatter_back,
                      fl=_ptv3.FusedLinear.use_fused_bias_grad, loss=_ptv3._FUSED_LOSS)
    _ptv3._FUSED_LOSS = False
    ops.sparse_conv = native_sparse_conv
    ops.layer_norm_supported = lambda x, c: False
    ops.segment_max = _segment_max
    ops.unpool_add = lambda parent, child, cluster, order, seg_len: parent + child[cluster]
    ops.drop_path_add = _drop_path_add
    ops.binding = lambda: None
    _ptv3.flash_attn_varlen_qkvpacked_func = fa_call
    _ptv3.serialized_gather = lambda x, order_pad, primary_pos, offset_host, K, dup=None: x[order_pad]
    _ptv3.serialized_scatter_back = lambda x_pad, primary_pos: x_pad[primary_pos]
    _ptv3.FusedLinear.use_fused_bias_grad = False
    try:
        yield
    finally:
        for k, v in saved.items():
            setattr(ops, k, v)
        _ptv3.flash_attn_varlen_qkvpacked_func = saved_ptv3["fa"]
        _ptv3.serialized_gather, _ptv3.serialized_scatter_back = saved_ptv3["g"], saved_ptv3["s"]
        _ptv3.FusedLinear.use_fused_bias_grad = saved_ptv3["fl"]
        _ptv3._FUSED_LOSS = saved_ptv3["loss"]


DESCRIPTION = ("same step on the reference's GPU stack: stock flash-attn {fa} (FA2 mma.sync kernels) for the patch "
               "attention, torch-native gather->mm->index_add_ rulebook convolution (spconv is not installable offline), torch "
               "LayerNorm/Linear/indexing glue; index-side tables from this repo's kernels in both arms")
