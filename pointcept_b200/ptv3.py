"""PT-v3m1 backbone on the CUDA operators: host-side mirror of
pointcept/models/point_transformer_v3/point_transformer_v3m1_base.py (module tree, parameter names and
shapes identical, so reference checkpoints load), used as the workload of bench.py and the parity tests.

Differences in HOW (not WHAT): serialization / padding tables / attention / CPE convolutions are the
libb2pc kernels; the padding tables and gather indices are built once per stage on the device without
the reference's per-scene python loop; pooling clusters come from the already-sorted order-0 codes
instead of torch.unique + torch.sort.
"""
import math
import os
from functools import partial

import torch
import torch.nn as nn

from . import ops
from .flash_attn_interface import flash_attn_varlen_qkvpacked_func
from .spconv import pytorch as spconv
from .structure import Point, PointModule, PointSequential


class DropPath(nn.Module):
    """Stochastic depth per row (timm.layers.DropPath semantics, as used at ptv3m1:313-315)."""

    def __init__(self, drop_prob=0.0, scale_by_keep=True):
        super().__init__()
        self.drop_prob, self.scale_by_keep = drop_prob, scale_by_keep

    def forward(self, x):
        if self.drop_prob == 0.0 or not self.training:
            return x
        keep = 1 - self.drop_prob
        mask = x.new_empty((x.shape[0],) + (1,) * (x.dim() - 1)).bernoulli_(keep)
        if keep > 0.0 and self.scale_by_keep:
            mask.div_(keep)
        return x * mask


class FusedLayerNorm(nn.LayerNorm):
    """nn.LayerNorm (same parameters / state_dict) whose forward + backward are single fused kernels for [N, C] point features."""

    emit_autocast_dtype = False   # set on instances whose only consumer is an autocast Linear (pre-norms of attention / MLP)

    def forward(self, x):
        if self.elementwise_affine and len(self.normalized_shape) == 1 and ops.layer_norm_supported(x, self.normalized_shape[0]):
            return ops.layer_norm(x, self.weight, self.bias, self.eps, self.emit_autocast_dtype)
        return super().forward(x)


class FusedLinear(nn.Linear):
    """nn.Linear (same parameters).  With ``FusedLinear.use_fused_bias_grad = True`` it routes through ops.linear (identical
    math, fp32 column-sum kernel for the bias gradient: 4.3 -> 1.8 ms of GPU time per PT-v3-base step).  Off by default:
    at 2 scenes per GPU the step is host-bound and a *Python* autograd.Function per Linear costs more host time than the
    kernel saves (measured 48.7 -> 56.5 ms per step), so by default it is used only through the compiled binding."""

    use_fused_bias_grad = None   # None: on exactly when the compiled binding is present (its C++ node is cheaper than autograd's)
    _b2pc_half_shadow = True     # ops.HalfShadows keeps half-precision copies of weight / bias for the autocast path

    def forward(self, x, bias_grad_elsewhere=False):
        """bias_grad_elsewhere: the caller routes the bias gradient through the fused residual kernel that consumes this
        layer's output (ops.fused_residual(..., x_bias=self.bias)); the bias then enters detached here."""
        on = FusedLinear.use_fused_bias_grad
        if on is None:
            on = ops.binding() is not None
        if on:
            w16 = b16 = None
            if torch.is_autocast_enabled():
                w16, b16 = ops.shadow_of(self, torch.get_autocast_dtype("cuda"))
            bias = self.bias.detach() if (bias_grad_elsewhere and self.bias is not None) else self.bias
            return ops.linear(x, self.weight, bias, w16, b16)
        assert not bias_grad_elsewhere
        return nn.functional.linear(x, self.weight, self.bias)


class _SerializedGather(torch.autograd.Function):
    """y = x[order_pad]  (rows into patch order, ptv3m1:188).  Every point sits at exactly one primary padded slot
    (primary_pos) and at most once more as a borrowed filler of its scene's last patch (dup_slots -> dup_points), so the
    backward is a gather plus a tiny unique-index add -- no sort-based index_put."""

    @staticmethod
    def forward(ctx, x, order_pad, primary_pos, dup_slots, dup_points):
        ctx.save_for_backward(primary_pos, dup_slots, dup_points)
        return x.index_select(0, order_pad)

    @staticmethod
    def backward(ctx, dy):
        primary_pos, dup_slots, dup_points = ctx.saved_tensors
        dx = dy.index_select(0, primary_pos)
        if dup_slots.numel() > 0:
            dx.index_add_(0, dup_points, dy.index_select(0, dup_slots))
        return dx, None, None, None, None


class _SerializedScatterBack(torch.autograd.Function):
    """y = x_pad[primary_pos]  (patch order back to point order, ptv3m1:216); backward writes each row to its unique slot."""

    @staticmethod
    def forward(ctx, x_pad, primary_pos):
        ctx.save_for_backward(primary_pos)
        ctx.t_pad = x_pad.shape[0]
        return x_pad.index_select(0, primary_pos)

    @staticmethod
    def backward(ctx, dy):
        (primary_pos,) = ctx.saved_tensors
        dx = dy.new_zeros((ctx.t_pad,) + tuple(dy.shape[1:]))
        dx.index_copy_(0, primary_pos, dy)
        return dx, None


def borrowed_slots(offset_host, K, device):
    """Padded slots that hold a BORROWED token (the last K - n%K slots of a padded scene repeat the K - n%K tokens in front of
    the scene's last patch, ptv3m1:144-154); host arithmetic on the scene sizes, no sync."""
    slots, op = [], 0
    for a, b in zip([0] + list(offset_host[:-1]), offset_host):
        n = b - a
        npad = ((n + K - 1) // K * K) if n > K else n
        if npad != n:
            slots.append(torch.arange(op + npad - (K - n % K), op + npad, device=device))
        op += npad
    return torch.cat(slots) if slots else torch.zeros(0, dtype=torch.long, device=device)


def serialized_gather(x, order_pad, primary_pos, offset_host, K, dup=None):
    """x[order_pad] with the structured (sort-free) backward; compiled node when the binding is built."""
    if dup is None:
        ds = borrowed_slots(offset_host, K, x.device)
        dup = (ds, order_pad[ds])
    B = ops.binding()
    if B is not None:
        return B.serialized_gather(x, order_pad, primary_pos, dup[0], dup[1])
    return _SerializedGather.apply(x, order_pad, primary_pos, dup[0], dup[1])


def serialized_scatter_back(x_pad, primary_pos):
    B = ops.binding()
    if B is not None:
        return B.serialized_scatter_back(x_pad, primary_pos)
    return _SerializedScatterBack.apply(x_pad, primary_pos)


class RPE(nn.Module):
    """Relative position bias of the non-flash branch (ptv3m1:29-48): per-axis tables indexed by the clamped grid offset of every
    (query, key) pair of a patch, summed over the three axes.  Parameter name and shape as in the reference (checkpoint ABI)."""

    def __init__(self, patch_size, num_heads):
        super().__init__()
        self.patch_size, self.num_heads = patch_size, num_heads
        self.pos_bnd = int((4 * patch_size) ** (1 / 3) * 2)
        self.rpe_num = 2 * self.pos_bnd + 1
        self.rpe_table = nn.Parameter(torch.zeros(3 * self.rpe_num, num_heads))
        nn.init.trunc_normal_(self.rpe_table, std=0.02)

    def forward(self, rel):                                                   # rel [P, K, K, 3] integer grid offsets
        axis_base = torch.arange(3, device=rel.device) * self.rpe_num
        rows = rel.clamp(-self.pos_bnd, self.pos_bnd) + self.pos_bnd + axis_base
        bias = self.rpe_table.index_select(0, rows.reshape(-1)).view(rows.shape + (-1,)).sum(3)   # [P, K, K, H]
        return bias.permute(0, 3, 1, 2)


class SerializedAttention(PointModule):
    """ptv3m1:51-222.  enable_flash=True (every stock config) is the operator path of this library; enable_flash=False is the
    reference's own eager branch (dense per-patch softmax with optional RPE bias and fp32 upcasts, ptv3m1:173-206) -- there is no
    third-party operator behind it in the reference either, so it is mirrored with the same torch ops on the patch tables
    built by the library."""

    def __init__(self, channels, num_heads, patch_size, qkv_bias=True, qk_scale=None, attn_drop=0.0, proj_drop=0.0,
                 order_index=0, enable_rpe=False, enable_flash=True, upcast_attention=False, upcast_softmax=False):
        super().__init__()
        assert channels % num_heads == 0
        self.enable_flash, self.enable_rpe = enable_flash, enable_rpe
        self.upcast_attention, self.upcast_softmax = upcast_attention, upcast_softmax
        if enable_flash:
            assert not enable_rpe, "Set enable_rpe to False when enable Flash Attention"
            assert not upcast_attention, "Set upcast_attention to False when enable Flash Attention"
            assert not upcast_softmax, "Set upcast_softmax to False when enable Flash Attention"
            if attn_drop != 0.0:
                raise NotImplementedError("attn_drop > 0 is not supported on the operator path (all PT-v3 configs use 0.0)")
            self.patch_size = patch_size
        else:
            self.patch_size_max, self.patch_size = patch_size, 0      # set per call to min(patch_size_max, smallest scene)
            self.attn_drop = nn.Dropout(attn_drop)
            self.softmax = nn.Softmax(dim=-1)
        self.channels, self.num_heads = channels, num_heads
        self.scale = qk_scale or (channels // num_heads) ** -0.5
        self.order_index = order_index
        self.qkv = FusedLinear(channels, channels * 3, bias=qkv_bias)
        self.proj = FusedLinear(channels, channels)
        self.proj_drop = nn.Dropout(proj_drop)
        self.rpe = RPE(patch_size, num_heads) if enable_rpe else None

    def _forward_dense(self, point):
        """non-flash branch (ptv3m1:173-206): every patch is a dense [K, K] softmax; the patch size shrinks to the smallest scene
        so that no mask is needed"""
        oh = point.host_offset()
        self.patch_size = min(min(b - a for a, b in zip([0] + list(oh[:-1]), oh)), self.patch_size_max)
        H, K, C = self.num_heads, self.patch_size, self.channels
        pad, unpad, _ = self.get_padding_and_inverse(point)
        order = point.serialized_order[self.order_index][pad]
        inverse = unpad[point.serialized_inverse[self.order_index]]
        qkv = self.qkv(point.feat)[order]
        q, k, v = qkv.reshape(-1, K, 3, H, C // H).permute(2, 0, 3, 1, 4).unbind(0)        # each [P, H, K, D]
        if self.upcast_attention:
            q, k = q.float(), k.float()
        logits = (q * self.scale) @ k.transpose(-2, -1)
        if self.enable_rpe:
            key = f"rel_pos_{self.order_index}"
            if key not in point:
                g = point.grid_coord[order].reshape(-1, K, 3)
                point[key] = g.unsqueeze(2) - g.unsqueeze(1)
            logits = logits + self.rpe(point[key])
        if self.upcast_softmax:
            logits = logits.float()
        prob = self.attn_drop(self.softmax(logits)).to(qkv.dtype)
        feat = (prob @ v).transpose(1, 2).reshape(-1, C)[inverse]
        point.feat = self.proj_drop(self.proj(feat))
        return point

    @torch.no_grad()
    def get_padding_and_inverse(self, point):
        if "pad" not in point or "unpad" not in point or "cu_seqlens_key" not in point:
            pad, unpad, cu = ops.patch_padding(point.offset, point.host_offset(), self.patch_size)
            point["pad"], point["unpad"], point["cu_seqlens_key"] = pad, unpad, cu
        return point["pad"], point["unpad"], point["cu_seqlens_key"]

    @torch.no_grad()
    def _gather_indices(self, point):
        key = f"_attn_idx_{self.order_index}"
        if key not in point:
            pad, unpad, _ = self.get_padding_and_inverse(point)
            order_pad = point.serialized_order[self.order_index][pad]
            primary_pos = unpad[point.serialized_inverse[self.order_index]]
            dup_slots = borrowed_slots(point.host_offset(), self.patch_size, pad.device)
            point[key] = (order_pad, primary_pos, dup_slots, order_pad[dup_slots])
        return point[key]

    # class switch: gather-fused serialized attention (one operator) when the compiled binding + tensor-core path apply
    fused = os.environ.get("B2PC_ATTN_FUSED", "1") != "0"

    @torch.no_grad()
    def _fused_tables(self, point):
        """int32 tables of the gather-fused operator: gidx[t] = point row read by padded slot t; sidx[t] = point row written by
        slot t (its primary slot) or -(r+1) for the r-th borrowed filler slot; dup_point[r] = the point behind filler r."""
        key = f"_attn_fused_{self.order_index}"
        if key not in point:
            order_pad, _, dup_slots, dup_points = self._gather_indices(point)
            gidx = order_pad.int()
            sidx = gidx.clone()
            if dup_slots.numel() > 0:
                sidx[dup_slots] = -(torch.arange(dup_slots.numel(), device=gidx.device, dtype=torch.int32) + 1)
            point[key] = (gidx, sidx, dup_points.int())
        return point[key]

    def forward(self, point, proj_bias_grad_elsewhere=False):
        if not self.enable_flash:
            return self._forward_dense(point)
        H, K, C = self.num_heads, self.patch_size, self.channels
        _, _, cu_seqlens = self.get_padding_and_inverse(point)
        B = ops.binding()
        ext = proj_bias_grad_elsewhere and self.proj_drop.p == 0.0
        if B is not None and SerializedAttention.fused and C // H == 16 and ops.get_impl() != 1 and point.feat.is_cuda:
            gidx, sidx, dup_point = self._fused_tables(point)
            qkv = self.qkv(point.feat)
            # bf16 at the operator boundary whatever the autocast dtype, exactly as the reference (ptv3m1:209)
            feat = B.serialized_attention(qkv.to(torch.bfloat16), gidx, sidx, dup_point, cu_seqlens, K, H, float(self.scale)).to(qkv.dtype)
            point.feat = self.proj(feat, bias_grad_elsewhere=True) if ext else self.proj_drop(self.proj(feat))
            return point
        order_pad, primary_pos, dup_slots, dup_points = self._gather_indices(point)
        qkv = serialized_gather(self.qkv(point.feat), order_pad, primary_pos, None, K, dup=(dup_slots, dup_points))
        # bf16 at the operator boundary whatever the autocast dtype, exactly as the reference (ptv3m1:209)
        feat = flash_attn_varlen_qkvpacked_func(qkv.to(torch.bfloat16).reshape(-1, 3, H, C // H), cu_seqlens, max_seqlen=K,
                                                softmax_scale=self.scale).reshape(-1, C)
        feat = serialized_scatter_back(feat.to(qkv.dtype), primary_pos)
        point.feat = self.proj(feat, bias_grad_elsewhere=True) if ext else self.proj_drop(self.proj(feat))
        return point


class MLP(nn.Module):
    def __init__(self, in_channels, hidden_channels=None, out_channels=None, act_layer=nn.GELU, drop=0.0):
        super().__init__()
        out_channels = out_channels or in_channels
        hidden_channels = hidden_channels or in_channels
        self.fc1 = FusedLinear(in_channels, hidden_channels)
        self.act = act_layer()
        self.fc2 = FusedLinear(hidden_channels, out_channels)
        self.drop = nn.Dropout(drop)

    def forward(self, x, fc2_bias_grad_elsewhere=False):
        exact_gelu = type(self.act) is nn.GELU and self.act.approximate == "none"
        if exact_gelu and self.fc1.bias is not None and ops.gelu_fused_ok(x) and isinstance(self.fc1, FusedLinear):
            # fc1's bias gradient = column sums of the GELU backward's result: produced by that kernel, no separate reduction
            h = ops.gelu(self.fc1(x, bias_grad_elsewhere=True), self.fc1.bias)
        else:
            h = self.fc1(x)
            h = ops.gelu(h) if exact_gelu else self.act(h)
        if fc2_bias_grad_elsewhere and self.drop.p == 0.0:
            return self.fc2(h, bias_grad_elsewhere=True)
        return self.drop(self.fc2(self.drop(h)))


class Block(PointModule):
    """ptv3m1:251-338: CPE (SubMConv3d k3 -> Linear -> LN) + attention + MLP, pre- or post-norm."""

    def __init__(self, channels, num_heads, patch_size=48, mlp_ratio=4.0, qkv_bias=True, qk_scale=None, attn_drop=0.0,
                 proj_drop=0.0, drop_path=0.0, norm_layer=nn.LayerNorm, act_layer=nn.GELU, pre_norm=True, order_index=0,
                 cpe_indice_key=None, enable_rpe=False, enable_flash=True, upcast_attention=False, upcast_softmax=False):
        super().__init__()
        self.channels, self.pre_norm = channels, pre_norm
        self.cpe = PointSequential(
            spconv.SubMConv3d(channels, channels, kernel_size=3, bias=True, indice_key=cpe_indice_key),
            FusedLinear(channels, channels),
            norm_layer(channels),
        )
        self.norm1 = PointSequential(norm_layer(channels))
        self.attn = SerializedAttention(channels=channels, patch_size=patch_size, num_heads=num_heads, qkv_bias=qkv_bias,
                                        qk_scale=qk_scale, attn_drop=attn_drop, proj_drop=proj_drop, order_index=order_index,
                                        enable_rpe=enable_rpe, enable_flash=enable_flash, upcast_attention=upcast_attention,
                                        upcast_softmax=upcast_softmax)
        self.norm2 = PointSequential(norm_layer(channels))
        self.mlp = PointSequential(MLP(in_channels=channels, hidden_channels=int(channels * mlp_ratio), out_channels=channels,
                                       act_layer=act_layer, drop=proj_drop))
        self.drop_path = PointSequential(DropPath(drop_path) if drop_path > 0.0 else nn.Identity())
        if pre_norm:
            for seq in (self.norm1, self.norm2):
                if isinstance(seq[0], FusedLayerNorm):
                    seq[0].emit_autocast_dtype = True

    # class switch: one fused residual kernel per sub-layer (csrc/fused.cuh) when the compiled binding is present
    fused = os.environ.get("B2PC_BLOCK_FUSED", "1") != "0"

    def _drop_rand(self, point, n, dev):
        """uniform randoms for DropPath (one per row), sliced from a pool filled by a single torch.rand per forward"""
        dp = self.drop_path[0]
        prob = dp.drop_prob if isinstance(dp, DropPath) else 0.0
        if prob == 0.0 or not self.training:
            return None, 1.0
        pool = point.get("_dp_pool")
        if pool is None or pool[1] + n > pool[0].numel() or pool[0].device != dev:
            pool = [torch.rand(max(8 * n, 1 << 20), device=dev), 0]
            point["_dp_pool"] = pool
        u = pool[0][pool[1]:pool[1] + n]
        pool[1] += n
        return u, 1.0 - prob

    def _forward_fused(self, point):
        """Same math as forward() below, pre-norm only: CPE(conv -> Linear) -> [LN + residual + LN] -> attention ->
        [DropPath + residual + LN] -> MLP -> [DropPath + residual (+ half copy for the next conv)]: 3 glue kernels per block."""
        ln = FusedLayerNorm
        amp = torch.is_autocast_enabled()
        r0 = point.feat
        if r0.dtype != torch.float32:
            r0 = r0.float()
        n, dev = r0.shape[0], r0.device
        # the three Linears whose outputs feed a fused residual kernel get their bias gradients from that kernel's backward
        # (column sums of dx) instead of a reduction of their own
        ext = self.attn.proj_drop.p == 0.0 and self.mlp[0].drop.p == 0.0 and isinstance(self.cpe[1], FusedLinear)
        sct = self.cpe[0](point.sparse_conv_feat)
        lin = self.cpe[1](sct.features, bias_grad_elsewhere=ext)
        r1, _, y1 = ops.fused_residual(r0, lin, None, 1.0, self.cpe[2], self.norm1[0], False, self.cpe[1].bias if ext else None)
        point.feat = y1
        point = self.attn(point, proj_bias_grad_elsewhere=ext)
        u, keep = self._drop_rand(point, n, dev)
        r2, _, y2 = ops.fused_residual(r1, point.feat, u, keep, None, self.norm2[0], False, self.attn.proj.bias if ext else None)
        m = self.mlp[0](y2, fc2_bias_grad_elsewhere=ext)
        u, keep = self._drop_rand(point, n, dev)
        r3, r16, _ = ops.fused_residual(r2, m, u, keep, None, None, amp and m.dtype != torch.float32, self.mlp[0].fc2.bias if ext else None)
        point.feat = r3
        point.sparse_conv_feat = sct.replace_feature(r3)
        if r16 is not None:
            point.sparse_conv_feat._features_half = r16
        return point

    def forward(self, point):
        if (Block.fused and self.pre_norm and isinstance(self.cpe[2], FusedLayerNorm) and isinstance(self.norm1[0], FusedLayerNorm)
                and isinstance(self.norm2[0], FusedLayerNorm) and ops.fused_residual_supported(point.feat, self.channels)):
            return self._forward_fused(point)
        shortcut = point.feat
        point = self.cpe(point)
        point.feat = shortcut + point.feat
        shortcut = point.feat
        dp = self.drop_path[0]
        dp_prob = dp.drop_prob if isinstance(dp, DropPath) else 0.0
        if self.pre_norm:
            point = self.norm1(point)
        point = self.attn(point)
        point.feat = ops.drop_path_add(shortcut, point.feat, dp_prob, self.training)      # shortcut + drop_path(attn)
        if not self.pre_norm:
            point = self.norm1(point)
        shortcut = point.feat
        if self.pre_norm:
            point = self.norm2(point)
        point = self.mlp(point)
        point.feat = ops.drop_path_add(shortcut, point.feat, dp_prob, self.training)      # shortcut + drop_path(mlp)
        if not self.pre_norm:
            point = self.norm2(point)
        point.sparse_conv_feat = point.sparse_conv_feat.replace_feature(point.feat)
        return point


class SerializedPooling(PointModule):
    """ptv3m1:341-444.  Clusters = runs of equal (code >> 3*pooling_depth) in the order-0 sorted sequence, so
    neither torch.unique nor a second sort is needed; one host sync for the (data dependent) cluster count."""

    def __init__(self, in_channels, out_channels, stride=2, norm_layer=None, act_layer=None, reduce="max",
                 shuffle_orders=True, traceable=True):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        assert stride == 2 ** (math.ceil(stride) - 1).bit_length()
        self.stride = stride
        assert reduce in ["sum", "mean", "min", "max"]
        self.reduce, self.shuffle_orders, self.traceable = reduce, shuffle_orders, traceable
        self.proj = FusedLinear(in_channels, out_channels)
        if norm_layer is not None:
            self.norm = PointSequential(norm_layer(out_channels))
        if act_layer is not None:
            self.act = PointSequential(act_layer())

    @torch.no_grad()
    def plan(self, src):
        """Index side of the pooling (feature independent): clusters, head rows, the pooled level's codes / orders / scene
        sizes.  `src` needs serialized_code/order/depth, batch, grid_coord, offset (+ host companions).  Contains the only
        host syncs of the pooling (cluster count, scene sizes), so PointTransformerV3.forward runs all plans up front, when
        the GPU queue is still empty, instead of stalling in the middle of the feature pipeline."""
        pooling_depth = (math.ceil(self.stride) - 1).bit_length()
        if pooling_depth > src["serialized_depth"]:
            pooling_depth = 0
        n = src["serialized_code"].shape[1]
        order0 = src["serialized_order"][0]
        n_scene = len(src["offset"])
        depth = src["serialized_depth"] - pooling_depth
        key_bits = 3 * depth + max(n_scene - 1, 1).bit_length()
        if order0.is_cuda and n > 0:
            # device plan: 4 small launches + ONE host read (cluster count and per-scene counts together)
            pp = ops.pool_plan(src["serialized_code"], order0, src["batch"], src["grid_coord"], pooling_depth, n_scene)
            cluster, head_pos, head_indices, lengths = pp["cluster"], pp["head_pos"], pp["head_indices"], pp["lengths"]
            code, batch, grid, counts_host = pp["code"], pp["batch"], pp["grid_coord"], pp["counts"]
        else:
            code = src["serialized_code"] >> pooling_depth * 3
            sc = code[0][order0]
            flag = torch.ones_like(sc, dtype=torch.bool)
            flag[1:] = sc[1:] != sc[:-1]
            cid_sorted = torch.cumsum(flag, 0) - 1
            cluster = torch.empty_like(cid_sorted)
            cluster[order0] = cid_sorted
            head_pos = torch.nonzero(flag).squeeze(1)                 # host sync: number of clusters
            head_indices = order0[head_pos]
            lengths = torch.diff(head_pos, append=head_pos.new_full((1,), n))
            code = code[:, head_indices]
            batch = src["batch"][head_indices]
            grid = src["grid_coord"][head_indices] >> pooling_depth
            counts_host = torch.bincount(batch, minlength=n_scene).tolist()
        order, inverse = ops.serialize_sort(code, key_bits)
        if self.shuffle_orders:
            perm = torch.randperm(code.shape[0]).tolist()
            code = torch.stack([code[i] for i in perm])
            order = torch.stack([order[i] for i in perm])
            inverse = torch.stack([inverse[i] for i in perm])
        off, acc = [], 0
        for c in counts_host:
            acc += c
            off.append(acc)
        out = dict(order0=order0, lengths=lengths, head_pos=head_pos, head_indices=head_indices, cluster=cluster,
                   pooling_depth=pooling_depth,
                   serialized_code=code, serialized_order=order, serialized_inverse=inverse, serialized_depth=depth, batch=batch,
                   grid_coord=grid, offset_host=off,
                   offset=torch.tensor(off, device=batch.device, dtype=src["offset"].dtype))
        if "grid_max_host" in src:
            out["grid_max_host"] = [g >> pooling_depth for g in src["grid_max_host"]]
        return out

    def forward(self, point):
        assert {"serialized_code", "serialized_order", "serialized_inverse", "serialized_depth"}.issubset(point.keys())
        pl = point.pop("_pool_plan", None)
        if pl is None:
            pl = self.plan(point)
        order0, lengths = pl["order0"], pl["lengths"]
        if self.reduce == "max":
            feat = ops.segment_max(self.proj(point.feat), order0, pl["head_pos"], lengths)
        else:
            feat = torch.segment_reduce(self.proj(point.feat)[order0], self.reduce, lengths=lengths, axis=0, unsafe=True)
        with torch.no_grad():
            coord = torch.segment_reduce(point.coord[order0], "mean", lengths=lengths, axis=0, unsafe=True)
        point_dict = dict(feat=feat, coord=coord)
        for k in ("grid_coord", "serialized_code", "serialized_order", "serialized_inverse", "serialized_depth", "batch", "offset",
                  "offset_host", "grid_max_host"):
            if k in pl:
                point_dict[k] = pl[k]
        for k in ("condition", "context", "_dp_pool"):
            if k in point:
                point_dict[k] = point[k]
        if self.traceable:
            point_dict["pooling_inverse"] = pl["cluster"]
            point_dict["pooling_parent"] = point
            point_dict["_pool_sorted"] = (order0, lengths)
        point = Point(point_dict)
        if getattr(self, "norm", None) is not None:
            point = self.norm(point)
        if getattr(self, "act", None) is not None:
            point = self.act(point)
        point.sparsify()
        return point


class SerializedUnpooling(PointModule):
    """ptv3m1:447-482 (including the m1 quirk: parent.sparse_conv_feat is not refreshed after the add)."""

    def __init__(self, in_channels, skip_channels, out_channels, norm_layer=None, act_layer=None, traceable=False):
        super().__init__()
        self.proj = PointSequential(FusedLinear(in_channels, out_channels))
        self.proj_skip = PointSequential(FusedLinear(skip_channels, out_channels))
        if norm_layer is not None:
            self.proj.add(norm_layer(out_channels))
            self.proj_skip.add(norm_layer(out_channels))
        if act_layer is not None:
            self.proj.add(act_layer())
            self.proj_skip.add(act_layer())
        self.traceable = traceable

    def forward(self, point):
        parent = point.pop("pooling_parent")
        inverse = point.pop("pooling_inverse")
        sorted_info = point.pop("_pool_sorted", None)
        point = self.proj(point)
        parent = self.proj_skip(parent)
        if sorted_info is not None:
            parent.feat = ops.unpool_add(parent.feat, point.feat, inverse, sorted_info[0], sorted_info[1])
        else:
            parent.feat = parent.feat + point.feat[inverse]
        if self.traceable:
            parent["unpooling_parent"] = point
        return parent


class Embedding(PointModule):
    def __init__(self, in_channels, embed_channels, norm_layer=None, act_layer=None):
        super().__init__()
        self.in_channels, self.embed_channels = in_channels, embed_channels
        self.stem = PointSequential(conv=spconv.SubMConv3d(in_channels, embed_channels, kernel_size=5, padding=1, bias=False,
                                                           indice_key="stem"))
        if norm_layer is not None:
            self.stem.add(norm_layer(embed_channels), name="norm")
        if act_layer is not None:
            self.stem.add(act_layer(), name="act")

    def forward(self, point):
        return self.stem(point)


class PointTransformerV3(PointModule):
    """ "PT-v3m1" (ptv3m1:518-714) with the same constructor arguments and defaults."""

    def __init__(self, in_channels=6, order=("z", "z-trans"), stride=(2, 2, 2, 2), enc_depths=(2, 2, 2, 6, 2),
                 enc_channels=(32, 64, 128, 256, 512), enc_num_head=(2, 4, 8, 16, 32), enc_patch_size=(48, 48, 48, 48, 48),
                 dec_depths=(2, 2, 2, 2), dec_channels=(64, 64, 128, 256), dec_num_head=(4, 4, 8, 16),
                 dec_patch_size=(48, 48, 48, 48), mlp_ratio=4, qkv_bias=True, qk_scale=None, attn_drop=0.0, proj_drop=0.0,
                 drop_path=0.3, pre_norm=True, shuffle_orders=True, enable_rpe=False, enable_flash=True,
                 upcast_attention=False, upcast_softmax=False, enc_mode=False, pdnorm_bn=False, pdnorm_ln=False,
                 pdnorm_decouple=True, pdnorm_adaptive=False, pdnorm_affine=True,
                 pdnorm_conditions=("ScanNet", "S3DIS", "Structured3D"), spatial_reorder=False):
        super().__init__()
        # spatial_reorder (not a reference option): lay the level-0 points out in memory along the first space-filling
        # curve so that the rulebook gathers and the [order] / [inverse] gathers of the attention hit nearby cache lines.
        # Results are permutation-equivalent; the returned ``feat`` is restored to the caller's point order.  Every OTHER
        # per-point entry of the returned Point (coord, grid_coord, batch, serialized_*, sparse_conv_feat, pooling_inverse of
        # level 1) stays in the spatial layout: index it through point["spatial_perm"] (spatial row -> caller row), or run with
        # spatial_reorder=False when a head needs more than ``feat``.  A prepared Point is single use (asserted).
        self.spatial_reorder = spatial_reorder
        if pdnorm_bn or pdnorm_ln:
            raise NotImplementedError("PDNorm (multi-dataset prompt training) is outside the PT-v3m1 hot path")
        self.num_stages = len(enc_depths)
        self.order = [order] if isinstance(order, str) else order
        self.enc_mode, self.shuffle_orders = enc_mode, shuffle_orders
        assert self.num_stages == len(stride) + 1 == len(enc_channels) == len(enc_num_head) == len(enc_patch_size)
        assert enc_mode or self.num_stages == len(dec_depths) + 1 == len(dec_channels) + 1 == len(dec_num_head) + 1
        bn_layer = partial(nn.BatchNorm1d, eps=1e-3, momentum=0.01)
        ln_layer, act_layer = FusedLayerNorm, nn.GELU
        self.embedding = Embedding(in_channels, enc_channels[0], norm_layer=bn_layer, act_layer=act_layer)

        def make_block(ch, heads, patch, dp, i, s):
            return Block(channels=ch, num_heads=heads, patch_size=patch, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias,
                         qk_scale=qk_scale, attn_drop=attn_drop, proj_drop=proj_drop, drop_path=dp, norm_layer=ln_layer,
                         act_layer=act_layer, pre_norm=pre_norm, order_index=i % len(self.order), cpe_indice_key=f"stage{s}",
                         enable_rpe=enable_rpe, enable_flash=enable_flash, upcast_attention=upcast_attention,
                         upcast_softmax=upcast_softmax)

        enc_dp = [x.item() for x in torch.linspace(0, drop_path, sum(enc_depths))]
        self.enc = PointSequential()
        for s in range(self.num_stages):
            dps = enc_dp[sum(enc_depths[:s]): sum(enc_depths[: s + 1])]
            enc = PointSequential()
            if s > 0:
                enc.add(SerializedPooling(enc_channels[s - 1], enc_channels[s], stride=stride[s - 1], norm_layer=bn_layer,
                                          act_layer=act_layer), name="down")
            for i in range(enc_depths[s]):
                enc.add(make_block(enc_channels[s], enc_num_head[s], enc_patch_size[s], dps[i], i, s), name=f"block{i}")
            if len(enc) != 0:
                self.enc.add(module=enc, name=f"enc{s}")
        if not enc_mode:
            dec_dp = [x.item() for x in torch.linspace(0, drop_path, sum(dec_depths))]
            self.dec = PointSequential()
            dec_channels = list(dec_channels) + [enc_channels[-1]]
            for s in reversed(range(self.num_stages - 1)):
                dps = dec_dp[sum(dec_depths[:s]): sum(dec_depths[: s + 1])]
                dps.reverse()
                dec = PointSequential()
                dec.add(SerializedUnpooling(dec_channels[s + 1], enc_channels[s], dec_channels[s], norm_layer=bn_layer,
                                            act_layer=act_layer), name="up")
                for i in range(dec_depths[s]):
                    dec.add(make_block(dec_channels[s], dec_num_head[s], dec_patch_size[s], dps[i], i, s), name=f"block{i}")
                self.dec.add(module=dec, name=f"dec{s}")

    @torch.no_grad()
    def prepare(self, data_dict):
        """Everything of the forward that depends only on coordinates: serialization, optional spatial re-layout, the
        level-0 sparse tensor and the index plan of every pooling stage (the only host syncs of the model).  Feature
        independent and gradient free, so a training loop can run it for batch i+1 on a side stream while batch i trains
        (bench.py does); forward() calls it itself when handed a raw dict."""
        point = Point(data_dict)
        point.serialization(order=self.order, shuffle_orders=self.shuffle_orders)
        if self.spatial_reorder:
            perm, restore = point.serialized_order[0], point.serialized_inverse[0]
            point.serialized_order = restore[point.serialized_order]      # new row of the p-th point of every order
            point.serialized_inverse = point.serialized_inverse[:, perm]
            point.serialized_code = point.serialized_code[:, perm]
            for k in ("coord", "grid_coord", "batch"):
                if k in point:
                    point[k] = point[k][perm]
            point["spatial_perm"], point["spatial_restore"] = perm, restore
        plans, src = [], point
        for s in range(1, self.num_stages):
            pl = getattr(self.enc, f"enc{s}").down.plan(src)
            plans.append(pl)
            src = pl
        point["_pool_plans"] = plans
        point["_prepared"] = True
        return point

    def _sync_half_shadows(self):
        """autocast path: refresh the half-precision shadows of every Linear / sparse-conv parameter with one launch"""
        if not torch.is_autocast_enabled() or ops.binding() is None:
            return
        sh = self.__dict__.get("_half_shadows")
        if sh is None:
            sh = ops.HalfShadows(self)
            self.__dict__["_half_shadows"] = sh
        sh.sync(torch.get_autocast_dtype("cuda"))

    def forward(self, data_dict):
        point = data_dict if isinstance(data_dict, Point) and data_dict.get("_prepared", False) else self.prepare(data_dict)
        if point.get("_consumed", False):
            raise RuntimeError("this prepared Point already went through forward(); prepare() a fresh one (its feat was re-laid out)")
        point["_consumed"] = True
        self._sync_half_shadows()
        if "_has_dp" not in self.__dict__:
            self.__dict__["_has_dp"] = any(isinstance(m, DropPath) and m.drop_prob > 0.0 for m in self.modules())
        if self.training and self.__dict__["_has_dp"] and Block.fused and ops.binding() is not None:
            # one torch.rand for every DropPath decision of this forward (two per block, one per row)
            sizes = [point.host_offset()[-1]] + [pl["offset_host"][-1] for pl in point["_pool_plans"]]
            need = 0
            for st in range(self.num_stages):
                need += 2 * sizes[st] * len([m for m in getattr(self.enc, f"enc{st}").children() if isinstance(m, Block)])
                if not self.enc_mode and st < self.num_stages - 1:
                    need += 2 * sizes[st] * len([m for m in getattr(self.dec, f"dec{st}").children() if isinstance(m, Block)])
            point["_dp_pool"] = [torch.rand(max(need, 1), device=point.feat.device), 0]
        restore = point.get("spatial_restore")
        if restore is not None:
            point.feat = point.feat[point["spatial_perm"]]
        point.sparsify()
        plans = point["_pool_plans"]
        point = self.embedding(point)
        for s in range(self.num_stages):
            if s > 0:
                point["_pool_plan"] = plans[s - 1]
            point = getattr(self.enc, f"enc{s}")(point)
        if not self.enc_mode:
            point = self.dec(point)
            if restore is not None:
                point.feat = point.feat[restore]
        return point


_FUSED_LOSS = os.environ.get("B2PC_LOSS_FUSED", "1") != "0"


class PTv3Segmentor(nn.Module):
    """backbone + linear head + cross-entropy: the part of DefaultSegmentorV2 (pointcept/models/default.py:41-95)
    the fwd+bwd benchmark needs.  Parameter names match (``backbone.*``, ``seg_head.*``)."""

    def __init__(self, num_classes=20, backbone_out_channels=64, **backbone_kwargs):
        super().__init__()
        self.backbone = PointTransformerV3(**backbone_kwargs)
        self.seg_head = nn.Linear(backbone_out_channels, num_classes) if num_classes > 0 else nn.Identity()

    def prepare(self, input_dict):
        return self.backbone.prepare(input_dict)

    def forward(self, input_dict):
        point = self.backbone(input_dict)
        seg_logits = self.seg_head(point.feat)
        out = dict(seg_logits=seg_logits)
        if "segment" in input_dict:
            if _FUSED_LOSS and seg_logits.is_cuda:    # one pass each way (csrc/loss.cuh) instead of log_softmax + nll_loss
                out["loss"] = ops.cross_entropy(seg_logits, input_dict["segment"], ignore_index=-1)
            else:
                out["loss"] = nn.functional.cross_entropy(seg_logits.float(), input_dict["segment"], ignore_index=-1)
        return out


def ptv3_base_config():
    """model kwargs of configs/scannet/semseg-pt-v3m1-0-base.py:11-47 ("PTv3-base")."""
    return dict(
        in_channels=6, order=("z", "z-trans", "hilbert", "hilbert-trans"), stride=(2, 2, 2, 2), enc_depths=(2, 2, 2, 6, 2),
        enc_channels=(32, 64, 128, 256, 512), enc_num_head=(2, 4, 8, 16, 32), enc_patch_size=(1024,) * 5,
        dec_depths=(2, 2, 2, 2), dec_channels=(64, 64, 128, 256), dec_num_head=(4, 4, 8, 16), dec_patch_size=(1024,) * 4,
        mlp_ratio=4, qkv_bias=True, qk_scale=None, attn_drop=0.0, proj_drop=0.0, drop_path=0.3, shuffle_orders=True,
        pre_norm=True, enable_rpe=False, enable_flash=True, upcast_attention=False, upcast_softmax=False, enc_mode=False,
    )
