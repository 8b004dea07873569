"""Data-parallel gradient exchange: the one collective on the hot path (SURVEY.md 8(a).12 / 8(e)).

The reference wraps the model in ``DistributedDataParallel`` (pointcept/engines/defaults.py:22-43, one process per GPU from
pointcept/engines/launch.py:73): an autograd hook per parameter (486 for PT-v3m1 base) copies each gradient into a bucket and
launches the bucket's all-reduce.  The training step is a chain of well over a thousand short launches that the host has to keep
ahead of; 486 hook calls per step are then paid in wall time, not hidden.  ``FlatGradReducer`` does the same exchange (average
of every gradient over the ranks, fp32, in place) with ONE autograd hook and at most two collectives per step:

* all gradients are packed into one flat fp32 buffer by one launch of ``b2pc_multi_cast`` (fp32 -> fp32: a multi-tensor copy,
  185 MB), laid out in the order the backward pass produces them (measured on the first step, agreed across ranks);
* when the gradient of the *trigger* parameter arrives -- the point of the backward pass at which ``early_fraction`` of the
  gradient bytes exist (for PT-v3 that is inside encoder stage 3: the wide, cheap stages are behind, the narrow full-resolution
  stages that take most of the time are still ahead) -- the prefix of the buffer is packed and its all-reduce starts on NCCL's
  stream, under the rest of the backward pass;
* ``finish()`` packs and reduces the small remainder, waits for the early collective and points every ``p.grad`` at its slice of
  the flat buffer, where the (fused) optimizer reads it.

NVLink / NVSwitch moves the whole 185 MB in about a millisecond, so two large messages beat many small buckets: the
exchange is sized for launch latency and overlap, not for link count.  No activation, rulebook or sort ever crosses GPUs.

The pack is CUDA only (no CPU fallback); the CPU tests inject a packer to exercise the protocol under gloo.
"""
import ctypes

import numpy as np
import torch
import torch.distributed as dist

from . import _lib

_BLOCK_ELEMS = 2048   # kCastBlockElems of csrc/fused.cuh


class _CudaPacker:
    """One launch of b2pc_multi_cast (fp32 destination = multi-tensor copy) per parameter group.  Counts, destinations and the
    block table of a group never change; per step only the gradient pointers are refreshed (one small pinned -> device copy)."""

    def __init__(self):
        self.groups = {}

    def __call__(self, name, grads, offsets, flat):
        n = len(grads)
        if n == 0:
            return
        if not flat.is_cuda:
            raise RuntimeError("FlatGradReducer packs on the GPU only (libb2pc has no CPU path)")
        st = self.groups.get(name)
        if st is None or st["n"] != n or st["base"] != flat.data_ptr():
            counts = np.fromiter((g.numel() for g in grads), dtype=np.int64, count=n)
            blocks = (counts + _BLOCK_ELEMS - 1) // _BLOCK_ELEMS
            pinned = torch.zeros((n, 4), dtype=torch.int64).pin_memory()
            tab = pinned.numpy()
            tab[:, 1] = flat.data_ptr() + 4 * np.asarray(offsets, dtype=np.int64)
            tab[:, 2] = counts
            tab[:, 3] = np.cumsum(blocks) - blocks
            st = dict(n=n, base=flat.data_ptr(), pinned=pinned, tab=tab, total_blocks=int(blocks.sum()), counts=counts, ev=None, calls=0,
                      dev=torch.empty((n, 4), dtype=torch.int64, device=flat.device))
            self.groups[name] = st
        if st["calls"] < 3:      # layouts are fixed after the first steps: validate there, trust afterwards
            for g, c in zip(grads, st["counts"]):
                if g.dtype != torch.float32 or not g.is_contiguous() or g.device != flat.device or g.numel() != c:
                    raise RuntimeError("FlatGradReducer takes contiguous fp32 gradients of fixed shape on the buffer's device")
        st["calls"] += 1
        if st["ev"] is not None:
            st["ev"].synchronize()     # the previous upload of this table finished long ago; never overwrite it in flight
        st["tab"][:, 0] = np.fromiter((g.data_ptr() for g in grads), dtype=np.int64, count=n)
        st["dev"].copy_(st["pinned"], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        st["ev"] = ev
        _lib.check(_lib.lib().b2pc_multi_cast(ctypes.c_void_p(st["dev"].data_ptr()), n, st["total_blocks"], 0,   # 0 = B2PC_F32
                                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "multi_cast(pack)")


class FlatGradReducer:
    def __init__(self, params, process_group=None, early_fraction=0.9, average=True, broadcast=True, pack=None):
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("FlatGradReducer: no parameters")
        if not dist.is_initialized():
            raise RuntimeError("FlatGradReducer needs an initialised process group (one process per GPU)")
        self.group = process_group
        self.world = dist.get_world_size(process_group)
        self.backend = dist.get_backend(process_group)
        self.early_fraction = float(early_fraction)
        self.average = average
        self._pack = pack or _CudaPacker()      # pack(group name, gradients, element offsets, flat buffer)
        dev = self.params[0].device
        if any(p.device != dev or p.dtype != torch.float32 for p in self.params):
            raise RuntimeError("FlatGradReducer takes fp32 parameters on one device")
        self.sizes = [(p.numel() + 3) // 4 * 4 for p in self.params]      # 16-byte aligned slices (vector loads in AdamW)
        self.flat = torch.zeros(sum(self.sizes), dtype=torch.float32, device=dev)
        self.order = None          # parameter indices in gradient-arrival order (set by the first step)
        self.offsets = None        # element offset of each parameter in the flat buffer
        self.views = None
        self.n_early = 0           # the first n_early entries of `order` form the early group
        self.early_end = 0         # element offset where the early group ends
        self._arrival = []
        self._calib_handles = []
        self._trigger_handle = None
        self._early_work = None
        self._early_done = False
        self.enabled = True
        self.stats = dict(steps=0, early_steps=0, late_steps=0)
        if broadcast:
            with torch.no_grad():
                for p in self.params:
                    dist.broadcast(p.data, 0, group=process_group)
        for i, p in enumerate(self.params):
            self._calib_handles.append(p.register_post_accumulate_grad_hook(self._make_arrival_hook(i)))

    # ---- first step: measure the order in which the backward pass produces the gradients -------------------------------------
    def _make_arrival_hook(self, i):
        def hook(_p):
            self._arrival.append(i)
        return hook

    def _build_layout(self):
        seen = set()
        order = [i for i in self._arrival if not (i in seen or seen.add(i))]
        if len(order) != len(self.params):
            missing = len(self.params) - len(order)
            raise RuntimeError(f"FlatGradReducer: {missing} parameter(s) received no gradient (every parameter must be used every "
                               "step, as with DistributedDataParallel(find_unused_parameters=False))")
        t = torch.tensor(order, dtype=torch.int64, device=self.flat.device if self.backend == "nccl" else "cpu")
        dist.broadcast(t, 0, group=self.group)          # all ranks adopt rank 0's order: the layout must be identical everywhere
        order = [int(v) for v in t.cpu()]
        if sorted(order) != list(range(len(self.params))):
            raise RuntimeError("FlatGradReducer: ranks disagree on the parameter list")
        self.order = order
        self.offsets = [0] * len(self.params)
        total, off = sum(self.sizes), 0
        self.n_early, self.early_end = 0, 0
        for k, i in enumerate(order):
            self.offsets[i] = off
            off += self.sizes[i]
            if self.n_early == 0 and self.early_fraction > 0 and off >= self.early_fraction * total and k + 1 < len(order):
                self.n_early, self.early_end = k + 1, off
        self.views = [self.flat[self.offsets[i]:self.offsets[i] + p.numel()].view_as(p) for i, p in enumerate(self.params)]
        for h in self._calib_handles:
            h.remove()
        self._calib_handles = []
        if self.n_early > 0:
            trigger = self.params[order[self.n_early - 1]]
            self._trigger_handle = trigger.register_post_accumulate_grad_hook(self._early_hook)

    # ---- the exchange ------------------------------------------------------------------------------------------------------------
    def _pack_group(self, name, idxs):
        grads = [self.params[i].grad for i in idxs]
        if any(g is None for g in grads):
            raise RuntimeError("FlatGradReducer: a parameter has no gradient at exchange time (the backward pass must produce "
                               "every gradient in the same order on every step and rank)")
        offs = [self.offsets[i] for i in idxs]
        if any(g.data_ptr() == self.views[i].data_ptr() for g, i in zip(grads, idxs)):
            # zero_grad(set_to_none=False): autograd accumulated into the flat slices in place; copy only what lives elsewhere
            keep = [k for k, (g, i) in enumerate(zip(grads, idxs)) if g.data_ptr() != self.views[i].data_ptr()]
            grads, offs, name = [grads[k] for k in keep], [offs[k] for k in keep], name + f"/{len(keep)}"
        self._pack(name, grads, offs, self.flat)

    def _all_reduce(self, t, async_op):
        if self.average and self.backend == "nccl":
            return dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group, async_op=async_op), False
        return dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group, async_op=async_op), self.average

    def _early_hook(self, _p):
        if not self.enabled or self._early_done or self.order is None:
            return
        if any(self.params[i].grad is None for i in self.order[:self.n_early]):
            return      # this rank's backward pass ran in another order: finish() issues the same collective, just not overlapped
        self._pack_group("early", self.order[:self.n_early])
        self._early_work, self._early_div = self._all_reduce(self.flat[:self.early_end], True)
        self._early_done = True
        self.stats["early_steps"] += 1

    @torch.no_grad()
    def finish(self):
        """Call after ``loss.backward()``: afterwards every ``p.grad`` is its slice of the flat buffer holding the rank average.
        Every rank issues the same collectives in the same order on every step (layout step: broadcast + one all-reduce; afterwards
        the early slice, then the rest) whether or not its own trigger fired, so ranks can never disagree on the sequence."""
        if not self.enabled:
            return
        self.stats["steps"] += 1
        if self.order is None:                                   # first step: lay the buffer out, one collective
            self._build_layout()
            self._arrival = []
            self._pack_group("all", self.order)
            _, div = self._all_reduce(self.flat, False)
            if div:
                self.flat.div_(self.world)
        else:
            lo = self.early_end if self.n_early > 0 else 0
            if self.n_early > 0 and not self._early_done:        # trigger did not fire / found a gradient missing: same collective, late
                self._pack_group("early", self.order[:self.n_early])
                self._early_work, self._early_div = self._all_reduce(self.flat[:lo], True)
                self._early_done = True
                self.stats["late_steps"] += 1
            self._pack_group("rest" if lo else "all", self.order[self.n_early:])
            _, div = self._all_reduce(self.flat[lo:], False)
            if div:
                self.flat[lo:].div_(self.world)
            if self._early_done:
                self._early_work.wait()
                if self._early_div:
                    self.flat[:lo].div_(self.world)
            self._early_work, self._early_done = None, False
        for p, v in zip(self.params, self.views):
            p.grad = v

    def remove(self):
        for h in self._calib_handles:
            h.remove()
        if self._trigger_handle is not None:
            self._trigger_handle.remove()
        self._calib_handles, self._trigger_handle = [], None
