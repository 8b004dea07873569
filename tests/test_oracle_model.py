"""oracle/ptv3_cpu.py (functional restatement) vs the UNMODIFIED reference PT-v3m1 run on CPU
(tests/golden/ptv3_tiny.npz, made by tools/gen_golden.py with spconv stood in by oracle/spconv_ref.py)."""
import os

import numpy as np
import torch

from oracle import fixture_dout, fixture_state_dict, ptv3_cpu


def _load(golden_dir):
    g = np.load(os.path.join(golden_dir, "ptv3_tiny.npz"))
    sd = fixture_state_dict(g)
    grads = {k[6:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("grad::")}
    return g, sd, grads


def test_cpu_model_matches_reference_forward_backward(golden_dir):
    g, sd, grads = _load(golden_dir)
    for k, v in sd.items():
        if v.is_floating_point():
            v.requires_grad_(True)
    out = ptv3_cpu.forward(sd, dict(grid_coord=g["grid_coord"], feat=g["feat"], offset=g["offset"]), ptv3_cpu.TINY_CFG,
                           bn_training=True)
    ref = torch.from_numpy(g["out"])
    assert out.shape == ref.shape
    rel = (out.detach() - ref).norm() / ref.norm()
    assert rel < 1e-5, rel
    out.backward(fixture_dout(g))
    for k, gr in grads.items():
        rel = (sd[k].grad - gr).norm() / gr.norm()
        assert rel < 1e-4, (k, rel)


def test_spunet_restatement_matches_unmodified_reference_model(golden_dir):
    """oracle/spunet_cpu.py vs tests/golden/spunet_tiny.npz: the UNMODIFIED reference SpUNetBase (spconv_unet_v1m1_base.py:88-280) run on
    CPU in training mode over oracle/spconv_ref.py (tools/gen_golden.py::gen_spunet_tiny) -- logits and all 101 parameter gradients."""
    import types
    from oracle import spunet_cpu
    g = np.load(os.path.join(golden_dir, "spunet_tiny.npz"))
    sd = fixture_state_dict(g)
    grads = {k[6:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("grad::")}
    for v in sd.values():
        if v.is_floating_point():
            v.requires_grad_(True)
    shape = types.SimpleNamespace(num_stages=len(g["layers"]) // 2, layers=tuple(int(v) for v in g["layers"]),
                                  channels=tuple(int(v) for v in g["channels"]))
    out = spunet_cpu.forward(sd, dict(grid_coord=g["grid_coord"], feat=g["feat"], offset=g["offset"]), shape)
    ref = torch.from_numpy(g["out"])
    assert out.shape == ref.shape
    assert (out.detach() - ref).norm() / ref.norm() < 1e-5
    out.backward(torch.from_numpy(g["dout"]))
    assert len(grads) == 101
    for k, gr in grads.items():
        assert sd[k].grad is not None, k
        assert (sd[k].grad - gr).norm() / gr.norm().clamp(min=1e-12) < 1e-4, k
