"""CPU oracle for the PTv3 / spconv hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``pointcept_b200/`` may import this
package; only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` do, and only as the checker / the CPU
baseline -- never as the thing shipped.

Pinning status (see DESIGN.md, "Oracle"):
  * serialization (z-order / Hilbert / encode / argsort), patch padding and the
    dense attention math are PINNED: ``tools/gen_golden.py`` imports the
    reference's own python files from a reference checkout and writes
    ``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks this
    restatement against those fixtures bit-exactly (integers) / to 1e-6 (fp32).
  * sparse convolution (rulebook + gather-GEMM-scatter): PARITY UNPINNED.  The
    arithmetic lives in third-party ``spconv-cu124`` (unpinned version,
    reference ``environment.yml:47``) whose source is not vendored in the
    reference and is not installable offline.  ``oracle/spconv_ref.py`` restates
    its published semantics (SURVEY.md Appendix A) anchored on the reference
    call sites.
"""


def seeded_state_dict(spec, seed):
    """[(name, shape)] -> {name: tensor}, the weights of the model fixtures (tests/golden/ptv3_tiny.npz, spunet_tiny.npz): BatchNorm
    running statistics at their initial values, every other tensor drawn from one seeded torch.Generator in ``spec`` order --
    1-D ``.weight`` 1 + 0.1 N(0, 1), other 1-D 0.1 N(0, 1), 2-D U(-1, 1) / sqrt(fan_in) like ``nn.Linear``, higher-D 0.05 N(0, 1)
    like the oracle's conv stand-in.  ``tools/gen_golden.py`` loads the same tensors into the reference model, so the fixtures
    store the seed instead of the weights."""
    import math
    import torch
    gen = torch.Generator().manual_seed(int(seed))
    sd = {}
    for name, shape in spec:
        if name.endswith("num_batches_tracked"):
            t = torch.zeros(shape, dtype=torch.int64)
        elif name.endswith("running_mean"):
            t = torch.zeros(shape)
        elif name.endswith("running_var"):
            t = torch.ones(shape)
        elif len(shape) == 1:
            t = (1.0 if name.endswith(".weight") else 0.0) + 0.1 * torch.randn(shape, generator=gen)
        elif len(shape) == 2:
            t = (torch.rand(shape, generator=gen) * 2 - 1) / math.sqrt(shape[1])
        else:
            t = 0.05 * torch.randn(shape, generator=gen)
        sd[name] = t
    return sd


def fixture_state_dict(g):
    """the state dict of a model fixture loaded with np.load (its ``sd_spec`` / ``sd_seed`` entries, see seeded_state_dict)"""
    import json
    return seeded_state_dict(json.loads(str(g["sd_spec"])), int(g["sd_seed"]))


def fixture_dout(g):
    """the output gradient of tests/golden/ptv3_tiny.npz: N(0, 1) of the output's shape from a seeded torch.Generator"""
    import torch
    return torch.randn(tuple(int(v) for v in g["out"].shape), generator=torch.Generator().manual_seed(int(g["dout_seed"])))
