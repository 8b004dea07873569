"""Generate tests/golden/*.npz by running the reference's OWN python code (CPU, this container).

    python tools/gen_golden.py

The reference (/root/reference) does not travel to the GPU box; these small fixtures do.
Covers SURVEY.md section 8(c): serialization codes for all four orders at several depths,
Point.serialization order/inverse, get_padding_and_inverse, and the non-flash dense
attention branch of SerializedAttention (fp32) -- forward output and input gradients.
spconv is absent from the reference tree and from this image: no fixture can be generated
for it (parity unpinned, see oracle/__init__.py).
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import ref_import  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def gen_serialization():
    ser = ref_import.load_serialization()
    out = {}
    rng = np.random.default_rng(1234)
    cases = {"d3": (3, 300, 1), "d9": (9, 4000, 4), "d10": (10, 3000, 2), "d12": (12, 3000, 3), "d16": (16, 2000, 5)}
    for name, (depth, n, nb) in cases.items():
        gc = rng.integers(0, 1 << depth, size=(n, 3)).astype(np.int32)
        gc[0] = 0
        gc[1] = (1 << depth) - 1
        b = np.sort(rng.integers(0, nb, size=n)).astype(np.int64)
        out[f"{name}_grid"] = gc
        out[f"{name}_batch"] = b
        out[f"{name}_depth"] = np.int64(depth)
        for order in ("z", "z-trans", "hilbert", "hilbert-trans"):
            code = ser.encode(torch.from_numpy(gc), torch.from_numpy(b), depth, order=order)
            out[f"{name}_{order}"] = code.numpy()
    # survey appendix B points
    P = np.array([(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 2, 3), (7, 7, 7)], dtype=np.int32)
    for depth in (3, 9, 16):
        for order in ("z", "z-trans", "hilbert", "hilbert-trans"):
            out[f"appB_d{depth}_{order}"] = ser.encode(torch.from_numpy(P), torch.zeros(6, dtype=torch.long), depth, order=order).numpy()
    out["appB_points"] = P
    np.savez_compressed(os.path.join(OUT, "serialization.npz"), **out)
    print("serialization.npz", len(out), "arrays")


def gen_point_and_padding():
    ref = ref_import.load_models(use_shims=False)
    Point = ref.structure.Point
    SA = ref.ptv3.SerializedAttention
    out = {}
    # Point.serialization on unique voxels (ties are implementation-defined, so avoid them)
    rng = np.random.default_rng(7)
    n_per = [1500, 700, 2300]
    gcs, bs = [], []
    for bi, n in enumerate(n_per):
        lin = rng.choice(64 * 64 * 64, size=n, replace=False)
        gcs.append(np.stack([lin // 4096, (lin // 64) % 64, lin % 64], 1))
        bs.append(np.full(n, bi))
    gc = np.concatenate(gcs).astype(np.int32)
    b = np.concatenate(bs).astype(np.int64)
    p = Point(grid_coord=torch.from_numpy(gc), batch=torch.from_numpy(b), feat=torch.zeros(len(b), 1))
    orders = ("z", "z-trans", "hilbert", "hilbert-trans")
    p.serialization(order=orders, shuffle_orders=False)
    out["ser_grid"] = gc
    out["ser_batch"] = b
    out["ser_depth"] = np.int64(p.serialized_depth)
    out["ser_code"] = p.serialized_code.numpy()
    out["ser_order"] = p.serialized_order.numpy()
    out["ser_inverse"] = p.serialized_inverse.numpy()

    # padding tables
    cases = {"a": ([5, 12], 4), "b": ([3, 11], 4), "c": ([8, 9], 4), "d": ([10], 4),
             "e": ([3000, 5000], 1024), "f": ([100, 1124, 1125, 4000], 1024), "g": ([1024, 2048, 2049], 1024),
             "h": ([48, 96, 97, 200], 48)}
    for name, (offset, K) in cases.items():
        attn = SA(channels=16, num_heads=1, patch_size=K, enable_flash=False, upcast_attention=True, upcast_softmax=True)
        attn.patch_size = K
        pt = Point(offset=torch.tensor(offset), feat=torch.zeros(offset[-1], 1))
        pad, unpad, cu = attn.get_padding_and_inverse(pt)
        out[f"pad_{name}_offset"] = np.array(offset, dtype=np.int64)
        out[f"pad_{name}_K"] = np.int64(K)
        out[f"pad_{name}_pad"] = pad.numpy()
        out[f"pad_{name}_unpad"] = unpad.numpy()
        out[f"pad_{name}_cu"] = cu.numpy()
    np.savez_compressed(os.path.join(OUT, "point_padding.npz"), **out)
    print("point_padding.npz", len(out), "arrays")

    # dense (non-flash) attention of the reference, fp32, with gradients.
    # scenes all >= K so the non-flash branch keeps K (ptv3m1:173-176).
    torch.manual_seed(0)
    K, C, H = 64, 32, 2
    offset = [200, 200 + 64, 200 + 64 + 333]
    N = offset[-1]
    attn = SA(channels=C, num_heads=H, patch_size=K, enable_flash=False, upcast_attention=True, upcast_softmax=True)
    gc = torch.from_numpy(np.stack([np.arange(N) % 32, (np.arange(N) // 32) % 32, np.arange(N) // 1024], 1).astype(np.int32))
    feat = torch.randn(N, C, requires_grad=True)
    pt = Point(offset=torch.tensor(offset), grid_coord=gc, feat=feat)
    pt.serialization(order=("z", "hilbert"), shuffle_orders=False)
    attn.order_index = 1
    # capture the packed qkv the reference feeds the attention core, and the core's output
    cap = {}
    qkv_lin = attn.qkv
    orig_fwd = qkv_lin.forward
    def qkv_fwd(x):
        y = orig_fwd(x)
        y.retain_grad()
        cap["qkv_full"] = y
        return y
    qkv_lin.forward = qkv_fwd
    proj_orig = attn.proj.forward
    def proj_fwd(x):
        x.retain_grad()
        cap["core_out_unpadded"] = x
        return proj_orig(x)
    attn.proj.forward = proj_fwd
    res = attn(pt)
    g = torch.randn_like(res.feat)
    res.feat.backward(g)
    pad, unpad, cu = pt["pad"], pt["unpad"], pt["cu_seqlens_key"]
    np.savez_compressed(
        os.path.join(OUT, "attention_dense.npz"),
        offset=np.array(offset), K=np.int64(K), H=np.int64(H), C=np.int64(C),
        scale=np.float64(attn.scale),
        order=pt.serialized_order[1].numpy(), inverse=pt.serialized_inverse[1].numpy(),
        pad=pad.numpy(), unpad=unpad.numpy(), cu=cu.numpy(),
        qkv_full=cap["qkv_full"].detach().numpy(),            # [N, 3C] before the [order] gather
        core_out=cap["core_out_unpadded"].detach().numpy(),    # [N, C] after the [inverse] gather
        d_core_out=cap["core_out_unpadded"].grad.numpy(),
        d_qkv_full=cap["qkv_full"].grad.numpy(),
    )
    print("attention_dense.npz")


def gen_attention_rpe():
    """the reference's non-flash branch with RPE (ptv3m1:29-48,173-206) as a whole module: state_dict, inputs, tables, output, grads"""
    ref = ref_import.load_models(use_shims=False)
    Point, SA = ref.structure.Point, ref.ptv3.SerializedAttention
    torch.manual_seed(11)
    C, H = 32, 2
    offset = [150, 150 + 48, 150 + 48 + 101]
    N = offset[-1]
    attn = SA(channels=C, num_heads=H, patch_size=64, enable_rpe=True, enable_flash=False, upcast_attention=True, upcast_softmax=True)
    with torch.no_grad():
        attn.rpe.rpe_table.normal_(0.0, 0.5)
    rng = np.random.default_rng(5)
    lin = rng.choice(24 * 24 * 24, size=N, replace=False)
    gc = torch.from_numpy(np.stack([lin // 576, (lin // 24) % 24, lin % 24], 1).astype(np.int32))
    feat = torch.randn(N, C, requires_grad=True)
    pt = Point(offset=torch.tensor(offset), grid_coord=gc, feat=feat)
    pt.serialization(order=("z", "hilbert"), shuffle_orders=False)
    attn.order_index = 1
    res = attn(pt)
    g = torch.randn_like(res.feat)
    res.feat.backward(g)
    out = {f"sd::{k}": v.detach().numpy() for k, v in attn.state_dict().items()}
    out.update(offset=np.array(offset), grid_coord=gc.numpy(), feat=feat.detach().numpy(), dout=g.numpy(), out=res.feat.detach().numpy(),
               dfeat=feat.grad.numpy(), d_rpe_table=attn.rpe.rpe_table.grad.numpy(), patch_size=np.int64(attn.patch_size),
               order=pt.serialized_order.numpy(), inverse=pt.serialized_inverse.numpy(),
               pad=pt["pad"].numpy(), unpad=pt["unpad"].numpy(), cu=pt["cu_seqlens_key"].numpy())
    np.savez_compressed(os.path.join(OUT, "attention_rpe.npz"), **out)
    print("attention_rpe.npz patch_size", attn.patch_size)


from oracle.ptv3_cpu import TINY_CFG  # noqa: E402


def _seeded_weights(model, seed):
    """load oracle.seeded_state_dict() into the reference model -> (the spec as a JSON string array, seed): the fixture stores
    these instead of the weights themselves"""
    import json
    from oracle import seeded_state_dict
    spec = [[k, list(v.shape)] for k, v in model.state_dict().items()]
    model.load_state_dict(seeded_state_dict(spec, seed))
    return np.array(json.dumps(spec)), np.int64(seed)


def gen_ptv3_tiny():
    """The UNMODIFIED reference PT-v3m1 (non-flash fp32 attention branch) run on CPU, with spconv stood in by
    oracle/spconv_ref.py.  Pins the model-level restatement (blocks, pooling, unpooling quirk, padding)."""
    ref = ref_import.load_models(use_shims="oracle")
    from pointcept_b200 import synth
    torch.manual_seed(3)
    cfg = dict(TINY_CFG, enable_flash=False, upcast_attention=True, upcast_softmax=True)
    model = ref.ptv3.PointTransformerV3(**cfg)
    model.train()
    # SerializedPooling is built with its own default shuffle_orders=True (ptv3m1:607-617 never forwards the
    # model-level flag), i.e. the reference is random by design below stage 0: pin it for the fixture.
    for m in model.modules():
        if hasattr(m, "shuffle_orders"):
            m.shuffle_orders = False
    spec, seed = _seeded_weights(model, 3)
    scenes = [synth.indoor_scene(11, target_voxels=1400), synth.indoor_scene(12, target_voxels=1000)]
    grid = np.concatenate([s[1] for s in scenes])
    coord = np.concatenate([s[0] for s in scenes])
    offset = np.cumsum([len(s[1]) for s in scenes])
    feat = torch.randn(len(grid), 6)
    out = model(dict(coord=torch.from_numpy(coord), grid_coord=torch.from_numpy(grid), feat=feat,
                     offset=torch.from_numpy(offset)))
    from oracle import fixture_dout
    g = fixture_dout(dict(out=out.feat, dout_seed=4))
    out.feat.backward(g)
    keep = ("embedding.stem.conv.weight", "enc.enc0.block0.cpe.0.weight", "enc.enc0.block1.attn.qkv.weight",
            "enc.enc1.down.proj.weight", "enc.enc2.block1.cpe.0.weight", "dec.dec0.block0.cpe.0.weight",
            "dec.dec0.up.proj_skip.0.weight", "dec.dec1.block1.attn.proj.weight")
    grads = {"grad::" + k: p.grad.numpy() for k, p in model.named_parameters() if k in keep}
    np.savez_compressed(os.path.join(OUT, "ptv3_tiny.npz"), coord=coord, grid_coord=grid, offset=offset, feat=feat.numpy(),
                        out=out.feat.detach().numpy(), dout_seed=np.int64(4), sd_spec=spec, sd_seed=seed, **grads)
    print("ptv3_tiny.npz", out.feat.shape, float(out.feat.abs().mean()))



def gen_grid_sample():
    """GridSample (pointcept/datasets/transform.py:840-958) run by the reference's own class on two raw synthetic scenes:
    everything the reference determines (hash keys, grid_coord of the sampled voxels in output order, inverse, counts, min_coord,
    fragment count, and its displacement at its own picks) for fnv / ravel hashes and two grid sizes."""
    t = ref_import.load_transform()
    rng = np.random.default_rng(7)
    scenes = []
    for n, ext in ((9000, (1.6, 1.2, 1.0)), (5001, (0.8, 2.0, 0.5))):
        # points on a few planes with jitter, centred so that negative coordinates occur (floor of negatives matters)
        c = rng.random((n, 3)) * np.asarray(ext) - np.asarray(ext) / 2
        wall = rng.integers(0, 3, n)
        c[np.arange(n), wall] = np.round(c[np.arange(n), wall]) + rng.normal(0, 0.004, n)
        scenes.append(c.astype(np.float32))
    out = {f"coord{i}": c for i, c in enumerate(scenes)}
    out["fnv_of_arange"] = t.GridSample.fnv_hash_vec(np.arange(30, dtype=np.int64).reshape(10, 3))
    for hash_type in ("fnv", "ravel"):
        for gs in (0.05, 0.02):
            for i, c in enumerate(scenes):
                tr = t.GridSample(grid_size=gs, hash_type=hash_type, mode="test", return_inverse=True, return_grid_coord=True,
                                  return_min_coord=True, return_displacement=True)
                parts = tr(dict(coord=c.copy(), index_valid_keys=["coord"]))
                tag = f"{hash_type}_{gs}_{i}"
                out[tag + "_inverse"] = parts[0]["inverse"]
                out[tag + "_grid_coord"] = parts[0]["grid_coord"]
                out[tag + "_min_coord"] = parts[0]["min_coord"]
                out[tag + "_n_fragments"] = np.int64(len(parts))
                out[tag + "_index0"] = parts[0]["index"]
                if hash_type == "fnv":
                    out[tag + "_displacement0"] = parts[0]["displacement"]
                out[tag + "_last_index"] = parts[-1]["index"]
    np.savez_compressed(os.path.join(OUT, "grid_sample.npz"), **out)
    print("grid_sample.npz", {k: v.shape for k, v in out.items() if k.endswith("_grid_coord")})


if __name__ == "__main__" and "--only-grid-sample" in sys.argv:
    assert ref_import.available(), "needs /root/reference"
    gen_grid_sample()
    sys.exit(0)


def gen_point_rope():
    """PointROPE by the reference's own pure-PyTorch class (litept_v1.py:66-125): LitePT's head_dim 18 and a wider head."""
    lp = ref_import.load_litept()
    gen = torch.Generator().manual_seed(11)
    out = {}
    for name, (n, h, d, base) in {"d18": (777, 4, 18, 100.0), "d48": (300, 2, 48, 50.0)}.items():
        tokens = torch.randn(1, h, n, d, generator=gen)
        pos = torch.randint(0, 700, (1, n, 3), generator=gen)
        rope = lp.PointROPE(freq=base)
        assert hasattr(rope, "apply_rope1d"), "expected the pure-PyTorch fallback class"
        y = rope(tokens, pos)
        out[name + "_tokens"] = tokens[0].transpose(0, 1).contiguous().numpy()      # [N, H, D]
        out[name + "_pos"] = pos[0].numpy()
        out[name + "_out"] = y[0].transpose(0, 1).contiguous().numpy()
        out[name + "_base"] = np.float32(base)
    np.savez_compressed(os.path.join(OUT, "point_rope.npz"), **out)
    print("point_rope.npz", {k: v.shape for k, v in out.items() if k.endswith("_out")})


def gen_spunet_tiny():
    """The UNMODIFIED reference SpUNet-v1m1 (spconv_unet_v1m1_base.py:88-280) run on CPU in training mode, with spconv stood in by
    oracle/spconv_ref.py (SubMConv3d k5 / k3 / k1, SparseConv3d k2 s2, SparseInverseConv3d k2, SparseSequential dispatch).  Pins the
    model-level restatement oracle/spunet_cpu.py (block structure, BatchNorm eps, skip concatenation order, indice_key pairing)."""
    ref = ref_import.load_models(use_shims="oracle")
    from pointcept_b200 import synth
    torch.manual_seed(5)
    cfg = dict(in_channels=6, num_classes=13, base_channels=8, channels=(8, 16, 16, 24, 24, 16, 16, 8), layers=(2, 1, 1, 1, 1, 1, 1, 2))
    model = ref.spunet.SpUNetBase(**cfg)
    model.train()
    spec, seed = _seeded_weights(model, 5)   # 1-D parameters perturbed away from (1, 0) so that every term is exercised
    b = synth.make_batch(2, seed=21, target_voxels=1200)
    out = model(dict(grid_coord=torch.from_numpy(b["grid_coord"]), feat=torch.from_numpy(b["feat"]), offset=torch.from_numpy(b["offset"])))
    g = torch.randn_like(out)
    out.backward(g)
    grads = {"grad::" + k: p.grad.numpy() for k, p in model.named_parameters()}
    np.savez_compressed(os.path.join(OUT, "spunet_tiny.npz"), grid_coord=b["grid_coord"], offset=b["offset"], feat=b["feat"],
                        out=out.detach().numpy(), dout=g.numpy(), layers=np.array(cfg["layers"]), channels=np.array(cfg["channels"]),
                        sd_spec=spec, sd_seed=seed, **grads)
    print("spunet_tiny.npz", out.shape, float(out.abs().mean()), len(grads), "parameter gradients")


def gen_dropin_abi():
    """reference_dropin.npz (one JSON string): parameter names / shapes of the reference's own PT-v3m1 (base config) and SpUNet-v1m1 (6 -> 20) built on
    the drop-in spconv / flash_attn modules, and what the reference's Point.sparsify() makes of a seeded point set."""
    import json
    from pointcept_b200.ptv3 import ptv3_base_config
    ref = ref_import.load_models(use_shims=True)
    shapes = lambda m: [[k, list(v.shape)] for k, v in m.state_dict().items()]   # noqa: E731
    g = torch.Generator().manual_seed(0)
    grid = torch.randint(0, 50, (100, 3), generator=g)
    feat = torch.randn(100, 6, generator=g)
    pt = ref.structure.Point(grid_coord=grid, feat=feat, offset=torch.tensor([60, 100]))
    pt.sparsify()
    x = pt.sparse_conv_feat
    out = dict(ptv3_base=shapes(ref.ptv3.PointTransformerV3(**ptv3_base_config())), spunet_6_20=shapes(ref.spunet.SpUNetBase(6, 20)),
               sparsify=dict(grid_coord=grid.tolist(), offset=[60, 100], indices=x.indices.tolist(), spatial_shape=[int(v) for v in x.spatial_shape],
                             batch_size=int(x.batch_size)))
    np.savez_compressed(os.path.join(OUT, "reference_dropin.npz"), json=np.array(json.dumps(out, separators=(",", ":"))))
    print("reference_dropin.npz", len(out["ptv3_base"]), len(out["spunet_6_20"]))


def gen_collate():
    """collate_fn.pt: the reference's own collate_fn (pointcept/datasets/utils.py:19-73) on the seeded CPU inputs of
    tests/test_host_logic.py::test_collate_fn_matches_the_reference_function (torch.save of tensors, dicts, lists and strings)."""
    import importlib.util
    import types
    saved = {k: sys.modules.get(k) for k in ("torch_scatter", "pointcept", "pointcept.models", "pointcept.models.utils")}
    try:
        sys.modules["torch_scatter"] = types.SimpleNamespace(scatter_min=None)
        for name in ("pointcept", "pointcept.models"):
            sys.modules[name] = types.ModuleType(name)
        sys.modules["pointcept.models.utils"] = types.SimpleNamespace(offset2batch=None)
        spec = importlib.util.spec_from_file_location("_ref_datasets_utils", os.path.join(ref_import.REF, "pointcept/datasets/utils.py"))
        ref = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ref)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    sys.path.insert(0, os.path.join(os.path.dirname(OUT)))
    from test_host_logic import collate_inputs
    inp = collate_inputs()
    strip = lambda d: {k: v for k, v in d.items() if k != "name"}     # noqa: E731  (the reference cannot re-collate lists of str)
    two = [ref.collate_fn([strip(d) for d in inp["batch"][:2]]), ref.collate_fn([strip(d) for d in inp["batch"][1:]])]
    out = dict(batch=ref.collate_fn([dict(d) for d in inp["batch"]]), two_in=two, two=ref.collate_fn([dict(d) for d in two]),
               tensors=ref.collate_fn(list(inp["tensors"])), numbers=ref.collate_fn([[1, 2], [3]]), strings=ref.collate_fn(["a", "b"]))
    torch.save(out, os.path.join(OUT, "collate_fn.pt"))
    print("collate_fn.pt", sorted(out))


if __name__ == "__main__" and "--only-dropin" in sys.argv:
    assert ref_import.available(), "needs /root/reference"
    gen_dropin_abi()
    gen_collate()
    sys.exit(0)

if __name__ == "__main__" and "--only-spunet" in sys.argv:
    assert ref_import.available(), "needs /root/reference"
    gen_spunet_tiny()
    sys.exit(0)

if __name__ == "__main__" and "--only-rope" in sys.argv:
    assert ref_import.available(), "needs /root/reference"
    gen_point_rope()
    sys.exit(0)

if __name__ == "__main__" and "--only-tiny" in sys.argv:
    gen_ptv3_tiny()
if __name__ == "__main__" and "--only-rpe" in sys.argv:
    assert ref_import.available(), "needs /root/reference"
    gen_attention_rpe()
    sys.exit(0)


if __name__ == "__main__":
    assert ref_import.available(), "needs /root/reference"
    os.makedirs(OUT, exist_ok=True)
    if "--only-tiny" not in sys.argv:
        gen_serialization()
        gen_point_and_padding()
        gen_grid_sample()
        gen_point_rope()
        gen_spunet_tiny()
        gen_dropin_abi()
        gen_collate()
        gen_ptv3_tiny()

