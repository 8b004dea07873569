"""ctypes binding of libb2pc.so (C ABI in include/b2pc.h).  No CPU fallback: if the library is
missing or a call is made without a CUDA device, this fails loudly."""
import ctypes
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb2pc.so")
CSRC = os.path.join(_HERE, "csrc")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared", "-Xlinker", "-soname=libb2pc.so"]
BINDING_DIR = os.path.join(_HERE, "_build_torch_binding")
BINDING_PATH = os.path.join(BINDING_DIR, "_b2pc_torch.so")

_lib = None

c_i32p = ctypes.c_void_p


class ProfileEntry(ctypes.Structure):
    _fields_ = [("id", ctypes.c_int), ("calls", ctypes.c_longlong), ("ms", ctypes.c_double), ("flops", ctypes.c_double),
                ("bytes", ctypes.c_double)]


PROFILE_NAMES = ["attn_fwd", "attn_bwd", "conv_gather_gemm", "conv_bwd_weight", "serialize_encode", "serialize_sort", "rulebook_subm",
                 "rulebook_strided", "patch_padding", "fused_residual", "layer_norm", "segment_max", "colsum", "other"]


def profile_collect():
    """-> {entry point name: dict(calls, ms, flops, bytes)} for the calls made since b2pc_profile_enable(1)"""
    buf = (ProfileEntry * 32)()
    n = lib().b2pc_profile_collect(buf, 32)
    return {PROFILE_NAMES[buf[i].id]: dict(calls=int(buf[i].calls), ms=buf[i].ms, flops=buf[i].flops, bytes=buf[i].bytes) for i in range(n)}
_SIGS = {
    "b2pc_version": (ctypes.c_int, []),
    "b2pc_last_error": (ctypes.c_char_p, []),
    "b2pc_launch_count": (ctypes.c_longlong, []),
    "b2pc_serialize_encode": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                                             ctypes.POINTER(ctypes.c_int), ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_serialize_sort_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int]),
    "b2pc_serialize_sort": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_patch_padding": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_int64,
                                          ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_patch_attn_fwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
    "b2pc_patch_attn_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int, ctypes.c_int]),
    "b2pc_patch_attn_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_int,
                                           ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                           ctypes.c_int, ctypes.c_void_p]),
    "b2pc_rulebook_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int]),
    "b2pc_rulebook_subm": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.POINTER(ctypes.c_int),
                                          ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int), ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_rulebook_strided_begin": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64] + [ctypes.POINTER(ctypes.c_int)] * 5 +
                                    [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_rulebook_strided_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64] + [ctypes.POINTER(ctypes.c_int)] * 3),
    "b2pc_rulebook_strided_finish": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64] + [ctypes.POINTER(ctypes.c_int)] * 5 +
                                     [ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                      ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_spconv_gather_gemm_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "b2pc_spconv_gather_gemm": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                               ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                               ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                               ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]),
    "b2pc_spconv_bwd_weight_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "b2pc_spconv_bwd_weight": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64,
                                              ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]),
    "b2pc_segment_max_fwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                            ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_segment_max_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int64,
                                            ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_layer_norm_fwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                                           ctypes.c_float, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_layer_norm_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int]),
    "b2pc_layer_norm_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_rowscale_add": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64,
                                         ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_rowscale": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p,
                                     ctypes.c_int, ctypes.c_void_p]),
    "b2pc_colsum_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int]),
    "b2pc_colsum": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                   ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_pool_plan_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64]),
    "b2pc_pool_plan": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                      ctypes.c_int] + [ctypes.c_void_p] * 9 + [ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_profile_enable": (None, [ctypes.c_int]),
    "b2pc_profile_collect": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "b2pc_serialized_attn_fwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                                ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p,
                                                ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_serialized_attn_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int64]),
    "b2pc_serialized_attn_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                                                ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_fused_residual_fwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p,
                                               ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_int64, ctypes.c_int,
                                               ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_fused_residual_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int]),
    "b2pc_fused_residual_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                               ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                               ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                               ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_multi_cast": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]),
    "b2pc_multi_adamw": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                        ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b2pc_gelu_fwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_gelu_bwd_colsum_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int]),
    "b2pc_gelu_bwd_colsum": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_gelu_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_grid_sample_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int, ctypes.c_int64]),
    "b2pc_grid_sample_plan": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int64,
                                             ctypes.POINTER(ctypes.c_double), ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 7 +
                              [ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_grid_sample_select": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_uint64,
                                                                      ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_grid_sample_displacement": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_int64, ctypes.POINTER(ctypes.c_double),
                                                                             ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
    "b2pc_gather_rows": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_knn_query": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_vote_accumulate": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "b2pc_point_rope": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                       ctypes.c_float, ctypes.c_float, ctypes.c_void_p]),
    "b2pc_cross_entropy_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int64]),
    "b2pc_cross_entropy_fwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int64,
                                              ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "b2pc_cross_entropy_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                              ctypes.c_int64, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
}
EXPORTS = tuple(_SIGS)


def build(verbose=False, extra_flags=()):
    """Compile libb2pc.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
    extra_flags = list(extra_flags)
    cmd = ["nvcc"] + NVCC_FLAGS + extra_flags + [os.path.join(CSRC, "b2pc.cu"), "-o", LIB_PATH]
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    subprocess.run(cmd, check=True, cwd=CSRC)
    return LIB_PATH


def build_torch_binding(verbose=False):
    """Compile the pybind/C++ autograd binding (csrc/torch_binding.cpp) in-tree against this torch; g++ only, no GPU needed."""
    from torch.utils import cpp_extension
    os.makedirs(BINDING_DIR, exist_ok=True)
    lib()  # libb2pc.so must be loaded (by soname) before the module that depends on it is imported
    return cpp_extension.load(name="_b2pc_torch", sources=[os.path.join(CSRC, "torch_binding.cpp")], build_directory=BINDING_DIR,
                              extra_cflags=["-O2", "-std=c++17"],
                              extra_ldflags=[f"-L{_HERE}", "-lb2pc"], with_cuda=True,
                              verbose=verbose)


_binding = None


def torch_binding():
    """The compiled binding if it has been built (and B2PC_BINDING != ctypes), else None: ops.py then uses the ctypes path.
    Both bindings call the same C ABI; neither is a CPU fallback."""
    global _binding
    if _binding is None:
        _binding = False
        if os.environ.get("B2PC_BINDING", "") != "ctypes" and os.path.exists(BINDING_PATH):
            import importlib.util
            import torch  # noqa: F401  (libtorch symbols)
            lib()
            spec = importlib.util.spec_from_file_location("_b2pc_torch", BINDING_PATH)
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            _binding = mod
    return _binding or None


def _stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(os.path.dirname(_HERE), "include", "b2pc.h")]
    return any(os.path.getmtime(s) > t for s in srcs if os.path.exists(s))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"pointcept_b200: {LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). There is no CPU or PyTorch fallback for these operators.")
        l = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
        for name, (res, args) in _SIGS.items():
            fn = getattr(l, name)  # raises AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(status, what):
    if status != 0:
        msg = lib().b2pc_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"b2pc {what} failed (status {status}): {msg}")
