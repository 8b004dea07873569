"""pointcept_b200 -- H100 (sm_90a) operators behind Pointcept's PT-v3 / SpUNet hot path.

``install()`` registers the drop-in modules under the import names the reference uses
(``spconv``, ``spconv.pytorch``, optionally ``flash_attn``, and with ``extras=True`` ``pointrope`` and ``pointops.knn_query``) so unmodified Pointcept model files
and configs resolve to these operators.
"""
import sys

__version__ = "0.1.0"


def install(flash_attn=True, extras=False):
    from . import spconv as _spconv
    sys.modules["spconv"] = _spconv
    sys.modules["spconv.pytorch"] = _spconv.pytorch
    sys.modules["spconv.pytorch.modules"] = _spconv.pytorch.modules
    sys.modules["spconv.pytorch.conv"] = _spconv.pytorch.conv
    sys.modules["spconv.pytorch.core"] = _spconv.pytorch.core
    if flash_attn:
        from . import flash_attn_interface as _fa
        import types
        m = types.ModuleType("flash_attn")
        m.flash_attn_varlen_qkvpacked_func = _fa.flash_attn_varlen_qkvpacked_func
        m.__version__ = "2.8.3+b2pc"
        m.flash_attn_interface = _fa
        sys.modules["flash_attn"] = m
        sys.modules["flash_attn.flash_attn_interface"] = _fa
    if extras:
        import types
        from . import pointops as _po, pointrope as _pr
        sys.modules["pointrope"] = _pr
        if "pointops" not in sys.modules:      # only the query the evaluation path of PT-v3 / SpUNet uses; never shadow a real pointops
            m = types.ModuleType("pointops")
            m.knn_query = _po.knn_query
            sys.modules["pointops"] = m
