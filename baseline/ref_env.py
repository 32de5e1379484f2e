"""Make the UNMODIFIED reference importable (test / bench infrastructure, never imported by the product).

``baseline/_ref/`` holds a ``pip install --target`` of the reference tree (``__graft_entry__.build()``
populates it where ``/root/reference`` exists; git-ignored, NOT gpurun-ignored, so it travels to the GPU
box).  ``activate()`` puts it on ``sys.path`` and stubs the two pure-Python dependencies the image lacks
(``omegaconf``: only type names are touched at import, ``modelopt/torch/utils/robust_json.py:31``;
``pulp``: only used by the NAS searcher, ``modelopt/torch/opt/searcher.py:32``) -- the shim of
SURVEY.md Appendix D.

``use_prebuilt_extensions()`` hands the reference's loader (``quantization/extensions.py:28-72``) the
reference's own CUDA extensions, compiled ahead of time for sm_90a from the reference sources by
``oracle/build_ref_ext.py`` with the flags the loader itself uses.  It only skips the JIT compile (minutes per
translation unit on a fresh box); the code that runs is the reference's.
"""

from __future__ import annotations

import importlib.machinery
import importlib.util
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_DIR = os.path.join(HERE, "_ref")
PREBUILT = os.path.join(ROOT, "oracle", "_ref")


def available() -> bool:
    return os.path.isdir(os.path.join(REF_DIR, "modelopt"))


def _stub_missing_deps() -> None:
    class _Any(types.ModuleType):
        def __getattr__(self, k):
            if k.startswith("__"):
                raise AttributeError(k)
            return type(k, (), {})

    for name in ("omegaconf", "pulp"):
        try:
            importlib.import_module(name)
        except ImportError:
            mod = _Any(name)
            if name == "omegaconf":
                mod.DictConfig = type("DictConfig", (dict,), {})
                mod.ListConfig = type("ListConfig", (list,), {})
            sys.modules[name] = mod


def activate():
    """Import and return ``modelopt.torch.quantization`` from ``baseline/_ref`` (RuntimeError if absent)."""
    if not available():
        raise RuntimeError("baseline/_ref is empty: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "where /root/reference exists")
    _stub_missing_deps()
    if REF_DIR not in sys.path:
        sys.path.insert(0, REF_DIR)
    import modelopt.torch.quantization as mtq

    if not os.path.abspath(mtq.__file__).startswith(REF_DIR):
        raise RuntimeError(f"modelopt resolved to {mtq.__file__}, not to baseline/_ref")
    return mtq


def _load_so(name: str):
    path = os.path.join(PREBUILT, name + ".so")
    if not os.path.exists(path):
        return None
    import torch  # noqa: F401  (the extension links libtorch)

    loader = importlib.machinery.ExtensionFileLoader(name, path)
    mod = importlib.util.module_from_spec(importlib.util.spec_from_loader(name, loader))
    loader.exec_module(mod)
    return mod


def use_prebuilt_extensions() -> dict:
    """Pre-seed the reference loader's cache (``get_cuda_ext.extension`` ...) with the ahead-of-time builds of
    its own sources.  Returns {name: loaded?}."""
    import torch

    activate()
    import modelopt.torch.quantization.extensions as ext

    out = {}
    if not torch.cuda.is_available():
        return out
    for fn, name in ((ext.get_cuda_ext, "modelopt_cuda_ext"), (ext.get_cuda_ext_fp8, "modelopt_cuda_ext_fp8"),
                     (ext.get_cuda_ext_mx, "modelopt_cuda_ext_mx")):
        if getattr(fn, "extension", None) is None:
            mod = _load_so(name)
            if mod is not None:
                fn.extension = mod
        out[name] = getattr(fn, "extension", None) is not None
    return out
