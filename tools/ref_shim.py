"""Import shim that makes the READ-ONLY reference checkout importable in the build container.

Only used by tools/gen_golden.py (fixture generation) — never by the product, tests, smoke() or bench.
The four shims are documented in SURVEY.md §8(c)/Appendix A; no reference file is modified or copied.
"""
import importlib.util
import os
import sys
import types

import torch  # noqa: F401  (must precede the matplotlib stub)

REF = os.environ["DPB200_REFERENCE"]   # path of the reference checkout


def install():
    import huggingface_hub
    import huggingface_hub.constants as hc

    if not hasattr(hc, "hf_cache_home"):
        hc.hf_cache_home = os.path.expanduser("~/.cache/huggingface")
    for name in ("HfFolder", "cached_download"):
        if not hasattr(huggingface_hub, name):
            setattr(huggingface_hub, name, type(name, (), {}))

    class _Plt(types.ModuleType):
        def __getattr__(self, k):
            if k.startswith("__"):
                raise AttributeError(k)
            return lambda *a, **kw: None

    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = _Plt("matplotlib.pyplot")
    sys.modules["matplotlib"] = mpl
    sys.modules["matplotlib.pyplot"] = mpl.pyplot

    orig = importlib.util.find_spec
    importlib.util.find_spec = lambda n, *a, **k: None if n == "transformers" else orig(n, *a, **k)
    sys.path[:0] = [os.path.join(REF, "ddpm_exp"), REF]
    import diffusers  # noqa: F401

    importlib.util.find_spec = orig
    import torch_pruning  # noqa: F401

    return diffusers, torch_pruning
