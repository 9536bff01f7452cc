"""emernerf_b200 -- H100-native (sm_90a) volumetric renderer for EmerNeRF's per-ray-batch hot path.

Drop-in for the reference's ``radiance_fields`` package and ``third_party.nerfacc_prop_net`` /
``third_party.tcnn_modules`` modules: same class names, constructor arguments, ``forward`` /
``render_rays`` / ``sampling`` signatures and state-dict keys, evaluated by hand-written CUDA kernels
behind the C ABI of ``include/emer_b200.h`` (``emernerf_b200/lib/libemer_b200.so``).

    import emernerf_b200
    emernerf_b200.install_dropin()          # before `train_emernerf.py` imports radiance_fields
    from radiance_fields import RadianceField, DensityField, build_density_field
    from radiance_fields.render_utils import render_rays
    from third_party.nerfacc_prop_net import PropNetEstimator, get_proposal_requires_grad_fn
"""
from __future__ import annotations

import sys

__version__ = "0.1.0"


def install_dropin() -> None:
    """Alias the reference's module names to this package in ``sys.modules`` so that
    ``train_emernerf.py`` / ``builders.py`` import the GPU path without modification."""
    import importlib
    import importlib.util
    import os
    import types

    from . import radiance_fields as rf
    from .third_party import nerfacc_compat, nerfacc_prop_net, tcnn_modules

    def reference_dirs(package: str):
        """Directories named ``package`` on sys.path that are not this package's (the reference checkout's)."""
        own = os.path.dirname(os.path.abspath(__file__))
        out = []
        for base in sys.path:
            d = os.path.join(base or os.getcwd(), package)
            if os.path.isdir(d) and not os.path.abspath(d).startswith(own) and d not in out:
                out.append(d)
        return out

    # The overridden modules resolve to this package; every OTHER submodule of the reference's packages
    # (radiance_fields.video_utils, third_party.feature_extractor: train_emernerf.py:23, datasets/...) keeps
    # resolving to the reference's own file through the package search path.
    sys.modules["radiance_fields"] = rf
    for d in reference_dirs("radiance_fields"):
        if d not in rf.__path__:
            rf.__path__.append(d)
    for sub in ("encodings", "mlp", "nerf_utils", "radiance_field", "render_utils"):
        sys.modules[f"radiance_fields.{sub}"] = importlib.import_module(f"{__name__}.radiance_fields.{sub}")
    tp = sys.modules.get("third_party")
    if tp is None:
        tp = types.ModuleType("third_party")
        tp.__path__ = []
        sys.modules["third_party"] = tp
    for d in reference_dirs("third_party"):
        if d not in list(tp.__path__):
            tp.__path__.append(d)
    sys.modules["third_party.nerfacc_prop_net"] = nerfacc_prop_net
    sys.modules["third_party.tcnn_modules"] = tcnn_modules
    tp.nerfacc_prop_net = nerfacc_prop_net
    tp.tcnn_modules = tcnn_modules
    # loss/base.py:7 does `from nerfacc import accumulate_along_rays`: answer it from the library's compositing
    # kernels unless the real package is installed (then it keeps working as it is)
    if "nerfacc" not in sys.modules and importlib.util.find_spec("nerfacc") is None:
        sys.modules["nerfacc"] = nerfacc_compat


def library_path() -> str:
    from . import _lib

    return _lib.lib_path()
