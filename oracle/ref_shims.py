"""Stand-in modules that let the reference's own Python hot path run on CPU.

TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.  Used ONLY where a checkout of
NVlabs/EmerNeRF is named by ``EMER_REFERENCE_ROOT``, by the fixture generators
``tests/golden/make_golden*.py``; no test and nothing on the GPU path needs it.

``install()`` injects, *before* any reference import:
  * ``omegaconf``                    -- name-only (``render_utils.py:9,296`` type annotation)
  * ``nerfacc`` (+ ``.data_specs``, ``.estimators.base``, ``.pdf``, ``.volrend``, ``.scan``)
                                     -- ``oracle.nerfacc_ref``
  * ``third_party.tcnn_modules``     -- ``oracle.tcnn_ref.Encoding``
and puts ``EMER_REFERENCE_ROOT`` on ``sys.path`` so that ``radiance_fields`` /
``third_party.nerfacc_prop_net`` resolve to the reference's files, unmodified.
"""
from __future__ import annotations

import os
import sys
import types

REFERENCE_ROOT = os.environ.get("EMER_REFERENCE_ROOT", "")


def reference_available() -> bool:
    return os.path.isfile(os.path.join(REFERENCE_ROOT, "radiance_fields", "radiance_field.py"))


def install() -> None:
    from . import nerfacc_ref, tcnn_ref

    if "omegaconf" not in sys.modules:
        m = types.ModuleType("omegaconf")
        m.OmegaConf = type("OmegaConf", (), {})
        sys.modules["omegaconf"] = m

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    top = mod(
        "nerfacc",
        accumulate_along_rays=nerfacc_ref.accumulate_along_rays,
        render_transmittance_from_density=nerfacc_ref.render_transmittance_from_density,
        render_weight_from_density=nerfacc_ref.render_weight_from_density,
    )
    top.__path__ = []  # mark as package
    mod("nerfacc.data_specs", RayIntervals=nerfacc_ref.RayIntervals, RaySamples=nerfacc_ref.RaySamples)
    est = mod("nerfacc.estimators")
    est.__path__ = []
    mod("nerfacc.estimators.base", AbstractEstimator=nerfacc_ref.AbstractEstimator)
    mod("nerfacc.pdf", importance_sampling=nerfacc_ref.importance_sampling,
        searchsorted=nerfacc_ref.searchsorted)
    mod("nerfacc.volrend",
        render_transmittance_from_density=nerfacc_ref.render_transmittance_from_density,
        render_weight_from_density=nerfacc_ref.render_weight_from_density,
        accumulate_along_rays=nerfacc_ref.accumulate_along_rays)
    mod("nerfacc.scan", exclusive_sum=nerfacc_ref.exclusive_sum)

    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    # the reference's third_party/ has no __init__.py -> namespace package; pre-seed the
    # tcnn binding shim so `import third_party.tcnn_modules as tcnn` never reaches the real
    # file (which raises without CUDA, tcnn_modules.py:36-39).
    import importlib

    tp = importlib.import_module("third_party")
    shim = mod("third_party.tcnn_modules", Encoding=tcnn_ref.Encoding)
    setattr(tp, "tcnn_modules", shim)


def uninstall() -> None:
    for k in list(sys.modules):
        if k == "omegaconf" or k.startswith("nerfacc") or k.startswith("third_party") \
                or k.startswith("radiance_fields"):
            m = sys.modules[k]
            f = getattr(m, "__file__", None)
            if f is None or f.startswith(REFERENCE_ROOT):
                del sys.modules[k]
    if REFERENCE_ROOT in sys.path:
        sys.path.remove(REFERENCE_ROOT)
