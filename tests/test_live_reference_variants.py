"""Constructor options and data-dict shapes beyond the four golden cases, and ray generation: the drop-in (host side
on CPU through tests/cabi_emulator.py) against what the REFERENCE's own code computed on the same inputs, stored under
tests/golden/ (tests/live_reference_variants.py --write, tests/golden/make_golden.py raygen).  The variants run in a
subprocess because the emulator is installed for the whole process there."""
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def test_option_variants_match_the_live_reference():
    r = subprocess.run([sys.executable, os.path.join(HERE, "live_reference_variants.py")], capture_output=True, text=True,
                       cwd=os.path.dirname(HERE), timeout=1500)
    assert r.returncode == 0, r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("JSON:")][-1]
    res = json.loads(line[5:])
    assert len(res) >= 20
    for name, v in res.items():
        for key, err in v["errors"].items():
            # rendered outputs and per-sample extras: same arithmetic on the same host -> rounding level;
            # gradients: summation order of the scatter / weight-gradient reductions
            tol = 2e-5 if key.startswith("grad/") or key == "prop_loss" else 2e-6
            assert err <= tol, (name, key, err)
    calls = {k: set(v["calls"]) for k, v in res.items()}
    # the fused tail must step aside where the kernel cannot take the layout ...
    for name in ("mean_embedding", "odd_geometry_width", "wide_embedding"):
        assert "emer_field_tail_fwd" not in calls[name], name
    # ... and be the path everywhere else
    for name in ("cam_embedding", "no_embedding", "bounded_aabb", "narrow_widths", "wide_heads"):
        assert "emer_field_tail_fwd" in calls[name], name
    assert "emer_linear_fwd" in calls["wide_heads"] and "emer_linear_bwd_weight" in calls["wide_heads"]


def test_raygen_module_matches_the_reference_get_rays(monkeypatch):
    """emernerf_b200.raygen.get_rays (host side through the emulator) against the reference's own function
    (datasets/base/pixel_source.py:39-76), bit for bit: its outputs on these seeded inputs, per-ray and shared camera
    matrices, are stored in tests/golden/raygen.npz (tests/golden/make_golden.py raygen)."""
    import numpy as np
    import torch

    import cabi_emulator
    from emernerf_b200 import raygen

    cabi_emulator.install(monkeypatch)
    z = np.load(os.path.join(HERE, "golden", "raygen.npz"))
    x, y, c2w, K = (torch.from_numpy(z[k]) for k in ("x", "y", "c2w", "K"))
    for tag, (c, k) in (("per_ray", (c2w, K)), ("shared", (c2w[0], K[0]))):
        got = raygen.get_rays(x, y, c, k)
        assert len(got) == 3
        for i, a in enumerate(got):
            assert torch.equal(a, torch.from_numpy(z[f"{tag}/{i}"])), (tag, i)
