"""The lidar scene-flow evaluation of emernerf_b200.metrics on the host (CPU suite): ``eval_lidar_flow`` runs the
drop-in field through tests/cabi_emulator.py and emer_lidar_flow_accumulate through tests/lidar_flow_emulator.py (its
fp64 restatement), and is checked against the reference's own results (tests/golden/lidar_flow.npz,
make_golden_lidar_flow.py): keys, key order and types, every per-frame count exactly, the statistics within 1e-6
relative and NaN where the reference gives NaN.  Also chunked frames, the gate's edge values, the argument errors, the
refusal of CPU tensors without the emulator, and ``LidarRaySampler.get_render_rays`` against the reference's frames."""
import math
import os
import types

import numpy as np
import pytest
import torch

import lidar_flow_cases as lc
import lidar_flow_emulator
from oracle import lidar_flow_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lidar_flow.npz")
REL = 1e-6


@pytest.fixture
def metrics(monkeypatch):
    lidar_flow_emulator.install(monkeypatch)
    from emernerf_b200 import metrics

    return metrics


def dropin_field(z):
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                               build_density_field=build_density_field)
    field = lc.fixture_field(ns, float(z["density_shift"]))
    # the seeded parameters are the reference's only if both fields have the same parameter names
    assert sorted(k for k, _ in field.named_parameters()) == z["parameters"].tolist()
    return field


def check_against_golden(metrics, z, case, field, device="cpu"):
    source, remove_ground, split = lc.CASES[case]
    lidar_set = lc.SplitSet(lc.load(z, source, device=device), split)
    sums = metrics._lidar_flow_sums(lidar_set, field, remove_ground).cpu().numpy()
    assert np.array_equal(lc.counts_of(sums), z[f"{case}/frame_counts"])
    got = metrics.eval_lidar_flow(lidar_set, field, remove_ground)
    assert list(got) == list(lidar_flow_ref.KEYS)
    assert all(type(v) is np.float64 for v in got.values())
    want = z[f"{case}/result"]
    for k, w in zip(lidar_flow_ref.KEYS, want):
        if math.isnan(w):
            assert math.isnan(got[k]), (case, k, got[k])
        else:
            assert abs(got[k] - w) <= REL * abs(w), (case, k, got[k], w)
    return got


@pytest.mark.parametrize("case", list(lc.CASES))
def test_against_reference_golden(metrics, case):
    z = np.load(GOLDEN)
    check_against_golden(metrics, z, case, dropin_field(z))


def test_chunks_add_up(metrics, monkeypatch):
    """Frames split into chunks that are not multiples of anything give the same counts and results."""
    z = np.load(GOLDEN)
    monkeypatch.setattr(metrics, "FLOW_CHUNK_POINTS", 97)
    check_against_golden(metrics, z, "drive", dropin_field(z))


class FlowStub(torch.nn.Module):
    """A flow field whose forward flow and dynamic density are given per point (by the point's x coordinate)."""

    def __init__(self, pred, density):
        super().__init__()
        self.pred, self.density = pred, density
        self.flow_xyz_encoder = True

    def query_flow(self, positions, normed_timestamps):
        rows = positions[:, 0].long()
        flow = torch.cat([self.pred[rows], torch.zeros(len(rows), 3)], -1)
        return {"forward_flow": flow[:, :3], "backward_flow": flow[:, 3:], "dynamic_density": self.density[rows]}


def stub_set(n=12, flows=True):
    src = lc.LidarSource()
    src.origins = torch.stack([torch.arange(n).float(), torch.zeros(n), torch.zeros(n)], -1)
    src.directions = torch.tensor([[0.0, 0.0, 1.0]]).repeat(n, 1)
    src.ranges = torch.zeros(n, 1)
    src._timesteps = torch.zeros(n, dtype=torch.int64)
    src._normalized_timestamps = torch.zeros(n)
    if flows:
        src.flows = torch.tensor([[0.5, 0.0, 0.0]]).repeat(n, 1)
        src.flow_classes = torch.zeros(n, dtype=torch.int64)
        src.grounds = torch.zeros(n, dtype=torch.bool)
    return lc.SplitSet(src, [0])


def test_gate_edge_values(metrics):
    """A density of exactly 0.2f is kept, a NaN density is kept, and a NaN prediction gives a NaN EPE, is neither
    accurate nor an outlier, and has an angle of pi / 2 -- as the reference's gate and statistics."""
    lidar_set = stub_set(4)
    pred = torch.tensor([[0.5, 0.0, 0.0], [0.5, 0.0, 0.0], [0.5, 0.0, 0.0], [float("nan"), 0.0, 0.0]])
    density = torch.tensor([0.2, float("nan"), 0.19999999, 1.0])
    field = FlowStub(pred, density)
    got = metrics._lidar_flow_sums(lidar_set, field, True)[0].tolist()
    # points 0 and 1 are kept (zero error), point 2 is gated to 0 (error 0.5), point 3 is NaN
    assert math.isnan(got[0])
    assert got[1:4] == [2.0, 2.0, 1.0]                  # strict, relaxed: points 0, 1; outlier: point 2 only
    assert got[5:] == [4.0, 4.0, 4.0]
    # angles: points 0 and 1 at the dot of their unit vectors, (0.5 / (0.5 + 1e-7))^2, the zero flow of point 2 and
    # the NaN of point 3 at a dot of 0
    aligned = math.acos((0.5 / (0.5 + 1e-7)) ** 2)
    assert math.isclose(got[4], 2 * aligned + math.pi, rel_tol=1e-12)
    ref = lidar_flow_ref.scene_flow_metrics(pred[None, 3:], lidar_set.datasource.flows[None, 3:])
    assert math.isnan(ref["EPE3D"]) and ref["acc3d_strict"] == 0.0 and ref["outlier"] == 0.0
    assert math.isclose(ref["angle_error"], math.pi / 2, rel_tol=1e-6)


def test_negative_gated_flow_gives_negative_zero(metrics):
    """pred *= 0 on a negative value is -0; the statistics do not see the sign, so the sums match a zero flow."""
    lidar_set = stub_set(2)
    a = metrics._lidar_flow_sums(lidar_set, FlowStub(torch.tensor([[-0.3, -1.0, 0.2]] * 2), torch.zeros(2)), True)
    b = metrics._lidar_flow_sums(lidar_set, FlowStub(torch.zeros(2, 3), torch.zeros(2)), True)
    assert torch.equal(a, b)


def test_filters_and_empty_frames(metrics, caplog):
    lidar_set = stub_set(6)
    src = lidar_set.datasource
    src.flow_classes[:2] = -1
    src.grounds[2] = True
    field = FlowStub(torch.tensor([[0.5, 0.0, 0.0]] * 6), torch.ones(6))
    got = metrics._lidar_flow_sums(lidar_set, field, True)[0].tolist()
    assert got[6:] == [3.0, 4.0]
    got = metrics._lidar_flow_sums(lidar_set, field, False)[0].tolist()
    assert got[6:] == [4.0, 4.0]
    src.flow_classes[:] = -1
    lidar_set.split_indices = [0, 5]                      # no labelled point, and an absent time index
    with caplog.at_level("INFO"):
        with pytest.warns(RuntimeWarning):
            out = metrics.eval_lidar_flow(lidar_set, field)
    assert sum("no valid points, skipping..." in r.message for r in caplog.records) == 2
    assert list(out) == list(lidar_flow_ref.KEYS) and all(math.isnan(v) for v in out.values())


def test_argument_errors(metrics):
    lidar_set = stub_set(3)
    field = FlowStub(torch.zeros(3, 3), torch.ones(3))
    with pytest.raises(ValueError, match="split_indices"):
        metrics.eval_lidar_flow(types.SimpleNamespace(datasource=lidar_set.datasource), field)
    with pytest.raises(ValueError, match="split_indices"):
        metrics.eval_lidar_flow(lidar_set.datasource, field)
    field.flow_xyz_encoder = None
    with pytest.raises(ValueError, match="flow branch"):
        metrics.eval_lidar_flow(lidar_set, field)
    with pytest.raises(ValueError, match="flows"):
        metrics.eval_lidar_flow(stub_set(3, flows=False), FlowStub(torch.zeros(3, 3), torch.ones(3)))


def test_cpu_tensors_are_refused():
    from emernerf_b200 import metrics

    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.eval_lidar_flow(stub_set(3), FlowStub(torch.zeros(3, 3), torch.ones(3)))


@pytest.mark.parametrize("source", ["drive", "unsorted"])
@pytest.mark.parametrize("with_flows", [True, False], ids=["7key", "4key"])
def test_render_rays_match_reference_frames(source, with_flows):
    """Every frame, and an absent time index, is torch.equal to the reference's get_render_rays (its rows of the
    source, stored by the generator, which checked them against the reference's outputs), for contiguous and
    interleaved timesteps and for sources with and without flow labels."""
    from emernerf_b200.raygen import LidarRaySampler

    z = np.load(GOLDEN)
    src = lc.load(z, source, with_flows=with_flows)
    sampler = LidarRaySampler(src)
    keys = lc.FRAME_KEYS if with_flows else lc.FRAME_KEYS[:4]
    for t in list(range(lc.N_SCANS)) + [lc.ABSENT]:
        got = sampler.get_render_rays(t)
        want = {k: getattr(src, lc.ATTRS[k])[lc.rows(z, source, t)] for k in keys}
        assert list(got) == list(keys)
        for k in keys:
            assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), (t, k)
        oracle = lidar_flow_ref.get_render_rays(src, t)
        assert all(torch.equal(got[k], oracle[k]) for k in keys)
    assert (sampler._frames[3] is None) == (source == "drive")      # slices for contiguous runs, gathers otherwise


def test_frame_table_follows_the_timesteps():
    """A new timesteps tensor or an in-place change rebuilds the table."""
    from emernerf_b200.raygen import LidarRaySampler

    src = stub_set(6).datasource
    sampler = LidarRaySampler(src)
    assert len(sampler.get_render_rays(0)["lidar_origins"]) == 6
    src._timesteps[3:] = 1
    assert torch.equal(sampler.get_render_rays(1)["lidar_origins"], src.origins[3:])
    src._timesteps = torch.tensor([2, 1, 2, 1, 2, 1])
    assert torch.equal(sampler.get_render_rays(2)["lidar_origins"], src.origins[[0, 2, 4]])
    assert len(sampler.get_render_rays(0)["lidar_origins"]) == 0
