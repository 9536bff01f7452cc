"""The few-shot occupancy evaluation of emernerf_b200.metrics on the host (CPU suite): ``collect_centroids`` and
``eval_few_shot_occ`` run the drop-in field through tests/cabi_emulator.py and the occupancy kernels through
tests/occupancy_emulator.py (their fp64 restatement), and are checked against the reference's own functions
(tests/golden/occupancy.npz, make_golden_occ.py): centroids to 1e-5 of each row's largest magnitude, every count and
so every accuracy exactly.  Also the argument errors, the reference's ZeroDivisionError and KeyError, and the
refusal of CPU tensors without the emulator."""
import os
import types

import numpy as np
import pytest
import torch

import occ_cases as oc
import occupancy_emulator

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "occupancy.npz")
CENTROID_REL = 1e-5


@pytest.fixture
def metrics(monkeypatch):
    occupancy_emulator.install(monkeypatch)
    from emernerf_b200 import metrics

    return metrics


def dropin_field(z, model):
    from emernerf_b200.radiance_fields import RadianceField, build_density_field
    from emernerf_b200.radiance_fields.encodings import HashEncoder

    ns = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                               build_density_field=build_density_field)
    field = oc.fixture_field(ns, model, float(z[f"{model}/density_shift"]))
    # the seeded parameters are the reference's only if both fields have the same parameter names
    assert sorted(k for k, _ in field.named_parameters()) == z[f"{model}/parameters"].tolist()
    return field


def check_against_golden(metrics, z, model, field, dataset, device):
    want_c = torch.from_numpy(z[f"{model}/centroids"])
    centroids, bank = metrics.collect_centroids(list(oc.TRAIN), dataset, field, device)
    assert centroids.dtype == torch.float32 and tuple(centroids.shape) == (oc.N_CLASSES, 64)
    assert bank.dtype == torch.int64 and bank.tolist() == list(range(oc.N_CLASSES))
    centroids = centroids.cpu()
    assert not want_c[oc.MISSING_TRAIN].any() and not centroids[oc.MISSING_TRAIN].any()
    scale = want_c.abs().amax(dim=-1, keepdim=True).clamp_min(1e-30)
    assert ((centroids - want_c).abs() / scale).max() <= CENTROID_REL
    got = metrics.eval_few_shot_occ(list(oc.TEST), dataset, field, device, centroids.to(device), bank)
    assert set(got) == {"micro_accuracy", "macro_accuracy", "per_class_accuracy", "cover_rate",
                        "num_measured_points", "num_total_points"}
    for k in ("num_measured_points", "num_total_points"):
        assert isinstance(got[k], int) and got[k] == int(z[f"{model}/{k}"]), k
    for k in ("micro_accuracy", "macro_accuracy", "cover_rate"):
        assert isinstance(got[k], float) and got[k] == float(z[f"{model}/{k}"]), k
    assert list(got["per_class_accuracy"]) == list(oc.LABEL_MAPPING.values())
    assert list(got["per_class_accuracy"].values()) == z[f"{model}/per_class_accuracy"].tolist()
    return got


@pytest.mark.parametrize("model", oc.MODELS)
def test_against_reference_golden(metrics, model):
    z = np.load(GOLDEN)
    field = dropin_field(z, model)
    dataset = oc.OccDataset(oc.load_frames(z, model))
    got = check_against_golden(metrics, z, model, field, dataset, torch.device("cpu"))
    assert got["per_class_accuracy"][oc.LABEL_MAPPING[oc.MISSING_TEST]] == 0.0
    assert 0 < got["num_measured_points"] < got["num_total_points"]


def test_chunks_add_up(metrics, monkeypatch):
    """Frames split into chunks that are not multiples of anything give the same counts and centroids."""
    z = np.load(GOLDEN)
    field = dropin_field(z, "static_feat")
    dataset = oc.OccDataset(oc.load_frames(z, "static_feat"))
    monkeypatch.setattr(metrics, "OCC_CHUNK_POINTS", 97)
    check_against_golden(metrics, z, "static_feat", field, dataset, torch.device("cpu"))


class FieldStub(torch.nn.Module):
    """Per-voxel density and features given by the dataset (columns 0 and 1.. of the positions' source rows)."""

    def __init__(self, density, feat):
        super().__init__()
        self.density, self.feat = density, feat

    def forward(self, positions, data_dict, **kw):
        rows = positions[:, 0].long()
        return {"density": self.density[rows][:, None], "dino_feat": self.feat[rows]}


def stub_case(n=40, c=8, k=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(n, c, generator=g)
    density = torch.rand(n, generator=g)
    labels = torch.randint(0, k, (n,), generator=g)
    coords = torch.stack([torch.arange(n).float(), torch.zeros(n), torch.zeros(n)], -1)
    ds = types.SimpleNamespace(label_mapping={j: f"c{j}" for j in range(k)},
                               get_occ=lambda i: (coords, labels, torch.zeros(n)))
    return FieldStub(density, feat), ds, labels


def test_density_threshold_is_strict_and_nan_fails(metrics):
    field, ds, labels = stub_case()
    field.density[:4] = torch.tensor([0.2, float("nan"), 0.20000001, 0.19999999])
    keep = field.density > 0.2
    centroids, _ = metrics.collect_centroids([0], ds, field, "cpu")
    for j in range(4):
        m = keep & (labels == j)
        want = field.feat[m].double().mean(0).float() if m.any() else torch.zeros(8)
        assert torch.allclose(centroids[j], want, rtol=1e-6, atol=1e-7)
    got = metrics.eval_few_shot_occ([0], ds, field, "cpu", centroids, torch.arange(4))
    assert got["num_measured_points"] == int(keep.sum()) and got["num_total_points"] == 40


def test_no_measured_voxel_raises_zero_division(metrics):
    field, ds, _ = stub_case()
    field.density.zero_()
    with pytest.raises(ZeroDivisionError):
        metrics.eval_few_shot_occ([0, 0], ds, field, "cpu", torch.rand(4, 8), torch.arange(4))
    centroids, _ = metrics.collect_centroids([0], ds, field, "cpu")
    assert not centroids.any()


def test_measured_label_outside_the_mapping_raises_key_error(metrics):
    field, ds, labels = stub_case()
    field.density.fill_(1.0)
    labels[7] = 4
    with pytest.raises(KeyError):
        metrics.eval_few_shot_occ([0], ds, field, "cpu", torch.rand(4, 8), torch.arange(4))
    field.density[7] = 0.0                          # filtered out first: no lookup, as in the reference
    metrics.eval_few_shot_occ([0], ds, field, "cpu", torch.rand(4, 8), torch.arange(4))


def test_no_train_frames_give_zero_centroids(metrics):
    _, ds, _ = stub_case()
    centroids, bank = metrics.collect_centroids([], ds, None, "cpu")
    assert tuple(centroids.shape) == (4, 64) and not centroids.any() and bank.tolist() == [0, 1, 2, 3]


@pytest.mark.parametrize("bad", ["channels", "wide", "classes", "bank", "mapping", "feature_width"])
def test_argument_errors(metrics, bad):
    field, ds, _ = stub_case(k=4)
    cen, bank = torch.rand(4, 8), torch.arange(4)
    if bad == "channels":
        field.feat = torch.randn(40, 6)
        with pytest.raises(ValueError):
            metrics.collect_centroids([0], ds, field, "cpu")
        return
    if bad == "wide":
        field.feat = torch.randn(40, 260)
        with pytest.raises(ValueError):
            metrics.collect_centroids([0], ds, field, "cpu")
        return
    if bad == "classes":
        ds.label_mapping = {j: f"c{j}" for j in range(33)}
        cen, bank = torch.rand(33, 8), torch.arange(33)
    elif bad == "bank":
        bank = torch.arange(3)
    elif bad == "mapping":
        ds.label_mapping = {j + 1: f"c{j}" for j in range(4)}
    else:
        cen = torch.rand(4, 12)
    with pytest.raises(ValueError):
        metrics.eval_few_shot_occ([0], ds, field, "cpu", cen, bank)


def test_cpu_tensors_are_refused():
    from emernerf_b200 import metrics

    field, ds, _ = stub_case()
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.collect_centroids([0], ds, field, "cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.eval_few_shot_occ([0], ds, field, "cpu", torch.rand(4, 8), torch.arange(4))
