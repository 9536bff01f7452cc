"""Generate tests/golden/occupancy.npz by running the REFERENCE's own collect_centroids and eval_few_shot_occ on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_occ.py

For each model of ``occ_cases.MODELS`` this builds the reference's own ``RadianceField`` (with the stand-ins of
``oracle.ref_shims``) in eval mode, evaluates it at the seeded candidate voxels of every frame, and composes the frames
from those values: voxels on both sides of the 0.2 density filter, a class missing from the train frames (a zero
centroid), a class missing from the test frames, labels outside the mapping on train voxels that pass the filter and
on test voxels that do not, and one test frame in which no voxel passes (the reference's ``continue``).  Voxels whose
density lies within 1e-4 relative of 0.2, and test voxels whose best two cosine similarities to the reference's
centroids lie within 1e-4, are dropped, so every count is well defined.  Then it runs the unmodified
``datasets/metrics.py`` functions on a dataset object serving those frames and writes, per model, the density shift
(the parameters are seeded by ``occ_cases.seed_parameters``), which candidates each frame keeps and their labels, the
centroids and the metrics.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

warnings.filterwarnings("ignore", category=FutureWarning)

from oracle import ref_shims  # noqa: E402

ref_shims.install()

import occ_cases as oc  # noqa: E402
from radiance_fields import RadianceField, build_density_field  # noqa: E402  (reference)
from radiance_fields.encodings import HashEncoder  # noqa: E402  (reference)

REF = types.SimpleNamespace(HashEncoder=HashEncoder, RadianceField=RadianceField,
                            build_density_field=build_density_field)


def load_reference_metrics():
    sk = types.ModuleType("skimage")
    sk.__path__ = []
    skm = types.ModuleType("skimage.metrics")
    skm.structural_similarity = None                  # not used by the occupancy evaluation
    sys.modules.update({"skimage": sk, "skimage.metrics": skm})
    spec = importlib.util.spec_from_file_location("reference_metrics",
                                                  os.path.join(ref_shims.REFERENCE_ROOT, "datasets", "metrics.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def field_values(field, index, coords):
    with torch.no_grad():
        out = field.forward(positions=coords, data_dict={"normed_timestamps": oc.normed_time(index, len(coords))},
                            combine_static_dynamic=True, query_feature_head=True, query_pe_head=False)
    return out["density"].squeeze(-1), out["dino_feat"]


def draw_labels(feat, g, proj, absent):
    """Labels that follow the features (argmax of a fixed projection) for 3 voxels in 4, random for the rest."""
    z = (feat.double() @ proj).clone()
    z[:, absent] = -float("inf")
    lab = z.argmax(-1)
    allowed = torch.tensor([j for j in range(oc.N_CLASSES) if j != absent])
    noisy = torch.rand(len(lab), generator=g) < 0.25
    lab[noisy] = allowed[torch.randint(0, len(allowed), (int(noisy.sum()),), generator=g)]
    return lab


def nearest_labels(feat, centroids, g, absent):
    """Test labels: the nearest centroid's class (cosine) for 3 voxels in 4, random for the rest."""
    q = feat.double() / (feat.double().norm(dim=-1, keepdim=True) + 1e-7)
    c = centroids.double() / (centroids.double().norm(dim=-1, keepdim=True) + 1e-7)
    return draw_labels(q @ c.T, g, torch.eye(oc.N_CLASSES, dtype=torch.float64), absent)


def cosine_gap(feat, centroids):
    """Best minus second-best cosine similarity in fp64, per voxel."""
    q = feat.double() / (feat.double().norm(dim=-1, keepdim=True) + 1e-7)
    c = centroids.double() / (centroids.double().norm(dim=-1, keepdim=True) + 1e-7)
    top = (q @ c.T).topk(2, dim=-1).values
    return top[:, 0] - top[:, 1]


def run_model(ref, model, store):
    """Seeded parameters, the density band widened and centred on the threshold (so that frames have voxels on both
    sides of the filter), then the frames and the reference's results."""
    field = oc.build_field(REF, model)
    oc.seed_parameters(field)
    field.eval()
    oc.widen_density(field)
    d, _ = field_values(field, 0, oc.candidates(0))
    shift = float(torch.log(d.median() / oc.THRESHOLD))
    oc.shift_density(field, shift)
    again = oc.fixture_field(REF, model, shift).state_dict()      # what the tests rebuild from the stored shift
    assert all(torch.equal(again[k], v) for k, v in field.state_dict().items())
    store[f"{model}/density_shift"] = np.array(shift, np.float64)
    store[f"{model}/parameters"] = np.array(sorted(k for k, _ in field.named_parameters()))
    g = torch.Generator().manual_seed(77)
    proj = torch.randn(64, oc.N_CLASSES, generator=g, dtype=torch.float64)
    frames = {}

    keeps = {}

    def compose(index, keep_rows, labels):
        keeps[index] = (keep_rows, labels)
        frames[index] = oc.frame(index, keep_rows, labels)

    for i in oc.TRAIN:
        d, f = field_values(field, i, oc.candidates(i))
        ok = (d - oc.THRESHOLD).abs() > oc.MARGIN * oc.THRESHOLD
        lab = draw_labels(f, g, proj, oc.MISSING_TRAIN)
        outside = torch.rand(len(lab), generator=g) < 0.03          # skipped by the centroid loop
        lab[outside] = oc.OUTSIDE
        compose(i, ok, lab[ok])
    dataset = oc.OccDataset(frames)
    centroids, label_bank = ref.collect_centroids(list(oc.TRAIN), dataset, field, torch.device("cpu"))

    for i in oc.TEST:
        d, f = field_values(field, i, oc.candidates(i))
        passes = d > oc.THRESHOLD
        ok = ((d - oc.THRESHOLD).abs() > oc.MARGIN * oc.THRESHOLD) & (~passes | (cosine_gap(f, centroids) > oc.MARGIN))
        if i == oc.EMPTY_TEST:
            ok &= ~passes
        lab = nearest_labels(f, centroids, g, oc.MISSING_TEST)
        outside = (torch.rand(len(lab), generator=g) < 0.05) & ~passes   # filtered out before the class lookup
        lab[outside] = oc.OUTSIDE
        compose(i, ok, lab[ok])
    dataset = oc.OccDataset(frames)
    result = ref.eval_few_shot_occ(list(oc.TEST), dataset, field, torch.device("cpu"), centroids, label_bank)

    for i, (c, l, t) in frames.items():
        store[f"{model}/frame{i}/keep"] = keeps[i][0].numpy()
        store[f"{model}/frame{i}/labels"] = keeps[i][1].numpy().astype(np.int8)
        d, _ = field_values(field, i, c)
        print(f"{model} frame {i}: {len(l)} voxels, {int((d > oc.THRESHOLD).sum())} pass the filter")
    store[f"{model}/centroids"] = centroids.numpy()
    store[f"{model}/label_bank"] = label_bank.numpy()
    for k in ("micro_accuracy", "macro_accuracy", "cover_rate", "num_measured_points", "num_total_points"):
        store[f"{model}/{k}"] = np.array(result[k])
    store[f"{model}/per_class_accuracy"] = np.array([result["per_class_accuracy"][n]
                                                     for n in oc.LABEL_MAPPING.values()], np.float64)
    print(model, {k: v for k, v in result.items() if k != "per_class_accuracy"})
    print(model, "per class", [round(v, 4) for v in result["per_class_accuracy"].values()])


def main():
    torch.set_num_threads(1)                       # a fixed CPU reduction order
    ref = load_reference_metrics()
    store = {}
    for model in oc.MODELS:
        run_model(ref, model, store)
    path = os.path.join(HERE, "occupancy.npz")
    np.savez_compressed(path, **store)
    print(f"occupancy: {len(store)} arrays, {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    assert ref_shims.reference_available(), "set EMER_REFERENCE_ROOT to a checkout of NVlabs/EmerNeRF"
    main()
