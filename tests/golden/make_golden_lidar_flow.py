"""Generate tests/golden/lidar_flow.npz by running the REFERENCE's own lidar frames, split wrapper, flow query and
scene-flow metrics on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_lidar_flow.py

``SceneLidarSource`` and ``SplitWrapper`` are loaded by file path, as make_golden_raybatch.py loads the sources.  The
Waymo source cannot be imported (its module needs imageio and skimage for video output), so a subclass of the base
source adds the override's three gathers (flows, flow classes, ground flags).  ``RadianceField.query_flow`` is the
reference's own field with the stand-ins of ``oracle.ref_shims``, and ``compute_scene_flow_metrics`` comes from the
reference's ``datasets/metrics.py``.  The driver's loop around them is ``oracle.lidar_flow_ref.eval_lidar_flow``.

For each source of ``lidar_flow_cases.SOURCES`` the labels are the reference field's gated flows plus noise at several
scales, so every threshold has points on both sides; points within 1e-4 relative of a threshold (error norm against
0.05, 0.1 and 0.3, relative error against 0.05 and 0.1, label norm against 0.1, dynamic density against 0.2) are
dropped.  The file keeps, per source, which candidates each scan keeps, their labels and the rows the reference's
``get_render_rays`` returns for every time index; per case, the reference's result, and per frame its statistics and
the counts behind them.

An all-ground frame (case ``all_ground``) has no point left after the ground removal, and the reference's
``query_flow`` raises on zero points (it reshapes an empty tensor with a -1 dimension); the generator checks that it
raises, then answers that frame's query with an empty prediction, so the reference's ``compute_scene_flow_metrics``
gives what it gives for an empty frame: NaN for every statistic.
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden_occ as mgo  # noqa: E402  (installs oracle.ref_shims, imports the reference's field)
import make_golden_raybatch as mgr  # noqa: E402

import cases  # noqa: E402
import lidar_flow_cases as lc  # noqa: E402
from oracle import lidar_flow_ref, ref_shims  # noqa: E402

PACKAGE = "reference_datasets_base"


def load_base(name: str):
    """datasets/base/<name>.py of the reference as a submodule of a stand-in package, so its relative imports
    resolve to the modules loaded here."""
    full = f"{PACKAGE}.{name}"
    if full in sys.modules:
        return sys.modules[full]
    mgr.load_reference("datasets/base/lidar_source.py", "_stubs_only")     # installs the data-loading stand-ins
    pkg = mgr._stub(PACKAGE)
    pkg.__path__ = [os.path.join(ref_shims.REFERENCE_ROOT, "datasets", "base")]
    spec = importlib.util.spec_from_file_location(full, os.path.join(pkg.__path__[0], f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[full] = mod
    spec.loader.exec_module(mod)
    return mod


def waymo_source(ls):
    class WaymoLidar(ls.SceneLidarSource):
        """The base source with the Waymo override's three extra gathers (datasets/waymo.py:341-356)."""

        def get_render_rays(self, time_idx):
            out = super().get_render_rays(time_idx)
            out["lidar_flow"] = self.flows[self.timesteps == time_idx]
            out["lidar_flow_class"] = self.flow_classes[self.timesteps == time_idx]
            out["lidar_ground"] = self.grounds[self.timesteps == time_idx]
            return out

    return mgr.bare(WaymoLidar)


def far(x, thresholds):
    return torch.stack([(x - t).abs() > lc.MARGIN * t for t in thresholds]).all(0)


def compose_scan(field, source, scan):
    """(keep, labels of the kept points) of one scan, from the reference field's gated flows."""
    c = lc.candidates(source, scan)
    pts = c["origins"] + c["ranges"] * c["directions"]
    t = torch.full((lc.POINTS,), scan, dtype=torch.int64).float() / (cases.N_TIMESTEPS + 1e-6 - 1)
    with torch.no_grad():
        out = field.query_flow(positions=pts, normed_timestamps=t)
    pred, dd = out["forward_flow"], out["dynamic_density"]
    gated = torch.where((dd < lc.THRESHOLD)[:, None], pred * 0, pred)
    labels = c["noise"] if bool(c["static"]) else gated + c["noise"]
    l2 = (gated.double() - labels.double()).norm(dim=-1)
    ln = labels.double().norm(dim=-1)
    rel = l2 / (ln + 1e-20)
    keep = far(l2, (0.05, 0.1, 0.3)) & far(rel, (0.05, 0.1)) & far(ln, (0.1,)) & far(dd.double(), (lc.THRESHOLD,))
    return keep, labels[keep].contiguous()


class EmptyFrameQuery:
    """The field, except that a query of zero points returns empty flows and densities."""

    def __init__(self, field):
        self.field = field

    def query_flow(self, positions, normed_timestamps):
        if positions.shape[0] == 0:
            return {"forward_flow": positions.new_zeros(0, 3), "dynamic_density": positions.new_zeros(0)}
        return self.field.query_flow(positions=positions, normed_timestamps=normed_timestamps)


def main():
    assert ref_shims.reference_available(), "set EMER_REFERENCE_ROOT to a checkout of NVlabs/EmerNeRF"
    torch.set_num_threads(1)
    ls, sw = load_base("lidar_source"), load_base("split_wrapper")
    ref_metrics = mgo.load_reference_metrics()
    field = lc.fixture_field(mgo.REF, 0.0)
    c0 = lc.candidates("drive", 0)
    with torch.no_grad():
        dd = field.query_flow(positions=c0["origins"] + c0["ranges"] * c0["directions"],
                              normed_timestamps=torch.zeros(lc.POINTS))["dynamic_density"]
    shift = float(torch.log(dd.median() / lc.THRESHOLD))
    field = lc.fixture_field(mgo.REF, shift)
    store = {"density_shift": np.array(shift, np.float64),
             "parameters": np.array(sorted(k for k, _ in field.named_parameters()))}
    sources = {}
    for source in lc.SOURCES:
        keeps, labels = {}, {}
        for scan in range(lc.N_SCANS):
            keeps[scan], labels[scan] = compose_scan(field, source, scan)
            store[f"{source}/scan{scan}/keep"] = keeps[scan].numpy()
            store[f"{source}/scan{scan}/labels"] = labels[scan].numpy()
        src = lc.fill(waymo_source(ls), source, keeps, labels)
        sources[source] = src
        for t in list(range(lc.N_SCANS)) + [lc.ABSENT]:
            rows = torch.nonzero(src.timesteps == t).squeeze(1)
            got = src.get_render_rays(t)
            assert list(got) == list(lc.FRAME_KEYS)
            assert all(torch.equal(v, getattr(src, lc.ATTRS[k])[rows]) for k, v in got.items()), (source, t)
            base = ls.SceneLidarSource.get_render_rays(src, t)
            assert list(base) == list(lc.FRAME_KEYS[:4]) and all(torch.equal(v, got[k]) for k, v in base.items())
            store[f"{source}/rows{t}"] = rows.numpy().astype(np.int16)
        print(f"{source}: {len(src.timesteps)} points")
    for case, (source, remove_ground, split) in lc.CASES.items():
        angle_n = []

        def recorded(pred, labels):
            angle_n.append(int((torch.sqrt(torch.sum(labels * labels, 2)) > 0.1).sum()))
            return ref_metrics.compute_scene_flow_metrics(pred, labels)

        frames = []
        wrapper = sw.SplitWrapper(sources[source], split_indices=split, split="full")
        model = field
        if case == "all_ground":
            try:
                lidar_flow_ref.eval_lidar_flow(wrapper, field, remove_ground)
                raise AssertionError("the reference's query_flow accepted an empty frame")
            except RuntimeError as e:
                print(f"{case}: the reference's query_flow raises on the empty frame ({str(e)[:60]}...)")
            model, angle_n = EmptyFrameQuery(field), []
        result = lidar_flow_ref.eval_lidar_flow(wrapper, model, remove_ground, flow_metrics=recorded, frames=frames)
        assert list(result) == list(lidar_flow_ref.KEYS) and all(type(v) is np.float64 for v in result.values())
        store[f"{case}/result"] = np.array([result[k] for k in lidar_flow_ref.KEYS], np.float64)
        per = np.full((len(frames), len(lidar_flow_ref.KEYS)), np.nan)
        counts = np.zeros((len(frames), 6), np.int64)        # strict, relaxed, outlier, angle count, counted, valid
        it = iter(angle_n)
        for f, rec in enumerate(frames):
            counts[f, 4:] = rec["counted"], rec["valid"]
            if rec["metrics"] is None:
                continue
            per[f] = [rec["metrics"][k] for k in lidar_flow_ref.KEYS]
            n = rec["counted"]
            counts[f, :3] = [round(rec["metrics"][k] * n) if n else 0 for k in ("acc3d_strict", "acc3d_relax",
                                                                                 "outlier")]
            counts[f, 3] = next(it)
        store[f"{case}/frame_metrics"] = per
        store[f"{case}/frame_counts"] = counts
        print(case, {k: round(float(v), 6) for k, v in result.items()}, counts.tolist())
    path = os.path.join(HERE, "lidar_flow.npz")
    np.savez_compressed(path, **store)
    print(f"lidar_flow: {len(store)} arrays, {os.path.getsize(path) / 1e3:.1f} kB")


if __name__ == "__main__":
    main()
