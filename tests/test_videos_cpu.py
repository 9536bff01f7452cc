"""The evaluation videos of emernerf_b200.video on the host (CPU suite): ``render_videos`` runs its kernel through
tests/video_emulator.py and is checked against the reference's own ``render_pixels`` + ``save_videos``
(tests/golden/videos.npz, make_golden_videos.py): the writers' paths, modes and fps, every frame byte for byte (depth
pixels the golden marks as not firm excepted), the returned frames and the separate mode's images.  Also the row
order and key skipping, the to8b dtype rule, the metrics, the writer thread's error path, and every ValueError.
"""
import logging
import os
import re
import threading

import numpy as np
import pytest
import torch

import video_emulator as emu
import videos_cases as vc

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "videos.npz")
ROOT = os.path.dirname(HERE)


class Recorder:
    """imageio stand-ins: writers that record path, mode, fps and frames, and imwrite calls."""

    def __init__(self, fail_at=None):
        self.writers, self.images, self.fail_at = [], [], fail_at

    def get_writer(self, path, **kw):
        rec = {"path": path, "mode": kw.get("mode"), "fps": kw.get("fps", -1), "frames": [], "closed": False}
        self.writers.append(rec)
        outer = self

        class W:
            def append_data(self, frame):
                if outer.fail_at is not None and len(rec["frames"]) == outer.fail_at:
                    raise OSError("disk full")
                rec["frames"].append(np.array(frame, copy=True))

            def close(self):
                rec["closed"] = True
        return W()

    def imwrite(self, path, image):
        self.images.append((path, np.array(image, copy=True)))


def golden_pca(z, case):
    fits = [torch.from_numpy(z[f"{case}/pca{k}"]) for k in range(2) if f"{case}/pca{k}" in z]
    return iter([(f[:-2], f[-2], f[-1]) for f in fits])


@pytest.fixture
def video(monkeypatch, tmp_path):
    emu.install(monkeypatch)
    monkeypatch.chdir(tmp_path)                          # the separate mode makes its image directories
    from emernerf_b200 import video
    from emernerf_b200.radiance_fields import render_utils

    monkeypatch.setattr(video, "load_turbo_lut", vc.turbo_lut)
    monkeypatch.setattr(render_utils, "render_rays", vc.fake_render_rays())
    return video


def run(video, monkeypatch, case, rec=None, **kw):
    z = np.load(GOLDEN)
    s = vc.spec(case)
    rec = rec or Recorder()
    fits = golden_pca(z, case)
    monkeypatch.setattr(video.voxels, "robust_pca", lambda features, m=2.5: next(fits))
    monkeypatch.setattr(video, "_get_writer", rec.get_writer)
    monkeypatch.setattr(video, "_imwrite", rec.imwrite)
    args = dict(save_seperate_video=s["separate"], save_images=s["save_images"], fps=10, verbose=False)
    args.update(kw)
    out = video.render_videos(vc.cfg, vc.model(case), None, None, vc.Dataset(case), vc.save_path(case), s["ts"],
                              s["keys"], s["cams"], **args)
    return z, rec, out


def same_bytes(got, want, firm, what):
    assert got.dtype == np.uint8 and got.shape == want.shape, (what, got.shape, want.shape)
    bad = (got != want).any(-1) & firm
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:5].tolist())


def check_case(z, case, rec, out):
    s = vc.spec(case)
    p = f"{case}/"
    results, frames = out
    assert results == {k: -1 for k in ("psnr", "ssim", "feat_psnr", "masked_psnr", "masked_ssim",
                                       "masked_feat_psnr")}
    want = [w.split("|") for w in z[p + "writers"]]
    assert [(w["path"], w["mode"], str(w["fps"])) for w in rec.writers] == [tuple(w) for w in want]
    assert all(w["closed"] for w in rec.writers)
    firm = z[p + "firm"]                                 # [ts, rows * H, cams * W]
    h = s["hw"][0]
    for j, w in enumerate(rec.writers):
        got = np.stack(w["frames"])
        rows = slice(j * h, (j + 1) * h) if s["separate"] else slice(None)
        same_bytes(got, z[p + f"w{j}"], firm[:, rows], f"{case} writer {j}")
    assert list(frames) == z[p + "returned_keys"].tolist()
    for j, (k, v) in enumerate(frames.items()):
        rows = slice(j * h, (j + 1) * h) if s["separate"] else slice(None)
        same_bytes(v, z[p + f"returned/{k}"], firm[s["ts"] // 2, rows], f"{case} returned {k}")
    # the reference writes a key's images for every timestep before the next key's; here they come per timestep
    paths = z[p + "image_paths"].tolist()
    assert sorted(x[0] for x in rec.images) == sorted(paths)
    for path, img in rec.images:
        n = paths.index(path)
        same_bytes(img, z[p + "images"][n], np.ones(img.shape[:2], bool), path)
    if rec.images:
        assert all(os.path.isdir(path.replace(".mp4", "")) for path in z[p + "opened"] if path in
                   [w["path"] for w in rec.writers])


@pytest.mark.parametrize("case", list(vc.CASES))
def test_against_reference_golden(video, monkeypatch, case):
    z, rec, out = run(video, monkeypatch, case)
    check_case(z, case, rec, out)


@pytest.mark.parametrize("case", list(vc.CASES))
def test_produced_keys_are_the_references(case):
    from emernerf_b200 import video

    z = np.load(GOLDEN)
    want = sorted(k.split("/", 2)[2] for k in z.files if k.startswith(f"{case}/products/"))
    got = video.produced_keys(vc.results(case, 0), vc.data(case, 0))
    assert sorted(set(got)) == want


def test_row_order_and_skipping():
    from emernerf_b200 import video

    produced = ["rgbs", "depths", "opacities", "gt_rgbs", "median_depths", "static_depths", "static_opacities"]
    keys = ["sky_masks", "missing", "rgbs", "median_depths", "static_depths", "dynamic_depths", "gt_sky_masks",
            "foo_depths", "rgbs"]
    rows = video.plan_rows(keys, produced + ["foo_depths"])
    assert rows == [("sky_masks", video.GRAY, "opacities"), ("rgbs", video.RGB, None),
                    ("median_depths", video.DEPTH, "opacities"), ("static_depths", video.DEPTH, "static_opacities"),
                    ("rgbs", video.RGB, None)]
    # an empty list is absent; dynamic_depths keeps its own opacities; separate mode has no sky_masks row
    rows = video.plan_rows(["dynamic_depths", "dynamic_rgbs", "sky_masks", "dynamic_rgb_on_static_dinos"],
                           ["dynamic_depths", "dynamic_opacities", "dynamic_rgb_on_static_dinos"], separate=True)
    assert rows == [("dynamic_depths", video.DEPTH, "dynamic_opacities"),
                    ("dynamic_rgb_on_static_dinos", video.BLEND, None)]


def _tiles(video, values, f64):
    t = torch.from_numpy(np.repeat(values[:, None], 3, axis=1).reshape(1, -1, 3).copy())
    frame = torch.zeros(1, t.shape[1], 3, dtype=torch.uint8)
    video.compose(frame, [(video.RGB, (t,), 0, False, f64)], 1, t.shape[1], 0, None)
    return frame.numpy()[0, :, 0]


def test_to8b_dtype_rule(video):
    """A float64 frame's tiles get 255 * x in float64, a float32 frame's in float32, each truncated as numpy does.  For
    float32 x in [0, 1] the two truncations agree (checked over every such float32; near_steps holds the values next
    to each k / 255, where they would part), so the rule changes no byte of an in-range value."""
    x = vc.near_steps()
    f32, f64 = _tiles(video, x, False), _tiles(video, x, True)
    assert np.array_equal(f32, (np.float32(255) * x).astype(np.uint8))
    assert np.array_equal(f64, (255 * x.astype(np.float64)).astype(np.uint8))
    assert np.array_equal(f32, f64)
    edge = np.array([np.nan, -0.0, -1e-7, 1.0, 1.0000001, np.inf, -np.inf, 0.5], np.float32)
    assert _tiles(video, edge, False).tolist() == [0, 0, 0, 255, 255, 255, 0, 127]
    assert _tiles(video, edge, True).tolist() == [0, 0, 0, 255, 255, 255, 0, 127]


def test_depth_curve_constants_are_numpys():
    src = open(os.path.join(ROOT, "emernerf_b200", "csrc", "video.cuh")).read()
    lo = float.fromhex(re.search(r"VIDEO_DEPTH_CURVE_LO = (\S+);", src).group(1))
    hi = float.fromhex(re.search(r"VIDEO_DEPTH_CURVE_HI = (\S+);", src).group(1))
    assert lo == -np.log(4.0 + 1e-6) and hi == -np.log(120 + 1e-6)


def test_depth_index_edges():
    nan, inf = float("nan"), float("inf")
    d = np.array([4.0, 120.0, 0.0, -1e-6, -1.0, nan, inf, 10.0, 10.0, 10.0, 10.0, 10.0], np.float32)
    op = np.array([1, 1, 1, 1, 1, 1, 1, 0, nan, inf, -0.5, 1.0000001], np.float32)
    i = emu.depth_index(d, op)
    assert i[[0, 2, 3]].tolist() == [255, 255, 255]          # at lo, 0 and -1e-6 (log 0): clipped to 1
    assert i[[1, 4, 5, 6, 7, 10]].tolist() == [0, 0, 0, 0, 0, 0]   # hi, NaN curves, inf, opacity 0 and negative
    assert i[8] == -1                                        # NaN opacity: "bad", black
    assert i[9] == 255                                       # inf opacity: over


def test_writer_exception_surfaces_and_no_thread_is_left(video, monkeypatch):
    before = {t.ident for t in threading.enumerate()}
    with pytest.raises(OSError, match="disk full"):
        run(video, monkeypatch, "one_cam", rec=Recorder(fail_at=1))
    assert {t.ident for t in threading.enumerate() if t.name == "emernerf-video-writer"} - before == set()
    assert not any(t.name == "emernerf-video-writer" for t in threading.enumerate())


def test_render_error_closes_writers(video, monkeypatch):
    from emernerf_b200.radiance_fields import render_utils

    base = vc.fake_render_rays()
    calls = []

    def failing(**kw):
        calls.append(1)
        if len(calls) == 4:
            raise RuntimeError("field failed")
        return base(**kw)

    monkeypatch.setattr(render_utils, "render_rays", failing)
    rec = Recorder()
    with pytest.raises(RuntimeError, match="field failed"):
        run(video, monkeypatch, "dynamic", rec=rec)
    assert rec.writers and all(w["closed"] for w in rec.writers)
    assert len(rec.writers[0]["frames"]) == 1                 # the first timestep was written
    assert not any(t.name == "emernerf-video-writer" for t in threading.enumerate())


def test_one_wait_per_frame(video, monkeypatch):
    del emu.WAITS[:]
    run(video, monkeypatch, "separate")
    assert len(emu.WAITS) == vc.spec("separate")["ts"]


def test_metrics_and_logs(video, monkeypatch, caplog):
    from emernerf_b200 import metrics

    with caplog.at_level(logging.INFO):
        z, rec, (results, _) = run(video, monkeypatch, "feature", compute_metrics=True, verbose=True)
    per = []
    for i in range(vc.n_images("feature")):
        r, d = vc.results("feature", i), vc.data("feature", i)
        per.append(metrics.image_metrics(r["rgb"], d["pixels"], None, r["dino_feat"], d["features"]))
    want = metrics.summarize(per)
    assert results == {k: want[k] for k in results}
    assert results["masked_psnr"] == -1 and results["psnr"] > 0 and results["feat_psnr"] > 0
    assert "Eval over 4 images:" in caplog.text and "\tFeature PSNR:" in caplog.text
    assert f"saved video to {vc.save_path('feature')}" in caplog.text


def test_argument_errors(video, monkeypatch):
    with pytest.raises(ValueError, match="images for"):
        run(video, monkeypatch, "dynamic", vis_indices=[0, 1, 2])
    s = vc.spec("dynamic")
    with pytest.raises(ValueError, match="five cameras"):
        video.render_videos(vc.cfg, vc.model("dynamic"), None, None, vc.Dataset("dynamic"), "x.mp4", 1, s["keys"], 5)
    with pytest.raises(ValueError, match="has a product"):
        run(video, monkeypatch, "dynamic", keys=["nothing"]) if False else video.render_videos(
            vc.cfg, vc.model("dynamic"), None, None, vc.Dataset("dynamic"), "x.mp4", 2, ["nothing"], 2)


def test_compose_validation(video):
    h, w = 4, 5
    frame = torch.zeros(2 * h, 2 * w, 3, dtype=torch.uint8)
    good = torch.rand(h, w, 3)
    one = torch.rand(h, w, 1)
    lut = torch.from_numpy(vc.turbo_lut())
    video.compose(frame, [(video.RGB, (good,), 1, False, False), (video.DEPTH, (one, one), 0, False, True)], h, w, 1,
                  lut)
    cases = [
        ([(video.RGB, (good.double(),), 0, False, False)], "float32"),
        ([(video.RGB, (torch.rand(w, h, 3).transpose(0, 1),), 0, False, False)], "contiguous"),
        ([(video.RGB, (torch.rand(h, w + 1, 3),), 0, False, False)], "shape"),
        ([(video.RGB, (one,), 0, False, False)], "shape"),
        ([(video.BLEND, (good, one), 0, False, False)], "inputs"),
        ([(video.RGB, (good,), 2, False, False)], "row"),
        ([(7, (good,), 0, False, False)], "kind"),
        ([(video.RGB, (good,), 0, False, False)] * 33, "tiles"),
        ([(video.DEPTH, (one, one), 0, False, True)], "turbo"),
        ([], "tiles"),
    ]
    for tiles, msg in cases:
        with pytest.raises(ValueError, match=msg):
            video.compose(frame, tiles, h, w, 0, None)
    with pytest.raises(ValueError, match="column"):
        video.compose(frame, [(video.RGB, (good,), 0, False, False)], h, w, 2, None)
    with pytest.raises(ValueError, match="rows"):
        video.compose(torch.zeros(2 * h + 1, 2 * w, 3, dtype=torch.uint8), [(video.RGB, (good,), 0, False, False)],
                      h, w, 0, None)
    with pytest.raises(ValueError, match="uint8"):
        video.compose(frame.float(), [(video.RGB, (good,), 0, False, False)], h, w, 0, None)


def test_cpu_tensors_are_refused():
    from emernerf_b200 import video

    frame = torch.zeros(4, 5, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA"):
        video.compose(frame, [(video.RGB, (torch.rand(4, 5, 3),), 0, False, False)], 4, 5, 0, None)


def test_turbo_loader_reads_matplotlib(monkeypatch):
    """load_turbo_lut reads matplotlib's map, falling back to cm.get_cmap; no colour data is kept in the package."""
    import sys
    import types

    from emernerf_b200 import video
    from oracle.video_ref import Colormap

    cmap = Colormap(vc.turbo_table())
    mpl = types.ModuleType("matplotlib")
    mpl.colormaps = {"turbo": cmap}
    monkeypatch.setitem(sys.modules, "matplotlib", mpl)
    assert np.array_equal(video.load_turbo_lut(), vc.turbo_lut())
    old = types.ModuleType("matplotlib")
    old.cm = types.SimpleNamespace(get_cmap=lambda name: cmap)
    monkeypatch.setitem(sys.modules, "matplotlib", old)
    monkeypatch.setitem(sys.modules, "matplotlib.cm", old.cm)
    assert np.array_equal(video.load_turbo_lut(), vc.turbo_lut())


@pytest.mark.parametrize("case", list(vc.CASES))
def test_oracle_is_the_references(monkeypatch, tmp_path, case):
    """oracle.video_ref (the H100 tests' and the benchmark's baseline) writes the reference's frames."""
    from emernerf_b200.flow_vis import scene_flow_to_rgb
    from oracle import video_ref

    emu.install(monkeypatch)
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **kw: self)
    z = np.load(GOLDEN)
    s = vc.spec(case)
    fits = golden_pca(z, case)
    rec = Recorder()
    out = video_ref.render_videos(
        vc.cfg, vc.model(case), None, None, vc.Dataset(case), vc.save_path(case), s["ts"], s["keys"], s["cams"],
        s["separate"], s["save_images"], 10, False, render_rays=vc.fake_render_rays(),
        robust_pca=lambda features, m=2.5: next(fits), scene_flow_to_rgb=scene_flow_to_rgb,
        cmap=video_ref.Colormap(vc.turbo_table()), get_writer=rec.get_writer, imwrite=rec.imwrite)
    check_case(z, case, rec, ({k: -1 for k in ("psnr", "ssim", "feat_psnr", "masked_psnr", "masked_ssim",
                                               "masked_feat_psnr")}, out))
