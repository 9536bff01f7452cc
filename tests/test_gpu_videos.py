"""The evaluation videos on the H100 (csrc/video.cu through emernerf_b200.video):

* kernel: every frame of tests/golden/videos.npz rebuilt by ``emer_video_compose`` from the reference's own products
  (the raw blend inputs from videos_cases), byte for byte, depth pixels the golden marks as not firm excepted;
* end to end: ``render_videos`` with real static, dynamic and flow_feat fields against ``oracle.video_ref`` (the
  reference's ``render`` + ``save_videos`` with the package's ``render_rays`` on the same device): every written frame
  byte for byte under the same depth bin-edge rule, and the returned frames;
* no host sync in the per-image loop, the same sync count for 2 timesteps as for 6 and one writer wait per frame,
  bit-identical repeated calls, and a writer exception raised in the caller with no thread left behind.
"""
import os
import sys
import threading
import warnings

import numpy as np
import pytest
import torch

import videos_cases as vc

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "videos.npz")
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))


class Recorder:
    def __init__(self, fail_at=None):
        self.writers, self.images, self.fail_at = [], [], fail_at

    def get_writer(self, path, **kw):
        rec = {"path": path, "kw": kw, "frames": [], "closed": False}
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


@pytest.fixture
def video(monkeypatch, tmp_path):
    from emernerf_b200 import video

    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(video, "load_turbo_lut", vc.turbo_lut)
    monkeypatch.setattr(video, "_LUT", {})
    return video


def same_bytes(got, want, firm, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = (got != want).any(-1) & firm
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:5].tolist())


@pytest.mark.parametrize("case", list(vc.CASES))
def test_kernel_against_golden(video, case):
    z = np.load(GOLDEN)
    s = vc.spec(case)
    h, w = s["hw"]
    prods = {k.split("/", 2)[2]: z[k] for k in z.files if k.startswith(f"{case}/products/")}
    rows = video.plan_rows(s["keys"], list(prods), s["separate"])
    assert [r[0] for r in rows] == z[f"{case}/rows"].tolist()
    any_depth = any(k == video.DEPTH for _, k, _ in rows)
    f64 = [k == video.DEPTH if s["separate"] else any_depth for _, k, _ in rows]
    lut = torch.from_numpy(vc.turbo_lut()).to(DEV)
    frame = torch.empty(len(rows) * h, s["cams"] * w, 3, dtype=torch.uint8, device=DEV)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV)  # noqa: E731
    got = []
    for t in range(s["ts"]):
        for c in range(s["cams"]):
            p = t * s["cams"] + c
            raw = vc.results(case, p)
            tiles = []
            for r, (key, kind, okey) in enumerate(rows):
                if kind == video.DEPTH:
                    ins = (dev(prods[key][p]), dev(prods[okey][p]))
                elif kind == video.GRAY:
                    ins = (dev(prods[okey if key == "sky_masks" else key][p]),)
                elif key == "dynamic_rgb_on_static_dinos":
                    ins = (dev(raw["dynamic_rgb"]), dev(raw["dynamic_opacity"]), dev(prods["static_dino_feats"][p]))
                elif key == "dynamic_dino_on_static_rgbs":
                    ins = (dev(prods["dynamic_dino_feats"][p]), dev(raw["dynamic_opacity"]),
                           dev(prods["static_rgbs"][p]))
                else:
                    ins = (dev(prods[key][p]),)
                tiles.append((kind, ins, r, key == "sky_masks", f64[r]))
            video.compose(frame, tiles, h, w, c, lut)
        got.append(frame.cpu().numpy())
    got = np.stack(got)
    firm = z[f"{case}/firm"]
    if s["separate"]:
        for j in range(len(rows)):
            same_bytes(got[:, j * h:(j + 1) * h], z[f"{case}/w{j}"], firm[:, j * h:(j + 1) * h], f"{case} {j}")
    else:
        same_bytes(got, z[f"{case}/w0"], firm, case)


# ------------------------------------------------------------------------------------------------------ end to end
KEYS = {
    "static": ["gt_rgbs", "rgbs", "depths", "median_depths", "gt_sky_masks", "sky_masks"],
    "dynamic": vc.DYNAMIC_KEYS,
    "flow_feat": ["gt_rgbs", "rgbs", "dynamic_rgbs", "depths", "dynamic_depths", "forward_flows", "backward_flows",
                  "dino_feats", "gt_dino_feats", "dino_feats_pe_free", "dino_pe", "static_dino_feats",
                  "dynamic_dino_feats", "dynamic_rgb_on_static_dinos", "dynamic_dino_on_static_rgbs", "sky_masks"],
}


def scene(variant, timesteps, downscale=1 / 16):
    import bench_videos as bv

    return bv.scene(variant, timesteps, downscale)


def firm_frames(R, keys, cams, ts, h, w, separate=False):
    """The firm masks of the oracle's frames from its own products (concatenated layout)."""
    from emernerf_b200 import video

    produced = [k for k, v in R.items() if len(v) > 0]
    masks = []
    for key, kind, okey in video.plan_rows(keys, produced, separate):
        m = np.ones((ts, h, cams * w), bool)
        if kind == video.DEPTH:
            for t in range(ts):
                for c in range(cams):
                    p = t * cams + c
                    m[t, :, c * w:(c + 1) * w] = vc.firm_tile(R[key][p], R[okey][p])
        masks.append(m)
    return np.concatenate(masks, axis=1)


def run_new(video, parts, ts, keys, rec, **kw):
    cfg, field, props, est, ds, cams = parts
    torch.manual_seed(0)
    return video.render_videos(cfg, field, est, props, ds, "out.mp4", ts, keys, cams, **kw)


def run_oracle(parts, ts, keys, rec, separate=False):
    from emernerf_b200 import flow_vis, voxels
    from emernerf_b200.radiance_fields.render_utils import render_rays
    from oracle import video_ref

    cfg, field, props, est, ds, cams = parts
    torch.manual_seed(0)
    func = lambda d: render_rays(radiance_field=field, proposal_estimator=est,  # noqa: E731
                                 proposal_networks=props, data_dict=d, cfg=cfg, return_decomposition=True)
    R = video_ref.render(ds, func, field, voxels.robust_pca, list(range(len(ds))), flow_vis.scene_flow_to_rgb)
    out = video_ref.save_videos(R, "out.mp4", ts, keys, cams, separate, False, 10, False,
                                video_ref.Colormap(vc.turbo_table()), rec.get_writer, rec.imwrite)
    return R, out


@pytest.mark.parametrize("variant", ["static", "dynamic", "flow_feat"])
def test_end_to_end_against_oracle(video, monkeypatch, variant):
    parts = scene(variant, 2)
    ts, cams, keys = 2, parts[-1], KEYS[variant]
    new, ref = Recorder(), Recorder()
    monkeypatch.setattr(video, "_get_writer", new.get_writer)
    _, frames = run_new(video, parts, ts, keys, new, verbose=False)
    R, want = run_oracle(parts, ts, keys, ref)
    h, w = R["rgbs"][0].shape[:2]
    firm = firm_frames(R, keys, cams, ts, h, w)
    assert len(new.writers) == len(ref.writers) == 1
    assert new.writers[0]["kw"] == ref.writers[0]["kw"] == {"mode": "I", "fps": 10}
    same_bytes(np.stack(new.writers[0]["frames"]), np.stack(ref.writers[0]["frames"]), firm, variant)
    same_bytes(frames["concatenated_frame"], want["concatenated_frame"], firm[ts // 2], variant)
    assert (~firm).sum() <= 0.001 * firm.size


def test_separate_videos_against_oracle(video, monkeypatch):
    parts = scene("dynamic", 2)
    keys = ["rgbs", "depths", "dynamic_depths", "sky_masks", "gt_sky_masks"]
    new, ref = Recorder(), Recorder()
    monkeypatch.setattr(video, "_get_writer", new.get_writer)
    _, frames = run_new(video, parts, 2, keys, new, save_seperate_video=True, verbose=False)
    R, want = run_oracle(parts, 2, keys, ref, separate=True)
    h, w = R["rgbs"][0].shape[:2]
    firm = firm_frames(R, keys, parts[-1], 2, h, w, separate=True)
    assert [x["path"] for x in new.writers] == [x["path"] for x in ref.writers]
    for j, (a, b) in enumerate(zip(new.writers, ref.writers)):
        same_bytes(np.stack(a["frames"]), np.stack(b["frames"]), firm[:, j * h:(j + 1) * h], a["path"])
    assert list(frames) == list(want)


def syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(w.message) for w in caught)


def test_no_sync_in_the_image_loop(video, monkeypatch):
    """The dynamic field has no PCA fit: with metrics off a whole call runs without a host sync in the caller."""
    parts = scene("dynamic", 2)
    rec = Recorder()
    monkeypatch.setattr(video, "_get_writer", rec.get_writer)
    run_new(video, parts, 2, KEYS["dynamic"], rec, verbose=False)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        run_new(video, parts, 2, KEYS["dynamic"], rec, verbose=False)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(rec.writers[-1]["frames"]) == 2


def test_syncs_do_not_grow_with_timesteps(video, monkeypatch):
    rec = Recorder()
    monkeypatch.setattr(video, "_get_writer", rec.get_writer)
    waits = []
    real_wait = video._wait
    monkeypatch.setattr(video, "_wait", lambda ev: (waits.append(1), real_wait(ev)))
    counts = {}
    for ts in (2, 6):
        parts = scene("flow_feat", ts)
        run_new(video, parts, ts, KEYS["flow_feat"], rec, compute_metrics=True, verbose=False)
        del waits[:]
        counts[ts] = syncs(lambda: run_new(video, parts, ts, KEYS["flow_feat"], rec, compute_metrics=True,
                                           verbose=False))
        assert len(waits) == ts
    assert counts[2] == counts[6], counts


def test_repeated_calls_are_bit_identical(video, monkeypatch):
    parts = scene("flow_feat", 2)
    recs = [Recorder(), Recorder()]
    out = []
    for rec in recs:
        monkeypatch.setattr(video, "_get_writer", rec.get_writer)
        out.append(run_new(video, parts, 2, KEYS["flow_feat"], rec, compute_metrics=True, verbose=False))
    assert out[0][0] == out[1][0]
    assert np.array_equal(np.stack(recs[0].writers[0]["frames"]), np.stack(recs[1].writers[0]["frames"]))


def test_writer_exception_surfaces_without_a_thread_left(video, monkeypatch):
    parts = scene("static", 6)
    rec = Recorder(fail_at=2)
    monkeypatch.setattr(video, "_get_writer", rec.get_writer)
    with pytest.raises(OSError, match="disk full"):
        run_new(video, parts, 6, KEYS["static"], rec, verbose=False)
    assert rec.writers[0]["closed"] and len(rec.writers[0]["frames"]) == 2
    assert not any(t.name == "emernerf-video-writer" for t in threading.enumerate())
