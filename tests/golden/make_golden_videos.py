"""Generate tests/golden/videos.npz by running the REFERENCE's own ``render_pixels`` and ``save_videos``
(radiance_fields/video_utils.py) on CPU.

Needs a checkout of the reference (NVlabs/EmerNeRF@8c051d7):

    EMER_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_videos.py

``video_utils.py`` is loaded unmodified, with the shims the voxel and flow-figure generators use
(``make_golden_voxels.load_visualization_tools``) and three stand-ins: an ``imageio`` whose writers record their
path, mode, fps and frames (and an ``imwrite`` that records its images); a ``matplotlib.cm`` whose turbo map is
``videos_cases.turbo_table()`` behind ``oracle.video_ref.Colormap``, a restatement of matplotlib 3.6.1's
``Colormap.__call__``; and a ``render_rays`` that returns ``videos_cases``' seeded products.  ``get_robust_pca`` is
the reference's, recorded, so the tests can inject its outputs.

Per case the file holds the writers' calls and frames, the returned frames, the separate mode's images, the PCA fits,
the lists ``render`` returned (the kernel's inputs), and the firm mask of every frame: False on a depth pixel whose
v * 256 lies within ``videos_cases.MARGIN`` of an integer from 1 to 255.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden_voxels as mgv  # noqa: E402  (installs oracle.ref_shims)
import videos_cases as vc  # noqa: E402
from oracle import ref_shims  # noqa: E402
from oracle.video_ref import Colormap  # noqa: E402


class Writer:
    def __init__(self, log, path, **kw):
        self.rec = {"path": path, "mode": kw.get("mode"), "fps": kw.get("fps", -1), "frames": [], "closed": False}
        log.append(self.rec)

    def append_data(self, frame):
        self.rec["frames"].append(np.array(frame, copy=True))

    def close(self):
        self.rec["closed"] = True


def load_video_utils(log, images):
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    vt = mgv.load_visualization_tools()
    cmap = Colormap(vc.turbo_table())
    vt.cm = types.SimpleNamespace(get_cmap=lambda name: cmap)
    vt.turbo_cmap = cmap
    sys.modules["utils.visualization_tools"] = vt
    mod("imageio", get_writer=lambda path, **kw: Writer(log, path, **kw),
        imwrite=lambda path, im: images.append((path, np.array(im, copy=True))))
    sk = mod("skimage")
    sk.__path__ = []
    mod("skimage.metrics", structural_similarity=None)
    mod("datasets.base", SplitWrapper=object)
    mod("datasets.metrics", compute_psnr=None)
    spec = importlib.util.spec_from_file_location(
        "reference_video_utils", os.path.join(ref_shims.REFERENCE_ROOT, "radiance_fields", "video_utils.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def rows_of(R, keys, separate):
    """The reference's rows: (key, opacity key or None)."""
    out = []
    for key in keys:
        if key == "sky_masks" and not separate:
            out.append((key, None))
            continue
        if key not in R or len(R[key]) == 0:
            continue
        okey = None
        if "depth" in key:
            okey = key.replace("depths", "opacities")
            if okey not in R:
                if "median" not in key:
                    continue
                okey = "opacities"
        out.append((key, okey))
    return out


def firm_masks(R, s, separate):
    """Per row: [ts, H, cams * W] firm masks."""
    h, w = s["hw"]
    out = []
    for key, okey in rows_of(R, s["keys"], separate):
        m = np.ones((s["ts"], h, s["cams"] * w), bool)
        if okey is not None:
            for i in range(s["ts"]):
                for c in range(s["cams"]):
                    p = i * s["cams"] + c
                    m[i, :, c * w:(c + 1) * w] = vc.firm_tile(R[key][p], R[okey][p])
        out.append((key, m))
    return out


def main():
    assert ref_shims.reference_available(), "set EMER_REFERENCE_ROOT to a checkout of NVlabs/EmerNeRF"
    torch.set_num_threads(1)
    torch.Tensor.cuda = lambda self, *a, **kw: self              # the reference moves each item to the device
    log, images = [], []
    vu = load_video_utils(log, images)
    os.chdir(tempfile.mkdtemp(prefix="make_golden_videos_"))   # the separate mode makes its image directories
    vu.render_rays = vc.fake_render_rays()
    store = {"turbo_table": vc.turbo_table(), "near_steps": vc.near_steps()}
    for case in vc.CASES:
        s = vc.spec(case)
        del log[:], images[:]
        fits = []
        reference_pca = vu.get_robust_pca

        def pca(features, m=2):
            out = reference_pca(features, m=m)
            fits.append(torch.cat([out[0], out[1][None], out[2][None]]).numpy())
            return out

        vu.get_robust_pca = pca
        torch.manual_seed(0)
        R = vu.render_pixels(vc.cfg, vc.model(case), None, vc.Dataset(case), proposal_networks=None,
                             compute_metrics=False, return_decomposition=True)
        vu.get_robust_pca = reference_pca
        got = vu.save_videos(R, vc.save_path(case), s["ts"], keys=s["keys"], num_cams=s["cams"],
                             save_seperate_video=s["separate"], save_images=s["save_images"], fps=10, verbose=False)
        p = f"{case}/"
        writers = [w for w in log if w["frames"]]     # the separate mode's writers of absent keys stay empty
        store[p + "writers"] = np.array([f"{w['path']}|{w['mode']}|{w['fps']}" for w in writers])
        store[p + "opened"] = np.array([w["path"] for w in log])
        for j, w in enumerate(writers):
            store[p + f"w{j}"] = np.stack(w["frames"])
        store[p + "returned_keys"] = np.array(list(got))
        for k, v in got.items():
            store[p + f"returned/{k}"] = v
        store[p + "image_paths"] = np.array([x[0] for x in images])
        if images:
            store[p + "images"] = np.stack([x[1] for x in images])
        for k, f in enumerate(fits):
            store[p + f"pca{k}"] = f
        for k, v in R.items():
            if isinstance(v, list) and len(v) > 0:
                store[p + f"products/{k}"] = np.stack(v)
        masks = firm_masks(R, s, s["separate"])
        store[p + "rows"] = np.array([k for k, _ in masks])
        store[p + "firm"] = np.concatenate([m for _, m in masks], axis=1)
        loose = sum(int((~m).sum()) for _, m in masks)
        print(f"{case}: {len(writers)} writers, frames {[store[p + f'w{j}'].shape for j in range(len(writers))]}, "
              f"{len(images)} images, {len(fits)} PCA fits, {loose} depth pixels not firm")
    path = os.path.join(HERE, "videos.npz")
    np.savez_compressed(path, **store)
    print(f"wrote {path}: {len(store)} arrays, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
