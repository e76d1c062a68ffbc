"""TEST INFRASTRUCTURE - generates tests/golden/rect_cases.npz by running the UNMODIFIED reference's rect training loader:
`LoadImagesAndLabels(path, img_size, batch_size, augment=True, hyp=hyp, rect=True, cache_images=True, stride=32, pad=0.0)`
(utils/datasets.py:347-439, load_image's INTER_LINEAR cache resize :629-643, __getitem__ :518-592 without mosaic) and a torch DataLoader
with its `collate_fn` (no sampler, no shuffle), as train.py:196-198 builds them for `--rect` without DDP.

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_rect.py

The reference runs as it is, with the two adjustments of oracle/make_golden_val_batches.py (`np.int = int`, a fresh images/ + labels/
tree per case).  The sources are synthetic BGR images written as PNG with ten DISTINCT aspect ratios, so that the aspect-ratio sort has no
ties and the fixture does not depend on the CPU's argsort.  At batch size 3 the sorted dataset makes a landscape-only batch, a mixed
(square shape) batch, a portrait-only batch and a partial last batch of one portrait image.  The cache resize shrinks, grows, keeps and
halves them; at img_size 100 (not a multiple of the stride) the letterbox also up-scales.  The file holds the sources and their labels
and, per case, the seeds, the reference's order (as source indices), its batch_shapes, per batch the uint8 images and float32 targets,
and the next `random` / `numpy.random` draw after the last batch.
"""
import json
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402
from oracle.make_golden_val_batches import write_tree  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
# (h, w), aspect ratios 0.4 .. 2.5, all distinct; long sides around 96: shrink, keep, grow, exact 2x
SHAPES = [(40, 100), (48, 96), (120, 200), (45, 60), (176, 160), (39, 30), (192, 128), (126, 70), (96, 48), (150, 60)]
SCRATCH = dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0, flipud=0.0,
               fliplr=0.5, mosaic=1.0, mixup=0.0)
BATCH_SIZE = 3
CASES = {  # name -> (img_size, seed, hyp overrides)
    "scratch": (96, 1, {}),
    "stress": (128, 2, dict(degrees=10.0, shear=5.0, scale=0.5, translate=0.1)),
    "flipud": (100, 3, dict(flipud=1.0, degrees=3.0)),
    "identity": (96, 4, dict(translate=0.0, scale=0.0, degrees=0.0, shear=0.0)),
}


def sources(seed=0):
    """textured images in 8x8 blocks with a flat block (hue / saturation edge cases); labels (n, 5) as the label files' text reads"""
    rs = np.random.RandomState(seed)
    imgs, labels = [], []
    for k, (h, w) in enumerate(SHAPES):
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), ((xx + yy) * 7 + 40 * k) % 256], -1)
        texture = np.kron(rs.randint(-40, 41, (h // 8 + 1, w // 8 + 1, 3)), np.ones((8, 8, 1), np.int64))[:h, :w]
        img = np.clip(base + texture, 0, 255).astype(np.uint8)
        img[h // 4:h // 2, w // 3:w // 2] = rs.randint(0, 256, 3)
        n = rs.randint(1, 5)
        lb = np.zeros((n, 5), np.float32)
        lb[:, 0] = rs.randint(0, 10, n)
        lb[:, 3:5] = rs.uniform(0.1, 0.6, (n, 2))
        lb[:, 1:3] = rs.uniform(0.3, 0.7, (n, 2))
        lb[0, 1], lb[0, 3] = lb[0, 3] / 2, lb[0, 3]                               # touches the left border
        rows = [[str(int(r[0]))] + [f"{v:.6f}" for v in r[1:]] for r in lb]
        imgs.append(img)
        labels.append(np.array(rows, dtype=np.float32))
    return imgs, labels


def main():
    import torch
    np.int = int                                   # removed in numpy 1.24; the reference's batch index and batch_shapes use it
    ref_shims.import_reference()
    import utils.datasets as ref_datasets          # the reference's module (sys.path set by import_reference)
    ar = np.array([h / w for h, w in SHAPES], np.float64)
    assert len(np.unique(ar)) == len(ar), "aspect ratios must be distinct"
    imgs, labels = sources()
    out, meta = {}, {}
    for k, (im, lb) in enumerate(zip(imgs, labels)):
        out[f"src_{k}"] = im
        out[f"labels_{k}"] = lb
    for name, (s, seed, over) in CASES.items():
        hyp = dict(SCRATCH, **over)
        with tempfile.TemporaryDirectory() as tmp:
            write_tree(tmp, imgs, labels)
            ds = ref_datasets.LoadImagesAndLabels(os.path.join(tmp, "images"), s, BATCH_SIZE, augment=True, hyp=hyp, rect=True,
                                                  cache_images=True, stride=32, pad=0.0)
            assert not ds.mosaic
            out[f"{name}_order"] = np.array([int(os.path.basename(f)[2:4]) for f in ds.img_files], np.int64)
            out[f"{name}_batch_shapes"] = np.asarray(ds.batch_shapes, np.int64)
            dl = torch.utils.data.DataLoader(ds, batch_size=BATCH_SIZE, num_workers=0, shuffle=False,
                                             collate_fn=ref_datasets.LoadImagesAndLabels.collate_fn)
            random.seed(seed)
            np.random.seed(seed)
            nb = 0
            for b, (img, targets, _, _) in enumerate(dl):
                out[f"{name}_img_{b}"] = img.numpy()
                out[f"{name}_targets_{b}"] = targets.numpy()
                nb += 1
            meta[name] = dict(img_size=s, seed=seed, hyp=hyp, batch_size=BATCH_SIZE, n_batches=nb, next_random=random.random(),
                              next_np=float(np.random.random()))
    out["meta_json"] = np.frombuffer(json.dumps(dict(shapes=SHAPES, cases=meta)).encode(), dtype=np.uint8)
    path = os.path.join(GOLD, "rect_cases.npz")
    np.savez_compressed(path, **out)
    print("rect", {k: (v["n_batches"], out[f"{k}_batch_shapes"].tolist()) for k, v in meta.items()}, os.path.getsize(path) / 1e3, "KB")


if __name__ == "__main__":
    main()
