"""TEST INFRASTRUCTURE - generates tests/golden/quad_cases.npz by running the UNMODIFIED reference's `--quad` training loader:
`LoadImagesAndLabels(path, img_size, batch_size, augment=True, hyp=hyp, rect=rect, cache_images=True, stride=32, pad=0.0)` and a torch
DataLoader with `LoadImagesAndLabels.collate_fn4` (num_workers=0, no sampler, no shuffle), as train.py:196-199 builds them for `--quad`
without DDP.

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_quad.py

The reference runs as it is, with the adjustments of oracle/make_golden_rect.py (`np.int = int`, a fresh images/ + labels/ tree per case).
The collate function handed to the DataLoader records the batch it is given, and the `random` state, before calling collate_fn4 itself.
Fourteen synthetic PNGs at batch size 8 give, per case, a full batch of 8 (two quads) and a partial batch of 6 (one quad; two items
dropped).  The sources have distinct aspect ratios, all <= 0.5 for the first eight and >= 2 for the last six, so the rect case has a
32x64 and a 64x32 batch and its order does not depend on the CPU's argsort.  Per case and batch the file holds the items before collation
(uint8 images and float32 targets, column 0 the item index, as collate_fn gives them), the `random` state collate_fn4 starts from, the
collated images and targets, and the next `random` / `numpy.random` draw after the batch.  The seeds are chosen so that every case has
both branches; the generator asserts it.
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
S = 64
BATCH_SIZE = 8
# (h, w): aspect ratios <= 0.5, then >= 2, all distinct
SHAPES = [(20, 64), (24, 64), (25, 60), (28, 64), (30, 64), (32, 64), (27, 60), (26, 56),
          (64, 32), (66, 30), (70, 28), (72, 24), (64, 26), (60, 25)]
SCRATCH = dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0, flipud=0.0,
               fliplr=0.5, mosaic=1.0, mixup=0.0)
CASES = {  # name -> (rect, seed, hyp overrides)
    "mosaic": (False, 3, dict(degrees=5.0)),
    "mixup": (False, 4, dict(mixup=1.0)),
    "rect": (True, 2, dict(flipud=0.5)),
}


def sources(seed=0):
    """textured images in 8x8 blocks; labels (n, 5) as the label files' text reads them"""
    rs = np.random.RandomState(seed)
    imgs, labels = [], []
    for k, (h, w) in enumerate(SHAPES):
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), ((xx + yy) * 7 + 40 * k) % 256], -1)
        texture = np.kron(rs.randint(-40, 41, (h // 8 + 1, w // 8 + 1, 3)), np.ones((8, 8, 1), np.int64))[:h, :w]
        imgs.append(np.clip(base + texture, 0, 255).astype(np.uint8))
        n = rs.randint(1, 4)
        lb = np.zeros((n, 5), np.float32)
        lb[:, 0] = rs.randint(0, 10, n)
        lb[:, 3:5] = rs.uniform(0.2, 0.6, (n, 2))
        lb[:, 1:3] = rs.uniform(0.3, 0.7, (n, 2))
        rows = [[str(int(r[0]))] + [f"{v:.6f}" for v in r[1:]] for r in lb]
        labels.append(np.array(rows, dtype=np.float32))
    return imgs, labels


def peek():
    """the next random.random() and np.random.random() without consuming them"""
    st, nst = random.getstate(), np.random.get_state()
    r, q = random.random(), float(np.random.random())
    random.setstate(st)
    np.random.set_state(nst)
    return r, q


def main():
    import torch
    np.int = int                                   # removed in numpy 1.24; the reference's rect batch index and batch_shapes use it
    ref_shims.import_reference()
    import utils.datasets as ref_datasets          # the reference's module (sys.path set by import_reference)
    ar = np.array([h / w for h, w in SHAPES])
    assert len(np.unique(ar)) == len(ar) and (ar[:8] <= 0.5).all() and (ar[8:] >= 2).all()
    imgs, labels = sources()
    out, meta = {}, {}
    for k, (im, lb) in enumerate(zip(imgs, labels)):
        out[f"src_{k}"] = im
        out[f"labels_{k}"] = lb
    for name, (rect, seed, over) in CASES.items():
        hyp = dict(SCRATCH, **over)
        records = []

        def collate(batch, records=records):
            items = torch.stack([b[0] for b in batch], 0).numpy().copy()
            targets = [b[1].clone() for b in batch]             # collate_fn4 writes column 0 of some of them in place
            for i, t in enumerate(targets):
                t[:, 0] = i
            state = random.getstate()
            n = len(batch) // 4
            tile = [random.random() >= 0.5 for _ in range(n)]  # the draws collate_fn4 is about to make
            random.setstate(state)
            res = ref_datasets.LoadImagesAndLabels.collate_fn4(batch)
            records.append(dict(items=items, targets=torch.cat(targets, 0).numpy(), state=np.array(state[1], np.int64), tile=tile,
                                next=peek()))
            return res

        with tempfile.TemporaryDirectory() as tmp:
            write_tree(tmp, imgs, labels)
            ds = ref_datasets.LoadImagesAndLabels(os.path.join(tmp, "images"), S, BATCH_SIZE, augment=True, hyp=hyp, rect=rect,
                                                  cache_images=True, stride=32, pad=0.0)
            assert ds.mosaic == (not rect)
            if rect:
                out[f"{name}_order"] = np.array([int(os.path.basename(f)[2:4]) for f in ds.img_files], np.int64)
                out[f"{name}_batch_shapes"] = np.asarray(ds.batch_shapes, np.int64)
            dl = torch.utils.data.DataLoader(ds, batch_size=BATCH_SIZE, num_workers=0, shuffle=False, collate_fn=collate)
            random.seed(seed)
            np.random.seed(seed)
            sizes = []
            for b, (img4, targets4, paths4, _) in enumerate(dl):
                r = records[b]
                assert len(paths4) == len(r["items"]) // 4 == len(img4)
                out[f"{name}_items_{b}"] = r["items"]
                out[f"{name}_targets_{b}"] = r["targets"]
                out[f"{name}_state_{b}"] = r["state"]
                out[f"{name}_img4_{b}"] = img4.numpy()
                out[f"{name}_targets4_{b}"] = targets4.numpy()
                sizes.append(len(r["items"]))
        tiles = [r["tile"] for r in records]
        assert sizes == [8, 6], sizes
        flat = [t for ts in tiles for t in ts]
        assert any(flat) and not all(flat), (name, tiles)        # both branches in every case
        meta[name] = dict(img_size=S, seed=seed, hyp=hyp, rect=rect, batch_size=BATCH_SIZE, n_batches=len(records), tiles=tiles,
                          next_random=[r["next"][0] for r in records], next_np=[r["next"][1] for r in records])
    out["meta_json"] = np.frombuffer(json.dumps(dict(shapes=SHAPES, cases=meta)).encode(), dtype=np.uint8)
    path = os.path.join(GOLD, "quad_cases.npz")
    np.savez_compressed(path, **out)
    print("quad", {k: v["tiles"] for k, v in meta.items()}, os.path.getsize(path) / 1e3, "KB")


if __name__ == "__main__":
    main()
