"""TEST INFRASTRUCTURE - generates tests/golden/val_batch_cases.npz by running the UNMODIFIED reference's rect validation loader:
`LoadImagesAndLabels(path, img_size, batch_size, augment=False, rect=True, cache_images=True, stride=32, pad=0.5)` (utils/datasets.py
:347-452, load_image's INTER_AREA cache resize :629-643, __getitem__ :518-592) and a torch DataLoader with its `collate_fn`, as
create_dataloader builds them for test().

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_val_batches.py

Two things are needed to run the reference with current libraries, neither touching its arithmetic:
  * `np.int = int`: LoadImagesAndLabels.__init__ uses `np.int`, which numpy 1.24 removed; it was an exact alias of the builtin;
  * every case builds its dataset in a fresh temporary images/ + labels/ tree, so that the reference writes its labels .cache file
    instead of loading one (torch.load's weights_only default would refuse it).

The sources are small synthetic BGR images written as PNG: landscape, portrait and square, sized so that at img_size 96 they take
every path of load_image (general INTER_AREA, integral 3x and 4x, exact 2x, no resize, INTER_LINEAR up-scaling), with a group of four
equal aspect ratios (numpy's argsort permutes ties in a CPU-dependent order; the group always falls within one batch).  Some images
have no label file and some an empty one.  The file holds the sources and their labels and, per case, the reference's img_files order
(as source indices), its cached images (by source index), its batch_shapes and per batch the images, targets, shapes and paths.
"""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
# (h, w); at img_size 96: the tie group of aspect ratio 0.5 (no resize, exact 2x, general area, up-scaling), then a general landscape,
# 4x, general, near-1 general, a square kept as is, general portrait, up-scaled portrait, 3x portrait and a tall general portrait
SHAPES = [(48, 96), (96, 192), (100, 200), (30, 60), (70, 112), (256, 384), (150, 200), (97, 99), (96, 96), (160, 120), (50, 35),
          (288, 192), (200, 90)]
CASES = {  # name -> (img_size, batch_size, single_cls)
    "main": (96, 4, False),
    "single_cls": (64, 5, True),
    "big_batch": (128, 32, False),
}


def sources(seed=0):
    """images of flat 13x13 blocks of random colours (aligned with no resize grid, so that every area weight shows at the block edges, and
    compressible) and a noise patch; labels (n, 5), None for a missing label file"""
    rs = np.random.RandomState(seed)
    imgs, labels = [], []
    for k, (h, w) in enumerate(SHAPES):
        img = np.kron(rs.randint(0, 256, (h // 13 + 1, w // 13 + 1, 3)), np.ones((13, 13, 1), np.int64))[:h, :w].astype(np.uint8)
        ph, pw = min(h, 12), min(w, 12)
        img[h // 3:h // 3 + ph, w // 3:w // 3 + pw] = rs.randint(0, 256, (ph, pw, 3))
        if k % 4 == 1:
            lb = None                                                     # no label file
        elif k % 4 == 3:
            lb = np.zeros((0, 5), np.float32)                             # an empty label file
        else:
            n = rs.randint(1, 5)
            lb = np.zeros((n, 5), np.float32)
            lb[:, 0] = rs.randint(0, 10, n)
            lb[:, 3:5] = rs.uniform(0.05, 0.5, (n, 2))
            lb[:, 1:3] = rs.uniform(0.25, 0.75, (n, 2))
            lb[0, 1], lb[0, 3] = lb[0, 3] / 2, lb[0, 3]                   # touches the left border
            rows = [[str(int(r[0]))] + [f"{v:.6f}" for v in r[1:]] for r in lb]
            lb = np.array(rows, dtype=np.float32)                         # the label file's text, read as cache_labels reads it
        imgs.append(img)
        labels.append(lb)
    return imgs, labels


def write_tree(root, imgs, labels):
    import cv2
    os.makedirs(os.path.join(root, "images"))
    os.makedirs(os.path.join(root, "labels"))
    for k, (im, lb) in enumerate(zip(imgs, labels)):
        cv2.imwrite(os.path.join(root, "images", f"im{k:02d}.png"), im)
        if lb is not None:
            with open(os.path.join(root, "labels", f"im{k:02d}.txt"), "w") as f:
                f.writelines(" ".join([str(int(r[0]))] + [f"{float(v):.6f}" for v in r[1:]]) + "\n" for r in lb)


def main():
    import torch
    np.int = int                                   # removed in numpy 1.24; the reference's batch index and batch_shapes use it
    ref_shims.import_reference()
    import utils.datasets as ref_datasets          # the reference's module (sys.path set by import_reference)
    imgs, labels = sources()
    out, meta = {}, {}
    for k, (im, lb) in enumerate(zip(imgs, labels)):
        out[f"src_{k}"] = im
        out[f"labels_{k}"] = lb if lb is not None else np.zeros((0, 5), np.float32)
    for name, (s, bs, single_cls) in CASES.items():
        with tempfile.TemporaryDirectory() as tmp:
            write_tree(tmp, imgs, labels)
            ds = ref_datasets.LoadImagesAndLabels(os.path.join(tmp, "images"), s, bs, augment=False, hyp=None, rect=True,
                                                  cache_images=True, single_cls=single_cls, stride=32, pad=0.5)
            order = [int(os.path.basename(f)[2:4]) for f in ds.img_files]
            ar = np.array([h / w for h, w in SHAPES], np.float64)[order]
            bi = np.arange(len(order)) // bs
            for v in np.unique(ar):                # the fixture must not depend on the order of ties
                assert len(set(bi[ar == v])) == 1, (name, v)
            out[f"{name}_order"] = np.array(order, np.int64)
            out[f"{name}_batch_shapes"] = np.asarray(ds.batch_shapes, np.int64)
            for pos, k in enumerate(order):
                out[f"{name}_cache_{k}"] = ds.imgs[pos]
            dl = torch.utils.data.DataLoader(ds, batch_size=min(bs, len(ds)), num_workers=0, shuffle=False,
                                             collate_fn=ref_datasets.LoadImagesAndLabels.collate_fn)
            nb = 0
            for b, (img, targets, paths, shapes) in enumerate(dl):
                out[f"{name}_img_{b}"] = img.numpy()
                out[f"{name}_targets_{b}"] = targets.numpy()
                out[f"{name}_paths_{b}"] = np.array([int(os.path.basename(p)[2:4]) for p in paths], np.int64)
                out[f"{name}_shapes_{b}"] = np.array([[h0, w0, g[0], g[1], p[0], p[1]] for (h0, w0), (g, p) in shapes], np.float64)
                nb += 1
            meta[name] = dict(img_size=s, batch_size=bs, single_cls=single_cls, n_batches=nb)
    out["meta_json"] = np.frombuffer(json.dumps(dict(shapes=SHAPES, cases=meta)).encode(), dtype=np.uint8)
    path = os.path.join(GOLD, "val_batch_cases.npz")
    np.savez_compressed(path, **out)
    print("val batches", {k: v["n_batches"] for k, v in meta.items()}, os.path.getsize(path) / 1e3, "KB")


if __name__ == "__main__":
    main()
