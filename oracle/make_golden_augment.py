"""TEST INFRASTRUCTURE - generates tests/golden/augment_cases.npz by running the UNMODIFIED reference's training item
(utils/datasets.py:518-593 `LoadImagesAndLabels.__getitem__` -> load_image / load_mosaic / random_perspective / augment_hsv, cv2 underneath)
on a stand-in dataset object that carries only the attributes those functions read.

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_augment.py

Sources are small synthetic BGR images of varied shapes (portrait, landscape, tiny) with boxes touching their borders, written as PNG
so that the reference's own `load_image` reads and resizes them.  The file holds the cached (resized) images at s = 96 and, for every
case, the seeds, the output images and float32 labels of consecutive items, and the next `random` / `numpy.random` draw after them.
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
SHAPES = [(72, 120), (120, 66), (30, 40), (96, 96), (50, 140), (150, 90), (48, 192)]   # at s = 96: shrink, grow, keep, exact 2x
SCRATCH = dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0, flipud=0.0,
               fliplr=0.5, mosaic=1.0, mixup=0.0)
CACHE_SIZE = 96
CASES = {  # name -> (img_size, seed, hyp overrides, items)
    "scratch": (96, 1, {}, 3),
    "stress": (128, 2, dict(degrees=10.0, shear=5.0, scale=0.5, translate=0.1), 3),
    "mixup": (96, 3, dict(mixup=1.0, degrees=5.0), 3),
    "flipud": (96, 4, dict(flipud=1.0, degrees=3.0), 3),
    "single": (128, 5, dict(mosaic=0.0, degrees=10.0, shear=2.0), 3),
}


def sources(seed=0):
    rs = np.random.RandomState(seed)
    imgs, labels = [], []
    for k, (h, w) in enumerate(SHAPES):
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), ((xx + yy) * 7 + 40 * k) % 256], -1)
        texture = np.kron(rs.randint(-40, 41, (h // 8 + 1, w // 8 + 1, 3)), np.ones((8, 8, 1), np.int64))[:h, :w]   # 8x8 blocks: compresses
        img = np.clip(base + texture, 0, 255).astype(np.uint8)
        img[h // 4:h // 2, w // 3:w // 2] = rs.randint(0, 256, 3)                 # a flat block: hue / saturation edge cases
        n = rs.randint(1, 5)
        lb = np.zeros((n, 5), np.float32)
        lb[:, 0] = rs.randint(0, 10, n)
        lb[:, 3:5] = rs.uniform(0.1, 0.6, (n, 2))
        lb[:, 1:3] = rs.uniform(0.2, 0.8, (n, 2))
        lb[0, 1], lb[0, 3] = lb[0, 3] / 2, lb[0, 3]                               # touches the left border
        if n > 1:
            lb[1, 2] = 1 - lb[1, 4] / 2                                           # touches the bottom border
        imgs.append(img)
        labels.append(lb)
    return imgs, labels


class StandIn:
    """the attributes LoadImagesAndLabels.__getitem__ / load_image / load_mosaic read (augment=True, rect=False, no image weights)"""

    def __init__(self, files, labels, img_size, hyp):
        self.img_files, self.labels, self.img_size, self.hyp = files, labels, img_size, hyp
        self.n = len(files)
        self.indices = range(self.n)
        self.segments = [[] for _ in range(self.n)]
        self.mosaic_border = [-img_size // 2, -img_size // 2]
        self.mosaic, self.augment, self.rect = True, True, False
        self.imgs = [None] * self.n
        self.img_hw0, self.img_hw = [None] * self.n, [None] * self.n


def main():
    import random

    import cv2
    ref_shims.import_reference()
    import utils.datasets as ref_datasets   # the reference's module (sys.path set by import_reference)
    imgs, labels = sources()
    out, meta = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        files = []
        for k, im in enumerate(imgs):
            files.append(os.path.join(tmp, f"src{k}.png"))
            cv2.imwrite(files[-1], im)
            out[f"src_{k}"] = im
            out[f"labels_{k}"] = labels[k]
        for name, (s, seed, over, n_items) in CASES.items():
            hyp = dict(SCRATCH, **over)
            ds = StandIn(files, [lb.copy() for lb in labels], s, hyp)
            for i in range(ds.n):                                   # cache_images: the reference's load_image
                ds.imgs[i], ds.img_hw0[i], ds.img_hw[i] = ref_datasets.load_image(ds, i)
                if s == CACHE_SIZE:                                  # one size is enough: the items pin the other through the outputs
                    out[f"cache{s}_{i}"] = ds.imgs[i]
            random.seed(seed)
            np.random.seed(seed)
            items = list(range(n_items))
            for i in items:
                img, lab, _, _ = ref_datasets.LoadImagesAndLabels.__getitem__(ds, i)
                out[f"{name}_img_{i}"] = img.numpy()
                out[f"{name}_lab_{i}"] = lab.numpy()[:, 1:].copy()
            meta[name] = dict(img_size=s, seed=seed, hyp=hyp, items=items, next_random=random.random(), next_np=float(np.random.random()))
    out["meta_json"] = np.frombuffer(json.dumps(dict(shapes=SHAPES, cases=meta)).encode(), dtype=np.uint8)
    path = os.path.join(GOLD, "augment_cases.npz")
    np.savez_compressed(path, **out)
    print("augment", {k: len(v["items"]) for k, v in meta.items()}, os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
