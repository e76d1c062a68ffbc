"""TEST INFRASTRUCTURE - generates tests/golden/image_weights_cases.npz from the UNMODIFIED reference's `--image-weights` pieces:
`utils.general.labels_to_class_weights` / `labels_to_image_weights` (utils/general.py:216-240), the standard library's
`random.choices(range(n), weights=iw, k=n)` as train.py:310-311 calls it, and `LoadImagesAndLabels.__getitem__` (utils/datasets.py:518-593)
on a stand-in dataset whose `indices` are the drawn list (so load_mosaic's `random.choices(self.indices, k=3)` picks partners from it).

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_image_weights.py

Both reference functions still say `np.int`, which numpy 2 removed: this process alone sets `np.int = int` before calling them.  The
per-epoch `cw = model.class_weights.cpu().numpy() * (1 - maps) ** 2 / nc` is train.py's own expression, written out in
oracle/restate_image_weights.epoch_cw.  Per case the file holds the labels, the class weights, and per epoch the maps, cw, image weights
and drawn indices (or the ValueError's message), then the next `random` and `numpy.random` draws.  The label sets are stored as the
arguments of oracle/restate_image_weights.synth_labels and a digest of what it made, and the augmented items' sources are the ones
tests/golden/augment_cases.npz already holds (make_golden_augment.sources()), so the file stays small.
"""
import json
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import make_golden_augment as mga, ref_shims  # noqa: E402
from oracle.restate_image_weights import epoch_cw, labels_digest, synth_labels  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")


def maps_of(rs, nc, ones=0):
    m = rs.uniform(0.0, 0.9, nc)
    m[rs.choice(nc, ones, replace=False)] = 1.0           # classes whose weight becomes exactly zero
    return m


# name -> (seed, n, nc, labels per image, share of empty images, fractional classes, single_cls, maps per epoch (callables of rs, nc))
CASES = {
    "nc1_single": (1, 60, 1, 3, 0.2, False, True, [lambda rs, nc: np.zeros(nc)]),
    "nc5": (2, 300, 5, 2, 0.3, False, False, [lambda rs, nc: maps_of(rs, nc, 2), lambda rs, nc: maps_of(rs, nc, 0)]),
    "nc10_city": (3, 2975, 10, 6, 0.05, False, False, [lambda rs, nc: np.zeros(nc), lambda rs, nc: maps_of(rs, nc, 3)]),
    "nc80": (4, 1500, 80, 7, 0.01, False, False, [lambda rs, nc: maps_of(rs, nc, 5), lambda rs, nc: maps_of(rs, nc, 0)]),
    "nc130": (5, 700, 130, 9, 0.1, True, False, [lambda rs, nc: maps_of(rs, nc, 10)]),
    "all_maps_one": (6, 100, 10, 3, 0.1, False, False, [lambda rs, nc: np.ones(nc)]),
    "n1": (7, 1, 3, 4, 0.0, False, False, [lambda rs, nc: maps_of(rs, nc, 1)]),
}
AUG_HYP = dict(mga.SCRATCH, mosaic=1.0, mixup=0.5, degrees=5.0)
AUG_CASES = {"aug_mosaic": (11, AUG_HYP, 96, 4), "aug_single": (12, dict(AUG_HYP, mosaic=0.0), 96, 2)}
AUG_EMPTY = (2, 5)          # source images without labels: never drawn


def main():
    import cv2
    ref_shims.import_reference()
    import utils.datasets as ref_datasets
    import utils.general as ref_general
    np.int = int                                                     # the reference's functions predate numpy 2
    out, meta = {}, {"cases": {}, "aug": {}}
    for name, (seed, n, nc, per, empty, frac, single, maps_fns) in CASES.items():
        spec = dict(seed=seed, n=n, nc=nc, per_image=per, empty=empty, frac=frac, single=single)
        labels = synth_labels(**spec)                               # single: the class column zeroed, as single_cls=True does
        rs = np.random.RandomState(seed + 100)                      # the maps' stream
        model_cw = ref_general.labels_to_class_weights(labels, nc) * nc    # train.py:255 (.to(device) aside)
        out[f"{name}_class_weights"] = ref_general.labels_to_class_weights(labels, nc).numpy()
        m = dict(seed=seed, nc=nc, n=n, epochs=len(maps_fns), errors=[], labels_spec=spec, labels_sha256=labels_digest(labels))
        random.seed(seed)
        np.random.seed(seed)
        for e, fn in enumerate(maps_fns):
            maps = fn(rs, nc)
            cw = epoch_cw(model_cw.cpu().numpy(), maps)
            iw = ref_general.labels_to_image_weights(labels, nc=nc, class_weights=cw)
            out[f"{name}_e{e}_maps"], out[f"{name}_e{e}_cw"], out[f"{name}_e{e}_iw"] = maps, cw, iw
            try:
                out[f"{name}_e{e}_indices"] = np.array(random.choices(range(n), weights=iw, k=n), np.int32)
                m["errors"].append(None)
            except ValueError as ex:
                m["errors"].append(str(ex))
        m["next_random"], m["next_np"] = random.random(), float(np.random.random())
        meta["cases"][name] = m

    imgs, labels = mga.sources()
    for k in AUG_EMPTY:
        labels[k] = np.zeros((0, 5), np.float32)
    nc = 10
    with tempfile.TemporaryDirectory() as tmp:
        files = []
        for k, im in enumerate(imgs):
            files.append(os.path.join(tmp, f"src{k}.png"))
            cv2.imwrite(files[-1], im)
        for name, (seed, hyp, s, n_items) in AUG_CASES.items():
            ds = mga.StandIn(files, [lb.copy() for lb in labels], s, hyp)
            for i in range(ds.n):
                ds.imgs[i], ds.img_hw0[i], ds.img_hw[i] = ref_datasets.load_image(ds, i)
            model_cw = ref_general.labels_to_class_weights(ds.labels, nc) * nc
            maps = np.linspace(0.0, 0.8, nc)
            random.seed(seed)
            np.random.seed(seed)
            cw = epoch_cw(model_cw.cpu().numpy(), maps)
            iw = ref_general.labels_to_image_weights(ds.labels, nc=nc, class_weights=cw)
            ds.indices = random.choices(range(ds.n), weights=iw, k=ds.n)
            out[f"{name}_indices"] = np.array(ds.indices, np.int32)
            for p in range(n_items):
                img, lab, _, _ = ref_datasets.LoadImagesAndLabels.__getitem__(ds, p)
                out[f"{name}_img_{p}"] = img.numpy()
                out[f"{name}_lab_{p}"] = lab.numpy()[:, 1:].copy()
            meta["aug"][name] = dict(seed=seed, hyp=hyp, img_size=s, items=n_items, nc=nc, maps=maps.tolist(),
                                     next_random=random.random(), next_np=float(np.random.random()))
    meta["aug_sources"], meta["aug_empty"] = len(imgs), list(AUG_EMPTY)
    out["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    path = os.path.join(GOLD, "image_weights_cases.npz")
    np.savez_compressed(path, **out)
    print("image_weights", list(meta["cases"]), list(meta["aug"]), os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
