"""TEST INFRASTRUCTURE - generates tests/golden/seg_val_cases.npz by running the UNMODIFIED reference's segmentation datasets with
mode='val' (SegmentationDataset.py: CitySegmentation and CityBddSegmentation through get_citys_loader / get_citysbdd_loader with an int
crop_size, as train_citysbdd.py:236-241 builds its segval loader) on a temporary tree of small synthetic sources.

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_seg_val.py

The sources are landscape, portrait and square, so that the short side is resized to the crop (64 or 63) from 2x to 4x above it and from
below it, and the centre crop's (w' - c) / 2 falls on k + 0.5 for even and odd k as well as on whole numbers.  The City+BDD tree holds two
JPEG items whose train-id masks hold 255 next to Cityscapes .png items; the Cityscapes masks hold every label id and 255.  Items are taken
with `dataset[i]` in the order of their file names (the dataset's own order is os.walk's, which depends on the file system), so the
file is the same wherever it is regenerated; the npz is written with fixed zip timestamps for the same reason.

Stored: every distinct source as PIL decoded it and mask once (`sources` maps a case's item to their keys), each item's output (images as
uint8 v with output == float32(v) / 255, labels as int16, both checked here), the geometry the reference used (the size of each
Image.resize call and the Image.crop box, recorded by wrapping those two PIL methods while the item is built), the next `random` / torch
draw after the items, and the exception of get_citys_loader / get_custom_loader with their default tuple crop_size.
"""
import io
import json
import os
import random
import sys
import tempfile
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
# (h, w) of the Cityscapes-style .png sources; with crop 64: (w' or h') - 64 = 67 (33.5), 49 (24.5), 0, 1 (0.5), 3 (1.5), 64, 51 (25.5)
CITY_SHAPES = [(128, 262), (71, 40), (100, 100), (48, 49), (256, 268), (256, 128), (72, 40), (50, 50)]
# (h, w) of the BDD-style .jpg sources (16:9, the 1280x720 aspect)
BDD_SHAPES = [(72, 128), (144, 256)]
CASES = {  # name -> (loader, crop_size, seed)
    "citys": ("citys", 64, 21),
    "citys_c63": ("citys", 63, 22),
    "citysbdd": ("citysbdd", 64, 23),
}
SEED = 5


def sources(shapes, trainid, seed):
    """uint8 RGB images with gradients, 16x16 noise blocks and a flat patch; masks of 4x4 blocks over every Cityscapes label id and 255
    (train ids 0..18 and 255 when `trainid`), with a column of single-pixel detail for the NEAREST index"""
    rs = np.random.RandomState(seed)
    imgs, masks = [], []
    ids = np.concatenate([np.arange(19 if trainid else 34), [255]])
    for k, (h, w) in enumerate(shapes):
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx * 255 // (w - 1), yy * 255 // (h - 1), ((xx + 2 * yy) * 5 + 60 * k) % 256], -1)
        texture = np.kron(rs.randint(-5, 6, (h // 16 + 1, w // 16 + 1, 3)) * 10, np.ones((16, 16, 1), np.int64))[:h, :w]
        img = np.clip(base + texture, 0, 255).astype(np.uint8)
        img[h // 4:h // 2, w // 3:w // 2] = rs.randint(0, 256, 3)
        m = np.kron(rs.choice(ids, (h // 4 + 1, w // 4 + 1)), np.ones((4, 4), np.int64))[:h, :w]
        m[:, :2] = ids[np.arange(h) % len(ids)][:, None]
        imgs.append(img)
        masks.append(m.astype(np.uint8))
    return imgs, masks


def write_tree(root):
    """citys/{leftImg8bit,gtFine}/val/aachen/a{k}_*.png; citysbdd/ the same plus .../val/bdd/b{k}_leftImg8bit.jpg with train-id .png
    masks; custom/{segimages,seglabels}/val/c0.png"""
    from PIL import Image
    city_imgs, city_masks = sources(CITY_SHAPES, False, SEED)
    bdd_imgs, bdd_masks = sources(BDD_SHAPES, True, SEED + 1)
    roots = {}
    for name, with_bdd in (("citys", False), ("citysbdd", True)):
        r = roots[name] = os.path.join(root, name)
        dirs = ["leftImg8bit/val/aachen", "gtFine/val/aachen"] + (["leftImg8bit/val/bdd", "gtFine/val/bdd"] if with_bdd else [])
        for d in dirs:
            os.makedirs(os.path.join(r, d))
        for k, (im, m) in enumerate(zip(city_imgs, city_masks)):
            Image.fromarray(im).save(os.path.join(r, "leftImg8bit/val/aachen", f"a{k}_leftImg8bit.png"))
            Image.fromarray(m).save(os.path.join(r, "gtFine/val/aachen", f"a{k}_gtFine_labelIds.png"))
        if with_bdd:
            for k, (im, m) in enumerate(zip(bdd_imgs, bdd_masks)):
                Image.fromarray(im).save(os.path.join(r, "leftImg8bit/val/bdd", f"b{k}_leftImg8bit.jpg"), quality=90)
                Image.fromarray(m).save(os.path.join(r, "gtFine/val/bdd", f"b{k}_gtFine_labelIds.png"))
    cus = roots["custom"] = os.path.join(root, "custom")
    for d in ("segimages/val", "seglabels/val"):
        os.makedirs(os.path.join(cus, d))
    Image.fromarray(city_imgs[0]).save(os.path.join(cus, "segimages/val", "c0.png"))
    Image.fromarray(np.where(city_masks[0] > 18, 255, city_masks[0]).astype(np.uint8)).save(os.path.join(cus, "seglabels/val", "c0.png"))
    return roots


class GeometryRecorder:
    """records the arguments of PIL's Image.resize and Image.crop while active (the reference's own calls are left to run)"""

    def __init__(self):
        from PIL import Image
        self.Image, self.calls = Image.Image, []
        self.resize, self.crop = Image.Image.resize, Image.Image.crop

    def __enter__(self):
        rec, resize, crop = self.calls, self.resize, self.crop

        def resize_(im, size, resample=None, *a, **k):
            rec.append(("resize", [int(v) for v in size], int(resample)))
            return resize(im, size, resample, *a, **k)

        def crop_(im, box=None):
            rec.append(("crop", [int(v) for v in box]))
            return crop(im, box)
        self.Image.resize, self.Image.crop = resize_, crop_
        return self

    def __exit__(self, *exc):
        self.Image.resize, self.Image.crop = self.resize, self.crop


def save_npz(path, arrays):
    """np.savez_compressed with fixed zip timestamps, so that the same arrays give the same bytes"""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k, a in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(a), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    import torch
    from PIL import Image
    ref_shims.import_reference()
    import SegmentationDataset as SD    # the reference's module (sys.path set by import_reference)
    out, meta, stored = {}, {}, {"src": [], "mask": []}

    def store(kind, a):                                         # each distinct decoded image / mask once
        for k, b in enumerate(stored[kind]):
            if a.shape == b.shape and np.array_equal(a, b):
                return k
        stored[kind].append(a)
        out[f"{kind}_{len(stored[kind]) - 1}"] = a
        return len(stored[kind]) - 1

    raises = {}
    with tempfile.TemporaryDirectory() as tmp:
        roots = write_tree(tmp)
        for name, (loader, crop, seed) in CASES.items():
            get = SD.get_citys_loader if loader == "citys" else SD.get_citysbdd_loader
            ds = get(root=roots[loader], split="val", mode="val", base_size=1024, crop_size=crop, workers=0, pin=False).dataset
            assert ds.mode == "val" and ds.crop_size == crop
            order = sorted(range(len(ds.images)), key=lambda i: os.path.basename(ds.images[i]))
            files, srcs, geoms = [], [], []
            for i in order:
                srcs.append((store("src", np.array(Image.open(ds.images[i]).convert("RGB"))), store("mask", np.array(Image.open(ds.mask_paths[i])))))
                files.append(os.path.basename(ds.images[i]))
            random.seed(seed)
            torch.manual_seed(seed)
            for j, i in enumerate(order):
                with GeometryRecorder() as g:
                    img, lab = ds[i]
                geoms.append(g.calls)
                v = torch.round(img * 255).to(torch.uint8)
                assert torch.equal(v.float() / 255, img) and img.dtype == torch.float32 and img.shape == (3, crop, crop), (name, i)
                out[f"{name}_img_{j}"] = v.numpy()
                assert lab.dtype == torch.int64 and lab.shape == (crop, crop) and torch.equal(lab.to(torch.int16).long(), lab)
                out[f"{name}_lab_{j}"] = lab.numpy().astype(np.int16)
            meta[name] = dict(loader=loader, crop_size=crop, seed=seed, files=files, sources=srcs, geometry=geoms,
                              next_random=random.random(), next_torch=float(torch.rand(1)))
        # the loaders' default crop_size is a tuple (get_custom_loader always passes (base_size, base_size)): mode='val' raises
        for name, make in (("get_citys_loader", lambda: SD.get_citys_loader(root=roots["citys"], split="val", mode="val", workers=0,
                                                                            pin=False)),
                           ("get_custom_loader", lambda: SD.get_custom_loader(root=roots["custom"], split="val", mode="val",
                                                                              base_size=64, workers=0, pin=False))):
            ds = make().dataset
            try:
                ds[0]
            except Exception as e:      # noqa: BLE001  (the type is what is recorded)
                raises[name] = dict(crop_size=list(ds.crop_size), type=type(e).__name__, message=str(e))
            else:
                raise AssertionError(f"{name}(mode='val') did not raise")
    out["meta_json"] = np.frombuffer(json.dumps(dict(cases=meta, raises=raises), sort_keys=True).encode(), dtype=np.uint8)
    path = os.path.join(GOLD, "seg_val_cases.npz")
    save_npz(path, out)
    print("seg val", {k: len(v["files"]) for k, v in meta.items()}, raises, os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
