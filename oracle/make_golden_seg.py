"""TEST INFRASTRUCTURE - generates tests/golden/seg_augment_cases.npz by running the UNMODIFIED reference's segmentation datasets
(SegmentationDataset.py: CitySegmentation, CityBddSegmentation, CustomSegmentation with the transforms of get_citys_loader,
get_citysbdd_loader and get_custom_loader) on a temporary tree of small synthetic images.

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_seg.py

Sources are about 256x128 (landscape and portrait) with base_size 128 and crop (128, 64), so that the drawn long sides (96..384) cover
down-scaling, up-scaling and padding.  The City+BDD tree holds one JPEG item, whose mask is mapped as train ids.  Items are taken with
`dataset[i]` in sequence (a DataLoader's shuffle would consume torch's generator).  The file holds every distinct source as PIL decoded it and mask once
(`sources` maps a case's item index to their keys), each
item's output (images as uint8 v with output == float32(v) / 255, labels as int16, both checked here), and the next `random` / torch draw.
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

GOLD = os.path.join(HERE, "..", "tests", "golden")
SHAPES = [(128, 256), (200, 120), (100, 250), (128, 256)]        # (h, w) of the sources
CASES = {  # name -> (loader, kind, base_size, crop_size, seed, items)
    "citys": ("citys", "train", 128, (128, 64), 11, [0, 1, 2, 3, 0, 1]),
    "citysbdd": ("citysbdd", "train", 128, (128, 64), 12, [0, 1, 2, 3, 4, 4]),
    "custom": ("custom", "train", 128, (128, 128), 13, [0, 1, 2, 0]),
    "testval": ("citys", "testval", 160, (128, 64), 14, [0, 3]),
}


def sources(seed=0):
    """uint8 RGB images with gradients, 16x16 noise blocks and a flat patch; label-id masks with every Cityscapes id and 255"""
    rs = np.random.RandomState(seed)
    imgs, masks = [], []
    for k, (h, w) in enumerate(SHAPES):
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx * 255 // (w - 1), yy * 255 // (h - 1), ((xx + 2 * yy) * 5 + 60 * k) % 256], -1)
        texture = np.kron(rs.randint(-5, 6, (h // 16 + 1, w // 16 + 1, 3)) * 10, np.ones((16, 16, 1), np.int64))[:h, :w]
        img = np.clip(base + texture, 0, 255).astype(np.uint8)
        img[h // 4:h // 2, w // 3:w // 2] = rs.randint(0, 256, 3)
        ids = np.concatenate([np.arange(34), [255]])
        m = np.kron(rs.choice(ids, (h // 4 + 1, w // 4 + 1)), np.ones((4, 4), np.int64))[:h, :w]
        m[:, :3] = np.arange(h)[:, None] % 34                               # single-pixel detail for the NEAREST index
        imgs.append(img)
        masks.append(m.astype(np.uint8))
    return imgs, masks


def write_tree(root, imgs, masks):
    """leftImg8bit/train/<city>/*_leftImg8bit.png + gtFine/train/<city>/*_gtFine_labelIds.png, one BDD-style .jpg, and the custom
    segimages/train + seglabels/train layout"""
    from PIL import Image
    city = os.path.join(root, "citys")
    for d in ("leftImg8bit/train/aachen", "gtFine/train/aachen"):
        os.makedirs(os.path.join(city, d))
    for k, (im, m) in enumerate(zip(imgs, masks)):
        Image.fromarray(im).save(os.path.join(city, "leftImg8bit/train/aachen", f"a{k}_leftImg8bit.png"))
        Image.fromarray(m).save(os.path.join(city, "gtFine/train/aachen", f"a{k}_gtFine_labelIds.png"))
    bdd = os.path.join(root, "citysbdd")
    for d in ("leftImg8bit/train/aachen", "gtFine/train/aachen", "leftImg8bit/train/bdd", "gtFine/train/bdd"):
        os.makedirs(os.path.join(bdd, d))
    for k, (im, m) in enumerate(zip(imgs, masks)):
        Image.fromarray(im).save(os.path.join(bdd, "leftImg8bit/train/aachen", f"a{k}_leftImg8bit.png"))
        Image.fromarray(m).save(os.path.join(bdd, "gtFine/train/aachen", f"a{k}_gtFine_labelIds.png"))
    tid = np.where(masks[1] > 18, 255, masks[1]).astype(np.uint8)             # BDD masks hold train ids and 255
    Image.fromarray(imgs[1]).save(os.path.join(bdd, "leftImg8bit/train/bdd", "b0_leftImg8bit.jpg"), quality=90)
    Image.fromarray(tid).save(os.path.join(bdd, "gtFine/train/bdd", "b0_gtFine_labelIds.png"))
    cus = os.path.join(root, "custom")
    for d in ("segimages/train", "seglabels/train"):
        os.makedirs(os.path.join(cus, d))
    for k, (im, m) in enumerate(zip(imgs, masks)):
        Image.fromarray(im).save(os.path.join(cus, "segimages/train", f"c{k}.png"))
        Image.fromarray(np.where(m > 18, 255, m).astype(np.uint8)).save(os.path.join(cus, "seglabels/train", f"c{k}.png"))
    return dict(citys=city, citysbdd=bdd, custom=cus)


def main():
    import torch
    from PIL import Image
    ref_shims.import_reference()
    import SegmentationDataset as SD    # the reference's module (sys.path set by import_reference)
    imgs, masks = sources()
    out, meta, stored = {}, {}, {"src": [], "mask": []}

    def store(kind, a):                                         # each distinct decoded image / mask once
        for k, b in enumerate(stored[kind]):
            if a.shape == b.shape and np.array_equal(a, b):
                return k
        stored[kind].append(a)
        out[f"{kind}_{len(stored[kind]) - 1}"] = a
        return len(stored[kind]) - 1

    with tempfile.TemporaryDirectory() as tmp:
        roots = write_tree(tmp, imgs, masks)
        for name, (loader, mode, base, crop, seed, items) in CASES.items():
            if loader == "citys":
                ds = SD.get_citys_loader(root=roots["citys"], mode=mode, base_size=base, crop_size=crop, workers=0, pin=False).dataset
            elif loader == "citysbdd":
                ds = SD.get_citysbdd_loader(root=roots["citysbdd"], mode=mode, base_size=base, crop_size=crop, workers=0, pin=False).dataset
            else:
                ds = SD.get_custom_loader(root=roots["custom"], mode=mode, base_size=base, workers=0, pin=False).dataset
            files, srcs = [], []
            for ip, mp in zip(ds.images, ds.mask_paths):       # os.walk order: item k of the dataset is src_/mask_ srcs[k]
                srcs.append((store("src", np.array(Image.open(ip).convert("RGB"))), store("mask", np.array(Image.open(mp)))))
                files.append(os.path.basename(ip))
            random.seed(seed)
            torch.manual_seed(seed)
            for j, i in enumerate(items):
                img, lab = ds[i]
                v = torch.round(img * 255).to(torch.uint8)
                assert torch.equal(v.float() / 255, img) and img.dtype == torch.float32, (name, i)
                out[f"{name}_img_{j}"] = v.numpy()
                assert lab.dtype == torch.int64 and torch.equal(lab.to(torch.int16).long(), lab)
                out[f"{name}_lab_{j}"] = lab.numpy().astype(np.int16)
            meta[name] = dict(loader=loader, mode=mode, base_size=base, crop_size=list(ds.crop_size), seed=seed, items=items, files=files, sources=srcs,
                              next_random=random.random(), next_torch=float(torch.rand(1)))
    out["meta_json"] = np.frombuffer(json.dumps(dict(cases=meta)).encode(), dtype=np.uint8)
    path = os.path.join(GOLD, "seg_augment_cases.npz")
    np.savez_compressed(path, **out)
    print("seg augment", {k: len(v["items"]) for k, v in meta.items()}, os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
