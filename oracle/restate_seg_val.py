"""TEST INFRASTRUCTURE - numpy restatement of one mode='val' segmentation item of the reference's PIL loader
(SegmentationDataset.py:96-116 `_val_sync_transform`, the per-item mask map of :203-205 / :287-293, and ToTensor), on top of the
Pillow arithmetic of restate_seg.py (`resize_bilinear`, `resize_nearest`, `mask_lut`, `to_tensor`).

tests/test_seg_val_host.py pins it to the reference's own items (tests/golden/seg_val_cases.npz, oracle/make_golden_seg_val.py); the
GPU tests compare the device path with it.
"""
from oracle.restate_seg import mask_lut, resize_bilinear, resize_nearest, to_tensor  # noqa: F401  (mask_lut: the tests' maps)


def val_geometry(w, h, crop):
    """(ow, oh, x1, y1) of `_val_sync_transform` for a w x h source: the short side resized to `crop`, the long side scaled and
    truncated, then the centre crop's corner with Python's round (half to even) on the resized size"""
    if w > h:
        oh = crop
        ow = int(1.0 * w * oh / h)
    else:
        ow = crop
        oh = int(1.0 * h * ow / w)
    x1 = int(round((ow - crop) / 2.))
    y1 = int(round((oh - crop) / 2.))
    return ow, oh, x1, y1


def val_item(img, mask, lut, crop):
    """dataset[i] for mode='val': (float32 (3, crop, crop), int64 (crop, crop))"""
    h, w = img.shape[:2]
    ow, oh, x1, y1 = val_geometry(w, h, crop)
    im = resize_bilinear(img, ow, oh)[y1:y1 + crop, x1:x1 + crop]
    m = resize_nearest(mask, ow, oh)[y1:y1 + crop, x1:x1 + crop]
    return to_tensor(im), lut[m]
