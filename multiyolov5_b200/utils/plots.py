"""Box drawing of detect.py behind the reference's names (reference utils/plots.py:57-68).  cv2 on the host, as in the reference: the boxes
are drawn on the decoded frame that is written out, after the device has scaled them to it."""
import cv2
import numpy as np


def plot_one_box(x, img, color=None, label=None, line_thickness=3):
    """reference utils/plots.py:57-68: one xyxy box, and a filled label box with its text, drawn on img in place (anti-aliased)"""
    tl = line_thickness or round(0.002 * (img.shape[0] + img.shape[1]) / 2) + 1
    color = color or [np.random.randint(0, 255) for _ in range(3)]
    c1, c2 = (int(x[0]), int(x[1])), (int(x[2]), int(x[3]))
    cv2.rectangle(img, c1, c2, color, thickness=tl, lineType=cv2.LINE_AA)
    if label:
        tf = max(tl - 1, 1)
        t_size = cv2.getTextSize(label, 0, fontScale=tl / 3, thickness=tf)[0]
        c2 = c1[0] + t_size[0], c1[1] - t_size[1] - 3
        cv2.rectangle(img, c1, c2, color, -1, cv2.LINE_AA)
        cv2.putText(img, label, (c1[0], c1[1] - 2), 0, tl / 3, [225, 255, 255], thickness=tf, lineType=cv2.LINE_AA)


def box_extent(x, img_shape, label=None, line_thickness=3):
    """the pixels plot_one_box(x, img, label=label, line_thickness=...) can change, as a list of (y0, y1, x0, x1) slices clipped to
    img_shape: the box and the label box, each grown by the line thickness plus 1 for the anti-aliased edge, the label box also by the
    text's descent below its baseline"""
    tl = line_thickness or round(0.002 * (img_shape[0] + img_shape[1]) / 2) + 1
    g = tl + 1
    (x1, y1), (x2, y2) = (int(x[0]), int(x[1])), (int(x[2]), int(x[3]))
    rects = [(min(y1, y2) - g, max(y1, y2) + g, min(x1, x2) - g, max(x1, x2) + g)]
    if label:
        tf = max(tl - 1, 1)
        (tw, th), base = cv2.getTextSize(label, 0, fontScale=tl / 3, thickness=tf)
        rects.append((y1 - th - 3 - g, y1 + base + tf + g, x1 - g, x1 + tw + tf + g))
    h, w = img_shape[:2]
    out = []
    for a, b, c, d in rects:
        a, b, c, d = max(a, 0), min(b + 1, h), max(c, 0), min(d + 1, w)
        if a < b and c < d:
            out.append((a, b, c, d))
    return out


def reblend(dst, mask, im0, rects, alpha=0.4, beta=0.6):
    """dst[r] = cv2.addWeighted(mask[r], alpha, im0[r], beta, 0) over the rectangles r (y0, y1, x0, x1): a blend of the undrawn frame
    becomes the blend of the drawn one, byte for byte, where drawing touched it"""
    for a, b, c, d in rects:
        dst[a:b, c:d] = cv2.addWeighted(mask[a:b, c:d], alpha, im0[a:b, c:d], beta, 0)
    return dst
