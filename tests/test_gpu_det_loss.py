"""H100: the fused detection loss (`myolo_det_loss`, csrc/detloss.cu) in isolation against its fp64 restatement: oracle/restate.py's
compute_det_loss on float64 predictions, whose target assignment makes the reference's float32 decisions.

Every case checks exactly: the valid-candidate count of every level and the winning (last valid) candidate of every cell, read from the
kernel's workspace; zero box and class gradients and zero objectness targets off the matched cells; no NaN left in the gradient (it and the
workspace are NaN before the call); the predictions untouched.  Within limits, per level: each channel group of the gradient (xy, wh,
objectness at matched cells, objectness at unmatched cells, classes) as max |ours - ref| over the group's max |ref|, so the small objectness
gradient of the unmatched cells is not measured against the box gradient of a few matched ones; the objectness targets of the matched cells;
the four loss items by relative error.

Cases that test a decision (the neighbour-cell rule, the anchor ratio test, the cell clamp, shared cells, coincident box edges) put it on its
boundary with values that are exact in fp32 and fp64: dyadic coordinates, on power-of-two grids or at products checked to be exact.  Random
cases keep random values, so no decision of theirs sits on a boundary."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import restate

pytestmark = pytest.mark.gpu

# about 4x the worst value over all cases on an H100 80GB HBM3 (700 W power limit): xy 6.8e-7 (neighbour_1x1), wh 1.8e-6 (na10_nt1200,
# many candidates summed into one cell), obj_m 3.2e-7, obj_u 1.7e-7, cls 2.5e-7, tobj 5.0e-7, items 7.6e-7 (train_step)
LIMITS = dict(xy=3e-6, wh=8e-6, obj_m=1.5e-6, obj_u=8e-7, cls=1e-6, tobj=2e-6, items=3e-6)
WORST = {}

ANCHORS_PX = [[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]]   # the models' P3-P5 anchors
STRIDES = (8, 16, 32)


def balance(nl):
    """ComputeLoss's per-level objectness weights (reference utils/loss.py:104)"""
    return {3: [4.0, 1.0, 0.4]}.get(nl, [4.0, 1.0, 0.25, 0.06, 0.02])[:nl]


def default_anchors(nl):
    """the models' anchors in grid units (pixels over stride: dyadic)"""
    return np.array([np.array(ANCHORS_PX[i], np.float32).reshape(3, 2) / STRIDES[i] for i in range(nl)], np.float32)


def dyadic_anchors(nl, na, seed):
    return (np.random.RandomState(seed).randint(6, 48, (nl, na, 2)) / 8.0).astype(np.float32)


def norm(g, n):
    """the float32 x with float32(x) * float32(n) == g exactly, the normalised coordinate of grid coordinate g; None if there is none"""
    g, n = np.float32(g), np.float32(n)
    x = g / n
    for _ in range(8):
        if x * n == g:
            return x
        x = np.nextafter(x, np.float32(np.inf) if x * n < g else np.float32(-np.inf))
    return None


class Case:
    """predictions (random unless set), targets, anchors in grid units and hyps of one call"""

    def __init__(self, shapes, anchors, nc=10, B=2, gr=1.0, mult=1.0, scale=None, seed=0, **hyp):
        self.shapes, self.anchors, self.nc, self.B, self.gr, self.mult, self.scale = shapes, anchors, nc, B, gr, mult, scale
        self.hyp = dict(dict(box=0.05, obj=1.0, cls=0.5, anchor_t=4.0, label_smoothing=0.0), **hyp)
        self.na = anchors.shape[1]
        self.rs = np.random.RandomState(seed)
        self.p = [(self.rs.randn(B, self.na, ny, nx, 5 + nc) * 1.5).astype(np.float32) for ny, nx in shapes]
        self.rows = []

    @property
    def targets(self):
        return np.array(self.rows, np.float32).reshape(-1, 6)

    def grid(self, l, b, gx, gy, gw, gh, cls=0):
        """a target given in grid units of level l"""
        ny, nx = self.shapes[l]
        row = [norm(gx, nx), norm(gy, ny), norm(gw, nx), norm(gh, ny)]
        assert None not in row, (gx, gy, gw, gh, self.shapes[l])
        self.rows.append([b, cls, *row])

    def random(self, n, images=None, wh=(0.02, 0.4)):
        rs = self.rs
        b = rs.randint(0, self.B, n) if images is None else rs.choice(images, n)
        for i in range(n):
            self.rows.append([b[i], rs.randint(0, self.nc), *rs.uniform(0.01, 0.99, 2), *rs.uniform(*wh, 2)])
        return self


# ---- the cases ---------------------------------------------------------------------------------------------------------------------------
def neighbour_case(ny, nx):
    """the neighbour-cell rule (gxy % 1 < 0.5 and gxy > 1, the same on gain - gxy) at and beside its boundaries in x and in y, and the cell
    clamp at normalised 0 and 1 (tbox then relative to the clamped cell: x = 1.0 in cell nx - 1)"""
    c = Case([(ny, nx)], np.array([[[1.0, 1.0], [2.0, 1.5]]], np.float32), B=2, seed=ny * 100 + nx)
    e = 2.0 ** -6

    def values(n):
        """the boundary values that are exact on a grid of n cells; a fractional part is tried at integer parts from n // 2 down"""
        v = [next((k + f for k in range(n // 2, -1, -1) if k + f <= n and norm(k + f, n) is not None), None)
             for f in (0.0, 0.5 - e, 0.5, 0.5 + e)]
        v += [1.0, 1.0 + e] + [n - d for d in (0.5, 1.0, 1.0 + e)] + [0.0, float(n)]
        return sorted({x for x in v if x is not None and 0.0 <= x <= n and norm(x, n) is not None})

    for i, gx in enumerate(values(nx)):
        c.grid(0, i % 2, gx, min(ny * 0.5 + 0.25, ny * 0.75), 1.0, 1.25)
    for i, gy in enumerate(values(ny)):
        c.grid(0, i % 2, min(nx * 0.5 + 0.25, nx * 0.75), gy, 1.25, 1.0)
    c.grid(0, 1, float(nx), float(ny), 1.5, 1.5)          # both coordinates at 1.0
    c.grid(0, 0, 0.0, 0.0, 1.5, 1.5)
    return c


def ratio_case(t):
    """max(r, 1/r) < anchor_t at the bound (rejected: the test is strict), at 1/anchor_t, one ulp inside either bound, and zero width or height
    (1/r = inf), against anchors of power-of-two sides so that every ratio is exact"""
    c = Case([(16, 32)], np.array([[[2.0, 2.0], [1.0, 4.0]]], np.float32), B=1, seed=int(t), anchor_t=float(t))
    t32 = np.float32(t)
    inside_hi = np.nextafter(t32, np.float32(0))
    inside_lo = np.nextafter(np.float32(1) / t32, np.float32(np.inf))
    while not np.maximum(inside_lo, np.float32(1) / inside_lo) < t32:
        inside_lo = np.nextafter(inside_lo, np.float32(np.inf))
    sides = [2.0 * t32, 2.0 / t32, 2.0 * inside_hi, 2.0 * inside_lo, 0.0]
    for i, s in enumerate(sides):
        assert np.float32(s) / np.float32(2.0) in (t32, np.float32(1) / t32, inside_hi, inside_lo, 0.0)
        c.grid(0, 0, 3.25 + 3 * i, 4.25, s, 2.0)
        c.grid(0, 0, 3.25 + 3 * i, 10.25, 2.0, s)
    return c


def shared_case():
    """cells reached by several candidates: identical targets; different targets through different offsets at both anchors; and a cell whose
    winner (the later candidate, offset x-1) has a negative CIoU - its objectness target clamps to 1 - gr - after a candidate with a positive one"""
    c = Case([(16, 32)], np.array([[[0.5, 0.5], [1.0, 1.0]]], np.float32), B=2, gr=0.5, seed=7)
    for _ in range(3):
        c.grid(0, 0, 10.3125, 3.6875, 0.75, 0.625, cls=2)
    c.grid(0, 0, 5.25, 8.375, 0.75, 0.75, cls=1)          # centre cell 5, x-1 neighbour cell 4
    c.grid(0, 0, 4.75, 8.375, 0.75, 0.75, cls=3)          # centre cell 4, x+1 neighbour cell 5
    c.grid(0, 1, 4.5, 8.5, 0.625, 0.625, cls=4)           # centre of cell (8, 4): positive CIoU against box logits 0
    c.grid(0, 1, 5.25, 8.5, 0.25, 0.25, cls=5)            # its x-1 candidate lands there later: disjoint from the prediction
    c.p[0][1, 0, 8, 4, :4] = 0.0
    c.random(10, images=[0, 1])
    return c


def ciou_case(kind):
    """one candidate of a chosen CIoU geometry at cell (gj, gi) = (4, 8) of image 0 with box logits 0 (prediction centred, of anchor size),
    plus random targets in image 1"""
    c = Case([(16, 32)], np.array([[[0.5, 0.5], [1.25, 1.625], [2.0, 3.75]]], np.float32), B=2, seed=11)
    gi, gj, d = 8, 4, 0.125
    aw, ah = 1.25, 1.625
    geo = dict(all=(0.5, 0.5, aw, ah),
               x1=(0.5 + d / 2, 0.5, aw + d, ah + 2 * d), x2=(0.5 - d / 2, 0.5, aw + d, ah + 2 * d),
               y1=(0.5, 0.5 + d / 2, aw + 2 * d, ah + d), y2=(0.5, 0.5 - d / 2, aw + 2 * d, ah + d),
               pred_contains=(0.53125, 0.53125, aw / 2, ah / 2), target_contains=(0.53125, 0.53125, 2 * aw, 2 * ah))
    a = 1
    if kind in geo:
        tx, ty, tw, th = geo[kind]
        c.grid(0, 0, gi + tx, gj + ty, tw, th)
    elif kind == "touching":                              # offset x-1 candidate: target [0.75, 1.25] against prediction [0.25, 0.75]
        a = 0
        c.grid(0, 0, gi + 1.0, gj + 0.5, 0.5, 0.75)
    elif kind == "disjoint":                              # target [1.125, 1.375] against [0.25, 0.75]
        a = 0
        c.grid(0, 0, gi + 1.25, gj + 0.5, 0.25, 0.75)
    elif kind == "saturated":                             # box logits +-30 at every cell of image 0: sigma is 0 or 1 in fp32
        c.random(12, images=[0])
        c.p[0][0, ..., :4] = c.rs.choice([-30.0, 30.0], c.p[0][0, ..., :4].shape)
    c.p[0][0, a, gj, gi, :4] = 0.0
    return c.random(12, images=[1])


def bce_case(gr):
    """objectness and class logits at 0, +-20 (softplus's threshold) and +-90, label smoothing 0.1"""
    c = Case([(16, 32), (8, 16), (4, 8)], default_anchors(3), B=2, gr=gr, seed=int(gr * 10), label_smoothing=0.1)
    for q in c.p:
        special = c.rs.rand(*q.shape[:-1], q.shape[-1] - 4) < 0.5
        vals = c.rs.choice([0.0, 20.0, -20.0, 90.0, -90.0], special.shape).astype(np.float32)
        q[..., 4:] = np.where(special, vals, q[..., 4:])
    return c.random(30)


def count_case(nl, na, nc, B, nt, shapes=None, images=None, seed=0, **kw):
    shapes = shapes or [(16 >> i, 32 >> i) for i in range(nl)]
    anchors = default_anchors(nl) if na == 3 else dyadic_anchors(nl, na, seed)
    return Case(shapes, anchors, nc=nc, B=B, seed=seed, **kw).random(nt, images=images)


def train_step_case():
    """the train step's shapes: 16 x 3 x 64x128 / 32x64 / 16x32, nc = 10, 160 boxes with a group of identical ones, loss scale on the device"""
    c = count_case(3, 3, 10, 16, 160, shapes=[(64, 128), (32, 64), (16, 32)], seed=5, mult=0.75, scale=1024.0, box=0.0375, cls=0.3125)
    c.rows[20:24] = [c.rows[20]] * 4
    return c


CASES = {
    **{f"neighbour_{ny}x{nx}": (lambda ny=ny, nx=nx: neighbour_case(ny, nx)) for ny, nx in [(16, 32), (13, 23), (2, 3), (1, 1)]},
    **{f"ratio_t{t}": (lambda t=t: ratio_case(t)) for t in (2, 4, 8)},
    "shared": shared_case,
    **{f"ciou_{k}": (lambda k=k: ciou_case(k)) for k in ("all", "x1", "x2", "y1", "y2", "touching", "disjoint", "pred_contains",
                                                         "target_contains", "saturated")},
    **{f"bce_gr{g}": (lambda g=g: bce_case(g)) for g in (1.0, 0.5, 0.0)},
    "nl1_na1_nc1_B1": lambda: count_case(1, 1, 1, 1, 20, seed=1),
    "nl2_na4_nc80": lambda: count_case(2, 4, 80, 2, 25, seed=2),
    "nl3_na10_nt1": lambda: count_case(3, 10, 10, 1, 1, seed=3),
    "nl3_na3_B16_nt0": lambda: count_case(3, 3, 10, 16, 0, shapes=[(8, 16), (4, 8), (2, 4)], seed=4),
    "targets_in_last_image": lambda: count_case(3, 3, 10, 16, 30, shapes=[(8, 16), (4, 8), (2, 4)], images=[15], seed=6),
    "na10_nt1200": lambda: count_case(3, 10, 10, 2, 1200, shapes=[(32, 64), (16, 32), (8, 16)], seed=8, mult=2.5, scale=0.5),
    "train_step": train_step_case,
    "rect_416x736": lambda: count_case(3, 3, 10, 2, 40, shapes=[(52, 92), (26, 46), (13, 23)], seed=9, mult=0.375, scale=None),
}


# ---- the kernel and the yardstick --------------------------------------------------------------------------------------------------------
def read_workspace(ws, B, na, shapes):
    """winner (int32) and tobj (fp32) of every level and nvalid[3] from the workspace of myolo_det_loss.  The layout is that of the six lines
    after `int64_t off = 0` in csrc/detloss.cu: the winner arrays of all levels, then the tobj arrays, then nvalid."""
    raw = ws.view(torch.uint8).cpu().numpy()
    cells = [B * na * ny * nx for ny, nx in shapes]
    off, winner, tobj = 0, [], []
    for n, (ny, nx) in zip(cells, shapes):
        winner.append(raw[off:off + 4 * n].view(np.int32).reshape(B, na, ny, nx)); off += 4 * n
    for n, (ny, nx) in zip(cells, shapes):
        tobj.append(raw[off:off + 4 * n].view(np.float32).reshape(B, na, ny, nx)); off += 4 * n
    return winner, tobj, raw[off:off + 12].view(np.int32).copy()


def run_kernel(c):
    """one myolo_det_loss call with every argument explicit; gradient and workspace NaN before it"""
    from multiyolov5_b200 import _lib
    L = _lib.lib()
    nl, B, na = len(c.shapes), c.B, c.na
    p = [torch.from_numpy(q).cuda() for q in c.p]
    dp = [torch.full_like(q, float("nan")) for q in p]
    tg = torch.from_numpy(c.targets).cuda()
    ny = (C.c_int32 * nl)(*[s[0] for s in c.shapes])
    nx = (C.c_int32 * nl)(*[s[1] for s in c.shapes])
    need = int(L.myolo_det_loss_workspace_bytes(B, na, nl, ny, nx))
    ws = torch.full(((need + 3) // 4,), float("nan"), device="cuda")
    items = torch.full((4,), float("nan"), device="cuda")
    scale = None if c.scale is None else torch.full((), c.scale, device="cuda")
    eps = c.hyp["label_smoothing"]
    h = c.hyp
    vp = C.c_void_p
    _lib.check(L.myolo_det_loss((vp * nl)(*[_lib.ptr(t) for t in p]), (vp * nl)(*[_lib.ptr(t) for t in dp]), _lib.ptr(tg), tg.shape[0], B,
                                na, 5 + c.nc, nl, ny, nx, (C.c_float * (nl * na * 2))(*c.anchors.reshape(-1).tolist()),
                                (C.c_float * nl)(*balance(nl)), h["box"], h["obj"], h["cls"], h["anchor_t"], c.gr, 1.0 - 0.5 * eps, 0.5 * eps,
                                c.mult, _lib.ptr(scale), _lib.ptr(items), _lib.ptr(ws), need, _lib.stream_ptr()))
    torch.cuda.synchronize()
    winner, tobj, nvalid = read_workspace(ws, B, na, c.shapes)
    return dict(dp=[d.cpu().numpy() for d in dp], items=items.cpu().numpy(), winner=winner, tobj=tobj, nvalid=nvalid,
                p_kept=all(np.array_equal(q.cpu().numpy().view(np.int32), q0.view(np.int32)) for q, q0 in zip(p, c.p)))


def reference(c, mutant=None):
    """compute_det_loss in fp64 and the gradient of loss_items[3] * mult * scale, which is what the kernel writes"""
    p = [torch.from_numpy(q).double().requires_grad_(True) for q in c.p]
    with np.errstate(divide="ignore"):                    # zero-width targets: 1 / r = inf, as in the kernel
        loss, items, asg = restate.compute_det_loss(p, c.targets, c.anchors, c.hyp, c.nc, gr=c.gr, assignment=True, mutant=mutant)
    (loss * (c.mult * (1.0 if c.scale is None else c.scale) / c.B)).backward()
    return dict(g=[q.grad.numpy() for q in p], items=items.numpy(), nvalid=[n for n, _, _ in asg], winner=[w for _, w, _ in asg],
                tobj=[t.numpy() for _, _, t in asg])


def compare(c, out, ref):
    """(failed exact checks, worst relative error of every limit group)"""
    fails, errs = [], {}

    def group(key, ours, theirs):
        ours, theirs = np.asarray(ours, np.float64), np.asarray(theirs, np.float64)
        den = np.abs(theirs).max() if theirs.size else 0.0
        e = np.abs(ours - theirs).max() / den if den > 0 else (0.0 if not np.any(ours) else np.inf)
        errs[key] = max(errs.get(key, 0.0), float(e))

    nl = len(c.shapes)
    if not out["p_kept"]:
        fails.append("p changed")
    if list(out["nvalid"][nl:]) != [0] * (3 - nl):
        fails.append(f"nvalid beyond level {nl}: {out['nvalid']}")
    for l in range(nl):
        m = ref["winner"][l] >= 0
        dp, g = out["dp"][l], ref["g"][l]
        if out["nvalid"][l] != ref["nvalid"][l]:
            fails.append(f"level {l}: nvalid {out['nvalid'][l]} != {ref['nvalid'][l]}")
        if not np.array_equal(out["winner"][l], ref["winner"][l]):
            fails.append(f"level {l}: winner differs at {int((out['winner'][l] != ref['winner'][l]).sum())} cells")
        if np.isnan(dp).any():
            fails.append(f"level {l}: NaN left in dp")
        if np.any(dp[~m][:, :4]) or np.any(dp[~m][:, 5:]) or np.any(out["tobj"][l][~m]):
            fails.append(f"level {l}: nonzero box / class gradient or tobj off the matched cells")
        group("xy", dp[..., :2], g[..., :2])
        group("wh", dp[..., 2:4], g[..., 2:4])
        group("obj_m", dp[..., 4][m], g[..., 4][m])
        group("obj_u", dp[..., 4][~m], g[..., 4][~m])
        group("cls", dp[..., 5:], g[..., 5:])
        group("tobj", out["tobj"][l][m], ref["tobj"][l][m])
    for i in range(4):
        if ref["items"][i] == 0.0:
            if out["items"][i] != 0.0:
                fails.append(f"item {i}: {out['items'][i]} != 0")
        else:
            errs["items"] = max(errs.get("items", 0.0), abs(float(out["items"][i]) - ref["items"][i]) / abs(ref["items"][i]))
    return fails, errs


def over_limit(errs):
    return max((e / LIMITS[k] for k, e in errs.items()), default=0.0)


_RUNS = {}


def run_case(name):
    if name not in _RUNS:
        c = CASES[name]()
        _RUNS[name] = (c, run_kernel(c), reference(c))
    return _RUNS[name]


def record(name, errs):
    for k, e in errs.items():
        WORST[k] = max(WORST.get(k, 0.0), e)
    print(f"\n{name}: " + " ".join(f"{k}={e:.2e}" for k, e in errs.items()) + f"  (worst so far: {WORST})")


# ---- the tests ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_det_loss_matches_fp64(name):
    c, out, ref = run_case(name)
    fails, errs = compare(c, out, ref)
    record(name, errs)
    assert not fails, fails
    assert all(e <= LIMITS[k] for k, e in errs.items()), errs


def test_boundary_cases_decide_as_intended():
    """the boundary cases exercise what they are named for: the ratio bound rejects, one ulp inside accepts, the shared cell's winner has a
    negative CIoU after a positive one, the clamped cell's box offset is 1.0, and x % 1 == 0.5 has no neighbour"""
    c, _, ref = run_case("ratio_t4")
    # 10 targets: 4 accepted by anchor 0 at their centre cells (1 ulp inside either bound, and the two exact sides 2, 2); the bound, 1 / bound
    # and zero sides are rejected by anchor 0
    w = ref["winner"][0][0, 0]
    assert sorted({int(v) % 10 for v in w[w >= 0].ravel()}) == [4, 5, 6, 7], sorted(w[w >= 0].ravel())
    c, _, ref = run_case("shared")
    assert ref["tobj"][0][1, 0, 8, 4] == 1.0 - c.gr
    assert ref["winner"][0][1, 0, 8, 4] // (c.na * len(c.rows)) == 1                   # offset x-1
    rows = restate.build_targets_loop(c.shapes, c.targets, c.anchors, c.hyp["anchor_t"])[0]
    first = [r for r in rows if (r[0], r[1], r[2], r[3]) == (1, 0, 8, 4)]
    assert len(first) == 2 and first[0][6] // (c.na * len(c.rows)) == 0
    c, _, _ = run_case("neighbour_16x32")
    rows = restate.build_targets_loop(c.shapes, c.targets, c.anchors, c.hyp["anchor_t"])[0]
    assert any(r[3] == 31 and r[4][0] == 1.0 for r in rows)                            # x = 1.0: cell nx - 1, offset 1.0
    assert not any(r[6] // (c.na * len(c.rows)) in (1, 3) and c.targets[r[6] % len(c.rows), 2] * 32 == 16.5 for r in rows)


# every mutant of the restatement, and the cases that must catch it
MUTANT_CASES = {
    "ties": ["ciou_all", "ciou_x1", "ciou_x2", "ciou_y1", "ciou_y2"],
    "half_le": ["neighbour_16x32"],
    "gt_ge": ["neighbour_16x32"],
    "unclamped": ["neighbour_16x32"],
    "first_wins": ["shared"],
    "alpha_grad": ["ciou_disjoint"],
    "balance": ["bce_gr1.0"],
    "gr": ["shared", "bce_gr0.5"],
    "cp_cn": ["bce_gr0.5"],
}


def test_det_loss_checks_catch_wrong_references():
    """the checks discriminate: against each deliberately wrong restatement (restate.DET_LOSS_MUTANTS) every case listed for it fails an
    exact check or misses a limit by at least 10x.  The mutants: the whole gradient to the prediction's edge at min / max ties, <= in the
    0.5 rule, >= 1 instead of > 1, the box offset relative to the unclamped cell, the first candidate of a cell winning, alpha differentiated,
    the other branch of the balance lookup (the nl = 3 weights elsewhere are the same first entries, so it shows at nl = 3), gr ignored,
    cp and cn swapped."""
    assert set(MUTANT_CASES) == set(restate.DET_LOSS_MUTANTS)
    print()
    for mutant, names in MUTANT_CASES.items():
        for name in names:
            c, out, _ = run_case(name)
            fails, errs = compare(c, out, reference(c, mutant))
            over = np.inf if fails else over_limit(errs)
            print(f"mutant {mutant:<10} on {name:<16}: " + (f"exact check fails ({fails[0]})" if fails else f"{over:.0f}x its limit"))
            assert over >= 10, (mutant, name, errs)


def _wrapper_check(crit, p, targets, anchors, hyp, nc, gr, mult, scale):
    """FusedComputeLoss(model)(p, targets, mult, scale) against the fp64 restatement with the same checks as a direct call"""
    B, na = p[0].shape[:2]
    shapes = [tuple(q.shape[2:4]) for q in p]
    dp, items = crit(p, targets, mult=mult, scale=scale)
    torch.cuda.synchronize()
    winner, tobj, nvalid = read_workspace(crit._ws, B, na, shapes)
    c = SimpleNamespace(p=[q.cpu().numpy() for q in p], targets=targets.cpu().numpy(), anchors=anchors, hyp=hyp, nc=nc, gr=gr,
                        mult=mult * B, scale=None if scale is None else float(scale), B=B, shapes=shapes)
    out = dict(dp=[d.cpu().numpy() for d in dp], items=items.cpu().numpy(), winner=winner, tobj=tobj, nvalid=nvalid, p_kept=True)
    return compare(c, out, reference(c))


def test_fused_compute_loss_plumbing_on_a_model():
    """FusedComputeLoss on the s/PSP model: mult * B, the anchors of the Detect buffer, ComputeLoss's balance, and every hyp it reads (box,
    obj, cls, anchor_t, label_smoothing, gr) away from their defaults, with a device loss scale"""
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils.loss import FusedComputeLoss
    model = Model("yolov5s_city_seg.yaml")
    hyp = dict(box=0.0625, obj=0.75, cls=0.375, anchor_t=2.0, label_smoothing=0.1, fl_gamma=0.0, cls_pw=1.0, obj_pw=1.0)
    model.hyp, model.gr = hyp, 0.5
    crit = FusedComputeLoss(model)
    assert crit.supported
    B, nc = 3, 10
    gen = torch.Generator().manual_seed(3)
    p = [(torch.randn((B, 3, 128 // s, 256 // s, 5 + nc), generator=gen) * 1.5).cuda() for s in STRIDES]
    tc = count_case(3, 3, nc, B, 40, seed=12)
    fails, errs = _wrapper_check(crit, p, torch.from_numpy(tc.targets).cuda(), model.model[-1].anchors.numpy(), hyp, nc, 0.5, 0.75,
                                 torch.full((), 256.0, device="cuda"))
    record("wrapper_model", errs)
    assert not fails, fails
    assert all(e <= LIMITS[k] for k, e in errs.items()), errs


def test_fused_compute_loss_reuses_its_workspace_across_shapes():
    """one FusedComputeLoss over the calls --multi-scale and --rect make: large, small, empty, large (and the anchors changed in place in
    between, as autoanchor does), on a two-level, four-anchor, one-class Detect; every call meets the checks of a fresh instance and the
    workspace only grows"""
    from multiyolov5_b200.models.yolo import Detect
    from multiyolov5_b200.utils.loss import FusedComputeLoss
    anchors = dyadic_anchors(2, 4, 13)
    det = Detect(nc=1, anchors=anchors.reshape(2, -1).tolist(), ch=(8, 8))
    hyp = dict(box=0.05, obj=1.0, cls=0.5, anchor_t=4.0, fl_gamma=0.0)
    crit = FusedComputeLoss(SimpleNamespace(hyp=hyp, gr=1.0, model=[det]))
    assert crit.supported
    calls = [(4, (32, 64), 300, 21), (1, (8, 16), 5, 22), (2, (16, 32), 0, 23), (4, (32, 64), 300, 24)]
    sizes = []
    for k, (B, (ny, nx), nt, seed) in enumerate(calls):
        if k == 3:
            det.anchors.mul_(1.25)
        gen = torch.Generator().manual_seed(seed)
        p = [(torch.randn((B, 4, ny >> i, nx >> i, 6), generator=gen) * 1.5).cuda() for i in range(2)]
        tc = count_case(2, 4, 1, B, nt, seed=seed)
        fails, errs = _wrapper_check(crit, p, torch.from_numpy(tc.targets).cuda(), det.anchors.numpy().copy(), dict(hyp, label_smoothing=0.0),
                                     1, 1.0, 1.0, None)
        record(f"wrapper_call{k}", errs)
        assert not fails, (k, fails)
        assert all(e <= LIMITS[k_] for k_, e in errs.items()), (k, errs)
        sizes.append(crit._ws.numel())
    assert sizes == sorted(sizes) and sizes[1] == sizes[0]
