"""The reference's autoanchor (utils/autoanchor.py:23-160): check how well the Detect anchors fit the training labels and, when the best
possible recall is below 0.98, replace them with k-means anchors evolved by a genetic algorithm.

Same names, signatures, printed lines and random draws as the reference:

    check_anchor_order(m)
    check_anchors(dataset, model, thr=4.0, imgsz=640)
    kmean_anchors(dataset, n=9, img_size=640, thr=4.0, gen=1000, verbose=True) -> (n, 2) float64 anchors

`dataset` is a `utils.datasets.DeviceImageCache` (its original (h0, w0) `shapes0` and float32 `labels`) or any object with the reference
dataset's `shapes` ((n, 2) [w, h]) and `labels`.  A path (`str`) raises NotImplementedError: loading data files is not built.

What runs where.  The ratio metric, scipy's k-means and the 1000-generation evolution run on the GPU.  The evolution is one persistent
kernel (csrc/autoanchor.cu), with every generation's mutation factors drawn up front on the host from `numpy.random` in the reference's
order and count (its loop never reads the anchors or the fitness).  `kmeans(wh / s, n, iter=30)` returns what scipy.cluster.vq.kmeans
returns, bit for bit, with all restarts in one launch (csrc/kmeans.cu) from starts drawn up front as scipy draws them; scipy is not needed
at run time.  So a seeded run leaves `numpy.random` and `random` where the reference leaves them, and the augmenters that draw next see the
same streams.  The numpy filtering and whitening, `print_results`' sort and the torch writes into the Detect buffers stay on the host.

Exactness.  Each generation's fitness is the fp32 mean of per-label terms, summed exactly in fp64 (DESIGN.md section 3b), and every
comparison runs in the dtype torch uses (fp64 where the reference divides an fp32 tensor by a float64 numpy array).  Torch's own fp32
`mean` rounds its cascade sum in a way that depends on the CPU, so the reference's fitness can differ by a few ulp between two machines;
the library's is the same on every run and GPU.

Updating the model.  New anchors are written in place into `anchor_grid` and `anchors`, as the reference does.  The writes move the buffers'
version counters, so inference plans built earlier re-read their anchors before the next forward, and the fused detection loss re-reads
them on its next call.

In the reference's training loop (train.py:151, 222-225) the call sits after ModelEMA is built and before `model.half().float()`; keep
that order:

    ema = ModelEMA(model)
    if not opt.noautoanchor:
        check_anchors(cache, model=model, thr=hyp['anchor_t'], imgsz=imgsz)
    model.half().float()

With several ranks the reference computes the anchors on rank 0 and relies on DDP's buffer broadcast, which this package does not do.
Broadcast them from rank 0 after the call:

    for b in (det.anchors, det.anchor_grid):
        torch.distributed.broadcast(b, src=0)
"""
import numpy as np
import torch

from .. import _lib
from .datasets import DeviceImageCache

_STATS = np.dtype([("n_best", "<i8"), ("n_x", "<i8"), ("sum_x", "<f8"), ("sum_best", "<f8"), ("sum_x_above", "<f8")])


def colorstr(*input):
    """ANSI colours as the reference's colorstr: colorstr('blue', 'hello') or colorstr('hello') (blue, bold)"""
    *args, string = input if len(input) > 1 else ("blue", "bold", input[0])
    colors = {"black": "\033[30m", "red": "\033[31m", "green": "\033[32m", "yellow": "\033[33m", "blue": "\033[34m", "magenta": "\033[35m",
              "cyan": "\033[36m", "white": "\033[37m", "end": "\033[0m", "bold": "\033[1m", "underline": "\033[4m"}
    return "".join(colors[x] for x in args) + f"{string}" + colors["end"]


def check_anchor_order(m):
    """reverse the anchors of Detect m when their area order disagrees with the stride order"""
    a = m.anchor_grid.prod(-1).view(-1)
    da = a[-1] - a[0]
    ds = m.stride[-1] - m.stride[0]
    if da.sign() != ds.sign():
        print("Reversing anchor order")
        m.anchors[:] = m.anchors.flip(0)
        m.anchor_grid[:] = m.anchor_grid.flip(0)


def dataset_shapes_labels(dataset):
    """(shapes (n, 2) float64 [w, h], labels) of a DeviceImageCache or a reference-style dataset"""
    if isinstance(dataset, str):
        raise NotImplementedError("autoanchor: loading a dataset from a path is not built; pass a utils.datasets.DeviceImageCache")
    if isinstance(dataset, DeviceImageCache):
        return np.array([(w0, h0) for h0, w0 in dataset.shapes0], dtype=np.float64).reshape(-1, 2), dataset.labels
    if not (hasattr(dataset, "shapes") and hasattr(dataset, "labels")):
        raise TypeError("autoanchor: dataset must be a DeviceImageCache or have the reference dataset's `shapes` and `labels`")
    return np.asarray(dataset.shapes, dtype=np.float64).reshape(-1, 2), dataset.labels


def _device(t=None):
    if not torch.cuda.is_available():
        raise _lib.MyoloError("autoanchor needs a CUDA device: multiyolov5_b200 has no CPU path")
    return t.device if t is not None and t.is_cuda else torch.device("cuda", torch.cuda.current_device())


def anchor_metric(wh, k, thr):
    """the reference's ratio metric of label wh (n, 2) against anchors k (na, 2) on the device: {n_best, n_x, sum_x, sum_best,
    sum_x_above} (counts of best > thr and x > thr, fp64 sums of x, best and x > thr).  `wh` is an fp32 / fp64 CUDA tensor; `k` a numpy
    float64 array (the metric then runs in fp64, as torch promotes it) or an fp32 / fp64 tensor; thr = 1 / anchor_t."""
    dev = _device(wh)
    k = torch.from_numpy(np.ascontiguousarray(k, dtype=np.float64)) if isinstance(k, np.ndarray) else k.detach()
    k = k.to(dev).contiguous()
    wh = wh.contiguous()
    codes = {torch.float32: _lib.F32, torch.float64: _lib.F64}
    if wh.dtype not in codes or k.dtype not in codes:
        raise TypeError("anchor_metric: wh and k must be float32 or float64")
    L = _lib.lib()
    ws = torch.empty(int(L.myolo_anchor_metric_workspace_bytes()), dtype=torch.uint8, device=dev)
    out = torch.empty(_STATS.itemsize, dtype=torch.uint8, device=dev)
    _lib.check(L.myolo_anchor_metric(_lib.ptr(wh), codes[wh.dtype], int(wh.shape[0]), _lib.ptr(k), codes[k.dtype], int(k.numel() // 2),
                                     float(thr), _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()))
    r = np.frombuffer(out.cpu().numpy().tobytes(), dtype=_STATS)[0]
    return {name: r[name].item() for name in _STATS.names}


def draw_mutations(gen, sh, mp=0.9, s=0.1):
    """the reference's `gen` mutation factors (gen, *sh) float64, drawn from numpy.random exactly as its evolution loop draws them"""
    npr = np.random
    out = np.empty((gen,) + tuple(sh), dtype=np.float64)
    for g in range(gen):
        v = np.ones(sh)
        while (v == 1).all():  # mutate until a change occurs (prevent duplicates)
            v = ((npr.random(sh) < mp) * npr.random() * npr.randn(*sh) * s + 1).clip(0.3, 3.0)
        out[g] = v
    return out


def evolve(wh, k0, v, thr):
    """the evolution on the device (myolo_anchor_evolve): wh (n, 2) fp32 CUDA labels, k0 (na, 2) float64 start anchors, v (gen, na, 2)
    float64 mutation factors, thr = 1 / anchor_t.  Returns (k float64 numpy, fitness of k0, final fitness, fg per generation fp32 numpy,
    accepted count)."""
    dev = _device(wh)
    wh = wh.to(dtype=torch.float32).contiguous()
    na = int(np.asarray(k0).size // 2)
    gen = int(v.shape[0])
    k0_d = torch.from_numpy(np.ascontiguousarray(k0, dtype=np.float64)).to(dev)
    v_d = torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(dev) if gen else None
    L = _lib.lib()
    n = int(wh.shape[0])
    need = int(L.myolo_anchor_evolve_workspace_bytes(n))
    if need < 0:
        raise _lib.MyoloError(f"myolo_anchor_evolve_workspace_bytes: {L.myolo_last_error().decode(errors='replace')}")
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    k_out = torch.empty(na * 2, dtype=torch.float64, device=dev)
    f_out = torch.empty(2, dtype=torch.float32, device=dev)
    fg = torch.empty(max(gen, 1), dtype=torch.float32, device=dev)
    acc = torch.empty(1, dtype=torch.int32, device=dev)
    _lib.check(L.myolo_anchor_evolve(_lib.ptr(wh), n, _lib.ptr(k0_d), na, _lib.ptr(v_d), gen, float(thr), _lib.ptr(k_out), _lib.ptr(f_out),
                                     _lib.ptr(fg), _lib.ptr(acc), _lib.ptr(ws), need, _lib.stream_ptr()))
    f = f_out.cpu().numpy()
    return (k_out.cpu().numpy().reshape(na, 2), np.float32(f[0]), np.float32(f[1]), fg.cpu().numpy()[:gen].copy(), int(acc.item()))


KMEANS_ITER_CAP = 1000      # scipy has no cap; restarts on label sets take 9 to about 130 Lloyd iterations


def kmeans_restarts(obs, idx, thresh=1e-5, max_iter=KMEANS_ITER_CAP):
    """every restart of scipy's k-means from the start rows idx (restarts, k) int, in one launch (myolo_kmeans) and one read-back:
    ([book (k'_r, d) float64 per restart], distortions (restarts,) float64, Lloyd iterations (restarts,) int32, index of scipy's winner).
    obs: (n, d) float64 numpy.  A restart still moving after max_iter iterations raises MyoloError."""
    n, d = obs.shape
    R, k = idx.shape
    dev = _device()
    L = _lib.lib()
    need = int(L.myolo_kmeans_workspace_bytes(n, k, R))
    if need < 0:
        raise _lib.MyoloError(f"kmeans: n = {n}, k = {k}, {R} restarts: no workspace size")
    obs_d = torch.from_numpy(np.ascontiguousarray(obs, dtype=np.float64)).to(dev)
    idx_d = torch.from_numpy(np.ascontiguousarray(idx, dtype=np.int64)).to(dev)
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    # one output buffer: books (R, k, d) f64 | dists (R) f64 | book_k (R) i32 | iters (R) i32 | best i32 | status i32
    nb = R * k * d * 8
    o_dist, o_bk, o_it, o_best = nb, nb + 8 * R, nb + 12 * R, nb + 16 * R
    out = torch.zeros(o_best + 8, dtype=torch.uint8, device=dev)
    p = out.data_ptr()
    _lib.check(L.myolo_kmeans(_lib.ptr(obs_d), n, d, _lib.ptr(idx_d), k, R, float(thresh), int(max_iter), p, p + o_bk, p + o_dist, p + o_it,
                              p + o_best, p + o_best + 4, _lib.ptr(ws), need, _lib.stream_ptr()))
    buf = out.cpu().numpy()
    books = buf[:nb].view(np.float64).reshape(R, k, d)
    book_k = buf[o_bk:o_it].view(np.int32)
    best, status = (int(v) for v in buf[o_best:].view(np.int32))
    if status & _lib.KMEANS_MAX_ITER:
        raise _lib.MyoloError(f"kmeans: a restart was still moving after {max_iter} Lloyd iterations")
    if status:
        raise _lib.MyoloError(f"kmeans: start indices outside [0, {n})")
    dists, iters = buf[o_dist:o_bk].view(np.float64).copy(), buf[o_it:o_best].view(np.int32).copy()
    return [books[r, :book_k[r]].copy() for r in range(R)], dists, iters, best


def kmeans(obs, k, iter=20, thresh=1e-5):
    """scipy.cluster.vq.kmeans(obs, k, iter, thresh) for an int k on the device, bit for bit: (code book (k', 2) float64, mean distance
    float64).  obs: (n, 2) float64 numpy, e.g. kmean_anchors' whitened `wh / s`.  Every restart's start is drawn up front from numpy's
    global state exactly as scipy draws them (`choice(n, k, replace=False)` per restart), so `numpy.random` ends where scipy leaves it and
    n < k raises numpy's ValueError from that call, as in scipy.  The checks before the draws raise scipy's ValueErrors."""
    obs = np.asarray(obs)
    if not np.isfinite(obs).all():
        raise ValueError("array must not contain infs or NaNs")
    if iter < 1:
        raise ValueError(f"iter must be at least 1, got {iter}")
    if k < 1:
        raise ValueError(f"Asked for {k} clusters.")
    if obs.dtype != np.float64 or obs.ndim != 2:
        raise TypeError("kmeans: obs must be a (n, d) float64 array")
    idx = np.stack([np.random.choice(obs.shape[0], k, replace=False) for _ in range(iter)])
    books, dists, _, best = kmeans_restarts(obs, idx, thresh)
    if best < 0:
        raise ValueError("kmeans: no restart has a finite distortion")
    return books[best], np.float64(dists[best])


def _mean32(count, n):
    """torch's fp32 mean of `n` values that sum to the integer `count` (exact in fp32 below 2^24): the sum divided by n in fp32"""
    return np.float32(np.float32(count) / np.float32(n))


def check_anchors(dataset, model, thr=4.0, imgsz=640):
    """check the anchors' fit to the labels (best possible recall), and recompute them when it is below 0.98"""
    prefix = colorstr("autoanchor: ")
    print(f"\n{prefix}Analyzing anchors... ", end="")
    m = model.module.model[-1] if hasattr(model, "module") else model.model[-1]  # Detect()
    shapes, labels = dataset_shapes_labels(dataset)
    dev = _device(m.anchors)
    shapes = imgsz * shapes / shapes.max(1, keepdims=True)
    scale = np.random.uniform(0.9, 1.1, size=(shapes.shape[0], 1))  # augment scale
    wh = torch.tensor(np.concatenate([l[:, 3:5] * s for s, l in zip(shapes * scale, labels)])).float().to(dev)  # wh
    n = int(wh.shape[0])

    def metric(k):  # (bpr, aat) as torch forms them: fp32 means of the counts
        st = anchor_metric(wh, k, 1. / thr)
        return _mean32(st["n_best"], n), _mean32(st["n_x"], n)

    anchors = m.anchor_grid.detach().reshape(-1, 2).float()  # current anchors
    bpr, aat = metric(anchors)
    print(f"anchors/target = {float(aat):.2f}, Best Possible Recall (BPR) = {float(bpr):.4f}", end="")
    if bpr < 0.98:  # threshold to recompute
        print(". Attempting to improve anchors, please wait...")
        na = m.anchor_grid.numel() // 2  # number of anchors
        try:
            anchors = kmean_anchors(dataset, n=na, img_size=imgsz, thr=thr, gen=1000, verbose=False)
        except _lib.MyoloError:
            raise  # a device failure is not a reason to keep the old anchors quietly
        except Exception as e:
            print(f"{prefix}ERROR: {e}")
        new_bpr = metric(anchors)[0]
        if new_bpr > bpr:  # replace anchors
            anchors = torch.tensor(anchors, device=m.anchors.device).type_as(m.anchors)
            m.anchor_grid[:] = anchors.clone().view_as(m.anchor_grid)  # for inference
            m.anchors[:] = anchors.clone().view_as(m.anchors) / m.stride.to(m.anchors.device).view(-1, 1, 1)  # loss
            check_anchor_order(m)
            print(f"{prefix}New anchors saved to model. Update model *.yaml to use these anchors in the future.")
        else:
            print(f"{prefix}Original anchors better than new anchors. Proceeding with original anchors.")
    print("")  # newline


def kmean_anchors(dataset, n=9, img_size=640, thr=4.0, gen=1000, verbose=True):
    """k-means anchors of the dataset's labels, evolved by the reference's genetic algorithm on the device.  thr: hyp['anchor_t'].
    Returns the (n, 2) float64 anchors, sorted small to large."""
    thr = 1. / thr
    prefix = colorstr("autoanchor: ")
    shapes, labels = dataset_shapes_labels(dataset)
    dev = _device()

    def print_results(k):
        k = k[np.argsort(k.prod(1))]  # sort small to large
        st = anchor_metric(wh0, k, thr)
        n_wh = int(wh0.shape[0])
        bpr, aat = _mean32(st["n_best"], n_wh), np.float32(_mean32(st["n_x"], n_wh * n) * np.float32(n))
        x_mean, best_mean = st["sum_x"] / (n_wh * n), st["sum_best"] / n_wh
        past = st["sum_x_above"] / st["n_x"] if st["n_x"] else float("nan")
        print(f"{prefix}thr={thr:.2f}: {float(bpr):.4f} best possible recall, {float(aat):.2f} anchors past thr")
        print(f"{prefix}n={n}, img_size={img_size}, metric_all={x_mean:.3f}/{best_mean:.3f}-mean/best, "
              f"past_thr={past:.3f}-mean: ", end="")
        for i, x in enumerate(k):
            print("%i,%i" % (round(x[0]), round(x[1])), end=",  " if i < len(k) - 1 else "\n")  # use in *.cfg
        return k

    # Get label wh
    shapes = img_size * shapes / shapes.max(1, keepdims=True)
    wh0 = np.concatenate([l[:, 3:5] * s for s, l in zip(shapes, labels)])  # wh

    # Filter
    i = (wh0 < 3.0).any(1).sum()
    if i:
        print(f"{prefix}WARNING: Extremely small objects found. {i} of {len(wh0)} labels are < 3 pixels in size.")
    wh = wh0[(wh0 >= 2.0).any(1)]  # filter > 2 pixels

    # Kmeans calculation
    print(f"{prefix}Running kmeans for {n} anchors on {len(wh)} points...")
    s = wh.std(0)  # sigmas for whitening
    k, dist = kmeans(wh / s, n, iter=30)  # points, mean distance
    if len(k) != n:
        print(f"{prefix}ERROR: scipy.cluster.vq.kmeans requested {n} points but returned only {len(k)}")
        raise AssertionError(None)
    k *= s
    wh = torch.tensor(wh, dtype=torch.float32).to(dev)  # filtered
    wh0 = torch.tensor(wh0, dtype=torch.float32).to(dev)  # unfiltered
    k = print_results(k)

    # Evolve: every generation's factors drawn first, then all generations in one kernel
    v = draw_mutations(gen, k.shape)
    k_dev, f0, _, fg, _ = evolve(wh, k, v, thr)
    if verbose:  # the accepted generations, replayed on the host (the same fp64 products) for the reference's prints
        f = f0
        for g in range(gen):
            if fg[g] > f:
                f, k = fg[g], (k.copy() * v[g]).clip(min=2.0)
                print_results(k)
        assert np.array_equal(k, k_dev)
    return print_results(k_dev)
