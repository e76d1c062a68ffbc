"""fp64 restatement of torch.nn.SyncBatchNorm in training mode (torch/nn/modules/_functions.py SyncBatchNorm.forward / backward) over
per-rank inputs, the semantics of the reference's --sync-bn (train.py:190-193) that the train plans' synchronised BatchNorm implements.

Forward: every rank r has n_r = B_r*H*W values per channel, its mean and biased variance; the ranks gather (n_r, mean_r, var_r), the
global mean and biased variance over N = sum n_r normalise each rank's batch, and the running statistics take the global mean and the
unbiased variance var * N / (N - 1).  Backward: each rank reduces sum dy and sum dy * (x - mean); both are summed over ranks; dx uses the
global sums and 1 / N, while d weight / d bias stay per rank (the data-parallel gradient all-reduce sums them)."""
import torch


def sync_bn_forward(xs, weight, bias, running_mean, running_var, momentum=0.03, eps=1e-3):
    """xs: list of per-rank (B_r, C, H, W) tensors.  Returns (ys, ctx, new_running_mean, new_running_var), all fp64."""
    xs = [x.double() for x in xs]
    counts = [x.numel() // x.shape[1] for x in xs]
    means = [x.mean((0, 2, 3)) for x in xs]
    vars_ = [x.var((0, 2, 3), unbiased=False) for x in xs]
    n = sum(counts)                                                         # all-gather of the records, then the combine
    mean = sum(c * m for c, m in zip(counts, means)) / n
    var = sum(c * (v + (m - mean) ** 2) for c, m, v in zip(counts, means, vars_)) / n
    invstd = 1.0 / torch.sqrt(var + eps)
    w, b = weight.double(), bias.double()
    ys = [(x - mean[None, :, None, None]) * (invstd * w)[None, :, None, None] + b[None, :, None, None] for x in xs]
    rm = (1 - momentum) * running_mean.double() + momentum * mean
    rv = (1 - momentum) * running_var.double() + momentum * var * n / (n - 1)
    return ys, (xs, mean, invstd, w, n), rm, rv


def sync_bn_backward(dys, ctx):
    """dys: per-rank gradients of the outputs.  Returns (dxs, dweights, dbiases), one per rank (fp64)."""
    xs, mean, invstd, w, n = ctx
    dys = [d.double() for d in dys]
    xmu = [x - mean[None, :, None, None] for x in xs]
    sum_dy = [d.sum((0, 2, 3)) for d in dys]                               # per rank
    sum_dy_xmu = [(d * xm).sum((0, 2, 3)) for d, xm in zip(dys, xmu)]
    g_dy, g_dy_xmu = sum(sum_dy), sum(sum_dy_xmu)                          # the all-reduce
    dxs = [(w * invstd)[None, :, None, None] * (d - (g_dy / n)[None, :, None, None]
                                                - xm * (invstd ** 2 * g_dy_xmu / n)[None, :, None, None])
           for d, xm in zip(dys, xmu)]
    return dxs, [s * invstd for s in sum_dy_xmu], sum_dy
