"""TEST INFRASTRUCTURE - the schedule of reference train.py restated over torch's real optimizers and LambdaLR, for tests to compare
multiyolov5_b200.train.LRSchedule against: the optimizer and its three groups (:114-137), the scheduler (:143-147), resume (:152-177),
the warm-up length and the scheduler's start (:260, :264), the warm-up statements of each iteration (:335-352), the step condition (:396)
and the scheduler's step at the epoch end (:428).  No model and no data: three one-element parameters stand for the three groups, and the
records are what the reference's statements leave in `optimizer.param_groups` at each iteration.
"""
import copy
import math
import warnings

import numpy as np
import torch


def cosine_ramp(y1, y2, steps):
    """reference utils/general.py one_cycle, written out here so that the oracle does not lean on the code under test"""
    return lambda x: ((1 - math.cos(x * math.pi / steps)) / 2) * (y2 - y1) + y1


def run(hyp, epochs, nb, total_batch_size, linear_lr=False, adam=False, start_epoch=0, optimizer_state=None, skip=(),
        on_epoch_end=None, nbs=64, warmup_min=800):
    """records [(epoch, i, ni, [lr0, lr1, lr2], momentum or None, accumulate, steps)] of every iteration that trains; `skip`: the
    (epoch, i) of batches the loop skips for holding one image.  optimizer_state: the checkpoint's ckpt['optimizer'] of a resumed run
    (start_epoch = its epoch + 1).  on_epoch_end(epoch, optimizer.state_dict()) after each scheduler step, where the checkpoint is taken."""
    hyp = dict(hyp)
    accumulate = max(round(nbs / total_batch_size), 1)
    hyp["weight_decay"] *= total_batch_size * accumulate / nbs
    p = [torch.nn.Parameter(torch.zeros(1)) for _ in range(3)]
    if adam:
        opt = torch.optim.Adam([p[0]], lr=hyp["lr0"], betas=(hyp["momentum"], 0.999))
    else:
        opt = torch.optim.SGD([p[0]], lr=hyp["lr0"], momentum=hyp["momentum"], nesterov=True)
    opt.add_param_group({"params": [p[1]], "weight_decay": hyp["weight_decay"]})
    opt.add_param_group({"params": [p[2]]})
    run_epochs = {"n": epochs}                   # the reference's linear lambda reads train()'s `epochs` when it is called
    if linear_lr:
        lf = lambda x: (1 - x / (run_epochs["n"] - 1)) * (1.0 - hyp["lrf"]) + hyp["lrf"]     # noqa: E731
    else:
        lf = cosine_ramp(1, hyp["lrf"], epochs)
    scheduler = torch.optim.lr_scheduler.LambdaLR(opt, lr_lambda=lf)
    if optimizer_state is not None:
        opt.load_state_dict(copy.deepcopy(optimizer_state))
        if epochs < start_epoch:
            epochs += start_epoch - 1
            run_epochs["n"] = epochs
    nw = max(round(hyp["warmup_epochs"] * nb), warmup_min)
    scheduler.last_epoch = start_epoch - 1
    skip = set(skip)
    out = []
    for epoch in range(start_epoch, epochs):
        for i in range(nb):
            if (epoch, i) in skip:
                continue
            ni = i + nb * epoch
            if ni <= nw:
                xi = [0, nw]
                accumulate = max(1, np.interp(ni, xi, [1, math.floor(nbs / total_batch_size)]).round())
                for j, g in enumerate(opt.param_groups):
                    start = hyp["warmup_bias_lr"] if j == 2 else 0.0
                    g["lr"] = np.interp(ni, xi, [start, g["initial_lr"] * lf(epoch)])
                    if "momentum" in g:
                        g["momentum"] = np.interp(ni, xi, [hyp["warmup_momentum"], hyp["momentum"]])
            g0 = opt.param_groups[0]
            out.append((epoch, i, ni, [g["lr"] for g in opt.param_groups], g0.get("momentum"), accumulate, ni % accumulate == 0))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")      # "lr_scheduler.step() before optimizer.step()": nothing is optimised here
            scheduler.step()
        if on_epoch_end is not None:
            on_epoch_end(epoch, copy.deepcopy(opt.state_dict()))
    return out
