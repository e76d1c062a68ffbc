"""TEST INFRASTRUCTURE - generates tests/golden/optim_cases.pt by running the UNMODIFIED reference's `train.train()` (train.py:44-542) on the
CPU for one short epoch, once with SGD and once with --adam, at yolov5s_city_seg.yaml over a tiny synthetic det + seg tree:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_optim.py

The run is observed, not edited: `torch.optim.Optimizer.add_param_group` is wrapped to keep the optimizer the run builds, `Model.__init__` to
keep the model instance, and `strip_optimizer` (which empties ckpt['optimizer'] after the last epoch, train.py:527-532) and the plotting
helpers (matplotlib / seaborn are import shims here, oracle/ref_shims.py) are replaced by no-ops in train.py's namespace.  `wandb` is made
unimportable, so the reference's logger runs without W&B as it does where wandb is not installed.  train.py's ComputeLoss is the
reference's utils/loss.py with the one in-memory fix of oracle/make_golden.py (its clamp_ bounds, which torch >= 1.12 rejects).

The full optimizer state of s/PSP is 31 MB (SGD) / 62 MB (Adam) of fp32, too large for a fixture.  Per run the file holds what last.pt's
ckpt['optimizer'] says about the mapping, exactly: its param_groups (every key and value, Python / numpy types as written), the
parameter names of each group in index order (from the run's own Model), each state entry's keys, shapes and dtypes, Adam's step values,
the state tensors of pg0 (BatchNorm weights) and pg2 (biases) in full, and a SHA-256 of every pg1 state tensor's bytes; plus the
scaled hyp the run trained with.
"""
import argparse
import copy
import hashlib
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402
from oracle.make_golden import load_reference_loss  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
IMGSZ, BATCH = 64, 4


def write_data(root):
    """det images/labels (oracle/make_golden_rect.py sources), a Cityscapes train + val tree (oracle/make_golden_seg.py sources), yamls"""
    import shutil
    import yaml
    from oracle import make_golden_rect, make_golden_seg
    from oracle.make_golden_val_batches import write_tree as write_det
    imgs, labels = make_golden_rect.sources()
    for d in ("det", "det_val"):      # two trees: the loader caches labels next to them and reads a cache back with torch.load's default
        write_det(os.path.join(root, d), imgs, [np.asarray(lb, np.float32) for lb in labels])   # weights_only, which rejects it
    simgs, smasks = make_golden_seg.sources()
    same = [k for k, im in enumerate(simgs) if im.shape == simgs[0].shape]     # the val loader stacks whole frames: one frame shape
    simgs, smasks = [simgs[k] for k in same] * 2, [smasks[k] for k in same] * 2
    city = make_golden_seg.write_tree(os.path.join(root, "seg"), simgs, smasks)["citys"]
    for sub in ("leftImg8bit", "gtFine"):
        shutil.copytree(os.path.join(city, sub, "train"), os.path.join(city, sub, "val"))
    data = dict(train=os.path.join(root, "det", "images"), val=os.path.join(root, "det_val", "images"), segtrain=city, segval=city, nc=10,
                names=[f"c{k}" for k in range(10)])
    with open(os.path.join(root, "data.yaml"), "w") as f:
        yaml.safe_dump(data, f)
    return os.path.join(root, "data.yaml")


def run(adam, data, root):
    import argparse as ap
    import torch
    import yaml
    import train as ref_train                                     # the reference's train.py (sys.path set by import_reference)
    kept = {}
    orig_add = torch.optim.Optimizer.add_param_group

    def add_param_group(self, group):
        kept["opt"] = self
        return orig_add(self, group)

    orig_init = ref_train.Model.__init__

    def model_init(self, *a, **k):
        orig_init(self, *a, **k)
        kept["model"] = self

    torch.optim.Optimizer.add_param_group = add_param_group
    ref_train.Model.__init__ = model_init
    saved = {k: getattr(ref_train, k) for k in ("ComputeLoss", "strip_optimizer", "plot_labels", "plot_images", "plot_results")}
    ref_train.ComputeLoss = load_reference_loss().ComputeLoss
    for k in ("strip_optimizer", "plot_labels", "plot_images", "plot_results"):
        setattr(ref_train, k, lambda *a, **kw: None)
    try:
        with open(os.path.join(ref_shims.REF_ROOT, "data", "hyp.scratch.yaml")) as f:
            hyp = yaml.safe_load(f)
        name = "adam" if adam else "sgd"
        opt = ap.Namespace(weights="", cfg=os.path.join(ref_shims.REF_ROOT, "models", "yolov5s_city_seg.yaml"), data=data, hyp="",
                           epochs=1, batch_size=BATCH, total_batch_size=BATCH, img_size=[IMGSZ, IMGSZ], rect=False, resume=False,
                           nosave=False, notest=True, noautoanchor=True, evolve=False, bucket="", cache_images=False, image_weights=False,
                           device="cpu", multi_scale=False, single_cls=False, adam=adam, sync_bn=False, local_rank=-1, workers=0,
                           project=root, entity=None, name=name, exist_ok=True, quad=False, linear_lr=False, label_smoothing=0.0,
                           upload_dataset=False, bbox_interval=-1, save_period=-1, artifact_alias="latest", world_size=1, global_rank=-1,
                           save_dir=os.path.join(root, name))
        ref_train.train(hyp, opt, torch.device("cpu"), None)
        ckpt = torch.load(os.path.join(root, name, "weights", "last.pt"), map_location="cpu", weights_only=False)
    finally:
        torch.optim.Optimizer.add_param_group = orig_add
        ref_train.Model.__init__ = orig_init
        for k, v in saved.items():
            setattr(ref_train, k, v)
    sd = ckpt["optimizer"]
    names = {id(p): n for n, p in kept["model"].named_parameters()}
    groups = [[names[id(p)] for p in g["params"]] for g in kept["opt"].param_groups]
    assert [len(g) for g in groups] == [len(g["params"]) for g in sd["param_groups"]]
    pg1 = set(sd["param_groups"][1]["params"])
    state = {}
    for i, st in sd["state"].items():
        e = {}
        for k, t in st.items():
            meta = dict(shape=tuple(t.shape), dtype=str(t.dtype), device=t.device.type)
            if k == "step":
                meta["value"] = t.clone()
            elif i in pg1:
                meta["sha256"] = hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()
            else:
                meta["value"] = t.clone()
            e[k] = meta
        state[i] = e
    return dict(param_groups=copy.deepcopy(sd["param_groups"]), names=groups, state=state, hyp=dict(hyp))


def main():
    argp = argparse.ArgumentParser()
    argp.add_argument("--out", default=os.path.join(GOLD, "optim_cases.pt"))
    args = argp.parse_args()
    import torch
    np.int = int                                   # removed in numpy 1.24; the reference's loaders use it
    sys.modules["wandb"] = None                    # the reference's W&B logger then takes its `wandb = None` path (no login, no network)
    ref_shims.import_reference()
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(ref_shims.REF_ROOT)               # the reference resolves its model / hyp yamls relative to its root
        try:
            for adam in (False, True):
                name = "adam" if adam else "sgd"
                os.makedirs(os.path.join(tmp, name + "_data"))
                out[name] = run(adam, write_data(os.path.join(tmp, name + "_data")), tmp)
        finally:
            os.chdir(cwd)
    torch.save(out, args.out)
    print("wrote", args.out, os.path.getsize(args.out), "bytes")


if __name__ == "__main__":
    main()
