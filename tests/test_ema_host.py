"""CPU: the host side of the device ModelEMA (utils.torch_utils): which state_dict entries the work table averages and in what order,
how the table cuts them into chunks, and the decay it hands the kernel.  The yardstick is tests/golden/ema_cases.pt, written by
oracle/make_golden_ema.py from the unmodified reference's ModelEMA and Model."""
import copy
import os

import pytest
import torch

from oracle import make_golden_ema as G

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ema_cases.pt")


@pytest.fixture(scope="module")
def cases():
    return torch.load(GOLD, weights_only=False)


def model_of(yml="yolov5s_city_seg.yaml"):
    from multiyolov5_b200.models.yolo import Model
    torch.manual_seed(0)
    return Model(yml)


def test_table_entries_are_the_references_averaged_keys(cases):
    """this Model's EMA averages exactly the keys the reference's ModelEMA averages, in its order: 377 for s/PSP (the 229 parameters, the
    146 BN running statistics and both anchor buffers), no num_batches_tracked"""
    from multiyolov5_b200.utils.torch_utils import ModelEMA, ema_entries
    model = model_of(cases["cfg"])
    ema = ModelEMA(model)
    entries = ema_entries(ema.ema, model)
    keys = [k for k, _, _ in entries]
    assert keys == cases["keys"] and len(keys) == 377
    assert [str(v.dtype) for _, v, _ in entries] == cases["dtypes"]
    assert sum(k.endswith(("running_mean", "running_var")) for k in keys) == 146
    assert sum(1 for _ in model.parameters()) == 229 and {"model.25.anchors", "model.25.anchor_grid"} <= set(keys)
    assert not any(k.endswith("num_batches_tracked") for k in keys)
    for _, v, s in entries:                                   # EMA side: the EMA's own tensors; source side: the model's
        assert v.data_ptr() != s.data_ptr()
    ema.ema.half()
    assert [str(v.dtype) for _, v, _ in ema_entries(ema.ema, model)] == ["torch.float16"] * 377


def test_table_refuses_what_the_kernel_cannot_average():
    """ValueError before any launch: a source that is not fp32, a shape mismatch, an entry missing from the model"""
    from multiyolov5_b200.utils.torch_utils import ema_entries
    model = model_of()
    ema = copy.deepcopy(model)
    with pytest.raises(ValueError, match="fp32"):
        ema_entries(ema, copy.deepcopy(model).half())
    other = copy.deepcopy(model)
    other.model[0].conv.conv.weight = torch.nn.Parameter(torch.zeros(3, 3, 1, 1))
    with pytest.raises(ValueError, match="shape"):
        ema_entries(ema, other)
    with pytest.raises(ValueError, match="counterpart"):
        ema_entries(ema, torch.nn.Linear(1, 1))


@pytest.mark.parametrize("chunk", [8, 8192])
def test_chunks_cover_every_element_once(chunk):
    """fake addresses: 1-element segments, every n % 4, sizes around the chunk size, fp32 and fp16 EMAs, unaligned and aligned bases.
    Every element of every segment is in exactly one chunk, paired with its own source element; no chunk is longer than `chunk`; every
    chunk starts a multiple of 4 elements into its segment, so it is as aligned as the segment's base."""
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils.torch_utils import ema_chunks
    sizes = [1, 2, 3, 4, 5, 6, 7, chunk - 1, chunk, chunk + 1, chunk + 3, 3 * chunk + 2, 0, 1]
    segs, base = [], 1 << 20
    for i, n in enumerate(sizes):
        dt = _lib.F16 if i % 3 == 1 else _lib.F32
        es = 2 if dt == _lib.F16 else 4
        ema, src = base + (i % 2) * es, base + (1 << 28) + (i % 5) * 4          # odd segments start off a 16-byte boundary
        segs.append((ema, src, n, dt))
        base += 16 * (n + 64)
    chunks = ema_chunks(segs, chunk=chunk)
    assert all(1 <= n <= chunk for _, _, n, _ in chunks)
    for ema, src, n, dt in segs:
        es = 2 if dt == _lib.F16 else 4
        mine = [c for c in chunks if ema <= c[0] < ema + max(n, 1) * es]
        assert all(c[3] == dt for c in mine)
        covered = []
        for e, s, k, _ in mine:
            assert (e - ema) % (4 * es) == 0                   # a multiple of 4 elements in: the segment's alignment is kept
            assert (s - src) // 4 == (e - ema) // es and (s - src) % 4 == 0
            covered += range((e - ema) // es, (e - ema) // es + k)
        assert sorted(covered) == list(range(n)), (n, dt)
    assert sum(n for _, _, n, _ in chunks) == sum(sizes)


def test_host_decay_equals_the_references(cases):
    """ModelEMA.decay over the fixture's sequence of update counts (jumps and resume included) gives the reference's d, as doubles"""
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    ema = ModelEMA(torch.nn.Linear(1, 1))
    updates, ds = 0, []
    for step in G.SEQUENCE:
        if step[0] == "update":
            for _ in range(step[1]):
                updates += 1
                ds.append(ema.decay(updates))
        elif step[0] == "jump":
            updates = step[1]
    assert len(ds) == len(cases["d"]) == G.n_updates() and updates == cases["updates"]
    assert [float(x) for x in cases["d"]] == ds
