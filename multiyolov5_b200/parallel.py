"""Multi-GPU plumbing of the path (SURVEY.md section 8e).  Inference shards by image: one process per GPU, independent
replicas, NO data-path collective; torch.distributed (NCCL on GPUs, gloo in CPU tests) is used only for the barrier and the
max-over-ranks time so that throughput is reported for the whole job.  Training (row a13) has ONE real exchange per optimiser step:
the sum of the flat gradient buffer over ranks (the reference wraps the model in DistributedDataParallel, train.py:243-245)."""
import torch
import torch.distributed as dist


def shard_range(n_items: int, world: int, rank: int):
    """contiguous, balanced shard [lo, hi) of a global batch (sizes differ by at most one)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def aggregate_throughput(images_local: int, ms_local: float, device=None) -> float:
    """whole-job images/s = sum of images over ranks / max of elapsed time over ranks."""
    t = torch.tensor([ms_local], dtype=torch.float64, device=device)
    n = torch.tensor([float(images_local)], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(n, op=dist.ReduceOp.SUM)
    return float(n.item() / (t.item() * 1e-3))


LAST_ALLREDUCE_PATH = "none"      # which route the last allreduce_flat_grads took (reported by bench.py's train record)


def nccl_comm_ptr(group=None, device=None):
    """the raw ncclComm_t of the process group's NCCL backend (what the C ABI's myolo_allreduce_grads takes), or None (gloo / no comm yet)"""
    try:
        pg = group if group is not None else dist.distributed_c10d._get_default_group()
        be = pg._get_backend(device or torch.device("cuda", torch.cuda.current_device()))
        ptr = int(be._comm_ptr())
        return ptr or None
    except Exception:
        return None


def allreduce_flat_grads(flat_grad: torch.Tensor, group=None, stream=None) -> int:
    """ONE collective per optimiser step over the contiguous gradient buffer (31 MB fp32 for s/PSP): SUM over ranks, in place.
    Averaging (DDP semantics) is folded into the optimiser's unscale factor, 1 / (loss scale x world size), so no extra pass over the
    buffer is needed.  On the NCCL backend the call goes through the library's own entry point (`myolo_allreduce_grads`: ncclAllReduce on
    the communicator torch created, enqueued on `stream` or the current stream); gloo (CPU tests) uses torch.distributed.
    Returns the world size used."""
    if not (dist.is_available() and dist.is_initialized()):
        return 1
    world = dist.get_world_size(group)
    if world > 1:
        comm = nccl_comm_ptr(group, flat_grad.device) if flat_grad.is_cuda and dist.get_backend(group) == "nccl" else None
        global LAST_ALLREDUCE_PATH
        if comm is not None:
            from . import _lib
            sp = stream.cuda_stream if stream is not None else _lib.stream_ptr()
            _lib.check(_lib.lib().myolo_allreduce_grads(_lib.ptr(flat_grad), flat_grad.numel(), comm, sp))
            LAST_ALLREDUCE_PATH = "myolo_allreduce_grads (ncclAllReduce on torch's communicator, issued by libmyolo_sm90a)"
        else:
            dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
            LAST_ALLREDUCE_PATH = f"torch.distributed.all_reduce ({dist.get_backend(group)})"
    return world
