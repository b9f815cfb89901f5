"""Ranks of a command under torchrun (train, pretrain; dynamic_train keeps its own copy of this pattern).

    ranks()                          (rank, world, local) from RANK / WORLD_SIZE / LOCAL_RANK; (0, 1, 0) when they are absent
    check_divisible(p, world, ...)   the global sizes that are split over the ranks, refused (p.error) when one is not a multiple of world
    process_group(world, local, backend)
                                     the process group of the run: none at world 1 (today's single-GPU path, untouched); otherwise
                                     set_device, init_process_group with a timeout unless a group exists, destroy_process_group always

Backends: "nccl" puts one rank on each GPU; "gloo" also lets several ranks share a GPU (rank r on device local % device_count), so a
two-rank run fits on one GPU.  The timeout bounds every collective: when one rank dies, the others fail their next collective within it
and exit instead of waiting forever."""
import contextlib
import datetime
import os

BACKENDS = ("nccl", "gloo")
TIMEOUT_S = 600


def ranks():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def check_divisible(p, world, **sizes):
    """p.error naming the first --flag whose global size is not a multiple of the number of ranks."""
    for k, v in sizes.items():
        if int(v) % world != 0:
            p.error("--%s %d must be divisible by the %d ranks (WORLD_SIZE): every rank takes an equal share" % (k, int(v), world))


def device_of(local, backend):
    """The CUDA device index of a rank: its LOCAL_RANK under NCCL, LOCAL_RANK modulo the visible devices under gloo."""
    import torch
    return local % torch.cuda.device_count() if backend == "gloo" else local


@contextlib.contextmanager
def process_group(world, local, backend="nccl", timeout_s=TIMEOUT_S):
    """Yields the rank's CUDA device index (0 at world 1, where nothing is set up)."""
    if world == 1:
        yield 0
        return
    import torch
    import torch.distributed as dist
    dev = device_of(local, backend)
    torch.cuda.set_device(dev)
    own = not dist.is_initialized()
    if own:
        dist.init_process_group(backend, timeout=datetime.timedelta(seconds=timeout_s),
                                device_id=torch.device("cuda", dev) if backend == "nccl" else None)
    try:
        yield dev
    finally:
        if own:
            dist.destroy_process_group()


def all_equal(t):
    """True on every rank when the flat tensor t is bit-identical on every rank (one all-gather)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size()
    t = t.contiguous().reshape(-1).view(torch.uint8)           # compared as bytes: NaN payloads too
    out = torch.empty(world * t.numel(), dtype=t.dtype, device=t.device)      # gloo wants the output flat, as the input
    dist.all_gather_into_tensor(out, t)
    out = out.view(world, -1)
    return all(torch.equal(out[0], out[r]) for r in range(1, world))
