"""The model-independent layer of the sequence-parallel forwards (hyi2v_sp.py, wan_sp.py): group and rank,
the rank slices of a sequence and their all-gather, the degree checks (each names the model its caller
passes), the fused-forward check on the blocks, and the Ulysses exchange every rank agrees on."""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

from . import ulysses as U

MAX_WORLD = 8        # the peer arrays of the fused exchange and of the attention epilogue


class _Local:
    """the group of the one-GPU forward: one rank, no process group, no exchange"""

    def __repr__(self):
        return "LOCAL"


LOCAL = _Local()


def world(group) -> tuple[int, int]:
    """(world size, rank) of `group` by the lookup the Ulysses exchange itself uses; (1, 0) for LOCAL"""
    return (1, 0) if group is LOCAL else U._group_size_rank(group)


def shard(x: torch.Tensor, dim: int, world: int, rank: int) -> torch.Tensor:
    """The contiguous slice `rank` of `world` along `dim`: rows [rank*n, min((rank+1)*n, len)) with
    n = ceil(len / world), zero-padded to n rows (no padding when the length divides by world)."""
    n = -(-x.shape[dim] // world)
    lo = min(rank * n, x.shape[dim])
    part = x.narrow(dim, lo, min(n, x.shape[dim] - lo))
    if part.shape[dim] == n:
        return part.contiguous()
    pad = list(x.shape)
    pad[dim] = n - part.shape[dim]
    return torch.cat([part, x.new_zeros(pad)], dim)


def shard_rows(L: int, world: int, rank: int, model: str) -> tuple[int, int]:
    """(n, real): rows per rank, n = ceil(L / world), and how many of rank `rank`'s n rows are real.
    Raises when some rank would hold no real row."""
    n = -(-L // world)
    if L - (world - 1) * n <= 0:
        raise ValueError(f"sequence-parallel {model}: {L} tokens over {world} ranks leave the last rank "
                         f"without a real row ({n} rows per rank)")
    return n, max(0, min(n, L - rank * n))


def gather_rows(x: torch.Tensor, L: int, P: int, group) -> torch.Tensor:
    """the [1, n, C] rows of every rank in rank order, then the first L"""
    if group is LOCAL:
        return x[:, :L]
    parts = [torch.empty_like(x) for _ in range(P)]
    dist.all_gather(parts, x.contiguous(), group=group)
    return torch.cat(parts, dim=1)[:, :L]


def check_degree(img_tokens: int, heads: int, world: int, model: str) -> None:
    """Whole head groups per rank and, for a non-zero img_tokens, whole image slices per rank (a route that
    pads its slices passes 0).  Under the ragged head split (ulysses.RAGGED_HEADS) heads >= world pass."""
    if U.ragged(heads, world) and heads < world:
        raise ValueError(f"sequence-parallel {model}: {heads} attention heads over {world} ranks leave a rank "
                         "without a head")
    if heads % world and not U.ragged(heads, world):
        raise ValueError(f"sequence-parallel {model}: {heads} attention heads do not split over "
                         f"{world} ranks (the degree must divide the head count)")
    if img_tokens % world:
        raise ValueError(f"sequence-parallel {model}: {img_tokens} image tokens do not split over "
                         f"{world} ranks (the degree must divide the image token count)")


def check_world(heads: int, world: int, model: str) -> None:
    """check_degree for a route that pads its slices, and at most MAX_WORLD ranks"""
    check_degree(0, heads, world, model)
    if world > MAX_WORLD:
        raise ValueError(f"sequence-parallel {model}: {world} ranks; the Ulysses exchange is built for at "
                         f"most {MAX_WORLD} (one NVLink box)")


def check_fused_blocks(modules, model: str, install_call: str, instance_forward: bool = True) -> None:
    """Every module runs the fused jenga_b200 forward of its class: an unpatched forward ignores jenga_sp,
    so every rank would attend over its own rows alone.  instance_forward: also refuse a foreign instance
    forward (the usp_attn_forward WanT2V / WanI2V(use_usp=True) bind), which would run instead."""
    for m in modules:
        cls = type(m)
        if not getattr(cls.forward, "__jenga_b200__", False):
            raise RuntimeError(f"{cls.__module__}.{cls.__name__}.forward is not the fused jenga_b200 forward: "
                               f"{install_call} must run before the {model} model module is imported")
        inst = m.__dict__.get("forward") if instance_forward else None
        if inst is not None and not getattr(getattr(inst, "__func__", inst), "__jenga_b200__", False):
            raise RuntimeError(f"{cls.__name__} has an instance forward ({getattr(inst, '__name__', inst)}) "
                               "that is not the jenga_b200 one: it would run instead of the sharded "
                               "self-attention (install(wan_sp=True) swaps usp_attn_forward)")


def default_attention(group, variant: str):
    """UlyssesFusedAttention(group, variant) when every rank of `group` (None: the default group) can map
    symmetric memory, else UlyssesCarvedAttention (also outside a process group).  The ranks agree by an
    all_reduce MIN, so none takes the fused exchange alone.  JENGA_ULYSSES=nccl picks the NCCL form."""
    ok = 0
    if (os.environ.get("JENGA_ULYSSES", "fused") != "nccl" and dist.is_initialized()
            and dist.get_backend(group) == "nccl"):
        try:
            import torch.distributed._symmetric_memory as symm
            symm.enable_symm_mem_for_group((group if group is not None else dist.group.WORLD).group_name)
            ok = 1
        except Exception:  # noqa: BLE001
            ok = 0
        t = torch.tensor([ok], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
        ok = int(t.item())
    return (U.UlyssesFusedAttention(group=group, variant=variant) if ok
            else U.UlyssesCarvedAttention(group=group, variant=variant))
