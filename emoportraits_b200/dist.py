"""Multi-GPU plumbing of the path (SURVEY.md §8e): driver frames are independent once the source identity has been
encoded, so the only exchange step is ONE broadcast per identity of the cached source state

    target_latent_volume  1 x 16 x 64 x 64 x 96 fp32 = 25.2 MB
    idt_embed             1 x 512 x 4 x 4 fp32      = 32 KB
    source theta          4 x 4 fp32                = 64 B

from the rank that ran the source pass (torch.distributed / NCCL over NVLink; `gloo` in the CPU tests).  After it every
rank runs its own frames; there is no data-path collective (frames are sharded round-robin, weak scaling).
The reference's own num_gpus > 1 inference branch (notebooks/infer.py:99-136) is not usable as a model for this.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
import torch.distributed as dist

from .config import HotPathConfig


def source_state_shapes(cfg: HotPathConfig):
    """The identity: the fields of a source state that a driver frame reads (Model.driver_pass), besides
    source_theta_dev, which is pred_source_theta[0] in every state (new_identity keeps it as that view).  The broadcast
    sends these, and a captured driver graph (Model.make_driver_graph) holds its own copy of them."""
    return {
        "target_latent_volume": (1, cfg.D, cfg.S, cfg.S, cfg.C),
        "idt_embed": (1, cfg.idt_channels, cfg.embed_size, cfg.embed_size),
        "pred_source_theta": (1, 4, 4),
    }


def new_identity(cfg: HotPathConfig, device, fields=None) -> SimpleNamespace:
    """zeroed fp32 identity buffers (source_state_shapes, or only the names in `fields`, which must include
    pred_source_theta), with source_theta_dev the view pred_source_theta[0]"""
    shapes = source_state_shapes(cfg)
    out = SimpleNamespace(**{k: torch.zeros(shapes[k], dtype=torch.float32, device=device) for k in (fields or shapes)})
    out.source_theta_dev = out.pred_source_theta[0]
    return out


def check_identity(st, cfg: HotPathConfig) -> None:
    """ValueError unless `st` carries every identity field as an fp32 tensor of the shape `cfg` gives it"""
    for k, shp in source_state_shapes(cfg).items():
        t = getattr(st, k, None)
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != shp or t.dtype != torch.float32:
            got = (tuple(t.shape), t.dtype) if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"not an identity of this model: {k} must be an fp32 tensor of shape {shp}, got {got}")


def broadcast_source_state(st, cfg: HotPathConfig, device, src: int = 0, group=None):
    """Rank `src` passes its source state; every rank returns a state usable by Model.driver_pass."""
    rank = dist.get_rank(group)
    shapes = source_state_shapes(cfg)
    # one flat buffer -> one collective
    total = sum(int(torch.tensor(s).prod()) for s in shapes.values())
    flat = torch.empty(total, dtype=torch.float32, device=device)
    if rank == src:
        off = 0
        for k, shp in shapes.items():
            t = getattr(st, k).reshape(-1)
            flat[off:off + t.numel()].copy_(t)
            off += t.numel()
    dist.broadcast(flat, src=src, group=group)
    out = new_identity(cfg, device)
    off = 0
    for k, shp in shapes.items():
        n = int(torch.tensor(shp).prod())
        getattr(out, k).copy_(flat[off:off + n].view(shp))
        off += n
    return out


def shard_frames(num_frames: int, rank: int, world: int):
    """frame indices rank `rank` processes: i == rank (mod world)"""
    return list(range(rank, num_frames, world))
