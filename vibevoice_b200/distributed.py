"""Multi-GPU plumbing (SURVEY 8e): prompts shard by batch across ranks -- one process per GPU, weights replicated, no
collective inside the generation loop -- and the finished waveforms are gathered to rank 0 with one exchange of lengths
(`all_gather`) and one `gather` of zero-padded samples.  Works on any `torch.distributed` backend (NCCL over NVLink on a
multi-GPU machine, gloo in the CPU tests)."""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.distributed as dist


def shard_prompts(n_prompts: int, rank: int, world: int) -> List[int]:
    """Prompt indices owned by `rank`: contiguous blocks, sizes differing by at most one."""
    base, rem = divmod(n_prompts, world)
    start = rank * base + min(rank, rem)
    return list(range(start, start + base + (1 if rank < rem else 0)))


def gather_waveforms(wavs: Sequence[Optional[torch.Tensor]], device=None, dst: int = 0) -> Optional[List[List[Optional[torch.Tensor]]]]:
    """wavs: this rank's outputs, each [1, T_i] float (or None).  Returns on `dst` a list (per rank) of lists of tensors
    (CPU), elsewhere None."""
    world, rank = dist.get_world_size(), dist.get_rank()
    device = device or (wavs[0].device if len(wavs) and wavs[0] is not None else torch.device("cpu"))
    lens = torch.tensor([(-1 if w is None else w.shape[-1]) for w in wavs], dtype=torch.int64, device=device)
    n_local = torch.tensor([len(wavs)], dtype=torch.int64, device=device)
    counts = [torch.zeros_like(n_local) for _ in range(world)]
    dist.all_gather(counts, n_local)
    max_n = int(max(c.item() for c in counts))
    lens_pad = torch.full((max_n,), -1, dtype=torch.int64, device=device)
    lens_pad[: len(wavs)] = lens
    all_lens = [torch.zeros_like(lens_pad) for _ in range(world)]
    dist.all_gather(all_lens, lens_pad)
    t_max = max(1, int(max(int(l.max().item()) for l in all_lens)))
    buf = torch.zeros(max_n, t_max, dtype=torch.float32, device=device)
    for i, w in enumerate(wavs):
        if w is not None:
            buf[i, : w.shape[-1]] = w.reshape(-1).to(device=device, dtype=torch.float32)
    out = [torch.empty_like(buf) for _ in range(world)] if rank == dst else None
    dist.gather(buf, out, dst=dst)
    if rank != dst:
        return None
    res = []
    for r in range(world):
        row = []
        for i in range(int(counts[r].item())):
            n = int(all_lens[r][i].item())
            row.append(None if n < 0 else out[r][i, :n].cpu()[None])
        res.append(row)
    return res
