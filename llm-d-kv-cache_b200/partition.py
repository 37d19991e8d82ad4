"""Host-side planning for the multi-GPU paths (pure Python, backend-agnostic: tested with gloo on CPU).

The offload path shards by KV partition: one engine per GPU over its own pool, no data-path collective
(the reference runs one engine per worker and separates ranks only by directory, file_mapper.py:60-67).
Migration has one exchange step; torch.distributed carries only its control plane (pool descriptors, block-id
lists, checksums), the bytes move over NVLink by peer stores from the gather kernel."""
from __future__ import annotations

from typing import Sequence

import numpy as np


def shard_range(n_items: int, world: int, rank: int) -> tuple:
    """Contiguous [lo, hi) share of n_items for this rank; shares differ by at most one item."""
    if world <= 0 or not 0 <= rank < world:
        raise ValueError("bad world/rank")
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def ring_peers(rank: int, world: int) -> tuple:
    """(destination, source) of this rank in the all-pairs ring r -> r+1."""
    return (rank + 1) % world, (rank - 1) % world


def fanout_plan(n_blocks: int, world: int, root: int = 0) -> dict:
    """Prefill -> decode hand-off from `root` to every other GPU: peer p receives its own n_blocks pages
    (different prefixes).  Returns {dst_rank: (src_lo, src_hi)} into the root's list of world-1 prefixes."""
    peers = [r for r in range(world) if r != root]
    return {p: (i * n_blocks, (i + 1) * n_blocks) for i, p in enumerate(peers)}


def _kv_heads_of(rank: int, tp: int, num_kv_heads: int, mla: bool) -> range:
    """Global KV heads a TP rank holds (vLLM's rule): a contiguous H/tp share when tp <= H, one head replicated on
    tp/H ranks when tp > H, the one latent head everywhere for MLA."""
    if mla:
        return range(0, 1)
    if tp <= num_kv_heads:
        if num_kv_heads % tp:
            raise ValueError(f"{num_kv_heads} KV heads do not split over TP={tp}")
        per = num_kv_heads // tp
        return range(rank * per, (rank + 1) * per)
    if tp % num_kv_heads:
        raise ValueError(f"TP={tp} is not a multiple of {num_kv_heads} KV heads")
    h = rank // (tp // num_kv_heads)
    return range(h, h + 1)


def tp_head_transfers(num_kv_heads: int, src_tp: int, dst_tp: int, mla: bool = False) -> list:
    """KV hand-off plan between a TP=src_tp pool set and a TP=dst_tp pool set of one model:
    [(src_rank, dst_rank, src_head0, dst_head0, n_heads)], head indices local to each rank's pool, one
    migrate.migrate_heads call each.  Every destination head is written exactly once; where several source ranks hold
    it (replicated heads), destination rank d reads from holders[d % len(holders)].  Consecutive heads from one source
    rank are merged into one transfer."""
    if num_kv_heads < 1 or src_tp < 1 or dst_tp < 1:
        raise ValueError("num_kv_heads and TP sizes must be >= 1")
    H = 1 if mla else num_kv_heads
    src_heads = [_kv_heads_of(r, src_tp, H, mla) for r in range(src_tp)]
    out = []
    for d in range(dst_tp):
        mine = _kv_heads_of(d, dst_tp, H, mla)
        for j, h in enumerate(mine):
            holders = [r for r in range(src_tp) if h in src_heads[r]]
            s = holders[d % len(holders)]
            sh = h - src_heads[s].start
            last = out[-1] if out else None
            if last and last[0] == s and last[1] == d and last[2] + last[4] == sh and last[3] + last[4] == j:
                out[-1] = (s, d, last[2], last[3], last[4] + 1)
            else:
                out.append((s, d, sh, j, 1))
    return out


def token_segments(src_ids, src_block_size: int, dst_ids, dst_block_size: int, n_tokens: int, src_start: int = 0,
                   dst_start: int = 0) -> np.ndarray:
    """Segments for migrate.migrate_tokens: token u < n_tokens of the transfer is at position src_start + u of the
    source request (block table src_ids, blocks of src_block_size tokens) and goes to position dst_start + u of the
    destination request.  Returns the maximal segments, an (n, 5) int64 array of [src_block, src_tok0, dst_block,
    dst_tok0, n_tokens], cut wherever either side crosses a block boundary.  All TP ranks of an instance share one block
    table, so one list serves every call of a tp_head_transfers plan."""
    Bs, Bd, n = int(src_block_size), int(dst_block_size), int(n_tokens)
    if Bs < 1 or Bd < 1 or n < 0 or src_start < 0 or dst_start < 0:
        raise ValueError("block sizes must be >= 1, the token count and starts >= 0")
    src_ids, dst_ids = np.asarray(src_ids, dtype=np.int64).reshape(-1), np.asarray(dst_ids, dtype=np.int64).reshape(-1)
    if n and (src_ids.size * Bs < src_start + n or dst_ids.size * Bd < dst_start + n):
        raise ValueError(f"{src_ids.size} source / {dst_ids.size} destination block ids do not cover tokens "
                         f"[{src_start}, +{n}) / [{dst_start}, +{n})")
    out, u = [], 0
    while u < n:
        sb, so = divmod(src_start + u, Bs)
        db, do = divmod(dst_start + u, Bd)
        k = min(Bs - so, Bd - do, n - u)
        out.append((src_ids[sb], so, dst_ids[db], do, k))
        u += k
    return np.array(out, dtype=np.int64).reshape(-1, 5)


def exchange_objects(obj, dist=None) -> list:
    """all_gather of one picklable object per rank (pool descriptors, checksums)."""
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return [obj]
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, obj)
    return out


def page_checksum_np(tensors: Sequence[np.ndarray], ids) -> int:
    """Order-independent 64-bit checksum of the listed pages (sum of little-endian u64 words mod 2^64)."""
    total = 0
    ids = np.asarray(ids, dtype=np.int64)
    for t in tensors:
        pages = np.ascontiguousarray(t[ids])
        total = (total + int(pages.view(np.uint64).sum(dtype=np.uint64))) & ((1 << 64) - 1)
    return total


def page_checksum_torch(tensors, ids_dev) -> int:
    import torch
    total = 0
    for t in tensors:
        pages = t[ids_dev].contiguous().view(torch.int64)
        total = (total + int(pages.sum().item())) & ((1 << 64) - 1)
    return total
