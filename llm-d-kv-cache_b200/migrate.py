"""Cross-GPU KV-block migration over NVLink (kvb.h section 5).  No reference counterpart: the
reference has no cross-GPU path (SURVEY §1); only the paged layout is shared.

One process per GPU.  The destination rank exports its KV tensors over CUDA IPC, the source rank
maps them and ONE kernel reads source pages and writes destination pages (gather fused with the
peer write and the scatter).  torch.distributed carries only the control plane (handles, ids)."""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from . import _lib
from ._lib import IpcMem, check
from .pool import KVPool, _ids_array, _stream_ptr


def export_pool(pool: KVPool) -> dict:
    """Picklable description of a pool's tensors (CUDA IPC handles), for the peer that will write/read it."""
    lib = _lib.load()
    mems = []
    for t in pool._tensors:
        m = IpcMem()
        check(lib.kvb_ipc_export(pool.device, t.data_ptr(), C.byref(m)))
        mems.append((bytes(m.handle), int(m.offset)))
    desc = {"device": pool.device, "num_blocks": pool.num_blocks, "frag_bytes": pool.frag_bytes, "mems": mems}
    if pool.geometry is not None:
        desc["geometry"] = tuple(pool.geometry)
    return desc


class RemotePool(KVPool):
    """A peer GPU's pool mapped into this process (pointers usable from ``local_device``)."""

    def __init__(self, desc: dict, local_device: int):
        lib = _lib.load()
        self._imported = []
        ptrs = []
        cache: dict = {}
        for handle, offset in desc["mems"]:
            base = cache.get(handle)
            if base is None:
                m = IpcMem()
                C.memmove(m.handle, handle, 64)
                m.offset = 0
                p = C.c_void_p()
                check(lib.kvb_ipc_import(local_device, C.byref(m), C.byref(p)))
                base = cache[handle] = p.value
                self._imported.append(base)
            ptrs.append(base + offset)
        super().__init__(None, local_device, ptrs=ptrs, num_blocks=desc["num_blocks"],
                         frag_bytes=desc["frag_bytes"], stride_bytes=desc["frag_bytes"], geometry=desc.get("geometry"))
        check(lib.kvb_pool_mark_peer(self.handle, 1))

    def close(self):
        super().close()
        for base in getattr(self, "_imported", []):
            _lib.load().kvb_ipc_close(self.device, base, 0)
        self._imported = []


def migrate_blocks(src: KVPool, dst: KVPool, src_ids: Sequence[int], dst_ids: Sequence[int], stream=None,
                   flags: int = 0) -> None:
    """src pages src_ids[i] -> dst pages dst_ids[i]; ``dst`` is a local pool or a RemotePool."""
    s, d = _ids_array(src_ids), _ids_array(dst_ids)
    if s.size != d.size:
        raise ValueError("src_ids and dst_ids differ in length")
    check(_lib.load().kvb_migrate_blocks(src.handle, dst.handle, s.ctypes.data_as(C.POINTER(C.c_int64)),
                                         d.ctypes.data_as(C.POINTER(C.c_int64)), s.size, _stream_ptr(stream), flags))


def migrate_heads(src: KVPool, dst: KVPool, src_ids: Sequence[int], dst_ids: Sequence[int], src_head0: int,
                  dst_head0: int, n_heads: int, stream=None, flags: int = 0) -> None:
    """Heads [src_head0, src_head0 + n_heads) of src pages src_ids[i] -> heads [dst_head0, dst_head0 + n_heads) of dst
    pages dst_ids[i], each pool in its own KV geometry (kvb.h section 5); the rest of each destination page is left
    alone.  Both pools need a geometry; partition.tp_head_transfers plans the calls of a TP resharding."""
    s, d = _ids_array(src_ids), _ids_array(dst_ids)
    if s.size != d.size:
        raise ValueError("src_ids and dst_ids differ in length")
    check(_lib.load().kvb_migrate_heads(src.handle, dst.handle, s.ctypes.data_as(C.POINTER(C.c_int64)),
                                        d.ctypes.data_as(C.POINTER(C.c_int64)), s.size, int(src_head0),
                                        int(dst_head0), int(n_heads), _stream_ptr(stream), flags))


_SEGMENT = np.dtype([("src_block", "<i8"), ("dst_block", "<i8"), ("src_tok0", "<i4"), ("dst_tok0", "<i4"),
                     ("n_tokens", "<i4"), ("pad", "<i4")])  # kvb_token_segment_t


def migrate_tokens(src: KVPool, dst: KVPool, segments, src_head0: int = 0, dst_head0: int = 0, n_heads=None,
                   stream=None, flags: int = 0) -> None:
    """Token segments between pools of different block sizes or at offsets inside a block (kvb.h section 5).
    ``segments`` is an (n, 5) integer array of rows [src_block, src_tok0, dst_block, dst_tok0, n_tokens]: tokens
    [src_tok0, +n_tokens) of source block src_block, heads [src_head0, +n_heads), go to tokens [dst_tok0, +n_tokens) of
    destination block dst_block, heads [dst_head0, +n_heads); nothing else of the destination is written.
    partition.token_segments plans the segments of a request.  n_heads=None means all heads and needs both pools to
    hold the same number."""
    seg = np.asarray(segments, dtype=np.int64)
    if seg.size == 0:
        seg = seg.reshape(0, 5)
    if seg.ndim != 2 or seg.shape[1] != 5:
        raise ValueError(f"segments must be an (n, 5) array, not {seg.shape}")
    if n_heads is None:
        gs, gd = src.geometry, dst.geometry
        if gs is None or gd is None or gs.heads != gd.heads:
            raise ValueError("n_heads=None needs both pools to carry a geometry with the same number of heads")
        n_heads = gs.heads
    lim = np.iinfo(np.int32)
    if seg.size and (seg[:, [1, 3, 4]].min() < lim.min or seg[:, [1, 3, 4]].max() > lim.max):
        raise ValueError("token offsets and counts must fit in 32 bits")
    rec = np.zeros(seg.shape[0], dtype=_SEGMENT)
    rec["src_block"], rec["src_tok0"], rec["dst_block"], rec["dst_tok0"], rec["n_tokens"] = seg.T
    check(_lib.load().kvb_migrate_tokens(src.handle, dst.handle, rec.ctypes.data_as(C.POINTER(_lib.TokenSegment)),
                                         rec.size, int(src_head0), int(dst_head0), int(n_heads), _stream_ptr(stream),
                                         flags))


def enable_peer_access(device: int, peer: int) -> None:
    check(_lib.load().kvb_enable_peer_access(device, peer))
