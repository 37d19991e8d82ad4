"""Paged-KV pool: T canonical tensors (num_blocks, page_bytes) + gather / scatter (kvb.h section 1)."""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Sequence

import numpy as np

from . import _lib
from ._lib import check


def _stream_ptr(stream) -> int:
    if stream is None:
        import torch
        return torch.cuda.current_stream().cuda_stream
    if isinstance(stream, int):
        return stream
    return stream.cuda_stream


def _ids_array(block_ids) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(block_ids, dtype=np.int64).reshape(-1))


_LAYOUTS = {"NHD": _lib.KV_LAYOUT_NHD, "HND": _lib.KV_LAYOUT_HND}


class KVGeometry(NamedTuple):
    """How one fragment holds the KV heads of a block (kvb.h section 5).  planes: 1 when K and V are separate
    tensors, 2 when they share a fragment; tokens: block size; heads: the KV heads this pool holds; head_bytes:
    head_size x element size; layout: "NHD" ([token][head][byte]) or "HND" ([head][token][byte])."""
    planes: int
    tokens: int
    heads: int
    head_bytes: int
    layout: str = "NHD"


class KVPool:
    """Borrowed view of the KV cache: list of CUDA tensors, each (num_blocks, page_size_bytes)
    (reference: TensorCopier ctor, csrc/storage/tensor_copier.cu:31-48).  ``geometry`` (a KVGeometry) lets the pool
    take part in head-slice migration (migrate.migrate_heads)."""

    def __init__(self, tensors: Sequence, device: int | None = None, *, ptrs=None, num_blocks=None,
                 frag_bytes=None, stride_bytes=None, geometry=None):
        lib = _lib.load()
        if ptrs is None:
            if not tensors:
                raise ValueError("TensorCopier: tensors is empty")
            t0 = tensors[0]
            if not t0.is_contiguous():
                raise ValueError("GPU tensor must be contiguous")
            frag_bytes = t0.stride(0) * t0.element_size()  # tensor_copier.cu:39
            stride_bytes = frag_bytes
            num_blocks = t0.shape[0]
            for t in tensors:
                if t.stride(0) * t.element_size() != frag_bytes or t.shape[0] != num_blocks:
                    raise ValueError("all KV tensors must share num_blocks and page bytes")
            device = t0.device.index if device is None else device
            ptrs = [t.data_ptr() for t in tensors]
        self._tensors = list(tensors) if tensors is not None else []  # keep storage alive
        self.device = int(device)
        self.num_tensors = len(ptrs)
        self.num_blocks = int(num_blocks)
        self.frag_bytes = int(frag_bytes)
        self.block_bytes = self.frag_bytes * self.num_tensors
        arr = (C.c_void_p * len(ptrs))(*ptrs)
        h = C.c_void_p()
        check(lib.kvb_pool_create(self.device, arr, len(ptrs), self.num_blocks, self.frag_bytes,
                                  int(stride_bytes), C.byref(h)))
        self.handle = h
        self.geometry = None
        if geometry is not None:
            self.set_geometry(geometry)

    def set_geometry(self, geometry) -> None:
        """Declare how each fragment holds its KV heads; planes x tokens x heads x head_bytes must be the fragment."""
        g = KVGeometry(*geometry)
        if g.layout not in _LAYOUTS:
            raise ValueError(f"layout must be 'NHD' or 'HND', not {g.layout!r}")
        c = _lib.KvGeometry(int(g.planes), int(g.tokens), int(g.heads), int(g.head_bytes), _LAYOUTS[g.layout], 0)
        check(_lib.load().kvb_pool_set_geometry(self.handle, C.byref(c)))
        self.geometry = g

    def close(self):
        if getattr(self, "handle", None):
            _lib.load().kvb_pool_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- host id lists (uploaded by the library)
    def gather(self, block_ids, packed, stream=None, flags: int = 0):
        ids = _ids_array(block_ids)
        check(_lib.load().kvb_gather_blocks(self.handle, ids.ctypes.data_as(C.POINTER(C.c_int64)), ids.size,
                                            packed.data_ptr(), _stream_ptr(stream), flags))

    def scatter(self, block_ids, packed, stream=None, flags: int = 0):
        ids = _ids_array(block_ids)
        check(_lib.load().kvb_scatter_blocks(self.handle, ids.ctypes.data_as(C.POINTER(C.c_int64)), ids.size,
                                             packed.data_ptr(), _stream_ptr(stream), flags))

    # -- device-resident id tensors (int64 CUDA tensors)
    def gather_dev(self, ids_dev, packed, stream=None, flags: int = 0):
        check(_lib.load().kvb_gather_blocks_dev(self.handle, ids_dev.data_ptr(), ids_dev.numel(),
                                                packed.data_ptr(), _stream_ptr(stream), flags))

    def scatter_dev(self, ids_dev, packed, stream=None, flags: int = 0):
        check(_lib.load().kvb_scatter_blocks_dev(self.handle, ids_dev.data_ptr(), ids_dev.numel(),
                                                 packed.data_ptr(), _stream_ptr(stream), flags))


class PinnedBuffer:
    """Pinned host memory from kvb_host_alloc: page-locked and placed on the NUMA node of the current CUDA device, so
    the copy engine (and the engine's fused host I/O) reads it at full PCIe rate without a staging copy."""

    def __init__(self, nbytes: int, huge_pages: bool = False):
        p = C.c_void_p()
        check(_lib.load().kvb_host_alloc_mode(int(nbytes), 1 if huge_pages else 0, C.byref(p)))
        self.ptr, self.nbytes = int(p.value), int(nbytes)

    def numpy(self, dtype=np.uint8) -> np.ndarray:
        """A view of the whole buffer; it must not outlive this object."""
        raw = (C.c_uint8 * self.nbytes).from_address(self.ptr)
        return np.frombuffer(raw, dtype=np.uint8).view(dtype)

    def free(self) -> None:
        if getattr(self, "ptr", 0):
            _lib.load().kvb_host_free(C.c_void_p(self.ptr))
            self.ptr = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
