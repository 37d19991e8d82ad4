"""CPU oracle for the offload path: file grouping, file naming, staging/file byte layout.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  numpy byte arithmetic; every function
cites the reference file:line (relative to /root/reference/kv_connectors/llmd_fs_backend).

The reference holds no golden *bytes* for this path (its tests only check that a load
returns what a store wrote, tests/test_fs_backend.py:353-411), so this layout statement is
taken from the code; tests/test_gpu_ref_interop.py cross-checks it against files written by the reference
engine itself (stored under tests/golden/).
"""
from __future__ import annotations

from typing import Sequence

import numpy as np

MIN_STAGING_BUFFER_SIZE = 16 * 1024 * 1024  # csrc/storage/thread_pool.cpp:35


def build_file_block_mapping(block_hashes: Sequence, block_ids: Sequence[int], gpu_blocks_per_file: int):
    """BaseStorageOffloadingHandler._build_file_block_mapping (llmd_fs_backend/worker.py:158-193).

    Returns (per-file hash list, per-file block-id lists): the first file takes
    ``len(ids) % bpf or bpf`` ids, every later file ``bpf``.
    """
    hashes, per_file = [], []
    n = len(block_ids)
    first = n % gpu_blocks_per_file or gpu_blocks_per_file
    start, size = 0, first
    for h in block_hashes:
        end = min(start + size, n)
        hashes.append(h)
        per_file.append(list(block_ids[start:end]))
        start += size
        size = gpu_blocks_per_file
    return hashes, per_file


def base_path(root_dir, model_name, gpu_block_size, gpu_blocks_per_file, tp_size, pp_size, pcp_size, rank, dtype) -> str:
    """FileMapper.__init__ (llmd_fs_backend/file_mapper.py:60-67)."""
    return (f"{root_dir}/{model_name}/block_size_{gpu_block_size}_blocks_per_file_{gpu_blocks_per_file}"
            f"/tp_{tp_size}_pp_size_{pp_size}_pcp_size_{pcp_size}/rank_{rank}/{dtype}")


def file_name(base: str, block_hash) -> str:
    """FileMapper.get_file_name (llmd_fs_backend/file_mapper.py:69-87)."""
    if isinstance(block_hash, (bytes, bytearray)):
        block_hash = int.from_bytes(block_hash, "big")
    hx = f"{block_hash & ((1 << 64) - 1):016x}"
    return f"{base}/{hx[:3]}/{hx[3:5]}/{hx}.bin"


def staging_size(num_tensors: int, frag_bytes: int, gpu_blocks_per_file: int) -> int:
    """Per-thread staging buffer == file size on the CPU path
    (storage_offload.cpp:160-171 calc_staging_bytes; thread_pool.cpp:229-231 max with 16 MiB;
    file_io.cpp:77 writes buf.size bytes)."""
    return max(num_tensors * frag_bytes * gpu_blocks_per_file, MIN_STAGING_BUFFER_SIZE)


def slot_offset(num_tensors: int, frag_bytes: int, gpu_blocks_per_file: int, n_blocks_in_file: int) -> int:
    """Byte offset of the first block of a file holding n blocks: tail-aligned within the
    ``bpf`` slots (tensor_copier.cu:75-76)."""
    return (gpu_blocks_per_file - n_blocks_in_file) * num_tensors * frag_bytes


def pack_blocks(tensors: Sequence[np.ndarray], block_ids: Sequence[int]) -> np.ndarray:
    """Packed bytes of the listed blocks, [block][tensor][fragment] (tensor_copier.cu:78-96).

    ``tensors``: T arrays of shape (num_blocks, frag_bytes) uint8 (the canonical KV tensors).
    """
    T = len(tensors)
    frag = tensors[0].shape[1]
    out = np.empty((len(block_ids), T, frag), dtype=np.uint8)
    ids = np.asarray(block_ids, dtype=np.int64)
    for t, ten in enumerate(tensors):
        out[:, t, :] = ten[ids]
    return out.reshape(-1)


def unpack_blocks(tensors: Sequence[np.ndarray], block_ids: Sequence[int], packed: np.ndarray) -> None:
    """Inverse of pack_blocks (H2D direction of tensor_copier.cu:50-97): in-place scatter."""
    T = len(tensors)
    frag = tensors[0].shape[1]
    src = packed.reshape(len(block_ids), T, frag)
    ids = np.asarray(block_ids, dtype=np.int64)
    for t, ten in enumerate(tensors):
        ten[ids] = src[:, t, :]  # later duplicates win, like sequential memcpys


def file_image(tensors: Sequence[np.ndarray], block_ids: Sequence[int], gpu_blocks_per_file: int,
               fill: int = 0) -> np.ndarray:
    """Full image of one reference file written by the CPU path (file_io.cpp:152-187):
    ``staging_size`` bytes, blocks tail-aligned at ``slot_offset``; bytes outside the
    written slots are whatever the staging buffer held (``fill`` here)."""
    T = len(tensors)
    frag = tensors[0].shape[1]
    img = np.full(staging_size(T, frag, gpu_blocks_per_file), fill, dtype=np.uint8)
    off = slot_offset(T, frag, gpu_blocks_per_file, len(block_ids))
    p = pack_blocks(tensors, block_ids)
    img[off:off + p.size] = p
    return img


def load_from_image(tensors: Sequence[np.ndarray], block_ids: Sequence[int], gpu_blocks_per_file: int,
                    img: np.ndarray) -> None:
    """read_blocks_from_file (file_io.cpp:190-225): take the tail-aligned ``len(block_ids)`` slots."""
    T = len(tensors)
    frag = tensors[0].shape[1]
    off = slot_offset(T, frag, gpu_blocks_per_file, len(block_ids))
    n = len(block_ids) * T * frag
    unpack_blocks(tensors, block_ids, img[off:off + n])
