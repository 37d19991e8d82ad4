"""StorageOffloadEngine — same constructor and methods as the reference's pybind class
(kv_connectors/llmd_fs_backend/csrc/storage/storage_offload_bindings.cpp:25-94), i.e. the
StorageEngine Protocol of llmd_fs_backend/worker.py:36-52, implemented by libkvb.so."""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from . import _lib
from ._lib import EngineOpts, EngineStats, check
from .pool import KVPool, _stream_ptr


class StorageOffloadEngine:
    """Async KV-block offload between the GPU KV cache and a storage tier.

    Positional arguments are the reference's (storage_offload_bindings.cpp:30-41).  Keyword-only
    extensions select the H100-native host tier:
      tier="file"        reference on-disk format under the given file paths (default, drop-in)
      tier="host_arena"  pinned host DRAM arena of ``host_arena_bytes`` keyed by the same path strings
    ``gds_mode`` (file tier) takes the reference's strings (gds_file_io.cpp:425-446): reads and/or writes then use its
    GDS file format (head-aligned, exactly n x block_bytes) through cuFile on the packed HBM chunk, one call per file;
    without a usable cuFile the same format goes through the pinned staging buffer.
    """

    def __init__(self, io_threads: int, gpu_blocks_per_file: int, tensors: Sequence, read_preferring_workers: int,
                 gds_mode: str = "disabled", max_write_queued_seconds: float = 10.0, *, tier: str = "file",
                 host_arena_bytes: int = 0, chunk_bytes: int = 0, copy_variant: int = 0,
                 strict_load_errors: bool = False, direct_host_io: bool = False, arena_huge_pages: bool = False):
        # reference parse_gds_mode (gds_file_io.cpp:425-446): unknown strings mean "disabled"
        gds_bits = {"read_only": 1, "write_only": 2, "read_write": 3, "bb_read_only": 5, "bb_write_only": 6,
                    "bb_read_write": 7}.get(gds_mode, 0)
        lib = _lib.load()
        self.pool = tensors if isinstance(tensors, KVPool) else KVPool(tensors)
        opts = EngineOpts()
        lib.kvb_engine_default_opts(C.byref(opts))
        opts.io_threads = int(io_threads)
        opts.gpu_blocks_per_file = int(gpu_blocks_per_file)
        opts.read_preferring_workers = int(read_preferring_workers)
        opts.max_write_queued_seconds = float(max_write_queued_seconds)
        opts.tier = {"file": _lib.TIER_FILE, "host_arena": _lib.TIER_HOST_ARENA}[tier]
        opts.copy_flags = int(copy_variant)
        opts.host_arena_bytes = int(host_arena_bytes)
        if chunk_bytes:
            opts.chunk_bytes = int(chunk_bytes)
        opts.strict_load_errors = 1 if strict_load_errors else 0
        opts.direct_host_io = 1 if direct_host_io else 0
        opts.arena_alloc_mode = 1 if arena_huge_pages else 0  # KVB_HOST_ALLOC_THP: arena on transparent huge pages
        opts.gds_mode = gds_bits if tier == "file" else 0
        h = C.c_void_p()
        check(lib.kvb_engine_create(self.pool.handle, C.byref(opts), C.byref(h)))
        self._h = h
        self.gpu_blocks_per_file = int(gpu_blocks_per_file)
        self.tier = tier

    # -- submit ---------------------------------------------------------------------------------
    def _submit(self, fn, job_id: int, files: Sequence[str], all_block_ids: Sequence[Sequence[int]], stream):
        if len(files) != len(all_block_ids):
            raise ValueError("files and block id lists differ in length")
        n = len(files)
        paths = (C.c_char_p * max(n, 1))(*[f.encode() for f in files])
        off = np.zeros(n + 1, dtype=np.int64)
        for i, ids in enumerate(all_block_ids):
            off[i + 1] = off[i] + len(ids)
        flat = np.empty(int(off[-1]), dtype=np.int64)
        for i, ids in enumerate(all_block_ids):
            flat[off[i]:off[i + 1]] = np.asarray(ids, dtype=np.int64)
        rc = fn(self._h, int(job_id), n, paths, flat.ctypes.data_as(C.POINTER(C.c_int64)),
                off.ctypes.data_as(C.POINTER(C.c_int64)), _stream_ptr(stream))
        if rc < 0:  # reference returns bool; errors are logged, not raised (storage_offload.cpp:338-347)
            import sys
            print(f"[kvb][ERROR] submit failed: {_lib.load().kvb_last_error().decode()}", file=sys.stderr)
            return False
        return True

    def async_store_gpu_blocks(self, job_id: int, dst_files, all_block_ids, stream=None) -> bool:
        return self._submit(_lib.load().kvb_engine_store, job_id, dst_files, all_block_ids, stream)

    def async_load_gpu_blocks(self, job_id: int, src_files, all_block_ids, stream=None) -> bool:
        return self._submit(_lib.load().kvb_engine_load, job_id, src_files, all_block_ids, stream)

    # -- completion -----------------------------------------------------------------------------
    def get_finished(self) -> list:
        cap = 256
        ids = (C.c_int64 * cap)()
        ok = (C.c_int32 * cap)()
        out = []
        while True:
            n = check(_lib.load().kvb_engine_poll(self._h, ids, ok, cap))
            out.extend((int(ids[i]), bool(ok[i])) for i in range(n))
            if n < cap:
                return out

    def wait_job(self, job_id: int) -> None:
        check(_lib.load().kvb_engine_wait(self._h, int(job_id)))

    def exists(self, file: str) -> bool:
        return bool(_lib.load().kvb_engine_exists(self._h, file.encode()))

    def lookup_prefix(self, files: Sequence[str]) -> int:
        """How many CONSECUTIVE entries of ``files`` from the start exist in this engine's tier — the whole
        ``SharedStorageOffloadingManager.lookup`` loop (manager.py:43-53) in one library call."""
        n = len(files)
        if n == 0:
            return 0
        paths = (C.c_char_p * n)(*[f.encode() for f in files])
        hits = C.c_int32()
        check(_lib.load().kvb_engine_lookup_prefix(self._h, n, paths, C.byref(hits)))
        return int(hits.value)

    def lookup_prefix_hashes(self, base_path: str, hashes: np.ndarray) -> int:
        """Same, from the low 64 bits of the block hashes (uint64 array): the library builds FileMapper's file names
        itself, so nothing per block is done in Python."""
        hashes = np.ascontiguousarray(hashes, dtype=np.uint64)
        if hashes.size == 0:
            return 0
        hits = C.c_int32()
        check(_lib.load().kvb_engine_lookup_prefix_hashes(self._h, base_path.encode(), hashes.ctypes.data, hashes.size,
                                                          C.byref(hits)))
        return int(hits.value)

    def arena_clear(self) -> None:
        check(_lib.load().kvb_engine_arena_clear(self._h))

    def stats(self) -> dict:
        s = EngineStats()
        check(_lib.load().kvb_engine_get_stats(self._h, C.byref(s)))
        return {n: int(getattr(s, n)) for n, _ in EngineStats._fields_}

    def shutdown(self) -> None:
        if getattr(self, "_h", None):
            _lib.load().kvb_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.shutdown()
        except Exception:
            pass
