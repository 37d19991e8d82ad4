"""llm-d-kv-cache_b200 — H100-native (sm_90a) KV-block hot path behind the reference's own surfaces.

The directory name is not a Python identifier; import it with
    kvb = importlib.import_module("llm-d-kv-cache_b200")
Host-side mirrors of the reference interfaces (same names / argument meaning / error behaviour):
    kvb.engine.StorageOffloadEngine      <- storage_offload.StorageOffloadEngine (pybind, csrc/storage)
    kvb.worker.{GPUToStorageHandler,StorageToGPUHandler,StorageOffloadingHandlers}, kvb.file_mapper.FileMapper
    kvb.kvblock.{ChunkedTokenDatabase,Index,PodEntry,...}  <- pkg/kvcache/kvblock
    kvb.indexer.{Indexer,LongestPrefixScorer}              <- pkg/kvcache
All compute goes through libkvb.so (include/kvb.h); importing this package without the built library fails.
"""
from . import _lib

lib = _lib.load()  # fail loudly if the CUDA library is absent

from . import pool, engine, file_mapper, mediums, worker, kvblock, indexer, migrate, partition, kvevents, manager, spec  # noqa: E402,F401

__all__ = ["lib", "pool", "engine", "file_mapper", "mediums", "worker", "kvblock", "indexer", "migrate", "partition", "kvevents", "manager", "spec"]
