#!/usr/bin/env python
"""BASELINE config #3: Llama-3-70B GQA paged-KV fp8-e4m3 (160 tensors x 16384 B, 2.5 MiB blocks), offload sweep.

Resident pool N = 16384 blocks (43 GB of the H100's 80 GB, beside a 21 GB packed slice).  For n in {1k, 4k, 16k}: device-resident
gather/scatter timing (CUDA events per launch) and end-to-end save+load through the engine API (host-arena tier).
{128k, 1M} blocks are CUMULATIVE: batches of 16k blocks cycled through a bounded 42 GB pinned arena
(1 M x 2.5 MiB = 2.6 TB cannot be resident on the host tier at once) — stated, not hidden.
One process per GPU under torchrun for the multi-GPU sweep (independent partitions, aggregate GB/s).
Prints one JSON object on rank 0."""
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

T, FRAG = 160, 16384
BLOCK = T * FRAG
POOL = int(os.environ.get("KVB_SWEEP_POOL", "16384"))
RESIDENT = [int(x) for x in os.environ.get("KVB_SWEEP_RESIDENT", "1000,4000,16000").split(",")]
CUMULATIVE = [int(x) for x in os.environ.get("KVB_SWEEP_CUMULATIVE", "128000,1000000").split(",") if x]
BATCH = 16000
BPF = 16


def drain(eng, job):
    while True:
        for j, ok in eng.get_finished():
            if j == job:
                assert ok
                return
        time.sleep(0.0005)


def main():
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    kvb = importlib.import_module("llm-d-kv-cache_b200")

    def sync():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
            torch.cuda.synchronize()

    def rmax(x):
        if dist is None:
            return x
        t = torch.tensor([x], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    big = torch.empty((T, POOL, FRAG), dtype=torch.uint8, device="cuda")
    big.random_(0, 256)
    tensors = list(big.unbind(0))
    pool = kvb.pool.KVPool(tensors)
    perm = np.random.default_rng(1 + rank).permutation(POOL).astype(np.int64)
    n_max = max(RESIDENT)
    # the packed staging for the device-resident arm is bounded: gather/scatter in slices of 8k blocks (21 GB)
    SLICE = 8000
    packed = torch.empty(min(n_max, SLICE) * BLOCK, dtype=torch.uint8, device="cuda")
    rows = []
    arena_blocks = max(min(n_max, BATCH), BATCH if CUMULATIVE else 0)
    eng = kvb.engine.StorageOffloadEngine(4, BPF, tensors, 3, "disabled", 0.0, tier="host_arena",
                                          host_arena_bytes=arena_blocks * BLOCK + (64 << 20), chunk_bytes=80 << 20)
    job = [0]

    def save_load(ids, tag):
        nf = len(ids) // BPF
        groups = [ids[i * BPF:(i + 1) * BPF].tolist() for i in range(nf)]
        files = [f"{tag}/{i:07d}" for i in range(nf)]
        job[0] += 1
        assert eng.async_store_gpu_blocks(job[0], files, groups)
        drain(eng, job[0])
        job[0] += 1
        assert eng.async_load_gpu_blocks(job[0], files, groups)
        drain(eng, job[0])
        eng.arena_clear()

    for n in RESIDENT:
        ids = perm[:n]
        ids_dev = torch.from_numpy(ids).cuda()
        # device-resident: sum of per-slice kernel times
        g_ms = s_ms = 0.0
        for rep in range(3):
            g_acc = s_acc = 0.0
            for lo in range(0, n, SLICE):
                sl = ids_dev[lo:lo + SLICE]
                a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                a.record()
                pool.gather_dev(sl, packed)
                b.record()
                pool.scatter_dev(sl, packed)
                c.record()
                torch.cuda.synchronize()
                g_acc += a.elapsed_time(b)
                s_acc += b.elapsed_time(c)
            if rep > 0:
                g_ms, s_ms = g_ms + g_acc / 2, s_ms + s_acc / 2
        g_ms, s_ms = rmax(g_ms), rmax(s_ms)
        payload = n * BLOCK
        row = {"blocks": n, "payload_gb": payload / 1e9, "gather_hbm_gbs": 2 * payload / g_ms / 1e6,
               "scatter_hbm_gbs": 2 * payload / s_ms / 1e6, "device_save_plus_load_gbs": world * 2 * payload / (g_ms + s_ms) / 1e6}
        if n <= arena_blocks:
            n16 = n // BPF * BPF
            save_load(ids[:n16], f"w{n}")
            sync()
            t0 = time.perf_counter()
            save_load(ids[:n16], f"r{n}")
            sync()
            dt = rmax(time.perf_counter() - t0)
            row["e2e_save_plus_load_gbs"] = world * 2 * n16 * BLOCK / dt / 1e9
            row["e2e_blocks_per_s"] = world * 2 * n16 / dt
        else:
            # larger than the arena: cycle batches (cumulative)
            sync()
            t0 = time.perf_counter()
            done = 0
            while done < n:
                m = min(BATCH, n - done) // BPF * BPF
                save_load(ids[done:done + m], f"c{n}_{done}")
                done += m
            sync()
            dt = rmax(time.perf_counter() - t0)
            row["e2e_save_plus_load_gbs"] = world * 2 * done * BLOCK / dt / 1e9
            row["e2e_blocks_per_s"] = world * 2 * done / dt
            row["e2e_mode"] = f"cumulative in batches of {BATCH} through a {arena_blocks}-block arena"
        rows.append(row)
        if rank == 0:
            print("#", json.dumps(row), file=sys.stderr, flush=True)

    for total in CUMULATIVE:
        sync()
        t0 = time.perf_counter()
        done, k = 0, 0
        while done < total:
            m = min(BATCH, total - done) // BPF * BPF
            start = (k * BATCH) % (POOL - BATCH)
            save_load(perm[start:start + m], f"cum{total}_{k}")
            done += m
            k += 1
        sync()
        dt = rmax(time.perf_counter() - t0)
        row = {"blocks": total, "cumulative": True, "payload_tb_each_way": done * BLOCK / 1e12,
               "e2e_save_plus_load_gbs": world * 2 * done * BLOCK / dt / 1e9, "e2e_blocks_per_s": world * 2 * done / dt,
               "seconds": dt, "e2e_mode": f"batches of {BATCH} blocks cycled through a {arena_blocks}-block pinned arena"}
        rows.append(row)
        if rank == 0:
            print("#", json.dumps(row), file=sys.stderr, flush=True)

    # restored data must still equal what was there (every save+load is an identity on the pool)
    chk = torch.from_numpy(perm[:64]).cuda()
    ref = big[:, chk].clone()
    save_load(perm[:64 // BPF * BPF], "final")
    assert torch.equal(big[:, chk], ref)
    eng.shutdown()
    if rank == 0:
        print(json.dumps({"config": "BASELINE #3: Llama-3-70B GQA fp8-e4m3 paged-KV, 160 tensors x 16384 B, 2.5 MiB blocks",
                          "n_gpus": world, "pool_blocks": POOL, "rows": rows}))
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
