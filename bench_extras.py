"""bench_extras.py — the parts of bench.py that are not BASELINE config #2's headline numbers.

Part of bench.py (imported by it and by nothing else): cross-GPU migration with byte-for-byte verification (config #4),
the 70B-fp8 block shape (config #3), and the index path (configs #1 and #5, KV-event ingest, manager lookup).  Every
section asserts parity before it reports a number.  The `oracle` imports below are bench.py's checker / cpu_baseline legs
(the oracle is the checker and the CPU baseline, never the thing measured)."""
from __future__ import annotations

import os
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))


# ---------------------------------------------------------------------------------------------------------------------
# small helpers shared with bench.py
def barrier_sync(dist):
    import torch
    torch.cuda.synchronize()
    if dist is not None:
        dist.barrier()
    torch.cuda.synchronize()


def max_over_ranks(dist, x: float) -> float:
    if dist is None:
        return x
    import torch
    t = torch.tensor([x], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gather_objects(dist, obj):
    if dist is None:
        return [obj]
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, obj)
    return out


def nvlink_counters(local_device: int):
    """Cumulative NVLink payload bytes (tx, rx) of this rank's GPU summed over its links, from NVML
    (NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX / _RX, KiB), else parsed from `nvidia-smi nvlink -gt d`.  None if the box
    exposes neither."""
    try:
        import pynvml
        import torch
        pynvml.nvmlInit()
        uuid = str(torch.cuda.get_device_properties(local_device).uuid)
        if not uuid.startswith("GPU-"):
            uuid = "GPU-" + uuid
        try:
            h = pynvml.nvmlDeviceGetHandleByUUID(uuid.encode())
        except Exception:
            h = pynvml.nvmlDeviceGetHandleByIndex(local_device)
        vals = pynvml.nvmlDeviceGetFieldValues(h, [(pynvml.NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX, 0xFFFFFFFF),
                                                   (pynvml.NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_RX, 0xFFFFFFFF)])
        out = []
        for v in vals:
            if v.nvmlReturn != 0:
                raise RuntimeError(f"nvml field {v.fieldId}: return {v.nvmlReturn}")
            out.append(int(v.value.ullVal) * 1024)
        return {"tx": out[0], "rx": out[1], "source": "nvml NVLINK_THROUGHPUT_DATA_TX/RX (all links)"}
    except Exception as e_nvml:
        try:
            import re
            import subprocess
            txt = subprocess.run(["nvidia-smi", "nvlink", "-gt", "d", "-i", str(local_device)], capture_output=True,
                                 text=True, timeout=20).stdout
            tx = sum(int(x) for x in re.findall(r"Data Tx:\s*(\d+)\s*KiB", txt)) * 1024
            rx = sum(int(x) for x in re.findall(r"Data Rx:\s*(\d+)\s*KiB", txt)) * 1024
            if tx or rx:
                return {"tx": tx, "rx": rx, "source": "nvidia-smi nvlink -gt d"}
        except Exception:
            pass
        return {"tx": None, "rx": None, "source": f"unavailable ({e_nvml})"}


def _delta(a, b, key):
    if not a or not b or a.get(key) is None or b.get(key) is None:
        return None
    return b[key] - a[key]


# ---------------------------------------------------------------------------------------------------------------------
# config #4: cross-GPU migration, any block shape
def _ring_verify(dist, rank, world, tensors, my_src_ids, ids_written_into_me, group=16) -> bool:
    """Byte-for-byte: what my ring source wrote into my pool must equal the pages it read.  Every rank ships the pages it
    SENT (plain torch indexing, none of our kernels) to its destination over NCCL and compares what it RECEIVES from its
    source with its own destination pages."""
    import torch
    dst_rank, src_rank = (rank + 1) % world, (rank - 1) % world
    s_idx = torch.from_numpy(np.asarray(my_src_ids)).cuda()
    d_idx = torch.from_numpy(np.asarray(ids_written_into_me)).cuda()
    ok = True
    for g in range(0, len(tensors), group):
        sent = torch.stack([t[s_idx] for t in tensors[g:g + group]])
        mine = torch.stack([t[d_idx] for t in tensors[g:g + group]])
        want = torch.empty_like(mine)
        ops = [dist.P2POp(dist.isend, sent, dst_rank), dist.P2POp(dist.irecv, want, src_rank)]
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        torch.cuda.synchronize()
        ok = ok and bool(torch.equal(want, mine))
        del sent, mine, want
    return ok


def _pair_verify(dist, rank, sender, receiver, tensors, ids_sender, ids_receiver, group=16):
    """Same check for one (sender, receiver) pair; returns the verdict on the receiver, None elsewhere."""
    import torch
    if rank == sender:
        idx = torch.from_numpy(np.asarray(ids_sender)).cuda()
        for g in range(0, len(tensors), group):
            dist.send(torch.stack([t[idx] for t in tensors[g:g + group]]), receiver)
        torch.cuda.synchronize()
        return None
    if rank == receiver:
        idx = torch.from_numpy(np.asarray(ids_receiver)).cuda()
        ok = True
        for g in range(0, len(tensors), group):
            mine = torch.stack([t[idx] for t in tensors[g:g + group]])
            want = torch.empty_like(mine)
            dist.recv(want, sender)
            torch.cuda.synchronize()
            ok = ok and bool(torch.equal(want, mine))
        return ok
    return None


def run_migration(kvb, dist, rank, world, local, tensors, pool, pool_blocks, block_bytes, n, steps, warmup,
                  reference_engine=None, blocks_per_file=16, shape_name="8B"):
    """Cross-GPU block migration over NVLink (BASELINE config #4): all-pairs ring r -> r+1, the same exchange through
    NCCL (gather -> send/recv -> scatter) as the library baseline, and — for world > 2 — fan-out rank 0 -> every peer.
    One kernel per destination reads local pages and writes the peer's pages (CUDA IPC mapping).  Every arm is verified
    BYTE FOR BYTE on the receiver after a run into zeroed destination pages; NVLink payload counters are read around
    the timed ring loop."""
    import torch
    part, mig = kvb.partition, kvb.migrate
    descs = part.exchange_objects(mig.export_pool(pool), dist)
    dst_rank, src_rank = part.ring_peers(rank, world)
    payload = n * block_bytes
    half = pool_blocks // 2
    # source pages: the LOWER half of my pool; destination pages: the UPPER half of the peer's pool, so that ring traffic
    # never overwrites pages that are being read
    src_ids = np.random.default_rng(10 + rank).permutation(half)[:n].astype(np.int64)
    dst_ids = (half + np.random.default_rng(20 + rank).permutation(half)[:n]).astype(np.int64)
    all_dst = gather_objects(dist, dst_ids.tolist())
    into_me = np.asarray(all_dst[src_rank], dtype=np.int64)            # where my ring source writes in MY pool
    into_me_dev = torch.from_numpy(into_me).cuda()
    remote = mig.RemotePool(descs[dst_rank], local)
    out = {"shape": shape_name, "blocks": n, "block_bytes": block_bytes, "bytes_per_destination": payload}

    def zero_dst():
        for t in tensors:
            t[into_me_dev] = 0
        barrier_sync(dist)

    def timed(fn, counters=False):
        for _ in range(warmup):
            fn()
        barrier_sync(dist)
        c0 = nvlink_counters(local) if counters else None
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        barrier_sync(dist)
        c1 = nvlink_counters(local) if counters else None
        return max_over_ranks(dist, a.elapsed_time(b)) / steps, c0, c1

    # ---- ring, our kernel
    ring = lambda: mig.migrate_blocks(pool, remote, src_ids, dst_ids)
    ring_ms, c0, c1 = timed(ring, counters=True)
    zero_dst()
    ring()
    barrier_sync(dist)
    oks = gather_objects(dist, _ring_verify(dist, rank, world, tensors, src_ids, into_me))
    tx, rx = _delta(c0, c1, "tx"), _delta(c0, c1, "rx")
    links = gather_objects(dist, {"tx": tx, "rx": rx})
    per_gpu = payload / ring_ms / 1e6
    out["ring"] = {
        "ms": ring_ms, "egress_gbs_per_gpu": per_gpu, "aggregate_gbs": world * per_gpu,
        "bit_exact": oks, "verified": "byte-for-byte on every receiver after a run into zeroed pages (torch.equal of the "
                                      "sender's pages shipped over NCCL against the receiver's destination pages)",
        "frac_of_450": per_gpu / 450.0,
        "roofline": {"bound": "nvlink", "achieved": per_gpu, "peak": 450.0, "unit": "GB/s", "frac": per_gpu / 450.0,
                     "peak_source": "NVLink 4 on H100 SXM (data sheet), per direction per GPU",
                     "traffic": {"what": "NVLink payload bytes per GPU over the timed loop (steps launches), NVML counters",
                                 "expected_tx_bytes": payload * steps, "tx_bytes": [x["tx"] for x in links],
                                 "rx_bytes": [x["rx"] for x in links], "source": (c1 or {}).get("source"),
                                 "tx_over_payload": [None if x["tx"] is None else x["tx"] / (payload * steps) for x in links]}},
    }
    assert all(oks), f"ring migration ({shape_name}) is not bit-exact on every receiver: {oks}"

    # ---- same exchange through NCCL: gather -> packed -> send/recv -> scatter (library baseline)
    packed_s = torch.empty(payload, dtype=torch.uint8, device="cuda")
    packed_r = torch.empty(payload, dtype=torch.uint8, device="cuda")
    src_dev = torch.from_numpy(src_ids).cuda()

    def nccl_step():
        pool.gather_dev(src_dev, packed_s)
        ops = [dist.P2POp(dist.isend, packed_s, dst_rank), dist.P2POp(dist.irecv, packed_r, src_rank)]
        for w in dist.batch_isend_irecv(ops):
            w.wait()
        pool.scatter_dev(into_me_dev, packed_r)

    nccl_ms, _, _ = timed(nccl_step)
    zero_dst()
    nccl_step()
    barrier_sync(dist)
    oks_n = gather_objects(dist, _ring_verify(dist, rank, world, tensors, src_ids, into_me))
    out["ring_nccl_staged"] = {"ms": nccl_ms, "egress_gbs_per_gpu": payload / nccl_ms / 1e6, "bit_exact": oks_n,
                               "note": "gather kernel -> ncclSend/ncclRecv of the packed buffer -> scatter kernel"}
    assert all(oks_n), f"NCCL-staged migration ({shape_name}) is not bit-exact: {oks_n}"
    del packed_s, packed_r

    # ---- fan-out: rank 0 pushes a different prefix to every peer, one kernel per peer on its own stream
    if world > 2:
        peers = [r for r in range(world) if r != 0]
        fan_src = {p: np.random.default_rng(30 + p).permutation(half)[:n].astype(np.int64) for p in peers}
        fan_dst = dst_ids if rank == 0 else None
        fan_dst = gather_objects(dist, None if fan_dst is None else fan_dst.tolist())[0]   # rank 0's list, for everybody
        fan_dst = np.asarray(fan_dst, dtype=np.int64)
        fan_dst_dev = torch.from_numpy(fan_dst).cuda()
        if rank == 0:
            remotes = {p: (remote if p == dst_rank else mig.RemotePool(descs[p], local)) for p in peers}
            streams = {p: torch.cuda.Stream() for p in peers}

            def fan():
                cur = torch.cuda.current_stream()
                ev = torch.cuda.Event()
                ev.record(cur)
                for p in peers:
                    streams[p].wait_event(ev)
                    mig.migrate_blocks(pool, remotes[p], fan_src[p], fan_dst, stream=streams[p])
                for p in peers:
                    cur.wait_stream(streams[p])
        else:
            def fan():
                pass
        fan_ms, f0, f1 = timed(fan, counters=True)
        if rank != 0:
            for t in tensors:
                t[fan_dst_dev] = 0
        barrier_sync(dist)
        fan()
        barrier_sync(dist)
        verdicts = {}
        for p in peers:
            v = _pair_verify(dist, rank, 0, p, tensors, fan_src[p], fan_dst)
            if v is not None:
                verdicts[p] = v
        allv = {}
        for d in gather_objects(dist, verdicts):
            allv.update(d)
        fan_ok = [bool(allv.get(p, False)) for p in peers]
        egress = len(peers) * payload / fan_ms / 1e6
        tx0 = gather_objects(dist, _delta(f0, f1, "tx"))[0]
        out["fanout_rank0"] = {"ms": fan_ms, "destinations": len(peers), "egress_gbs_rank0": egress,
                               "frac_of_450": egress / 450.0, "bit_exact": fan_ok,
                               "verified": "byte-for-byte on each of the destinations after a run into zeroed pages",
                               "roofline": {"bound": "nvlink", "achieved": egress, "peak": 450.0, "unit": "GB/s",
                                            "frac": egress / 450.0,
                                            "traffic": {"expected_tx_bytes_rank0": len(peers) * payload * steps,
                                                        "tx_bytes_rank0": tx0,
                                                        "tx_over_payload": None if not tx0 else tx0 / (len(peers) * payload * steps)}}}
        assert all(fan_ok), f"fan-out migration ({shape_name}) is not bit-exact on every destination: {fan_ok}"
        if rank == 0:
            for p, r in remotes.items():
                if r is not remote:
                    r.close()
    barrier_sync(dist)
    remote.close()

    # ---- status quo for the same hand-off with the reference: no cross-GPU path exists, a block reaches another GPU by
    # being stored by the source worker and loaded by the destination worker through the shared tier (here /dev/shm)
    if reference_engine is not None:
        import shutil
        ref_dir = f"/dev/shm/kvb_ref_migrate_{shape_name}"
        nf = n // blocks_per_file
        files = [f"{ref_dir}/{i:06d}.bin" for i in range(nf)]
        sid = np.random.default_rng(10).permutation(half)[:n].astype(np.int64)   # rank 0's source pages
        did = (half + np.random.default_rng(21).permutation(half)[:n]).astype(np.int64)
        grp = lambda ids: [[int(x) for x in ids[i * blocks_per_file:(i + 1) * blocks_per_file]] for i in range(nf)]
        t_store = t_load = 0.0
        try:
            eng = None
            if rank in (0, 1):
                eng = reference_engine.StorageOffloadEngine(min(64, os.cpu_count() or 1), blocks_per_file,
                                                            [t.view(torch.int8) for t in tensors], 48, "disabled", 0.0)
            barrier_sync(dist)
            if rank == 0:
                shutil.rmtree(ref_dir, ignore_errors=True)
                t0 = time.perf_counter()
                eng.async_store_gpu_blocks(1, files, grp(sid))
                _drain(eng, 1)
                t_store = time.perf_counter() - t0
            barrier_sync(dist)
            if rank == 1:
                t0 = time.perf_counter()
                eng.async_load_gpu_blocks(2, files, grp(did))
                _drain(eng, 2)
                t_load = time.perf_counter() - t0
            barrier_sync(dist)
            t_store, t_load = max_over_ranks(dist, t_store), max_over_ranks(dist, t_load)
            out["via_host_reference_engine"] = {
                "gbs": payload / (t_store + t_load) / 1e9, "store_s": t_store, "load_s": t_load,
                "note": "GPU0 -> /dev/shm -> GPU1 with the unmodified reference engine (store on rank 0, then load on rank 1)"}
            del eng
        except Exception as e:  # never let the comparison take the bench down
            out["via_host_reference_engine"] = {"error": repr(e)}
        if rank == 0:
            shutil.rmtree(ref_dir, ignore_errors=True)
        barrier_sync(dist)
    return out


def _drain(eng, job_id, timeout=900.0, sleep=0.0005):
    t0 = time.perf_counter()
    while time.perf_counter() - t0 < timeout:
        for jid, ok in eng.get_finished():
            if jid == job_id:
                if not ok:
                    raise RuntimeError(f"job {job_id} failed")
                return
        if sleep:
            time.sleep(sleep)
    raise TimeoutError(f"job {job_id}")


# ---------------------------------------------------------------------------------------------------------------------
# config #3: Llama-3-70B GQA paged-KV fp8-e4m3 — 160 tensors x 16 KiB fragments, 2.5 MiB blocks
C3_T, C3_FRAG = 160, 16384
HBM_DATASHEET_GBS = 3350.0   # H100 SXM HBM3, NVIDIA data sheet (not a measurement)
C3_BLOCK = C3_T * C3_FRAG
C3_BLOCKS = int(os.environ.get("KVB_BENCH_C3_BLOCKS", "10000"))
C3_POOL = int(os.environ.get("KVB_BENCH_C3_POOL", "12288"))
C3_E2E_BLOCKS = int(os.environ.get("KVB_BENCH_C3_E2E_BLOCKS", "4000"))


def run_config3(kvb, dist, rank, world, local, steps, warmup, peak, peak_src, reference_engine=None, migrate=True):
    """70B-fp8 block shape: gather / scatter of 10 000 blocks (26.2 GB per pass, pool + packed buffer fit 80 GB of HBM) against the HBM roofline, end-to-end
    save+load of 4 000 blocks through the engine (host arena), and — with peers — the migration of a 32k-token context
    (2048 blocks, 5.37 GB).  One pool per rank (weak scaling), restore checked bit-exact."""
    import torch
    big = torch.empty((C3_T, C3_POOL, C3_FRAG), dtype=torch.uint8, device="cuda")
    big.random_(0, 256, generator=torch.Generator(device="cuda").manual_seed(142 + rank))
    tensors = list(big.unbind(0))
    pool = kvb.pool.KVPool(tensors)
    ids_np = np.random.default_rng(3 + rank).permutation(C3_POOL)[:C3_BLOCKS].astype(np.int64)
    ids_dev = torch.from_numpy(ids_np).cuda()
    payload = C3_BLOCKS * C3_BLOCK
    packed = torch.empty(payload, dtype=torch.uint8, device="cuda")
    sum0 = int(big.view(torch.int64).sum().item())
    k = max(3, min(steps, 10))
    for _ in range(max(3, warmup)):
        pool.gather_dev(ids_dev, packed)
        pool.scatter_dev(ids_dev, packed)
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(k)]
    barrier_sync(dist)
    for e in evs:
        e[0].record()
        pool.gather_dev(ids_dev, packed)
        e[1].record()
        pool.scatter_dev(ids_dev, packed)
        e[2].record()
    barrier_sync(dist)
    g_ms = max_over_ranks(dist, float(np.mean([e[0].elapsed_time(e[1]) for e in evs])))
    s_ms = max_over_ranks(dist, float(np.mean([e[1].elapsed_time(e[2]) for e in evs])))
    # proof: save, ZERO the saved pages, load, whole-pool checksum
    pool.gather_dev(ids_dev, packed)
    big[:, ids_dev] = 0
    assert int(big.view(torch.int64).sum().item()) != sum0
    pool.scatter_dev(ids_dev, packed)
    assert int(big.view(torch.int64).sum().item()) == sum0, "config #3: gather/scatter did not restore the pool bit-exact"
    del packed
    torch.cuda.empty_cache()
    achieved = 2 * payload / g_ms / 1e6
    out = {
        "workload": "BASELINE config #3: Llama-3-70B GQA paged-KV fp8-e4m3, 160 tensors x 16384 B fragments, 2.5 MiB blocks",
        "blocks": C3_BLOCKS, "pool_blocks": C3_POOL, "payload_bytes": payload, "steps": k,
        "l2_policy": f"inputs_exceed_l2 ({payload / 1e9:.1f} GB per pass vs 50 MB L2)",
        "gather_ms": g_ms, "scatter_ms": s_ms,
        "device_save_plus_load_gbs": world * 2 * payload / (g_ms + s_ms) / 1e6, "bit_exact": True,
        "roofline": {"kernel": "paged_copy_bulk_kernel<gather>, 16 KiB fragments", "bound": "hbm", "achieved": achieved,
                     "peak": peak, "unit": "GB/s", "frac": achieved / peak, "peak_source": peak_src,
                     "algorithmic_bytes_per_launch": 2 * payload, "scatter_achieved": 2 * payload / s_ms / 1e6,
                     "frac_of_datasheet": achieved / HBM_DATASHEET_GBS, "traffic": _traffic("gather_traffic_70b.json")},
    }
    # ---- end to end through the engine API (host arena), 4 000 blocks
    bpf = 16
    n16 = C3_E2E_BLOCKS // bpf * bpf
    groups = [ids_np[i * bpf:(i + 1) * bpf].tolist() for i in range(n16 // bpf)]
    eng = kvb.engine.StorageOffloadEngine(4, bpf, tensors, 3, "disabled", 0.0, tier="host_arena",
                                          host_arena_bytes=n16 * C3_BLOCK + (64 << 20), chunk_bytes=80 << 20)
    try:
        def save_load(tag, zero=False):
            files = [f"{tag}/{i:06d}" for i in range(len(groups))]
            assert eng.async_store_gpu_blocks(1, files, groups)
            _drain(eng, 1)
            t_mid = time.perf_counter()
            if zero:
                big[:, ids_dev[:n16]] = 0
                torch.cuda.synchronize()
            t_mid2 = time.perf_counter()
            assert eng.async_load_gpu_blocks(2, files, groups)
            _drain(eng, 2)
            eng.arena_clear()
            return t_mid, t_mid2
        save_load("w", zero=True)
        assert int(big.view(torch.int64).sum().item()) == sum0, "config #3: engine save+load did not restore the pool"
        barrier_sync(dist)
        t0 = time.perf_counter()
        t_mid, _ = save_load("t")
        barrier_sync(dist)
        dt = max_over_ranks(dist, time.perf_counter() - t0)
        st = max_over_ranks(dist, t_mid - t0)
        out["e2e"] = {"value": world * 2 * n16 * C3_BLOCK / dt / 1e9, "unit": "GB/s", "blocks": n16, "tier": "host_arena",
                      "store_gbs": world * n16 * C3_BLOCK / st / 1e9,
                      "load_gbs": world * n16 * C3_BLOCK / max(dt - st, 1e-9) / 1e9,
                      "h2d_bytes": n16 * C3_BLOCK, "d2h_bytes": n16 * C3_BLOCK, "bit_exact": True}
    finally:
        eng.shutdown()
    if world > 1 and migrate:
        out["migration_70b"] = run_migration(kvb, dist, rank, world, local, tensors, pool, C3_POOL, C3_BLOCK, 2048,
                                             max(3, min(steps, 10)), max(3, warmup), reference_engine=None,
                                             shape_name="70B-fp8")
    pool.close()
    del tensors, big
    torch.cuda.empty_cache()
    return out


def _traffic(name):
    """dram read+write bytes per launch from the committed ncu capture of the same kernel at the same size, or None."""
    import json
    p = os.path.join(ROOT, "profiles", name)
    try:
        return json.load(open(p)).get("dram_bytes_per_launch_bench")
    except Exception:
        return None


# ---------------------------------------------------------------------------------------------------------------------
# configs #1 and #5, ingest, manager lookup (rank 0 only: replicas, no exchange)
N_KEYS = int(os.environ.get("KVB_INDEX_KEYS", "10000000"))
N_PROMPTS, N_TOK, BS, N_PODS = 1024, 1000, 16, 64
MODEL = "meta-llama/Llama-3-8B"
SM_HZ = 1.98e9   # H100 SXM maximum SM clock


def _med(fn, iters=9, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def run_index_configs(kvb):
    """BASELINE configs #5 (1024 prompts x 64 pods against a 10 M-key index) and #1 (one 1000-token prompt, 4 pods):
    fused tokens -> scores through the C ABI with HOST buffers in and out, bit-exact against the oracle's C restatement
    at full size, which is also timed on the host cores as the CPU baseline."""
    import torch
    from oracle import kvblock_oracle_c as oc          # checker + CPU baseline
    K = kvb.kvblock
    lib = kvb.lib
    rng = np.random.default_rng(2)
    tp = K.ChunkedTokenDatabase(BS, "")
    tokens = rng.integers(0, 128256, N_PROMPTS * N_TOK).astype(np.uint32)
    off = np.arange(0, (N_PROMPTS + 1) * N_TOK, N_TOK, dtype=np.int64)
    parents = np.full(N_PROMPTS, tp.get_init_hash(MODEL), dtype=np.uint64)
    keys_c, koff = oc.hash_batch(tokens, off, parents, BS)              # oracle keys (C restatement)
    keys_g, koff_g = tp.tokens_to_kv_block_keys_batch([tokens[off[i]:off[i + 1]] for i in range(N_PROMPTS)], MODEL)
    assert np.array_equal(keys_c, keys_g) and np.array_equal(koff, koff_g), "hash parity broken at full size"
    nk = N_TOK // BS
    total_keys = int(koff[-1])

    # ---- index build: prompt prefixes + random background keys, 1..10 entries per key, 80% gpu / 20% cpu.
    # The calls are prepared first so that the timed region is the index build and nothing else.
    pods = ["10.0.%d.%d" % (i // 8, i % 8) for i in range(N_PODS)]
    idx = K.Index(expected_keys=N_KEYS + (1 << 16))
    for p in pods:
        idx.pods.get(p)
    tier_id = {"gpu": idx._tier_id("gpu"), "cpu": idx._tier_id("cpu")}
    n_patterns = 512
    bg = rng.integers(1, 1 << 63, N_KEYS, dtype=np.int64).astype(np.uint64)
    pat_of = rng.integers(0, n_patterns, N_KEYS)
    order = np.argsort(pat_of, kind="stable")
    bounds = np.searchsorted(pat_of[order], np.arange(n_patterns + 1))
    calls = []                                                            # (keys, [(pod index, tier)])
    for pt in range(n_patterns):
        ks = np.ascontiguousarray(bg[order[bounds[pt]:bounds[pt + 1]]])
        if ks.size:
            calls.append((ks, [(int(rng.integers(0, N_PODS)), "gpu" if rng.random() < 0.8 else "cpu")
                               for _ in range(int(rng.integers(1, 11)))]))
    depth = rng.integers(0, nk + 1, N_PROMPTS)
    for i in range(N_PROMPTS):
        d = int(depth[i])
        if d == 0:
            continue
        chain = np.ascontiguousarray(keys_c[koff[i]:koff[i] + d])
        for _ in range(int(rng.integers(1, 5))):
            dd = int(rng.integers(1, d + 1))
            calls.append((chain[:dd], [(int(rng.integers(0, N_PODS)), "gpu" if rng.random() < 0.8 else "cpu")]))
    entry_arrays = [[K.PodEntry(pods[p], t) for p, t in ents] for _, ents in calls]
    n_add_keys = sum(int(ks.size) for ks, _ in calls)
    t0 = time.perf_counter()
    for (ks, _), ents in zip(calls, entry_arrays):
        idx.add(None, ks, ents)
    t_queue = time.perf_counter() - t0
    idx.flush()
    t_build = time.perf_counter() - t0
    st = idx.stats()
    n_index = st["live_keys"]
    # the same build on the host (oracle C restatement, one thread: its table is not concurrent)
    cix = oc.load().kvo_index_new(1 << int(np.ceil(np.log2(N_KEYS * 2.5))))
    t0 = time.perf_counter()
    for ks, ents in calls:
        for p, t in ents:
            oc.load().kvo_index_add(cix, ks.ctypes.data, ks.size, p, tier_id[t])
    t_build_cpu = time.perf_counter() - t0

    # ---- config #5: fused tokens -> scores (pinned host buffers in and out) vs the C restatement on all cores
    pin_tok = kvb.pool.PinnedBuffer(tokens.nbytes)       # kvb_host_alloc: pinned on the GPU's NUMA node
    tok_pin = pin_tok.numpy(np.uint32)
    tok_pin[:] = tokens
    pin_out = kvb.pool.PinnedBuffer(N_PROMPTS * 4 + N_PROMPTS * 13 * 2 + N_PROMPTS * 13 * 8 + 512)
    raw = pin_out.numpy(np.uint8)
    o_n = raw[:N_PROMPTS * 4].view(np.int32)
    o_p = raw[N_PROMPTS * 4:N_PROMPTS * 4 + N_PROMPTS * 26].view(np.uint16)
    base = (N_PROMPTS * 30 + 255) // 256 * 256
    o_s = raw[base:base + N_PROMPTS * 104].view(np.float64)
    out_pinned = (o_n, o_p, o_s)
    out = idx.score_tokens_flat(BS, tok_pin, off, parents, out=out_pinned)
    w = np.ones(256)
    w[tier_id["cpu"]] = 0.8
    c_n, c_p, c_s = np.zeros(N_PROMPTS, np.int32), np.zeros(N_PROMPTS * 13, np.uint16), np.zeros(N_PROMPTS * 13, np.float64)
    oc.load().kvo_score_batch(cix, keys_c.ctypes.data, koff.ctypes.data, N_PROMPTS, w.ctypes.data, c_n.ctypes.data,
                              c_p.ctypes.data, c_s.ctypes.data, 0)
    mism = 0
    for p in range(N_PROMPTS):
        g = {int(out[1][p * 13 + j]): float(out[2][p * 13 + j]) for j in range(int(out[0][p]))}
        c = {int(c_p[p * 13 + j]): float(c_s[p * 13 + j]) for j in range(int(c_n[p]))}
        mism += g != c
    assert mism == 0, f"config #5: {mism} prompts differ from the oracle at full size"

    # the call as a host-language shim makes it: arguments bound once, pinned buffers declared (KVB_SCORE_PINNED_IO)
    raw5 = _raw_call(kvb, idx, tok_pin, off, parents, out_pinned, kvb._lib.SCORE_PINNED_IO)
    launches0 = lib.kvb_launch_count()
    t_fused_pinned = _med(raw5, iters=25, warm=8)
    launches = (lib.kvb_launch_count() - launches0) // 33
    t_fused_py = _med(lambda: idx.score_tokens_flat(BS, tok_pin, off, parents, out=out_pinned), iters=15, warm=5)
    t_two_kernels = _med(_raw_call(kvb, idx, tok_pin, off, parents, out_pinned,
                                   kvb._lib.SCORE_PINNED_IO | kvb._lib.SCORE_TWO_KERNELS | kvb._lib.SCORE_COPY_TOKENS), iters=15, warm=5)
    pg_out = (np.zeros(N_PROMPTS, np.int32), np.zeros(N_PROMPTS * 13, np.uint16), np.zeros(N_PROMPTS * 13, np.float64))
    t_fused_pageable = _med(lambda: idx.score_tokens_flat(BS, tokens, off, parents, out=pg_out), iters=9, warm=3)
    # device time of the two kernels inside the fused call (CUDA events recorded by the library on its own stream)
    hus, sus, fus = [], [], []
    L = kvb._lib
    for _ in range(15):
        _score_timed(kvb, idx, tok_pin, off, parents, out_pinned, L.SCORE_TWO_KERNELS | L.SCORE_COPY_TOKENS)
        s2 = idx.stats()
        hus.append(s2["last_hash_us"])
        sus.append(s2["last_score_us"])
        _score_timed(kvb, idx, tok_pin, off, parents, out_pinned, 0)
        fus.append(idx.stats()["last_hash_us"])
    hash_stage_us, score_us, fused_kernel_us = float(np.median(hus)), float(np.median(sus)), float(np.median(fus))
    # hash kernel alone: everything resident in HBM, CUDA events on the launching stream, back-to-back launches
    d_tok, d_off, d_par = (torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a.view(np.int64)).cuda()
                           for a in (tokens, off, parents))
    d_koff = torch.from_numpy(koff_g).cuda()
    d_keys = torch.empty(total_keys, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream()

    def hash_dev():
        kvb._lib.check(lib.kvb_hash_token_blocks_dev(0, d_tok.data_ptr(), d_off.data_ptr(), d_par.data_ptr(), N_PROMPTS, BS,
                                                     None, None, d_keys.data_ptr(), d_koff.data_ptr(), total_keys, stream.cuda_stream))
    for _ in range(20):
        hash_dev()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(100)]
    torch.cuda.synchronize()
    for a, b in evs:
        a.record(stream)
        hash_dev()
        b.record(stream)
    torch.cuda.synchronize()
    t_hash_kernel = float(np.median([a.elapsed_time(b) for a, b in evs])) * 1e-3
    # The same kernel inside a LONG burst with the SM clock sampled while it runs (NVML): a 50 us kernel timed in a 6 ms
    # burst runs before the clock has ramped (~1.45 GHz observed in round 1), which says more about the power state than
    # about the kernel.  ~0.3 s of back-to-back launches, the last 100 timed, clock read during them.
    hash_warm = {"us": None, "sm_mhz": None}
    try:
        if os.environ.get("KVB_BENCH_NO_BURST"):   # 6 100 launches: far too many to replay under ncu
            raise RuntimeError("skipped: KVB_BENCH_NO_BURST is set")
        import pynvml
        pynvml.nvmlInit()
        h_nv = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        for _ in range(6000):
            hash_dev()
        evs2 = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(100)]
        mhz = []
        for i, (a, b) in enumerate(evs2):
            a.record(stream)
            hash_dev()
            b.record(stream)
            if i % 10 == 0:
                mhz.append(pynvml.nvmlDeviceGetClockInfo(h_nv, pynvml.NVML_CLOCK_SM))
        torch.cuda.synchronize()
        hash_warm = {"us": float(np.median([a.elapsed_time(b) for a, b in evs2])) * 1e3, "sm_mhz": float(np.median(mhz)),
                     "sm_max_mhz": float(pynvml.nvmlDeviceGetMaxClockInfo(h_nv, pynvml.NVML_CLOCK_SM)),
                     "how": "6000 back-to-back launches (~0.3 s), then 100 timed with CUDA events; SM clock from NVML during them"}
    except Exception as e:  # the number above stands on its own
        hash_warm["error"] = repr(e)
    assert np.array_equal(d_keys.cpu().numpy().view(np.uint64), keys_c), "device-resident hash differs from the oracle"
    vote_floor = (N_TOK // BS) * (8 * 61 + 80 + 15) / SM_HZ
    cores = os.cpu_count() or 1
    sweep = [t for t in (1, 8, 32, 64, 128, 256) if t <= cores]
    hash_by_t = {t: _med(lambda t=t: oc.hash_batch(tokens, off, parents, BS, threads=t), iters=5, warm=2) for t in sweep}
    score_by_t = {t: _med(lambda t=t: oc.load().kvo_score_batch(cix, keys_c.ctypes.data, koff.ctypes.data, N_PROMPTS,
                                                                  w.ctypes.data, c_n.ctypes.data, c_p.ctypes.data,
                                                                  c_s.ctypes.data, t), iters=5, warm=2) for t in sweep}
    t_c_best = min(hash_by_t.values()) + min(score_by_t.values())
    probe_bytes = total_keys * 64
    cfg5 = {
        "workload": "BASELINE config #5: 1024 prompts x 1000 tokens, 64 pods, 10 M-key index, longest-prefix match",
        "prompts": N_PROMPTS, "pods": N_PODS, "index_keys": int(n_index), "keys_scored": total_keys,
        "bit_exact_vs_oracle": True,
        "fused_tokens_to_scores_ms": t_fused_pinned * 1e3, "prompts_per_s": N_PROMPTS / t_fused_pinned,
        "keys_per_s": total_keys / t_fused_pinned, "kernels_per_call": int(launches),
        "fused_pageable_buffers_ms": t_fused_pageable * 1e3, "fused_through_python_wrapper_ms": t_fused_py * 1e3,
        "two_kernels_after_token_copy_ms": t_two_kernels * 1e3,
        "api": "kvb_index_score_tokens_batch (C ABI, arguments bound once): pinned host tokens read in place by ONE fused launch, "
               "(pod, score) pairs written to pinned host memory, recency refreshed (default), completion word instead of a stream sync",
        "h2d_bytes_per_call": int(tokens.nbytes + off.nbytes + parents.nbytes), "d2h_bytes_per_call": N_PROMPTS * (4 + 13 * 10),
        "fused_kernel_us_in_call": fused_kernel_us,
        "two_kernel_mode": {"token_copy_plus_hash_us": hash_stage_us, "score_kernel_us": score_us},
        "hash_kernel": {"device_resident_us": t_hash_kernel * 1e6, "keys_per_s": total_keys / t_hash_kernel,
                        "bound": "latency of dependent warp instructions (vote rounds), not HBM",
                        "floor_us": vote_floor * 1e6, "frac_of_floor": vote_floor / t_hash_kernel,
                        "floor": "62 blocks x (8 rounds x 61 + 4 REDUX 80 + multiply 15) cycles at 1.98 GHz",
                        "in_a_long_burst": dict(hash_warm, frac_of_floor=(vote_floor * 1e6 / hash_warm["us"]) if hash_warm.get("us") else None)},
        "roofline": {"kernel": "index_score_kernel", "bound": "hbm", "achieved": probe_bytes / (score_us * 1e-6) / 1e9 if score_us else None,
                     "peak": None, "unit": "GB/s", "frac": None, "traffic": _traffic("score_traffic.json"),
                     "algorithmic_bytes_per_launch": probe_bytes,
                     "note": "random 64 B probes (2 sectors each) followed by a serial float64 walk per prompt: latency-bound, "
                             "the HBM fraction is reported by bench.py against the measured copy peak for completeness"},
        "cpu_baseline": {"kind": "port", "cores": cores, "unit": "ms", "value": t_c_best * 1e3,
                         "hash_ms_by_threads": {str(k): v * 1e3 for k, v in hash_by_t.items()},
                         "score_ms_by_threads": {str(k): v * 1e3 for k, v in score_by_t.items()},
                         "sample": "the whole batch; best thread count per phase (OpenMP team start-up dominates at 128+)",
                         "note": "plain-C restatement without Go's allocations/mutexes: faster than the reference would be"},
        "speedup_vs_best_cpu": t_c_best / t_fused_pinned,
        "index_build": {"keys_added": int(n_add_keys), "add_calls": len(calls), "queue_s": t_queue, "total_s": t_build,
                        "keys_per_s": n_add_keys / t_build, "flushes_parallel": st["flushes_parallel"],
                        "flushes_sequential": st["flushes_sequential"], "rehashes": st["rehashes"],
                        "table_slots": st["table_slots"],
                        "cpu_c_restatement_1_thread_s": t_build_cpu, "where": "Add/Evict applied by kernels, no host copy"},
    }

    # ---- small batches against the same 10 M-key index: 4 / 16 / 64 prompts per call (the table kernel takes up to 32)
    small = {}
    for nb in (4, 16, 64):
        off_b, par_b = np.ascontiguousarray(off[:nb + 1]), np.ascontiguousarray(parents[:nb])
        for a in out_pinned:
            a[:] = 0
        call_b = _raw_call(kvb, idx, tok_pin, off_b, par_b, out_pinned, kvb._lib.SCORE_PINNED_IO)
        call_b()
        for p in range(nb):
            g = {int(o_p[p * 13 + j]): float(o_s[p * 13 + j]) for j in range(int(o_n[p]))}
            c = {int(c_p[p * 13 + j]): float(c_s[p * 13 + j]) for j in range(int(c_n[p]))}
            assert g == c, f"small batch of {nb}: prompt {p} differs from the oracle"
        t_b = _med(call_b, iters=200, warm=30)
        kb_, nb_, pb_, sb_ = np.zeros(nb * nk, np.uint64), np.zeros(nb, np.int32), np.zeros(nb * 13, np.uint16), np.zeros(nb * 13, np.float64)
        koff_b = np.ascontiguousarray(koff[:nb + 1])

        def c_small(threads):
            oc.load().kvo_hash_batch(tokens.ctypes.data, off_b.ctypes.data, par_b.ctypes.data, nb, BS, None, None, kb_.ctypes.data,
                                     koff_b.ctypes.data, threads)
            oc.load().kvo_score_batch(cix, kb_.ctypes.data, koff_b.ctypes.data, nb, w.ctypes.data, nb_.ctypes.data, pb_.ctypes.data,
                                      sb_.ctypes.data, threads)
        t_c1 = _med(lambda: c_small(1), iters=40, warm=5)
        t_cn = _med(lambda: c_small(min(nb, os.cpu_count() or 1)), iters=40, warm=5)
        small[str(nb)] = {"us_per_call": t_b * 1e6, "prompts_per_s": nb / t_b, "bit_exact_vs_oracle": True,
                          "cpu_c_restatement_us": {"1_thread": t_c1 * 1e6, "%d_threads" % min(nb, os.cpu_count() or 1): t_cn * 1e6}}
    cfg5["small_batches"] = small

    # ---- the index AT CAPACITY: exact-LRU eviction; an add-only batch is applied in parallel with its victims planned up
    # front (DESIGN.md section 5, "Planned")
    cap = 1 << 20
    idx_c = K.Index(size=cap, expected_keys=cap)
    fill = rng.integers(1, 1 << 62, cap + 200_100, dtype=np.int64).astype(np.uint64)
    ent_c = [K.PodEntry(pods[0], "gpu")]
    idx_c.add(None, fill[:cap], ent_c)
    idx_c.flush()
    idx_c.add(None, fill[cap:cap + 100], ent_c)        # first batch at capacity: builds the order array, allocates the planner
    idx_c.flush()
    t0 = time.perf_counter()
    idx_c.add(None, fill[cap + 100:], ent_c)
    idx_c.flush()
    t_cap = time.perf_counter() - t0
    st_c = idx_c.stats()
    assert st_c["live_keys"] == cap and st_c["lru_evictions"] == 200_100, st_c
    survivors = idx_c.lookup(fill[[0, 200_099, 200_100, cap - 1, cap, cap + 200_099]])
    assert set(int(k) for k in survivors) == {int(fill[200_100]), int(fill[cap - 1]), int(fill[cap]), int(fill[cap + 200_099])}
    cfg5["index_at_capacity"] = {"size": cap, "new_keys": 200_000, "seconds": t_cap, "keys_per_s": 200_000 / t_cap,
                                 "lru_evictions": st_c["lru_evictions"] - 100, "order_builds": st_c["order_builds"],
                                 "flushes_planned": st_c["flushes_planned"], "plan_fallbacks": st_c["plan_fallbacks"],
                                 "exact": "the 200 000 oldest keys were evicted, in insertion order (checked on the boundaries)"}
    # a mixed batch at capacity: 150 000 new keys interleaved with 30 000 removals of resident keys' only pod (those keys
    # disappear, so live moves both ways inside the batch); queued first, the flush is what is timed
    fresh = rng.integers(1, 1 << 62, 150_000, dtype=np.int64).astype(np.uint64)
    gone = fill[cap - 30_000:cap]                      # among the newest residents: not evicted by this batch
    for c in range(30):
        idx_c.add(None, fresh[c * 5000:(c + 1) * 5000], ent_c)
        for k in gone[c * 1000:(c + 1) * 1000]:
            idx_c.evict(int(k), K.REQUEST_KEY, ent_c)
    t0 = time.perf_counter()
    idx_c.flush()
    t_mix = time.perf_counter() - t0
    st_m = idx_c.stats()
    # live peaks after the 30th group of adds: 29 x (5000 - 1000) + 5000 above Size -> 121 000 evictions; the last 1000
    # removals come after the last insertion and leave the index 1000 short of full
    assert st_m["live_keys"] == cap - 1000 and st_m["lru_evictions"] == 200_100 + 121_000, st_m
    assert len(idx_c.lookup(gone[::1000])) == 0 and len(idx_c.lookup(fresh[::1000])) == 150
    cfg5["index_at_capacity"]["mixed_batch"] = {
        "ops": 180_000, "adds": 150_000, "removals_that_delete_a_key": 30_000, "flush_seconds": t_mix,
        "ops_per_s": 180_000 / t_mix, "lru_evictions": st_m["lru_evictions"] - st_c["lru_evictions"],
        "flushes_planned": st_m["flushes_planned"] - st_c["flushes_planned"],
        "plan_fallbacks": st_m["plan_fallbacks"] - st_c["plan_fallbacks"]}
    idx_c.close()

    # ---- config #1: one prompt, 4 pods
    idx1 = K.Index()
    tok1 = np.random.default_rng(0).integers(0, 128256, 1000).astype(np.uint32)
    off1 = np.array([0, 1000], dtype=np.int64)
    par1 = parents[:1].copy()
    k1, _ = oc.hash_batch(tok1, off1, par1, BS)
    for i in range(4):
        idx1.add(None, k1[: 62 * (i + 1) // 4], [K.PodEntry("pod-%d" % i, "gpu")])
    idx1.add(None, k1[:20], [K.PodEntry("pod-3", "cpu")])
    pin1 = kvb.pool.PinnedBuffer(4096)
    t1buf = pin1.numpy(np.uint32)[:1000]
    t1buf[:] = tok1
    pin1o = kvb.pool.PinnedBuffer(1024)
    r1 = pin1o.numpy(np.uint8)
    o1 = (r1[:4].view(np.int32), r1[64:64 + 26].view(np.uint16), r1[256:256 + 104].view(np.float64))
    idx1.score_tokens_flat(BS, t1buf, off1, par1, out=o1)
    got = {idx1.pods.names[int(o1[1][j])]: float(o1[2][j]) for j in range(int(o1[0][0]))}
    assert got == {"pod-0": 15.0, "pod-1": 31.0, "pod-2": 46.0, "pod-3": 62.0}, got
    raw1 = _raw_call(kvb, idx1, t1buf, off1, par1, o1, kvb._lib.SCORE_PINNED_IO)
    raw1()
    got_raw = {idx1.pods.names[int(o1[1][j])]: float(o1[2][j]) for j in range(int(o1[0][0]))}
    assert got_raw == got, got_raw
    t1 = _med(raw1, iters=500, warm=50)
    t1_wrapped = _med(lambda: idx1.score_tokens_flat(BS, t1buf, off1, par1, out=o1), iters=300, warm=50)
    ix = kvb.indexer.Indexer(tp, idx1)
    t1_py = _med(lambda: ix.score_tokens(tok1, MODEL), iters=100, warm=10)
    cix1 = oc.load().kvo_index_new(1 << 10)
    for i in range(4):
        oc.load().kvo_index_add(cix1, k1.ctypes.data, 62 * (i + 1) // 4, i, 0)
    n1, p1, s1 = np.zeros(1, np.int32), np.zeros(13, np.uint16), np.zeros(13, np.float64)

    def c_one():
        kk, ko = oc.hash_batch(tok1, off1, par1, BS, threads=1)
        oc.load().kvo_score_batch(cix1, kk.ctypes.data, ko.ctypes.data, 1, w.ctypes.data, n1.ctypes.data, p1.ctypes.data,
                                  s1.ctypes.data, 1)
    t1_c = _med(c_one, iters=300, warm=50)
    cfg1 = {"workload": "BASELINE config #1: ScoreTokens, one 1000-token prompt, 16-token blocks, 4 pods",
            "keys": 62, "us_per_call": t1 * 1e6, "calls_per_s": 1.0 / t1, "python_wrapper_us_per_call": t1_wrapped * 1e6,
            "python_indexer_us_per_call": t1_py * 1e6,
            "api": "kvb_index_score_tokens_batch through the C ABI with bound arguments and pinned buffers: one fused launch, the "
                   "prompt's offsets and parent in the kernel arguments, tokens read in place, completion word",
            "known_answer": got, "bit_exact_vs_known_answer": True,
            "cpu_baseline": {"kind": "port", "cores": 1, "unit": "us", "value": t1_c * 1e6,
                             "sample": "the same call, C restatement on one core"},
            "note": "one prompt is ONE serial chain of 62 dependent block hashes; the table kernel (hash_spec_kernel) moves the "
                    "token bytes off that chain (FNV-1a is linear above the byte it xors into), the chain keeps ~310 cycles per block"}
    for b in (pin_tok, pin_out, pin1, pin1o):
        b.free()
    idx.close()
    idx1.close()
    return cfg1, cfg5


def _raw_call(kvb, idx, tokens, off, parents, out, flags):
    fn = idx._lib.kvb_index_score_tokens_batch
    args = (idx._h, tokens.ctypes.data, off.ctypes.data, parents.ctypes.data, len(off) - 1, BS, None, None, None, 0, int(flags),
            out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data)

    def call():
        rc = fn(*args)
        assert rc == 0, rc
    return call


def _score_timed(kvb, idx, tokens, off, parents, out, flags=0):
    n = len(off) - 1
    idx._check(idx._lib.kvb_index_score_tokens_batch(
        idx._h, tokens.ctypes.data, off.ctypes.data, parents.ctypes.data, n, BS, None, None, None, 0,
        kvb._lib.SCORE_TIME_KERNELS | int(flags), out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data))


def run_ingest(kvb):
    """KV-event ingest (SURVEY §8f rank 1): BlockStored / BlockRemoved streams of 64 pods through EventProcessor.process_many
    (device hashing + device index updates) next to the oracle's restatement of pool.go:253-398, same stream, final index
    state compared on a sample."""
    from oracle import kvblock_oracle as ko
    from oracle import kvevents_oracle as keo
    K, E = kvb.kvblock, kvb.kvevents
    rng = np.random.default_rng(5)
    n_pods, ev_per_pod, blocks_per_ev = 64, 24, 8
    work, owork = [], []
    h = 1
    for p in range(n_pods):
        evs, oevs, parent, stored = [], [], 0, []
        for e in range(ev_per_pod):
            if stored and rng.random() < 0.15:
                victim = stored.pop(int(rng.integers(0, len(stored))))
                evs.append(E.BlockRemovedEvent([victim], "gpu"))
                oevs.append(keo.BlockRemoved([victim], "gpu"))
                continue
            hashes = list(range(h, h + blocks_per_ev))
            h += blocks_per_ev
            toks = [int(t) for t in rng.integers(0, 128256, blocks_per_ev * BS)]
            evs.append(E.BlockStoredEvent(hashes, toks, parent, "gpu"))
            oevs.append(keo.BlockStored(hashes, toks, parent, "gpu"))
            parent = hashes[-1]
            stored.extend(hashes)
        work.append(("pod-%d" % p, MODEL, evs))
        owork.append(("pod-%d" % p, MODEL, oevs))
    n_events = sum(len(w[2]) for w in work)
    n_keys = sum(len(e.block_hashes) for w in work for e in w[2] if isinstance(e, E.BlockStoredEvent))
    tp = K.ChunkedTokenDatabase(BS, "")
    idx = K.Index()
    proc = E.EventProcessor(idx, tp)
    t0 = time.perf_counter()
    proc.process_many(work)
    idx.flush()
    dt = time.perf_counter() - t0
    # the same batch through the native entry point (kvb_index_ingest_events): Python only flattens the batch
    idx_n = K.Index()
    proc_n = E.EventProcessor(idx_n, tp)
    proc_n.process_many_native(work[:2])          # warm: interners, scratch
    idx_n.close()
    idx_n = K.Index()
    proc_n = E.EventProcessor(idx_n, tp)
    t0 = time.perf_counter()
    flat = proc_n.flatten_events(work)            # Python: event objects -> the C-ABI arrays
    t1 = time.perf_counter()
    proc_n.ingest_flat(flat)                      # ONE library call
    idx_n.flush()
    t2 = time.perf_counter()
    dt_n, dt_call = t2 - t0, t2 - t1
    oidx, otp = ko.InMemoryIndex(), ko.TokenProcessor(BS, "")
    t0 = time.perf_counter()
    for pod, model, evs in owork:
        keo.process_event_batch(oidx, otp, evs, pod, model)
    dt_o = time.perf_counter() - t0
    assert len(idx) == len(oidx.data), "ingest: index sizes differ from the oracle"
    sample = list(oidx.data.d.keys())[:: max(1, len(oidx.data) // 500)]
    got = {k: sorted((e.pod_identifier, e.device_tier) for e in v) for k, v in idx.lookup(sample).items()}
    want = {k: sorted((e.pod_identifier, e.device_tier) for e in v) for k, v in oidx.lookup(sample).items()}
    assert got == want, "ingest: index contents differ from the oracle"
    assert len(idx_n) == len(oidx.data), "native ingest: index sizes differ from the oracle"
    got_n = {k: sorted((e.pod_identifier, e.device_tier) for e in v) for k, v in idx_n.lookup(sample).items()}
    assert got_n == want, "native ingest: index contents differ from the oracle"
    # CPU baseline closer to the reference's cost: hashing by the oracle's C restatement (one thread, event by event, chained
    # parents) — its index is not part of this figure, so it flatters the CPU
    from oracle import kvblock_oracle_c as oc
    root = tp.get_init_hash(MODEL)
    t0 = time.perf_counter()
    for pod, model, evs in owork:
        last = {}
        for ev in evs:
            if isinstance(ev, keo.BlockStored):
                toks = np.asarray(ev.tokens, dtype=np.uint32)
                par = np.asarray([last.get(ev.parent_hash, root)], dtype=np.uint64)
                ks, _ = oc.hash_batch(toks, np.asarray([0, toks.size], dtype=np.int64), par, BS, threads=1)
                if ks.size:
                    last[ev.block_hashes[-1]] = int(ks[-1])
    dt_c = time.perf_counter() - t0
    idx.close()
    idx_n.close()
    return {"events": n_events, "block_keys": n_keys, "pods": n_pods, "events_per_s": n_events / dt, "keys_per_s": n_keys / dt,
            "seconds": dt, "api": "EventProcessor.process_many (Python host logic; device hashing, device index updates)",
            "native": {"events_per_s": n_events / dt_n, "keys_per_s": n_keys / dt_n, "seconds": dt_n,
                       "library_call_only": {"events_per_s": n_events / dt_call, "keys_per_s": n_keys / dt_call, "seconds": dt_call,
                                             "what": "kvb_index_ingest_events + flush on the already flattened batch: what a host-"
                                                     "language shim that decodes into these arrays pays"},
                       "api": "kvb_index_ingest_events: one library call for the decoded batch (parents, hashing per round, engine map, "
                              "device index ops); Python only flattens the events", "bit_exact_vs_oracle": True},
            "cpu_c_hash_only_1_thread": {"events_per_s": n_events / dt_c, "seconds": dt_c,
                                          "what": "the hashing of the same stream by the oracle's C restatement, event by event on one "
                                                  "core (no index work): a floor for a single reference worker shard"},
            "bit_exact_vs_oracle": True,
            "cpu_baseline": {"kind": "port", "cores": 1, "unit": "events/s", "value": n_events / dt_o,
                             "sample": "the same stream through the oracle's pure-Python restatement of pool.go:253-398"}}


def run_manager_lookup(kvb, n_hashes=2048):
    """SharedStorageOffloadingManager.lookup over 2048 block hashes, all offloaded: ONE kvb_engine_lookup_prefix call
    against the reference's per-block existence loop (manager.py:43-53), host-arena tier (small scratch pool)."""
    import torch
    bpf = 1
    tensors = [torch.zeros((64, 4096), dtype=torch.uint8, device="cuda") for _ in range(4)]
    fm = kvb.file_mapper.FileMapper("/kvb_bench_lookup", "m", 16, bpf, 1, 1, 1, 0, "torch.uint8")
    eng = kvb.engine.StorageOffloadEngine(2, bpf, tensors, 1, "disabled", 0.0, tier="host_arena",
                                          host_arena_bytes=n_hashes * 4 * 4096 + (8 << 20))
    try:
        hashes = [int(i + 1).to_bytes(8, "little") for i in range(n_hashes)]
        files = [fm.get_file_name(h) for h in hashes]
        assert eng.async_store_gpu_blocks(1, files, [[i % 64] for i in range(n_hashes)])
        _drain(eng, 1)
        batch = kvb.manager.SharedStorageOffloadingManager(fm, engine=eng)
        loop = kvb.manager.SharedStorageOffloadingManager(fm, exists=eng.exists)
        assert batch.lookup(hashes) == loop.lookup(hashes) == n_hashes
        assert batch.lookup(hashes[:100] + [b"\xff" * 8] + hashes[100:]) == loop.lookup(hashes[:100] + [b"\xff" * 8] + hashes[100:]) == 100
        t_batch = _med(lambda: batch.lookup(hashes), iters=20, warm=3)
        t_loop = _med(lambda: loop.lookup(hashes), iters=10, warm=2)
        low64 = kvb.file_mapper.hashes_low64(hashes)
        t_c_only = _med(lambda: eng.lookup_prefix_hashes(fm.base_path, low64), iters=20, warm=3)
        return {"hashes": n_hashes, "one_call_us": t_batch * 1e6, "per_block_loop_us": t_loop * 1e6,
                "library_call_only_us": t_c_only * 1e6, "speedup": t_loop / t_batch, "tier": "host_arena",
                "same_answer_as_the_loop": True,
                "note": "one_call = manager.lookup(block_hashes): bytes hashes -> uint64 (vectorised) -> ONE C call that builds "
                        "the file names and probes the arena; per_block_loop = the reference's loop (manager.py:43-53) with "
                        "one existence probe per block"}
    finally:
        eng.shutdown()
