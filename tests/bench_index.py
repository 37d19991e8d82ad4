#!/usr/bin/env python
"""BASELINE configs #1 and #5: block-key hashing + index lookup + longest-prefix scoring.

  #5  1024 prompts x 1000 tokens, 64 pods, 10 M-entry index: fused tokens -> scores on the GPU through the C ABI
      (host buffers in, host buffers out), next to the oracle's C restatement on all host cores, results compared
      bit-exact at full size.
  #1  one 1000-token prompt, 16-token blocks, 4 pods: latency of one ScoreTokens call.
Prints one JSON object; the summary is kept under profiles/."""
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

kvb = importlib.import_module("llm-d-kv-cache_b200")
from oracle import kvblock_oracle_c as oc  # noqa: E402  (CPU baseline + full-size parity check)

N_KEYS = int(os.environ.get("KVB_INDEX_KEYS", "10000000"))
N_PROMPTS, N_TOK, BS, N_PODS = 1024, 1000, 16, 64
MODEL = "meta-llama/Llama-3-8B"


def med(fn, iters=7, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    torch.cuda.set_device(0)
    K = kvb.kvblock
    rng = np.random.default_rng(2)
    tp = K.ChunkedTokenDatabase(BS, "")
    tokens = rng.integers(0, 128256, N_PROMPTS * N_TOK).astype(np.uint32)
    off = np.arange(0, (N_PROMPTS + 1) * N_TOK, N_TOK, dtype=np.int64)
    parents = np.full(N_PROMPTS, tp.get_init_hash(MODEL), dtype=np.uint64)
    keys_c, koff = oc.hash_batch(tokens, off, parents, BS)              # oracle keys (C restatement)
    keys_g, koff_g = tp.tokens_to_kv_block_keys_batch([tokens[off[i]:off[i + 1]] for i in range(N_PROMPTS)], MODEL)
    assert np.array_equal(keys_c, keys_g) and np.array_equal(koff, koff_g), "hash parity broken at full size"
    nk = N_TOK // BS

    # ---- index: prompt prefixes + random background keys, 1..10 entries per key, 80% gpu / 20% cpu
    pods = ["10.0.%d.%d" % (i // 8, i % 8) for i in range(N_PODS)]
    t0 = time.perf_counter()
    idx = K.Index(expected_keys=N_KEYS + (1 << 16))
    cix = oc.load().kvo_index_new(1 << int(np.ceil(np.log2(N_KEYS * 2.5))))
    for p in pods:
        idx.pods.get(p)
    tier_id = {"gpu": idx._tier_id("gpu"), "cpu": idx._tier_id("cpu")}
    n_patterns = 512
    bg = rng.integers(1, 1 << 63, N_KEYS, dtype=np.int64).astype(np.uint64)
    pat_of = rng.integers(0, n_patterns, N_KEYS)
    order = np.argsort(pat_of, kind="stable")
    bounds = np.searchsorted(pat_of[order], np.arange(n_patterns + 1))
    for pt in range(n_patterns):
        ks = np.ascontiguousarray(bg[order[bounds[pt]:bounds[pt + 1]]])
        if ks.size == 0:
            continue
        ents = [(int(rng.integers(0, N_PODS)), "gpu" if rng.random() < 0.8 else "cpu") for _ in range(int(rng.integers(1, 11)))]
        idx.add(None, ks, [K.PodEntry(pods[p], t) for p, t in ents])
        for p, t in ents:
            oc.load().kvo_index_add(cix, ks.ctypes.data, ks.size, p, tier_id[t])
    depth = rng.integers(0, nk + 1, N_PROMPTS)
    for i in range(N_PROMPTS):
        d = int(depth[i])
        if d == 0:
            continue
        chain = np.ascontiguousarray(keys_c[koff[i]:koff[i] + d])
        for _ in range(int(rng.integers(1, 5))):
            dd = int(rng.integers(1, d + 1))
            p, t = int(rng.integers(0, N_PODS)), ("gpu" if rng.random() < 0.8 else "cpu")
            idx.add(None, chain[:dd], [K.PodEntry(pods[p], t)])
            oc.load().kvo_index_add(cix, chain.ctypes.data, dd, p, tier_id[t])
    t_build_host = time.perf_counter() - t0
    t0 = time.perf_counter()
    kvb._lib.check(kvb.lib.kvb_index_flush(idx._h, None))
    t_flush = time.perf_counter() - t0
    n_index = len(idx)

    # ---- config #5: fused tokens -> scores (host in, host out) vs C restatement on all cores
    out = idx.score_tokens_flat(BS, tokens, off, parents)
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
    assert mism == 0, f"{mism} prompts differ from the oracle at full size"

    launches0 = kvb.lib.kvb_launch_count()
    t_fused = med(lambda: idx.score_tokens_flat(BS, tokens, off, parents, out=out))
    launches = (kvb.lib.kvb_launch_count() - launches0) // 9
    # same call with the tokens in pinned host memory (kvb_host_alloc / cudaHostAlloc): no staging memcpy
    pin1 = kvb.pool.PinnedBuffer(tokens.nbytes)  # kvb_host_alloc: pinned on the GPU's NUMA node
    tok_pin = pin1.numpy(np.uint32)
    tok_pin[:] = tokens
    t_fused_pinned = med(lambda: idx.score_tokens_flat(BS, tok_pin, off, parents, out=out))
    # 8x the batch (8192 prompts): fixed per-call costs amortise
    reps = 8
    pin8 = kvb.pool.PinnedBuffer(tokens.nbytes * reps)
    tok8 = pin8.numpy(np.uint32)
    tok8[:] = np.tile(tokens, reps)
    off8 = np.arange(0, (N_PROMPTS * reps + 1) * N_TOK, N_TOK, dtype=np.int64)
    par8 = np.tile(parents, reps)
    t_fused8 = med(lambda: idx.score_tokens_flat(BS, tok8, off8, par8), iters=5)
    t_hash_gpu = med(lambda: kvb._lib.check(kvb.lib.kvb_hash_token_blocks(
        0, tokens.ctypes.data, off.ctypes.data, parents.ctypes.data, N_PROMPTS, BS, None, None, keys_g.ctypes.data,
        koff_g.ctypes.data, None)))
    # kernel alone: everything resident in HBM, CUDA events on the launching stream
    d_tok, d_off, d_par = (torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a.view(np.int64)).cuda()
                           for a in (tokens, off, parents))
    d_koff = torch.from_numpy(koff_g).cuda()
    d_keys = torch.empty(int(koff_g[-1]), dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream()

    def hash_dev():
        kvb._lib.check(kvb.lib.kvb_hash_token_blocks_dev(0, d_tok.data_ptr(), d_off.data_ptr(), d_par.data_ptr(), N_PROMPTS, BS,
                                                         None, None, d_keys.data_ptr(), d_koff.data_ptr(), int(koff_g[-1]), st.cuda_stream))
    for _ in range(5):
        hash_dev()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(50)]
    torch.cuda.synchronize()
    for a, b in evs:
        a.record(st)
        hash_dev()
        b.record(st)
    torch.cuda.synchronize()
    t_hash_kernel = float(np.median([a.elapsed_time(b) for a, b in evs])) * 1e-3
    assert np.array_equal(d_keys.cpu().numpy().view(np.uint64), keys_c), "device-resident hash differs from the oracle"
    # latency floors (DESIGN.md section 4), all chains concurrent so the LONGEST chain bounds the launch:
    #  - byte-serial formulation (lane per prompt): one dependent xor -> 64-bit multiply per CBOR byte, 12.3 cycles per
    #    byte on a lone in-order warp (model constant; tools/micro/hash_phase_profile.cu measures it)
    #  - vote-round formulation (warp per prompt, the kernel used for <= 1536 prompts): per block 8 rounds of
    #    IMAD -> LOP3 -> LOP3.P -> VOTE -> LOP3 -> POPC -> SHL -> LOP3 (61 cycles) + 4x REDUX and recombine (80) + the
    #    64-bit multiply (15)  (model constants; tools/micro/warp_chain_latency.cu measures them)
    full = tokens.reshape(N_PROMPTS, N_TOK)[:, : (N_TOK // BS) * BS]
    width = np.where(full < 24, 1, np.where(full < 256, 2, np.where(full < 65536, 3, 5)))
    chain_bytes = width.sum(axis=1) + (N_TOK // BS) * (1 + 9 + 1 + 1)        # 0x83, uint64 parent, array head, null extra
    sm_hz = 1.98e9   # H100 SXM maximum SM clock
    byte_floor = float(chain_bytes.max()) * 12.3 / sm_hz
    vote_floor = (N_TOK // BS) * (8 * 61 + 80 + 15) / sm_hz
    cores = os.cpu_count() or 1
    # CPU baseline = the BEST thread count for each phase (OpenMP team start-up dominates a 0.1 ms job at 128 threads)
    sweep = [t for t in (1, 4, 8, 16, 32, 64, 128, 256) if t <= cores]
    hash_by_t = {t: med(lambda t=t: oc.hash_batch(tokens, off, parents, BS, threads=t), iters=5, warm=2) for t in sweep}
    score_by_t = {t: med(lambda t=t: oc.load().kvo_score_batch(cix, keys_c.ctypes.data, koff.ctypes.data, N_PROMPTS,
                                                                 w.ctypes.data, c_n.ctypes.data, c_p.ctypes.data,
                                                                 c_s.ctypes.data, t), iters=5, warm=2) for t in sweep}
    t_c_hash_all, t_c_hash_1 = min(hash_by_t.values()), hash_by_t[1]
    t_c_score_all, t_c_score_1 = min(score_by_t.values()), score_by_t[1]
    total_keys = int(koff[-1])
    cfg5 = {
        "prompts": N_PROMPTS, "tokens_per_prompt": N_TOK, "pods": N_PODS, "index_keys": n_index, "keys_scored": total_keys,
        "bit_exact_vs_oracle": True,
        "gpu_fused_tokens_to_scores_ms": t_fused * 1e3, "gpu_prompts_per_s": N_PROMPTS / t_fused,
        "gpu_keys_per_s": total_keys / t_fused, "gpu_kernels_per_call": int(launches),
        "gpu_hash_only_host_to_host_ms": t_hash_gpu * 1e3,
        "hash_kernel": {"device_resident_us": t_hash_kernel * 1e6, "keys_per_s": total_keys / t_hash_kernel,
                        "kernel": "hash_chain_kernel_wpc (warp per prompt)" if N_PROMPTS <= 1536 and not os.environ.get("KVB_HASH_KERNEL")
                        else "hash_chain_kernel_2w (lane per prompt)",
                        "bound": "latency of dependent warp instructions, not HBM", "sm_hz": sm_hz,
                        "longest_chain_cbor_bytes": int(chain_bytes.max()),
                        "floor_us": {"byte_serial_12.3_cycles_per_byte": byte_floor * 1e6,
                                     "vote_rounds_583_cycles_per_block": vote_floor * 1e6},
                        "frac_of_vote_round_floor": vote_floor / t_hash_kernel,
                        "hbm_bytes": int(tokens.nbytes + total_keys * 8)},
        "gpu_fused_pinned_tokens_ms": t_fused_pinned * 1e3, "gpu_prompts_per_s_pinned": N_PROMPTS / t_fused_pinned,
        "gpu_fused_8192_prompts_pinned_ms": t_fused8 * 1e3, "gpu_prompts_per_s_8192": N_PROMPTS * reps / t_fused8,
        "gpu_keys_per_s_8192": total_keys * reps / t_fused8,
        "bytes_per_call": {"h2d_tokens": int(tokens.nbytes), "probe_bytes_64B_per_key": total_keys * 64, "d2h_scores": N_PROMPTS * 13 * 10 + N_PROMPTS * 4},
        "cpu_c_restatement": {"cores": cores, "hash_ms_best_threads": t_c_hash_all * 1e3, "hash_ms_1_core": t_c_hash_1 * 1e3,
                              "score_ms_best_threads": t_c_score_all * 1e3, "score_ms_1_core": t_c_score_1 * 1e3,
                              "total_ms_best_threads": (t_c_hash_all + t_c_score_all) * 1e3,
                              "hash_ms_by_threads": {str(k): v * 1e3 for k, v in hash_by_t.items()},
                              "score_ms_by_threads": {str(k): v * 1e3 for k, v in score_by_t.items()},
                              "note": "plain-C restatement without Go's allocations/mutexes: faster than the reference would be"},
        "speedup_vs_best_cpu": (t_c_hash_all + t_c_score_all) / t_fused_pinned,
        "speedup_vs_1_core": (t_c_hash_1 + t_c_score_1) / t_fused_pinned,
        "index_build": {"host_add_s": t_build_host, "device_flush_s": t_flush},
    }

    # ---- config #1: one prompt, 4 pods
    idx1 = K.Index()
    tok1 = np.random.default_rng(0).integers(0, 128256, 1000).astype(np.uint32)
    off1 = np.array([0, 1000], dtype=np.int64)
    par1 = parents[:1].copy()
    k1, _ = oc.hash_batch(tok1, off1, par1, BS)
    for i in range(4):
        idx1.add(None, k1[: 62 * (i + 1) // 4], [K.PodEntry("pod-%d" % i, "gpu")])
    idx1.add(None, k1[:20], [K.PodEntry("pod-3", "cpu")])
    o1 = idx1.score_tokens_flat(BS, tok1, off1, par1)
    got = {idx1.pods.names[int(o1[1][j])]: float(o1[2][j]) for j in range(int(o1[0][0]))}
    assert got == {"pod-0": 15.0, "pod-1": 31.0, "pod-2": 46.0, "pod-3": 62.0}, got
    t1 = med(lambda: idx1.score_tokens_flat(BS, tok1, off1, par1, out=o1), iters=200, warm=20)
    ix = kvb.indexer.Indexer(tp, idx1)
    t1_py = med(lambda: ix.score_tokens(tok1, MODEL), iters=100, warm=10)
    cix1 = oc.load().kvo_index_new(1 << 10)
    for i in range(4):
        oc.load().kvo_index_add(cix1, k1.ctypes.data, 62 * (i + 1) // 4, i, 0)
    n1, p1, s1 = np.zeros(1, np.int32), np.zeros(13, np.uint16), np.zeros(13, np.float64)

    def c_one():
        kk, ko = oc.hash_batch(tok1, off1, par1, BS, threads=1)
        oc.load().kvo_score_batch(cix1, kk.ctypes.data, ko.ctypes.data, 1, w.ctypes.data, n1.ctypes.data, p1.ctypes.data, s1.ctypes.data, 1)
    t1_c = med(c_one, iters=200, warm=20)
    cfg1 = {"tokens": 1000, "keys": 62, "pods": 4, "gpu_c_abi_us_per_call": t1 * 1e6, "gpu_python_indexer_us_per_call": t1_py * 1e6,
            "cpu_c_restatement_1core_us_per_call": t1_c * 1e6,
            "note": "a single 62-block chain is one serial FNV chain: the GPU has no parallelism to use and pays launch + PCIe "
                    "latency; the device path wins on batches (config #5), not on one prompt"}
    print(json.dumps({"config5_batch_scoring": cfg5, "config1_score_tokens": cfg1}))


if __name__ == "__main__":
    main()
