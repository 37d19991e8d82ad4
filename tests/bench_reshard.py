#!/usr/bin/env python
"""Head-slice migration (kvb_migrate_heads) against the plain page migration (kvb_migrate_blocks), HBM -> HBM on one
GPU: a 32k-token prefix (2048 blocks of 16 tokens) in the Llama-3-8B fp16 shape (64 tensors, 8 KV heads of 256 B) and
the Llama-3-70B fp8 shape (160 tensors, 8 KV heads of 128 B).  Arms:
    migrate_blocks       whole pages, TP=1 -> TP=1
    split_tp1_tp2_nhd    two migrate_heads calls, heads 0-3 and 4-7 into two 4-head NHD pools
    split_tp1_tp2_hnd    the same into two 4-head HND pools
    merge_tp2_tp1        two 4-head NHD pools into one 8-head pool
    split_tp1_tp8        eight one-head pools (256 B runs in the 8B shape)
Each arm is checked byte for byte against a torch index / permute reference before it is timed.  With two or more
GPUs the NHD split also runs into pools on GPU 1, peer-mapped and written over NVLink.
    python tests/bench_reshard.py [--iters 20] [--warmup 3]      -> one JSON line"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

HBM_PEAK = 3.35e12        # H100 SXM data sheet, bytes/s
NVLINK_PEAK = 450e9       # NVLink 4, per direction
N_BLOCKS, B = 2048, 16
SHAPES = {"llama3_8b_fp16": dict(T=64, H=8, E=256), "llama3_70b_fp8": dict(T=160, H=8, E=128)}


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})", "max_sm_clock": "unknown"}


def timed(fn, iters: int, warmup: int) -> float:
    """Median ms of fn() over iters calls, each between two CUDA events on the current stream."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def heads(t: torch.Tensor, n: int, H: int, E: int, layout: str) -> torch.Tensor:
    """(n, frag) rows -> (n, B, H, E) in either layout."""
    v = t.view(n, B, H, E) if layout == "NHD" else t.view(n, H, B, E).permute(0, 2, 1, 3)
    return v


def run_shape(kvb, T: int, H: int, E: int, iters: int, warmup: int, peer: bool) -> dict:
    mig, KVPool = kvb.migrate, kvb.pool.KVPool
    n, frag = N_BLOCKS, B * H * E
    g = torch.Generator(device="cuda").manual_seed(T)
    src_t = torch.empty((T, n, frag), dtype=torch.uint8, device="cuda")
    src_t.random_(0, 256, generator=g)
    big_t = torch.empty_like(src_t)
    halves_t = [torch.empty((T, n, frag // 2), dtype=torch.uint8, device="cuda") for _ in range(2)]
    rng = np.random.default_rng(T)
    sids, dids, mids = (rng.permutation(n).astype(np.int64) for _ in range(3))
    sd, dd, md = (torch.from_numpy(x).cuda() for x in (sids, dids, mids))
    src = KVPool(list(src_t.unbind(0)), geometry=(1, B, H, E, "NHD"))
    big = KVPool(list(big_t.unbind(0)), geometry=(1, B, H, E, "NHD"))
    half_nhd = [KVPool(list(h.unbind(0)), geometry=(1, B, H // 2, E, "NHD")) for h in halves_t]
    half_hnd = [KVPool(list(h.unbind(0)), geometry=(1, B, H // 2, E, "HND")) for h in halves_t]
    eighth_t = big_t.view(T, n, 8, frag // 8).permute(2, 0, 1, 3)      # 8 one-head pools carved from big_t
    eighths = [KVPool([eighth_t[d, t] for t in range(T)], ptrs=[eighth_t[d, t].data_ptr() for t in range(T)],
                      device=0, num_blocks=n, frag_bytes=frag // 8, stride_bytes=frag, geometry=(1, B, 1, E, "NHD"))
               for d in range(8)]
    hh = H // 2

    def check(name, pairs):
        for got, want in pairs:
            if not torch.equal(got, want):
                raise AssertionError(f"{name}: bytes differ from the torch reference")

    def ref_src(t):
        return heads(src_t[t][sd], n, H, E, "NHD")

    arms = {
        "migrate_blocks": (lambda: mig.migrate_blocks(src, big, sids, dids),
                           lambda: [(big_t[t][dd], src_t[t][sd]) for t in range(T)]),
        "split_tp1_tp2_nhd": (lambda: [mig.migrate_heads(src, half_nhd[d], sids, dids, d * hh, 0, hh) for d in (0, 1)],
                              lambda: [(heads(halves_t[d][t][dd], n, hh, E, "NHD"), ref_src(t)[:, :, d * hh:(d + 1) * hh])
                                       for d in (0, 1) for t in range(T)]),
        "split_tp1_tp2_hnd": (lambda: [mig.migrate_heads(src, half_hnd[d], sids, dids, d * hh, 0, hh) for d in (0, 1)],
                              lambda: [(heads(halves_t[d][t][dd], n, hh, E, "HND"), ref_src(t)[:, :, d * hh:(d + 1) * hh])
                                       for d in (0, 1) for t in range(T)]),
        # the halves hold the NHD split (re-made before this arm); they merge into rows mids of big
        "merge_tp2_tp1": (lambda: [mig.migrate_heads(half_nhd[s], big, dids, mids, 0, s * hh, hh) for s in (0, 1)],
                          lambda: [(heads(big_t[t][md], n, H, E, "NHD"), ref_src(t)) for t in range(T)]),
        "split_tp1_tp8": (lambda: [mig.migrate_heads(src, eighths[d], sids, dids, d, 0, 1) for d in range(8)],
                          lambda: [(eighth_t[d, t][dd], heads(src_t[t][sd], n, H, E, "NHD")[:, :, d].reshape(n, -1))
                                   for d in range(8) for t in range(T)]),
    }
    moved = n * T * frag
    out = {"blocks": n, "tensors": T, "heads": H, "head_bytes": E, "frag_bytes": frag, "moved_bytes": moved,
           "hbm_bytes": 2 * moved}
    for name, (fn, ref) in arms.items():
        big_t.fill_(0xA5)
        for h in halves_t:
            h.fill_(0x5A)
        if name == "merge_tp2_tp1":
            arms["split_tp1_tp2_nhd"][0]()
        fn()
        torch.cuda.synchronize()
        check(name, ref())
        ms = timed(fn, iters, warmup)
        out[name] = {"ms": round(ms, 4), "moved_GBps": round(moved / ms / 1e6, 1),
                     "hbm_GBps": round(2 * moved / ms / 1e6, 1),
                     "fraction_of_hbm_peak": round(2 * moved / (ms * 1e-3) / HBM_PEAK, 3), "checked": True}
    if peer:
        out["cross_gpu_split_tp1_tp2_nhd"] = cross_gpu(kvb, src, src_t, sids, sd, T, H, E, iters, warmup)
    else:
        out["cross_gpu_split_tp1_tp2_nhd"] = "not measured (one GPU)"
    return out


def cross_gpu(kvb, src, src_t, sids, sd, T, H, E, iters, warmup) -> dict:
    """The NHD split into two 4-head pools on GPU 1, described on GPU 0 (peer-mapped) and written over NVLink."""
    n, frag, hh = N_BLOCKS, B * H * E, H // 2
    kvb.migrate.enable_peer_access(0, 1)
    remote_t = [torch.full((T, n, frag // 2), 0x5A, dtype=torch.uint8, device="cuda:1") for _ in range(2)]
    remote = [kvb.pool.KVPool(list(r.unbind(0)), device=0, geometry=(1, B, hh, E, "NHD")) for r in remote_t]

    def fn():
        for d in (0, 1):
            kvb.migrate.migrate_heads(src, remote[d], sids, sids, d * hh, 0, hh)

    fn()
    torch.cuda.synchronize()
    for d in (0, 1):
        for t in range(T):
            want = heads(src_t[t][sd], n, H, E, "NHD")[:, :, d * hh:(d + 1) * hh].to("cuda:1")
            if not torch.equal(heads(remote_t[d][t][sd.to("cuda:1")], n, hh, E, "NHD"), want):
                raise AssertionError("cross-GPU split: bytes differ from the torch reference")
    ms = timed(fn, iters, warmup)
    moved = n * T * frag
    return {"ms": round(ms, 4), "moved_GBps": round(moved / ms / 1e6, 1),
            "fraction_of_nvlink_per_direction": round(moved / (ms * 1e-3) / NVLINK_PEAK, 3), "checked": True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reshard needs a CUDA device")
    torch.cuda.set_device(0)
    kvb = importlib.import_module("llm-d-kv-cache_b200")
    peer = torch.cuda.device_count() >= 2
    res = {"metric": "kv_head_reshard", "card": card(), "gpus": torch.cuda.device_count(), "iters": args.iters,
           "warmup": args.warmup, "hbm_peak_Bps": HBM_PEAK, "nvlink_peak_Bps_per_direction": NVLINK_PEAK}
    for name, kw in SHAPES.items():
        res[name] = run_shape(kvb, iters=args.iters, warmup=args.warmup, peer=peer, **kw)
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
