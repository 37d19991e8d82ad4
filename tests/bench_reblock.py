#!/usr/bin/env python
"""Token-segment migration (kvb_migrate_tokens) against the plain page migration (kvb_migrate_blocks), HBM -> HBM on
one GPU: a 32 768-token request in the Llama-3-8B fp16 shape (64 tensors, 8 KV heads of 256 B) and the Llama-3-70B fp8
shape (160 tensors, 8 KV heads of 128 B).  Arms:
    migrate_blocks         whole 16-token pages, B16 -> B16 (the same bytes; the reference rate)
    b16_to_b64_nhd         16-token blocks into 64-token blocks, NHD -> NHD
    b64_to_b16_nhd         64 -> 16, NHD -> NHD
    b16_to_b64_nhd_to_hnd  16 -> 64, NHD -> HND (runs of one head)
    b64_to_b16_start8      64 -> 16 starting 8 tokens into the source request: segments of 16 tokens, and of 8 where a
                           destination block straddles a source block boundary
    tp1_b16_to_tp2_b64     TP=1 16-token blocks into two TP=2 64-token pools: the tp_head_transfers plan, one segment
                           list for both calls
Each arm is checked byte for byte against a torch index / permute reference before it is timed.  With two or more
GPUs the 16 -> 64 NHD arm also runs into a pool on GPU 1, peer-mapped and written over NVLink.
    python tests/bench_reblock.py [--iters 30] [--warmup 5]      -> one JSON line"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tests.bench_reshard import HBM_PEAK, NVLINK_PEAK, card, timed  # noqa: E402

N_TOKENS = 32768
SHAPES = {"llama3_8b_fp16": dict(T=64, H=8, E=256), "llama3_70b_fp8": dict(T=160, H=8, E=128)}


def seq(rows: torch.Tensor, ids, B: int, H: int, E: int, layout: str) -> torch.Tensor:
    """Blocks ids of (num_blocks, B*H*E) rows -> the request's tokens, (len(ids) * B, H, E)."""
    r = rows[torch.from_numpy(np.asarray(ids, dtype=np.int64)).to(rows.device)]
    v = r.view(-1, B, H, E) if layout == "NHD" else r.view(-1, H, B, E).transpose(1, 2)
    return v.reshape(-1, H, E)


def run_shape(kvb, T: int, H: int, E: int, iters: int, warmup: int, peer: bool) -> dict:
    mig, KVPool, part = kvb.migrate, kvb.pool.KVPool, kvb.partition
    n16, n64 = N_TOKENS // 16, N_TOKENS // 64 + 1      # one spare 64-token block for the transfer starting at 8
    g = torch.Generator(device="cuda").manual_seed(T)

    def tensors(n, B, heads):
        t = torch.empty((T, n, B * heads * E), dtype=torch.uint8, device="cuda")
        t.random_(0, 256, generator=g)
        return t

    a16, b16, a64 = tensors(n16, 16, H), tensors(n16, 16, H), tensors(n64, 64, H)
    halves = [tensors(n64, 64, H // 2) for _ in range(2)]
    P16 = lambda t: KVPool(list(t.unbind(0)), geometry=(1, 16, H, E, "NHD"))  # noqa: E731
    src16, dst16 = P16(a16), P16(b16)
    p64 = KVPool(list(a64.unbind(0)), geometry=(1, 64, H, E, "NHD"))
    p64_hnd = KVPool(list(a64.unbind(0)), geometry=(1, 64, H, E, "HND"))      # the same memory read as HND
    tp2 = [KVPool(list(h.unbind(0)), geometry=(1, 64, H // 2, E, "NHD")) for h in halves]
    rng = np.random.default_rng(T)
    s16, d16 = rng.permutation(n16), rng.permutation(n16)
    s64 = rng.permutation(n64)
    d64 = s64[:n64 - 1]
    plan = part.token_segments
    seg_16_64 = plan(s16, 16, d64, 64, N_TOKENS)
    seg_64_16 = plan(d64, 64, d16, 16, N_TOKENS)
    seg_64_16_s8 = plan(s64, 64, d16, 16, N_TOKENS, src_start=8)
    tp = part.tp_head_transfers(H, 1, 2)

    def ref16(t):
        return seq(a16[t], s16, 16, H, E, "NHD")

    arms = {
        "migrate_blocks": (lambda: mig.migrate_blocks(src16, dst16, s16, d16),
                           lambda t: (b16[t][torch.from_numpy(d16).cuda()], a16[t][torch.from_numpy(s16).cuda()]),
                           len(s16)),
        "b16_to_b64_nhd": (lambda: mig.migrate_tokens(src16, p64, seg_16_64),
                           lambda t: (seq(a64[t], d64, 64, H, E, "NHD"), ref16(t)), len(seg_16_64)),
        "b64_to_b16_nhd": (lambda: mig.migrate_tokens(p64, dst16, seg_64_16),
                           lambda t: (seq(b16[t], d16, 16, H, E, "NHD"), seq(a64[t], d64, 64, H, E, "NHD")),
                           len(seg_64_16)),
        "b16_to_b64_nhd_to_hnd": (lambda: mig.migrate_tokens(src16, p64_hnd, seg_16_64),
                                  lambda t: (seq(a64[t], d64, 64, H, E, "HND"), ref16(t)), len(seg_16_64)),
        "b64_to_b16_start8": (lambda: mig.migrate_tokens(p64, dst16, seg_64_16_s8),
                              lambda t: (seq(b16[t], d16, 16, H, E, "NHD"),
                                         seq(a64[t], s64, 64, H, E, "NHD")[8:8 + N_TOKENS]), len(seg_64_16_s8)),
        "tp1_b16_to_tp2_b64": (lambda: [mig.migrate_tokens(src16, tp2[d], seg_16_64, sh, dh, nh)
                                        for (_, d, sh, dh, nh) in tp],
                               lambda t: (torch.cat([seq(halves[d][t], d64, 64, H // 2, E, "NHD") for d in (0, 1)], 1),
                                          ref16(t)), len(seg_16_64)),
    }
    moved = N_TOKENS * T * H * E
    out = {"tokens": N_TOKENS, "tensors": T, "heads": H, "head_bytes": E, "moved_bytes": moved, "hbm_bytes": 2 * moved}
    for name, (fn, ref, n_segs) in arms.items():
        b16.fill_(0xA5)
        for h in halves:
            h.fill_(0x5A)
        fn()
        torch.cuda.synchronize()
        for t in range(T):
            got, want = ref(t)
            if not torch.equal(got, want):
                raise AssertionError(f"{name}: tensor {t} differs from the torch reference")
        ms = timed(fn, iters, warmup)
        out[name] = {"segments": n_segs, "ms": round(ms, 4), "moved_GBps": round(moved / ms / 1e6, 1),
                     "hbm_GBps": round(2 * moved / ms / 1e6, 1),
                     "fraction_of_hbm_peak": round(2 * moved / (ms * 1e-3) / HBM_PEAK, 3), "checked": True}
    base = out["migrate_blocks"]["ms"]
    for name in arms:
        out[name]["ratio_to_migrate_blocks"] = round(base / out[name]["ms"], 3)
    if peer:
        out["cross_gpu_b16_to_b64_nhd"] = cross_gpu(kvb, src16, a16, s16, d64, seg_16_64, T, H, E, iters, warmup)
    else:
        out["cross_gpu_b16_to_b64_nhd"] = "not measured (one GPU)"
    return out


def cross_gpu(kvb, src16, a16, s16, d64, segs, T, H, E, iters, warmup) -> dict:
    """16 -> 64 NHD into a pool on GPU 1, described on GPU 0 (peer-mapped) and written over NVLink."""
    kvb.migrate.enable_peer_access(0, 1)
    remote_t = torch.full((T, N_TOKENS // 64 + 1, 64 * H * E), 0x5A, dtype=torch.uint8, device="cuda:1")
    remote = kvb.pool.KVPool(list(remote_t.unbind(0)), device=0, geometry=(1, 64, H, E, "NHD"))

    def fn():
        kvb.migrate.migrate_tokens(src16, remote, segs)

    fn()
    torch.cuda.synchronize()
    for t in range(T):
        if not torch.equal(seq(remote_t[t], d64, 64, H, E, "NHD"), seq(a16[t], s16, 16, H, E, "NHD").to("cuda:1")):
            raise AssertionError("cross-GPU 16 -> 64: bytes differ from the torch reference")
    ms = timed(fn, iters, warmup)
    moved = N_TOKENS * T * H * E
    return {"ms": round(ms, 4), "moved_GBps": round(moved / ms / 1e6, 1),
            "fraction_of_nvlink_per_direction": round(moved / (ms * 1e-3) / NVLINK_PEAK, 3), "checked": True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reblock needs a CUDA device")
    torch.cuda.set_device(0)
    kvb = importlib.import_module("llm-d-kv-cache_b200")
    peer = torch.cuda.device_count() >= 2
    res = {"metric": "kv_token_reblock", "card": card(), "gpus": torch.cuda.device_count(), "iters": args.iters,
           "warmup": args.warmup, "hbm_peak_Bps": HBM_PEAK, "nvlink_peak_Bps_per_direction": NVLINK_PEAK}
    for name, kw in SHAPES.items():
        res[name] = run_shape(kvb, iters=args.iters, warmup=args.warmup, peer=peer, **kw)
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
