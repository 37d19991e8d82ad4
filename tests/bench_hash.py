#!/usr/bin/env python
"""Device-resident timing of the block-key hash kernels (CUDA events around back-to-back launches) for the three kernel
families, with a parity check of every configuration against the oracle's C restatement.
    python tests/bench_hash.py [prompts ...]      -> one JSON line"""
import importlib
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from oracle import kvblock_oracle_c as oc  # noqa: E402  (checker)


def main():
    torch.cuda.set_device(0)
    kvb = importlib.import_module("llm-d-kv-cache_b200")
    lib = kvb.lib
    sizes = [int(x) for x in sys.argv[1:]] or [1, 4, 16, 64, 132, 1024]
    bs, ntok = 16, 1000
    rng = np.random.default_rng(2)
    out = {}
    for n in sizes:
        tokens = rng.integers(0, 128256, n * ntok).astype(np.uint32)
        off = np.arange(0, (n + 1) * ntok, ntok, dtype=np.int64)
        parents = rng.integers(1 << 40, 1 << 62, n).astype(np.uint64)
        want, koff = oc.hash_batch(tokens, off, parents, bs)
        d_tok = torch.from_numpy(tokens.view(np.int32)).cuda()
        d_off, d_par, d_koff = (torch.from_numpy(a.view(np.int64)).cuda() for a in (off, parents, koff))
        d_keys = torch.empty(int(koff[-1]), dtype=torch.int64, device="cuda")
        st = torch.cuda.current_stream()

        def launch():
            kvb._lib.check(lib.kvb_hash_token_blocks_dev(0, d_tok.data_ptr(), d_off.data_ptr(), d_par.data_ptr(), n, bs, None, None,
                                                         d_keys.data_ptr(), d_koff.data_ptr(), int(koff[-1]), st.cuda_stream))
        row = {}
        for family in ("spec", "chain_s1", "chain_s1_merged", "wpc", "lanes"):
            if family == "spec" and n > 64:
                continue
            for k in ("KVB_HASH_STAGERS", "KVB_HASH_MERGED", "KVB_HASH_KERNEL"):
                os.environ.pop(k, None)
            if family.startswith("chain"):
                os.environ["KVB_HASH_STAGERS"] = "2" if "_s2" in family else "1"
                os.environ["KVB_HASH_MERGED"] = "1" if "merged" in family else "0"
            else:
                os.environ["KVB_HASH_KERNEL"] = family
            d_keys.zero_()
            for _ in range(50):
                launch()
            torch.cuda.synchronize()
            assert np.array_equal(d_keys.cpu().numpy().view(np.uint64), want), (n, family)
            reps = 300
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            for _ in range(reps):
                launch()
            b.record(st)
            torch.cuda.synchronize()
            back_to_back = a.elapsed_time(b) / reps * 1e3
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(100)]
            for x, y in evs:
                x.record(st)
                launch()
                y.record(st)
            torch.cuda.synchronize()
            row[family] = {"us_back_to_back": round(back_to_back, 2),
                                         "us_median_single": round(float(np.median([x.elapsed_time(y) for x, y in evs])) * 1e3, 2)}
        for k in ("KVB_HASH_STAGERS", "KVB_HASH_MERGED", "KVB_HASH_KERNEL"):
            os.environ.pop(k, None)
        out[str(n)] = row
    print(json.dumps({"block_size": bs, "tokens_per_prompt": ntok, "blocks_per_chain": ntok // bs, "bit_exact_vs_oracle": True,
                      "prompts": out}))


if __name__ == "__main__":
    main()
