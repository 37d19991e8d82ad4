"""Block keys from the device hash kernel must be identical to the reference's (golden vectors) and to the oracle."""
import numpy as np
import pytest

from oracle import kvblock_oracle as o

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["auto", "lanes", "wpc", "chain", "spec"])
def hash_kernel_family(request, monkeypatch):
    """Every test runs twice: default dispatch (warp-per-chain kernel for small batches of block size 4/8/16) and with
    the lane-per-prompt kernels forced (KVB_HASH_KERNEL is read on every launch)."""
    if request.param in ("lanes", "wpc", "chain", "spec"):   # "spec": the table kernel for batches of up to 64 prompts;   # "wpc": round 1's warp kernel (the default); "chain": round 2's chain kernel, hash-only form
        monkeypatch.setenv("KVB_HASH_KERNEL", request.param)
    else:
        monkeypatch.delenv("KVB_HASH_KERNEL", raising=False)
    return request.param


def _oracle_features(kvb_feats):
    return None if kvb_feats is None else [
        None if f is None else o.BlockExtraFeatures([o.MMHash(m.hash) for m in f.mm_hashes]) for f in kvb_feats]


def test_golden_text(kvb, torch_cuda, golden):
    t = golden["text"]
    tp = kvb.kvblock.ChunkedTokenDatabase(t["block_size"], t["hash_seed"])
    assert tp.get_init_hash(t["model"]) == o.TokenProcessor(t["block_size"], t["hash_seed"]).get_init_hash(t["model"])
    assert tp.tokens_to_kv_block_keys(0, t["tokens"], t["model"]) == t["request_keys"]


def test_golden_multimodal(kvb, torch_cuda, golden):
    m = golden["multimodal"]
    K = kvb.kvblock
    ph = {k: [K.PlaceholderRange(r["offset"], r["length"]) for r in v] for k, v in m["mm_placeholders"].items()}
    feats = K.compute_block_extra_features(m["mm_hashes"], ph, m["block_size"], len(m["tokens"]))
    tp = K.ChunkedTokenDatabase(m["block_size"], m["hash_seed"])
    assert tp.tokens_to_kv_block_keys(0, m["tokens"], m["model"], feats) == m["request_keys"]


@pytest.mark.parametrize("bs", [1, 4, 16, 17, 23, 24, 64, 255, 256, 300])
def test_random_batches_match_oracle(kvb, torch_cuda, bs):
    rng = np.random.default_rng(bs)
    tp = kvb.kvblock.ChunkedTokenDatabase(bs, "seed-%d" % bs)
    otp = o.TokenProcessor(bs, "seed-%d" % bs)
    prompts, models, parents = [], [], []
    for i in range(37):
        n = int(rng.integers(0, 6 * bs + 3))
        width = rng.choice([5, 8, 16, 17, 32])          # exercises 1/2/3/5-byte CBOR ints
        prompts.append(rng.integers(0, 1 << width, n, dtype=np.uint64).astype(np.uint32))
        models.append("model-%d" % (i % 3))
        cands = [0, 0, 5, 200, 70000, 1 << 33, (1 << 64) - 1]
        parents.append(cands[int(rng.integers(0, len(cands)))])
    keys, off = tp.tokens_to_kv_block_keys_batch(prompts, models, parents)
    for i, p in enumerate(prompts):
        want = otp.tokens_to_kv_block_keys(parents[i], [int(x) for x in p], models[i]) or []
        assert [int(k) for k in keys[off[i]:off[i + 1]]] == want


def test_edge_tokens_and_empty(kvb, torch_cuda):
    tp = kvb.kvblock.ChunkedTokenDatabase(16, "")
    otp = o.TokenProcessor(16, "")
    edge = [0, 23, 24, 255, 256, 65535, 65536, 0xFFFFFFFF] * 4
    assert tp.tokens_to_kv_block_keys(0, edge, "m") == otp.tokens_to_kv_block_keys(0, edge, "m")
    assert tp.tokens_to_kv_block_keys(0, [], "m") is None
    assert tp.tokens_to_kv_block_keys(0, list(range(15)), "m") is None          # no full block -> nil
    keys, off = tp.tokens_to_kv_block_keys_batch([[], list(range(16)), []], "m")
    assert list(off) == [0, 0, 1, 1] and int(keys[0]) == otp.tokens_to_kv_block_keys(0, list(range(16)), "m")[0]
    with pytest.raises(ValueError):
        kvb.kvblock.ChunkedTokenDatabase(0)
    with pytest.raises(ValueError):
        tp.tokens_to_kv_block_keys(0, list(range(32)), "m", [None])              # extraFeatures length mismatch


def test_multimodal_random(kvb, torch_cuda):
    K = kvb.kvblock
    rng = np.random.default_rng(11)
    tp, otp = K.ChunkedTokenDatabase(8, "s"), o.TokenProcessor(8, "s")
    prompts, feats = [], []
    for i in range(12):
        n = int(rng.integers(8, 200))
        prompts.append(rng.integers(0, 200000, n).astype(np.uint32))
        hashes = {"image": ["%064x" % int(rng.integers(1, 1 << 62)) for _ in range(3)],
                  "audio": ["au-%d" % i]}
        ph = {"image": [K.PlaceholderRange(int(rng.integers(0, n)), int(rng.integers(1, 40))) for _ in range(3)],
              "audio": [K.PlaceholderRange(int(rng.integers(0, n)), 5)]}
        feats.append(None if i % 4 == 0 else K.compute_block_extra_features(hashes, ph, 8, n))
    keys, off = tp.tokens_to_kv_block_keys_batch(prompts, "m", None, feats)
    for i, p in enumerate(prompts):
        want = otp.tokens_to_kv_block_keys(0, [int(x) for x in p], "m", _oracle_features(feats[i])) or []
        assert [int(k) for k in keys[off[i]:off[i + 1]]] == want


def test_long_context_chain_property(kvb, torch_cuda):
    """32k-context prompt (2048 keys): chaining in one call == continuing from a parent key mid-way."""
    rng = np.random.default_rng(5)
    toks = rng.integers(0, 128256, 32768).astype(np.uint32)
    tp = kvb.kvblock.ChunkedTokenDatabase(16, "")
    full = tp.tokens_to_kv_block_keys(0, toks, "meta-llama/Llama-3-8B")
    assert len(full) == 2048 and len(set(full)) == 2048
    tail = tp.tokens_to_kv_block_keys(full[999], toks[16000:], "meta-llama/Llama-3-8B")
    assert tail == full[1000:]
    sample = o.TokenProcessor(16, "").tokens_to_kv_block_keys(0, [int(x) for x in toks[:1600]], "meta-llama/Llama-3-8B")
    assert sample == full[:100]


@pytest.mark.parametrize("n_prompts", [1, 31, 1320, 1321, 1536, 1537, 5000])
def test_dispatch_boundary_batches_match_c_oracle(kvb, torch_cuda, n_prompts):
    """Batch sizes either side of the warp-per-chain / lane-per-prompt dispatch threshold, ragged lengths, mixed token
    widths and short parents, against the oracle's C restatement."""
    from oracle import kvblock_oracle_c as oc
    rng = np.random.default_rng(n_prompts)
    lens = rng.integers(0, 200, n_prompts)
    off = np.zeros(n_prompts + 1, np.int64)
    off[1:] = np.cumsum(lens)
    width = rng.choice([5, 8, 16, 17, 32], int(off[-1]))
    tokens = (rng.integers(0, 1 << 32, int(off[-1]), dtype=np.uint64) & ((np.uint64(1) << width.astype(np.uint64)) - np.uint64(1))).astype(np.uint32)
    parents = rng.integers(0, 1 << 63, n_prompts, dtype=np.int64).astype(np.uint64)
    parents[::7] = rng.integers(0, 70000, parents[::7].size).astype(np.uint64)     # short CBOR heads for the parent
    for bs in (4, 8, 16):
        want, woff = oc.hash_batch(tokens, off, parents, bs)
        tp = kvb.kvblock.ChunkedTokenDatabase(bs, "")
        got = np.empty(int(woff[-1]), np.uint64)
        goff = np.empty(n_prompts + 1, np.int64)
        kvb._lib.check(kvb.lib.kvb_hash_token_blocks(0, tokens.ctypes.data, off.ctypes.data, parents.ctypes.data, n_prompts,
                                                     bs, None, None, got.ctypes.data, goff.ctypes.data, None))
        assert np.array_equal(goff, woff) and np.array_equal(got, want), bs
