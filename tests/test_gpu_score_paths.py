"""The fused tokens -> scores launch (kvb_index_score_tokens_batch) on every path its dispatcher can take, against the
oracle.

Paths are picked with the per-call environment switches (KVB_HASH_KERNEL, KVB_HASH_SPEC, KVB_HASH_MERGED,
KVB_CHAIN_FETCH, KVB_SPEC_SCORE_BATCH) and the KVB_SCORE_* flags.  The table ("spec") kernel and the chain kernel cannot
be told apart from outside, so every path states which kernel the documented thresholds select, and every call checks
the launch count that choice implies (1 for the fused forms, 2 for hash + score).

Scenarios put the index in a state that hits one edge each (S1 owners ... S6 inputs, R recency).  Expected results come
from the Python oracle (InMemoryIndex.lookup + longest_prefix_score); block keys come from the oracle's C restatement,
which tests/test_oracle_c.py pins to the Python oracle.  Scores are float64 and compared bit for bit: the kernels add in
the order of the reference's loop.  Every fused result must also be array-identical (count, pod order, scores) to
kvb_index_score_batch on the oracle's keys.

The scenario builders are plain Python; the unmarked tests at the end prove on the oracle alone that each scenario can
tell a right kernel from the wrong one it targets."""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass, field
from typing import NamedTuple

import numpy as np
import pytest

from oracle import kvblock_oracle as o
from oracle import kvblock_oracle_c as oc

MAX_ENT = 13
SPEC_MAX_KEYS = 16384           # hash_kernels.cu kSpecMaxKeys
FUSE_MAX_PROMPTS = 1536         # index.cu score_common: fuse = n_prompts <= 1536
SCORE_NO_TOUCH, SCORE_TWO_KERNELS, SCORE_PINNED_IO = 2, 16, 32
ENV_VARS = ("KVB_HASH_KERNEL", "KVB_HASH_SPEC", "KVB_HASH_MERGED", "KVB_CHAIN_FETCH", "KVB_SPEC_SCORE_BATCH")
MODEL, MODEL2 = "m", "m2"
DEFAULT_WEIGHTS = {"gpu": 1.0, "cpu": 0.8}


# ------------------------------------------------------------------------------------------------------------ paths
class Path(NamedTuple):
    id: str
    env: dict
    flags: int
    sizes: tuple   # (fewest, most) prompts per call
    bss: tuple     # block sizes
    doc: str       # which kernel the documented thresholds select


FUSED_BS = (4, 8, 16)
# table-kernel paths: batches are split to fit its 16 384 keys where the prompt count allows; a batch that cannot fit
# (S4 at 17+ prompts) goes to the chain kernel, and each call's message names the kernel the thresholds selected
SPEC_BS = (4, 8, 16, 1, 3, 64, 256)
PATHS = [
    Path("spec-1", {}, 0, (1, 1), SPEC_BS,
         "one prompt: table kernel with the 16-prompt argument block (default: <= 32 prompts, <= 16384 keys)"),
    Path("spec-2to16", {}, 0, (2, 16), SPEC_BS, "2-16 prompts: table kernel, 16-prompt argument block"),
    Path("spec-17to32", {}, 0, (17, 32), SPEC_BS, "17-32 prompts: table kernel, 64-prompt argument block (default)"),
    Path("spec-33to64", {"KVB_HASH_KERNEL": "spec"}, 0, (33, 64), SPEC_BS,
         "33-64 prompts with KVB_HASH_KERNEL=spec: table kernel, 64-prompt argument block"),
    Path("spec-batch1", {"KVB_SPEC_SCORE_BATCH": "1"}, 0, (2, 16), SPEC_BS, "table kernel, scorer takes 1+ keys a round"),
    Path("spec-batch7", {"KVB_SPEC_SCORE_BATCH": "7"}, 0, (2, 16), SPEC_BS, "table kernel, scorer takes 7+ keys a round"),
    Path("spec-batch32", {"KVB_SPEC_SCORE_BATCH": "32"}, 0, (2, 16), SPEC_BS, "table kernel, scorer takes full tiles"),
    Path("chain-merged", {"KVB_HASH_SPEC": "0"}, 0, (1, 48), FUSED_BS,
         "KVB_HASH_SPEC=0: chain kernel, merged first bits (default up to 512 prompts)"),
    Path("chain-merged-on", {"KVB_HASH_SPEC": "0", "KVB_HASH_MERGED": "1"}, 0, (1, 48), FUSED_BS,
         "chain kernel, merged forced on"),
    Path("chain-128x2", {"KVB_HASH_SPEC": "0", "KVB_HASH_MERGED": "0"}, 0, (1, 48), FUSED_BS,
         "chain kernel, merged forced off, default token fetch 128 tokens x 2 chunks ahead"),
    Path("chain-256x2", {"KVB_HASH_SPEC": "0", "KVB_HASH_MERGED": "0", "KVB_CHAIN_FETCH": "256x2"}, 0, (1, 48), FUSED_BS,
         "unmerged chain kernel, 256-token chunks x 2 ahead"),
    Path("chain-256x4", {"KVB_HASH_SPEC": "0", "KVB_HASH_MERGED": "0", "KVB_CHAIN_FETCH": "256x4"}, 0, (1, 48), FUSED_BS,
         "unmerged chain kernel, 256-token chunks x 4 ahead"),
    Path("chain-128x6", {"KVB_HASH_SPEC": "0", "KVB_HASH_MERGED": "0", "KVB_CHAIN_FETCH": "128x6"}, 0, (1, 48), FUSED_BS,
         "unmerged chain kernel, 128-token chunks x 6 ahead"),
    Path("two-kernels", {}, SCORE_TWO_KERNELS, (1, 48), FUSED_BS + (5,),
         "KVB_SCORE_TWO_KERNELS: hash kernel, then index_score_kernel"),
]


def _spec_wanted(env: dict, n: int) -> bool:
    if "KVB_HASH_KERNEL" in env:
        return env["KVB_HASH_KERNEL"] == "spec"
    return env.get("KVB_HASH_SPEC") != "0" and n <= 32


def selected_kernel(env: dict, flags: int, n: int, bs: int, total_keys: int) -> str:
    """What the documented dispatch runs for one call: no key at all -> the score kernel alone; fused (<= 1536 prompts,
    no KVB_SCORE_TWO_KERNELS) -> the table kernel when it is wanted and the batch fits it (<= 64 prompts, <= 16384 keys),
    else the chain kernel for block sizes 4 / 8 / 16; otherwise hash + score."""
    if total_keys == 0:
        return "score kernel only"
    if n <= FUSE_MAX_PROMPTS and not flags & SCORE_TWO_KERNELS:
        if _spec_wanted(env, n) and n <= 64 and total_keys <= SPEC_MAX_KEYS:
            return "table kernel"
        if bs in (4, 8, 16):
            return "chain kernel"
    return "hash + score"


def expected_launches(env: dict, flags: int, n: int, bs: int, total_keys: int) -> int:
    return 2 if selected_kernel(env, flags, n, bs, total_keys) == "hash + score" else 1


def _use_env(monkeypatch, env: dict):
    for v in ENV_VARS:
        monkeypatch.delenv(v, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


# -------------------------------------------------------------------------------------------------------- scenarios
@dataclass
class Scenario:
    name: str
    bs: int
    prompts: list                     # uint32 arrays
    parents: list                     # literal parent hash of each prompt
    extras: list                      # per prompt: None, or the encoded extra item of every block (b"" = nil)
    adds: list                        # [(keys, [(pod, tier, speculative), ...])] in order
    filters: list                     # pod filters every batch is scored with (None = no filter)
    weights: dict = field(default_factory=lambda: dict(DEFAULT_WEIGHTS))
    pod_cache_size: int = 13
    n_names: int = 0                  # "p0" .. "p{n-1}" are interned first, so that pod "p<i>" has id i
    extra_batches: list = field(default_factory=list)   # prompt groups that are also scored on their own
    io_variants: bool = False         # also score with prompt_off[0] != 0 and from pinned tokens at an odd start
    plan: dict = field(default_factory=dict)            # what the builder meant: checked by the self-checks
    keys: list = None
    expected: dict = None


def hash_keys(prompts, parents, bs, extras=None):
    """Block keys of every prompt (the oracle's C restatement)."""
    off = np.zeros(len(prompts) + 1, dtype=np.int64)
    np.cumsum([len(p) for p in prompts], out=off[1:])
    toks = np.concatenate([np.asarray(p, dtype=np.uint32) for p in prompts]) if off[-1] else np.zeros(1, np.uint32)
    extra = eoff = None
    if extras is not None and any(e is not None for e in extras):
        chunks = []
        for p, e in zip(prompts, extras):
            chunks.extend(e if e is not None else [b""] * (len(p) // bs))
        eoff = np.zeros(len(chunks) + 1, dtype=np.int64)
        np.cumsum([len(c) for c in chunks], out=eoff[1:])
        extra = np.frombuffer(b"".join(chunks) or b"\0", dtype=np.uint8).copy()
    keys, koff = oc.hash_batch(toks, off, np.asarray(parents, dtype=np.uint64), bs, extra, eoff, threads=4)
    return [[int(k) for k in keys[koff[i]:koff[i + 1]]] for i in range(len(prompts))]


def _init(bs, model=MODEL):
    return o.TokenProcessor(bs, "").get_init_hash(model)


def _tokens(rng, n):
    # mixed CBOR widths: 1-, 2-, 3- and 5-byte heads
    return rng.integers(0, 1 << int(rng.choice([5, 8, 16, 17, 20])), n, dtype=np.int64).astype(np.uint32)


def _seq_sum(ws):
    s = 0.0
    for w in ws:
        s += w
    return s


def build_s1(bs):
    """S1 owners: 13 distinct pods on key 0 (two owner groups of the walker) leaving at tile edges and deep; one pod on
    two tiers, one speculative; a pod that holds keys 1.. but not key 0 is never reported."""
    rng = np.random.default_rng(1000 + bs)
    L = 230
    prompt = _tokens(rng, L * bs + bs // 2)
    keys = hash_keys([prompt], [_init(bs)], bs)[0]
    depths = [1, 2, 31, 32, 33, 63, 64, 65, 95, 96, 97, 200, L]
    adds, plan = [], {}
    for j, d in enumerate(depths):
        tier = "cpu" if j == 7 else "gpu"
        adds.append((keys[:d], [("own-%d" % j, tier, j == 3)]))
        plan["own-%d" % j] = float(d)
    adds.append((keys[10:50], [("own-7", "gpu", False)]))         # second tier of own-7 (depth 65), heavier on 10..49
    plan["own-7"] = _seq_sum([1.0 if 10 <= i < 50 else 0.8 for i in range(depths[7])])
    adds.append((keys[1:150], [("late", "gpu", False)]))
    return Scenario("S1", bs, [prompt], [_init(bs)], [None], adds, [None, ["own-12", "own-0", "own-8", "late"]],
                    plan={"scores": plan, "depths": depths})


S2_WEIGHTS = {"gpu": 0.1, "cpu": 1 / 3, "disk": 0.7, "zero": 0.0}


def build_s2(bs):
    """S2 tiers and weights: weights float64 cannot hold exactly, a zero weight, an unknown tier (weight 1.0), pods
    moving between tiers along the chain, a pod on two tiers at once (the larger weight counts)."""
    rng = np.random.default_rng(2000 + bs)
    p0, p1 = _tokens(rng, 120 * bs + 1), _tokens(rng, 45 * bs)
    k0, k1 = hash_keys([p0, p1], [_init(bs)] * 2, bs)
    adds = []
    tiers = np.random.default_rng(5).choice(["gpu", "cpu", "disk"], 110)   # pod-a: moves between tiers key by key
    for s in range(110):
        adds.append((k0[s:s + 1], [("pod-a", str(tiers[s]), False)]))
    adds.append((k0[40:50], [("pod-a", "disk", False)]))             # on two tiers there
    adds.append((k0[:50], [("pod-b", "zero", False)]))
    adds.append((k0[20:90], [("pod-b", "nvme", False)]))             # unknown tier: 1.0
    adds.append((k0[:77], [("pod-c", "zero", False)]))               # scores 0.0, still reported
    adds.append((k0[:33], [("pod-d", "cpu", False)]))
    adds.append((k0[33:70], [("pod-d", "gpu", False)]))
    adds.append((k1[:45], [("pod-a", "cpu", False)]))
    adds.append((k1[:5], [("pod-e", "disk", False)]))
    return Scenario("S2", bs, [p0, p1], [_init(bs)] * 2, [None, None], adds, [None, ["pod-c", "pod-a"]],
                    weights=dict(S2_WEIGHTS), pod_cache_size=10)


def build_s3(bs):
    """S3 holes: key 0 absent with later keys present (no pod reported); a key missing at depth j with keys j+1..
    present, for j at and around the tile edges: the score must not resume after the hole."""
    rng = np.random.default_rng(3000 + bs)
    pa, pb, pc = _tokens(rng, 40 * bs), _tokens(rng, 100 * bs), _tokens(rng, 100 * bs + bs - 1)
    ka, kb, kc = hash_keys([pa, pb, pc], [_init(bs)] * 3, bs)
    adds = [(ka[1:40], [("pod-a", "gpu", False)]),
            (kb[:20] + kb[21:], [("pod-a", "gpu", False), ("pod-b", "cpu", False)])]
    holes = {"pod-a": 31, "pod-f": 32, "pod-c": 33, "pod-d": 63, "pod-b": 64, "pod-e": 65}
    for pod, j in holes.items():
        adds.append((kc[:j] + kc[j + 1:], [(pod, "gpu", False)]))
    return Scenario("S3", bs, [pa, pb, pc], [_init(bs)] * 3, [None] * 3, adds, [None, ["pod-b", "pod-f"]],
                    plan={"holes": holes})


def build_s4(bs):
    """S4 long context: a 32 768-token prompt, at block size 16 a 131 072-token one, and eight 8k-token prompts
    sharing a 4k-token prefix (many CTAs probe and stamp the same buckets).  Pods leave deep, after several wraps of
    the 64-key rings."""
    rng = np.random.default_rng(4000 + bs)
    prompts = [_tokens(rng, 32768)]
    if bs == 16:
        prompts.append(_tokens(rng, 131072))
    shared = _tokens(rng, 4096)
    prompts += [np.concatenate([shared, _tokens(rng, 4096)]) for _ in range(8)]
    keys = hash_keys(prompts, [_init(bs)] * len(prompts), bs)
    n0, npre, first = len(keys[0]), 4096 // bs, 2 if bs == 16 else 1
    adds, depths = [], []

    def hold(ks, d, pod, tier="gpu"):
        adds.append((ks[:d], [(pod, tier, False)]))
        depths.append(d)
    hold(keys[0], n0, "deep-0")
    hold(keys[0], n0 * 3 // 4 + 1, "deep-1", "cpu")
    hold(keys[0], n0 // 2 + 3, "deep-2")
    hold(keys[0], 200, "deep-3")
    hold(keys[0], 129, "deep-4", "cpu")
    if bs == 16:
        hold(keys[1], len(keys[1]), "huge-0")
        hold(keys[1], 5000, "huge-1")
        hold(keys[1], 4097, "huge-2", "cpu")
    hold(keys[first], npre, "pre-a")
    hold(keys[first], len(keys[first]), "pre-b")
    hold(keys[first + 3], npre + 100, "pre-c", "cpu")
    hold(keys[first + 7], npre + 70, "pre-d")
    return Scenario("S4", bs, prompts, [_init(bs)] * len(prompts), [None] * len(prompts), adds,
                    [None, ["deep-2", "huge-1", "pre-c"]], plan={"depths": depths})


S5_IDS = (0, 31, 32, 2047, 2048, 65534)


def build_s5(bs):
    """S5 filters: 65 535 pod names interned (ids 0..65534, 65535 is reserved); keys held by ids in the first and last
    bitmap words and on both sides of word and 2048-id boundaries; filters that change, repeat after another one,
    exclude every owner, or name no known pod."""
    rng = np.random.default_rng(5000 + bs)
    p0, p1 = _tokens(rng, 150 * bs + 3), _tokens(rng, 40 * bs)
    k0, k1 = hash_keys([p0, p1], [_init(bs)] * 2, bs)
    depth = {0: 150, 31: 70, 32: 33, 2047: 64, 2048: 100, 65534: 5}
    adds = [(k0[:depth[i]], [("p%d" % i, "gpu" if i % 2 == 0 else "cpu", False)]) for i in S5_IDS]
    adds += [(k1, [("p65534", "gpu", False)]), (k1[:20], [("p2048", "gpu", False)])]
    filters = [None, ["p0", "p31"], ["p32", "p2047", "p2048"], ["p0", "p31"], ["p65534"], ["p1", "p5000", "p65533"],
               ["nobody"], ["p31", "p0"], None, ["p65534", "nobody"], ["nobody", "p32"]]
    return Scenario("S5", bs, [p0, p1], [_init(bs)] * 2, [None, None], adds, filters, n_names=65535)


def build_s6(bs):
    """S6 inputs: caller-chosen parents (short CBOR forms < 2^32 take the byte-serial branch) and two models in one
    batch, multimodal extras, empty and shorter-than-a-block prompts in between; a batch of prompts without a full
    block (empty and bs-1 tokens), and a batch of empty prompts only."""
    rng = np.random.default_rng(6000 + bs)
    parents = [0, 23, 24, 255, 256, 65535, 65536, (1 << 32) - 1, 1 << 32, _init(bs), _init(bs, MODEL2),
               0x9E3779B97F4A7C15]
    prompts, pars, extras, no_block, empty = [], [], [], [], []
    for i, par in enumerate(parents):
        nb = int(rng.integers(3, 41))
        p = _tokens(rng, nb * bs + int(rng.integers(0, bs)))
        prompts.append(p)
        pars.append(par)
        extras.append([o.encode_extra_suffix(o.BlockExtraFeatures([o.MMHash("img-%d-%d" % (i, b))])) if b < 2 else b""
                       for b in range(nb)] if i % 3 == 1 else None)
        short = _tokens(rng, 0 if i % 2 == 0 else bs - 1)
        no_block.append(len(prompts))
        if len(short) == 0:
            empty.append(len(prompts))
        prompts.append(short)
        pars.append(par)
        extras.append(None)
    keys = hash_keys(prompts, pars, bs, extras)
    adds = []
    for i, ks in enumerate(keys):
        for r in range(int(rng.integers(1, 4)) if ks else 0):
            d = int(rng.integers(1, len(ks) + 1))
            adds.append((ks[:d], [("pod-%d" % ((i + r) % 7), "gpu" if r % 2 == 0 else "cpu", False)]))
    return Scenario("S6", bs, prompts, pars, extras, adds, [None, ["pod-1", "pod-4", "pod-6"]],
                    extra_batches=[no_block, empty], io_variants=True)


BUILDERS = {"S1": build_s1, "S2": build_s2, "S3": build_s3, "S4": build_s4, "S5": build_s5, "S6": build_s6}
SCENARIO_BS = {"S4": (4, 8, 16)}        # the long-context scenario at the block sizes a server uses


def oracle_index(sc: Scenario) -> o.InMemoryIndex:
    oidx = o.InMemoryIndex(pod_cache_size=sc.pod_cache_size)
    for ks, ents in sc.adds:
        oidx.add(None, ks, [o.PodEntry(*e) for e in ents])
    return oidx


@functools.lru_cache(maxsize=None)
def scenario(name: str, bs: int) -> Scenario:
    """The scenario with its keys and the oracle's result for every (filter, prompt)."""
    sc = BUILDERS[name](bs)
    sc.keys = hash_keys(sc.prompts, sc.parents, bs, sc.extras)
    oidx = oracle_index(sc)
    sc.expected = {}
    for fi, flt in enumerate(sc.filters):
        for i, ks in enumerate(sc.keys):
            sc.expected[fi, i] = o.longest_prefix_score(ks, oidx.lookup(ks, flt or ()), sc.weights) if ks else {}
    return sc


def batches(sc: Scenario, lo: int, hi: int, key_cap=None):
    """Groups of lo..hi prompt indices covering every prompt (repeating prompts where a path needs more); with key_cap,
    a group is closed early once it has lo prompts and the next one would take it past key_cap keys."""
    out = []
    for g in [list(range(len(sc.prompts)))] + sc.extra_batches:
        if len(g) < lo:
            g = (g * -(-lo // len(g)))[:lo]
        b, nk = [], 0
        for i in g:
            k = len(sc.keys[i])
            if b and (len(b) == hi or (key_cap is not None and len(b) >= lo and nk + k > key_cap)):
                out.append(b)
                b, nk = [], 0
            b.append(i)
            nk += k
        if len(b) < lo:
            b = b + g[:lo - len(b)]
        out.append(b)
    return out


# ----------------------------------------------------------------------------------------------------- GPU helpers
def _outs(n):
    n = max(n, 1)
    return (np.zeros(n, np.int32), np.zeros(n * MAX_ENT, np.uint16), np.zeros(n * MAX_ENT, np.float64))


def fused_raw(idx, bs, tokens, off, parents, extra, eoff, flt, flags, out):
    n = len(off) - 1
    filt, nf = idx._filter(flt)
    idx._check(idx._lib.kvb_index_score_tokens_batch(
        idx._h, tokens.ctypes.data, off.ctypes.data, parents.ctypes.data, n, bs,
        None if extra is None else extra.ctypes.data, None if eoff is None else eoff.ctypes.data,
        None if filt is None else filt.ctypes.data, nf, flags, out[0].ctypes.data, out[1].ctypes.data,
        out[2].ctypes.data))
    return out


def keys_raw(idx, key_lists, flt):
    """kvb_index_score_batch (index_score_kernel, fixed 32-key tiles) on the oracle's keys; read-only."""
    n = len(key_lists)
    flat = np.asarray([k for ks in key_lists for k in ks] or [0], dtype=np.uint64)
    koff = np.zeros(n + 1, np.int64)
    np.cumsum([len(ks) for ks in key_lists], out=koff[1:])
    filt, nf = idx._filter(flt)
    out = _outs(n)
    idx._check(idx._lib.kvb_index_score_batch(idx._h, flat.ctypes.data, koff.ctypes.data, n,
                                              None if filt is None else filt.ctypes.data, nf, SCORE_NO_TOUCH,
                                              out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data))
    return out


def decode(idx, out, p):
    base = p * MAX_ENT
    return {idx.pods.names[int(out[1][base + j])]: float(out[2][base + j]) for j in range(int(out[0][p]))}


def assert_same_arrays(a, b, n, what):
    assert np.array_equal(a[0][:n], b[0][:n]), what
    for p in range(n):
        k, s = int(a[0][p]), p * MAX_ENT
        assert np.array_equal(a[1][s:s + k], b[1][s:s + k]), (what, p)
        assert np.array_equal(a[2][s:s + k].view(np.uint64), b[2][s:s + k].view(np.uint64)), (what, p)


def assemble(sc: Scenario, ids):
    """Flat tokens, prompt offsets, parents and (if any prompt has them) encoded extras of a batch."""
    ps = [sc.prompts[i] for i in ids]
    off = np.zeros(len(ids) + 1, np.int64)
    np.cumsum([len(p) for p in ps], out=off[1:])
    tokens = np.concatenate(ps + [np.zeros(1, np.uint32)]).astype(np.uint32)   # one spare token: never empty
    parents = np.asarray([sc.parents[i] for i in ids], dtype=np.uint64)
    extra = eoff = None
    if any(sc.extras[i] is not None for i in ids):
        chunks = []
        for i in ids:
            chunks.extend(sc.extras[i] if sc.extras[i] is not None else [b""] * (len(sc.prompts[i]) // sc.bs))
        eoff = np.zeros(len(chunks) + 1, np.int64)
        np.cumsum([len(c) for c in chunks], out=eoff[1:])
        extra = np.frombuffer(b"".join(chunks) or b"\0", dtype=np.uint8).copy()
    return tokens, off, parents, extra, eoff


_held: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """Memory other modules' tensors left in torch's cache is handed back before this module's indexes are made; the
    last index is closed when the module is done."""
    try:
        import torch
        if torch.cuda.is_available():
            torch.cuda.empty_cache()
    except ImportError:
        pass
    yield
    for idx in _held.values():
        idx.close()
    _held.clear()


def gpu_index(kvb, name: str, bs: int):
    """The scenario's state in a device index.  Cases run scenario by scenario, so the index is built once per scenario
    and block size and closed when the next one is needed; nothing here runs at capacity, so the recency stamps of
    earlier calls do not change later results."""
    if (name, bs) in _held:
        return _held[name, bs]
    for old in _held.values():
        old.close()
    _held.clear()
    sc = scenario(name, bs)
    K = kvb.kvblock
    idx = K.Index(pod_cache_size=sc.pod_cache_size, expected_keys=sum(len(ks) for ks in sc.keys) + 64)
    for i in range(sc.n_names):
        assert idx.pods.get("p%d" % i) == i
    kvb.indexer.Indexer(K.ChunkedTokenDatabase(bs, ""), idx,
                        backend_configs=[kvb.indexer.KVCacheBackendConfig(t, w) for t, w in sc.weights.items()])
    for ks, ents in sc.adds:
        idx.add(None, ks, [K.PodEntry(*e) for e in ents])
    idx.flush()
    _held[name, bs] = idx
    return idx


def check_batch(kvb, idx, sc: Scenario, ids, fi, path: Path, layout="plain"):
    """One fused call: launch count, every prompt against the oracle, arrays against the score kernel."""
    lib = kvb.lib
    tokens, off, parents, extra, eoff = assemble(sc, ids)
    pin = None
    if layout == "offset":                    # prompt_off[0] != 0 through the C ABI
        tokens = np.concatenate([np.asarray([7, 70000, 1 << 31], np.uint32), tokens])
        off = off + 3
    elif layout == "pinned":                  # pinned tokens read in place, starting 4 bytes into the allocation
        pin = kvb.pool.PinnedBuffer((tokens.size + 2) * 4 + 64)
        view = pin.numpy(np.uint32)[1:1 + tokens.size]
        view[:] = tokens
        tokens = view
    n = len(ids)
    total_keys = int(sum(len(sc.keys[i]) for i in ids))
    flt = sc.filters[fi]
    what = (sc.name, sc.bs, path.id, path.doc, selected_kernel(path.env, path.flags, n, sc.bs, total_keys), layout, fi, n)
    c0 = lib.kvb_launch_count()
    got = fused_raw(idx, sc.bs, tokens, off, parents, extra, eoff, flt, path.flags, _outs(n))
    assert lib.kvb_launch_count() - c0 == expected_launches(path.env, path.flags, n, sc.bs, total_keys), what
    if pin is not None:
        del tokens, view
        pin.free()
    for p, i in enumerate(ids):
        assert decode(idx, got, p) == sc.expected[fi, i], what + (p, i)
    assert_same_arrays(got, keys_raw(idx, [sc.keys[i] for i in ids], flt), n, what)


def _cases():
    out = []
    for name in BUILDERS:                 # scenario and block size outermost: one index serves all paths in a row
        for bs in SCENARIO_BS.get(name, sorted({b for p in PATHS for b in p.bss})):
            for path in PATHS:
                if bs in path.bss:
                    out.append(pytest.param(path, name, bs, id="%s-%s-bs%d" % (path.id, name, bs)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("path,name,bs", _cases())
def test_fused_path_matches_oracle(kvb, torch_cuda, monkeypatch, path, name, bs):
    """Every scenario on every path; `path.doc` states which kernel the documented thresholds select, and the launch
    count each call makes is checked against that choice."""
    _use_env(monkeypatch, path.env)
    sc = scenario(name, bs)
    idx = gpu_index(kvb, name, bs)
    for fi in range(len(sc.filters)):
        for ids in batches(sc, *path.sizes, key_cap=SPEC_MAX_KEYS if path.id.startswith("spec") else None):
            for layout in (("plain", "offset", "pinned") if sc.io_variants else ("plain",)):
                check_batch(kvb, idx, sc, ids, fi, path, layout)


# ------------------------------------------------------------------------------------------- spec kernel's key cap
@pytest.mark.gpu
@pytest.mark.parametrize("bs,launches", [(16, 1), (5, 2)])
def test_spec_key_cap_falls_back(kvb, torch_cuda, monkeypatch, bs, launches):
    """Three prompts (the table kernel's default range) with 18 000 keys, more than its 16 384-key tables: block size
    16 goes to the chain kernel (one launch), block size 5 has no chain kernel and is hashed and scored (two)."""
    _use_env(monkeypatch, {})
    rng = np.random.default_rng(77 + bs)
    prompts = [_tokens(rng, 6000 * bs + 1) for _ in range(3)]
    keys = hash_keys(prompts, [_init(bs)] * 3, bs)
    adds = []
    for i, ks in enumerate(keys):
        adds += [(ks, [("a%d" % i, "gpu", False)]), (ks[:4000], [("b%d" % i, "cpu", False)]),
                 (ks[:1], [("c", "gpu", False)])]
    sc = Scenario("cap", bs, prompts, [_init(bs)] * 3, [None] * 3, adds, [None])
    sc.keys = keys
    oidx = oracle_index(sc)
    sc.expected = {(0, i): o.longest_prefix_score(ks, oidx.lookup(ks)) for i, ks in enumerate(keys)}
    K = kvb.kvblock
    idx = K.Index(pod_cache_size=13, expected_keys=20000)
    for ks, ents in adds:
        idx.add(None, ks, [K.PodEntry(*e) for e in ents])
    idx.flush()                                          # the adds' apply kernels are not the call's launches
    assert sum(len(k) for k in keys) > SPEC_MAX_KEYS
    assert expected_launches({}, 0, 3, bs, 18000) == launches
    check_batch(kvb, idx, sc, [0, 1, 2], 0, Path("default", {}, 0, (3, 3), (bs,), "over the table kernel's key cap: chain kernel, or hash + score"))


# ------------------------------------------------------------------------------- large batches, a sequence of calls
@functools.lru_cache(maxsize=None)
def _pool(n=2100, bs=16):
    """n short prompts (0..12 blocks) and their oracle results on an index with 20 pods at random depths."""
    rng = np.random.default_rng(99)
    lens = rng.integers(0, 13 * bs, n)
    lens[::97] = 0
    prompts = [_tokens(rng, int(x)) for x in lens]
    keys = hash_keys(prompts, [_init(bs)] * n, bs)
    adds = []
    for i, ks in enumerate(keys):
        for r in range(int(rng.integers(0, 4)) if ks else 0):
            d = int(rng.integers(1, len(ks) + 1))
            adds.append((ks[:d], [("pod-%d" % int(rng.integers(0, 20)), "gpu" if rng.random() < 0.7 else "cpu", False)]))
    sc = Scenario("pool", bs, prompts, [_init(bs)] * n, [None] * n, adds, [None])
    sc.keys = keys
    oidx = oracle_index(sc)
    sc.expected = {(0, i): o.longest_prefix_score(ks, oidx.lookup(ks)) if ks else {} for i, ks in enumerate(keys)}
    return sc


def _pool_index(kvb, sc):
    K = kvb.kvblock
    idx = K.Index(expected_keys=1 << 15)
    for ks, ents in sc.adds:
        idx.add(None, ks, [K.PodEntry(*e) for e in ents])
    idx.flush()
    return idx


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1537, 2100])
def test_two_kernel_form_above_1536_prompts(kvb, torch_cuda, monkeypatch, n):
    """More than 1536 prompts: the hash kernel and index_score_kernel, by default (two launches)."""
    _use_env(monkeypatch, {})
    sc = _pool()
    idx = _pool_index(kvb, sc)
    ids = list(range(n))
    assert expected_launches({}, 0, n, 16, sum(len(sc.keys[i]) for i in ids)) == 2
    check_batch(kvb, idx, sc, ids, 0, Path("default", {}, 0, (n, n), (16,), "hash + score above 1536 prompts"))


SEQ_PATHS = [({}, 0), ({"KVB_HASH_SPEC": "0"}, 0), ({"KVB_HASH_MERGED": "1"}, SCORE_PINNED_IO),
             ({"KVB_HASH_MERGED": "0", "KVB_CHAIN_FETCH": "256x4"}, 0), ({"KVB_HASH_KERNEL": "spec"}, SCORE_PINNED_IO),
             ({}, SCORE_TWO_KERNELS), ({"KVB_SPEC_SCORE_BATCH": "1"}, 0)]


@pytest.mark.gpu
def test_sequence_of_distinct_calls_into_poisoned_pinned_outputs(kvb, torch_cuda, monkeypatch):
    """60 fused calls in a row, 1 / 5 / 40 / 700 / 1600 prompts on seven paths in turn (every size meets every path),
    each into pinned output buffers written in place and poisoned before the call: a result read before the completion
    word is valid, or a done counter left over from the previous call, shows up as poison or a stale result.  Each call
    is checked once."""
    sc = _pool()
    idx = _pool_index(kvb, sc)
    lens = np.asarray([len(p) for p in sc.prompts])
    off_all = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off_all[1:])
    tin = kvb.pool.PinnedBuffer(int(off_all[-1]) * 4 + 64)
    tokens = tin.numpy(np.uint32)[:int(off_all[-1])]
    tokens[:] = np.concatenate(sc.prompts)
    nmax = 1600
    b1 = (nmax * 4 + 255) // 256 * 256
    b2 = b1 + (nmax * 26 + 255) // 256 * 256
    pout = kvb.pool.PinnedBuffer(b2 + nmax * 104)
    raw = pout.numpy(np.uint8)
    out = (raw[:nmax * 4].view(np.int32), raw[b1:b1 + nmax * 26].view(np.uint16), raw[b2:b2 + nmax * 104].view(np.float64))
    parents = np.full(nmax, _init(16), np.uint64)
    rng = np.random.default_rng(5)
    sizes = [1, 5, 40, 700, 1600]
    for call in range(60):
        n = sizes[call % len(sizes)]
        env, flags = SEQ_PATHS[call % len(SEQ_PATHS)]
        _use_env(monkeypatch, env)
        start = int(rng.integers(0, len(lens) - n + 1))
        off = off_all[start:start + n + 1].copy()                   # prompt_off[0] != 0: the call starts mid-buffer
        raw[:] = 0xA5
        total_keys = int(sum(len(sc.keys[i]) for i in range(start, start + n)))
        c0 = kvb.lib.kvb_launch_count()
        fused_raw(idx, 16, tokens, off, parents[:n], None, None, None, flags, out)
        what = (call, n, env, flags)
        assert kvb.lib.kvb_launch_count() - c0 == expected_launches(env, flags, n, 16, total_keys), what
        for p in range(n):
            want = sc.expected[0, start + p]
            assert int(out[0][p]) == len(want) and decode(idx, out, p) == want, what + (p,)
    del tokens, out, raw
    tin.free()
    pout.free()


# ---------------------------------------------------------------------------------------- R: recency at capacity
R_PATHS = [Path("spec", {}, 0, (1, 8), (4,), "<= 32 prompts: table kernel"),
           Path("chain-merged", {"KVB_HASH_SPEC": "0"}, 0, (1, 8), (4,), "chain kernel, merged (<= 512 prompts)"),
           Path("chain-unmerged", {"KVB_HASH_SPEC": "0", "KVB_HASH_MERGED": "0"}, 0, (1, 8), (4,), "chain kernel, unmerged"),
           Path("two-kernels", {}, SCORE_TWO_KERNELS, (1, 8), (4,), "hash kernel + index_score_kernel")]
R_FILTERS = [None, None, ["r1", "r3"], ["nobody"]]
R_SIZE = 300
R_KEYS = 96                      # three 32-key tiles per prompt


@functools.lru_cache(maxsize=None)
def r_scenario(bs=4):
    """R: a 300-key index with 3 pods per key, fed more keys than it holds.  Prompts have 96 keys, three tiles of the
    walker.  Most adds either hold a prefix that ends inside the first tile or hold keys from the second or third tile
    without key 0, so a scored prompt's pods are gone before its last tiles and the keys found there are refreshed
    only by a kernel that keeps stamping after the prefix.  Some batches hold the same prompt twice with another in
    between (the last use must win)."""
    rng = np.random.default_rng(31)
    base = [_tokens(rng, R_KEYS * bs) for _ in range(6)]
    chains = []
    for i in range(12):                                  # odd chains share their first half with the one before
        half = R_KEYS // 2 * bs
        chains.append(base[i // 2] if i % 2 == 0 else np.concatenate([base[i // 2][:half], _tokens(rng, half)]))
    keys = hash_keys(chains, [_init(bs)] * len(chains), bs)
    ops = []
    for step in range(130):
        r = rng.random()
        if r < 0.6:
            c = int(rng.integers(0, len(chains)))
            kind = rng.random()
            if kind < 0.45:                              # a prefix that ends inside the first tile
                lo, hi = 0, int(rng.integers(1, 32))
            elif kind < 0.9:                             # keys past the first tile, key 0 absent
                lo = int(rng.integers(1, R_KEYS - 8))
                hi = int(rng.integers(max(lo + 1, 40), R_KEYS + 1))
            else:                                        # the whole chain
                lo, hi = 0, R_KEYS
            ops.append(("add", c, lo, hi, "r%d" % int(rng.integers(0, 6)), "gpu" if rng.random() < 0.7 else "cpu"))
        else:
            ids = [int(x) for x in rng.integers(0, len(chains), int(rng.integers(1, 5)))]
            if rng.random() < 0.5:
                ids = ids + [int(rng.integers(0, len(chains))), ids[0]]
            ops.append(("score", ids, len([x for x in ops if x[0] == "score"]) % len(R_PATHS),
                        R_FILTERS[int(rng.integers(0, len(R_FILTERS)))]))
    universe = list(dict.fromkeys(k for ks in keys for k in ks))
    return chains, keys, ops, universe


def _peek(oidx, ks, flt):
    """Lookup without touching the LRU."""
    out, f = {}, set(flt or ())
    for k in ks:
        pods = oidx.data.d.get(k)
        if pods is None:
            continue
        if not f:
            out[k] = pods.keys()
        else:
            for p in pods.keys():
                if p.pod_identifier in f:
                    out.setdefault(k, []).append(p)
    return out


def _prefix_len(ks, found):
    """Keys on the consecutive prefix of the longest-staying reported pod (0 when key 0 reports nobody)."""
    owners = {e.pod_identifier for e in found.get(ks[0], ())}
    d = 0
    for k in ks:
        owners &= {e.pod_identifier for e in found.get(k, ())}
        if not owners:
            break
        d += 1
    return d


def r_oracle_score(oidx, ks, flt, refresh):
    """Score one prompt.  refresh: 'all' (Lookup's data.Get on every found key); 'none'; 'tiles' (a scorer that stops
    stamping once the prefix has ended: the 32-key tile in which it ends is stamped whole, later tiles are not);
    'tiles-any' (the same with tiles of any size: at most the 31 keys after the end are stamped)."""
    if refresh == "all":
        return o.longest_prefix_score(ks, oidx.lookup(ks, flt or ()))
    found = _peek(oidx, ks, flt)
    res = o.longest_prefix_score(ks, found)
    if refresh != "none":
        d = _prefix_len(ks, found)
        upto = 32 * (d // 32 + 1) if refresh == "tiles" else d + 32
        for k in ks[:upto]:
            oidx.data.get(k)
    return res


def r_replay(refresh, bs=4):
    """The R sequence on the oracle: per step, the survivors (key -> entries) and the scores of scoring steps.
    refresh: a mode of r_oracle_score, or a dict path id -> mode."""
    chains, keys, ops, universe = r_scenario(bs)
    oidx = o.InMemoryIndex(size=R_SIZE, pod_cache_size=3)
    states, scores = [], []
    for op in ops:
        if op[0] == "add":
            _, c, lo, hi, pod, tier = op
            oidx.add(None, keys[c][lo:hi], [o.PodEntry(pod, tier)])
            scores.append(None)
        else:
            _, ids, pi, flt = op
            mode = refresh if isinstance(refresh, str) else refresh.get(R_PATHS[pi].id, "all")
            scores.append([r_oracle_score(oidx, keys[i], flt, mode) for i in ids])
        states.append({k: list(v.keys()) for k, v in oidx.data.d.items()})
    return states, scores


@pytest.mark.gpu
@pytest.mark.parametrize("touch", [True, False], ids=["touch", "no-touch"])
def test_recency_refreshed_by_fused_kernels(kvb, torch_cuda, monkeypatch, touch):
    """Scoring at capacity on the table, merged-chain, unmerged-chain and two-kernel paths: every key found is
    refreshed, also after every pod has left the prefix, and the last use in a batch wins; so after each step the
    surviving keys and their entries equal the oracle's (read back without refreshing).  With touch_lru=False scoring
    refreshes nothing."""
    K = kvb.kvblock
    bs = 4
    chains, keys, ops, universe = r_scenario(bs)
    states, scores = r_replay("all" if touch else "none", bs)
    idx = K.Index(size=R_SIZE, pod_cache_size=3, expected_keys=R_SIZE)
    flags_touch = 0 if touch else SCORE_NO_TOUCH
    for step, op in enumerate(ops):
        if op[0] == "add":
            _, c, lo, hi, pod, tier = op
            idx.add(None, keys[c][lo:hi], [K.PodEntry(pod, tier)])
        else:
            _, ids, pi, flt = op
            path = R_PATHS[pi]
            _use_env(monkeypatch, path.env)
            ps = [chains[i] for i in ids]
            off = np.zeros(len(ids) + 1, np.int64)
            np.cumsum([len(p) for p in ps], out=off[1:])
            c0 = kvb.lib.kvb_launch_count()
            out = fused_raw(idx, bs, np.concatenate(ps), off, np.full(len(ids), _init(bs), np.uint64), None, None, flt,
                            path.flags | flags_touch, _outs(len(ids)))
            tk = sum(len(keys[i]) for i in ids)
            assert kvb.lib.kvb_launch_count() - c0 == expected_launches(path.env, path.flags, len(ids), bs, tk), step
            assert [decode(idx, out, p) for p in range(len(ids))] == scores[step], (step, path.id)
        want = states[step]
        got = {}
        for k in universe:
            e = idx.host_peek(k)
            if e is not None:
                got[k] = [(x.pod_identifier, x.device_tier, x.speculative) for x in e]
        assert got == {k: [(x.pod_identifier, x.device_tier, x.speculative) for x in v] for k, v in want.items()}, step
    assert idx.stats()["lru_evictions"] > 20


# ------------------------------------------------------------------------------ scenario self-checks (no GPU needed)
def test_s1_plan_reaches_the_oracle():
    sc = scenario("S1", 16)
    want = sc.expected[0, 0]
    assert len(want) == 13 and "late" not in want
    assert want == sc.plan["scores"]
    assert set(sc.expected[1, 0]) == {"own-12", "own-0", "own-8"}       # the pod without key 0 stays out when filtered in


def _tile_reversed(ws, tile):
    s = 0.0
    for t in range(0, len(ws), tile):
        for w in reversed(ws[t:t + tile]):
            s += w
    return s


def test_s2_sums_depend_on_the_order_of_additions():
    """A kernel that adds a pod's weights in any other order than key order gets a different float64 sum."""
    sc = scenario("S2", 16)
    oidx = oracle_index(sc)
    ks = sc.keys[0]
    found = oidx.lookup(ks)
    sens_fsum, sens_rev32, sens_rev4 = set(), set(), set()
    for pod, score in sc.expected[0, 0].items():
        ws = []
        for k in ks:
            mine = [S2_WEIGHTS.get(e.device_tier, 1.0) for e in found.get(k, ()) if e.pod_identifier == pod]
            if not mine:
                break
            ws.append(max(mine))
        assert _seq_sum(ws) == score
        if math.fsum(ws) != score:
            sens_fsum.add(pod)
        if _tile_reversed(ws, 32) != score:
            sens_rev32.add(pod)
        if _tile_reversed(ws, 4) != score:
            sens_rev4.add(pod)
    assert sens_fsum and sens_rev32 and sens_rev4, (sens_fsum, sens_rev32, sens_rev4)
    assert sc.expected[0, 0]["pod-c"] == 0.0                          # zero weight: reported, scores nothing


def test_s3_holes_stop_the_score():
    sc = scenario("S3", 8)
    assert sc.expected[0, 0] == {}
    assert sc.expected[0, 1] == {"pod-a": 20.0, "pod-b": _seq_sum([0.8] * 20)}
    assert sc.expected[0, 2] == {p: float(j) for p, j in sc.plan["holes"].items()}


def test_s4_pods_leave_after_the_key_rings_wrap():
    for bs in (4, 16):
        sc = scenario("S4", bs)
        assert min(sc.plan["depths"]) > 64
        assert len(sc.keys[0]) == 32768 // bs
        got = sc.expected[0, 0]
        assert got["deep-3"] == 200.0 and got["deep-0"] == float(len(sc.keys[0]))
    assert len(scenario("S4", 16).keys[1]) == 8192


def test_s5_filters_select_by_high_ids():
    sc = scenario("S5", 16)
    by = {tuple(f) if f else None: sc.expected[fi, 0] for fi, f in enumerate(sc.filters)}
    assert set(by[None]) == {"p%d" % i for i in S5_IDS}
    assert set(by["p32", "p2047", "p2048"]) == {"p32", "p2047", "p2048"}
    assert by["p1", "p5000", "p65533"] == {} and by["nobody", ] == {}
    assert by["p65534", ] == {"p65534": 5.0}


def test_r_refresh_variants_leave_different_survivors():
    """R tells the kernels apart from a scorer that stops stamping once the prefix has ended, on each fused path alone
    (the table kernel's 32-key tiles; the chain kernel's tiles of any size), and from one that stamps nothing."""
    def diff(a, b):
        return sum(set(x) != set(y) for x, y in zip(a, b))
    full, _ = r_replay("all")
    assert diff(full, r_replay({"spec": "tiles"})[0]) > 0
    assert diff(full, r_replay({"chain-merged": "tiles-any"})[0]) > 0
    assert diff(full, r_replay({"chain-unmerged": "tiles-any"})[0]) > 0
    assert diff(full, r_replay("none")[0]) > 0
    chains, keys, ops, universe = r_scenario()
    assert all(len(ks) == R_KEYS for ks in keys) and len(universe) > 2 * R_SIZE


def test_dispatch_model_matches_documented_thresholds():
    assert expected_launches({}, 0, 32, 3, 100) == 1 and expected_launches({}, 0, 33, 3, 100) == 2
    assert expected_launches({"KVB_HASH_KERNEL": "spec"}, 0, 64, 3, 100) == 1
    assert expected_launches({}, 0, 1536, 16, 10) == 1 and expected_launches({}, 0, 1537, 16, 10) == 2
    assert expected_launches({}, SCORE_TWO_KERNELS, 5, 16, 10) == 2 and expected_launches({}, 0, 5, 16, 0) == 1
