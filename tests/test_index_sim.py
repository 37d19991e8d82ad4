"""The index's device-side mutation logic (csrc/index.cu: op queue -> sort -> per-key replay, the sequential at-capacity
path with its LRU order array, rehash, recency stamps) checked against the oracle WITHOUT a GPU: the same source is
compiled by g++ with -DKVB_HOST_SIM (tests/cpp/sim_cuda.h: malloc for device memory, loops for kernels) and driven
through the product's own Python binding.  The GPU tests (tests/test_gpu_index.py) run the same scenarios on the real
kernels; this file exists so that a logic error shows up before a GPU is spent on it."""
import ctypes as C
import importlib
import os
import sys

import numpy as np
import pytest

from oracle import kvblock_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SIM_NAMES = ["kvb_index_create", "kvb_index_destroy", "kvb_index_set_tier_weight", "kvb_index_add", "kvb_index_evict",
             "kvb_index_get_request_key", "kvb_index_num_keys", "kvb_index_flush", "kvb_index_get_stats",
             "kvb_index_lookup", "kvb_index_host_peek"]


@pytest.fixture(scope="module")
def sim():
    spec = importlib.util.spec_from_file_location("build_index_sim", os.path.join(ROOT, "tests", "cpp", "build_index_sim.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    lib = C.CDLL(mod.build())
    kvb = importlib.import_module("llm-d-kv-cache_b200")
    kvb._lib.bind(lib, SIM_NAMES)
    lib.kvb_last_error = lambda: b"(host simulation)"
    return kvb, lib


def _as_tuples(d):
    return {int(k): [(e.pod_identifier, e.device_tier, bool(e.speculative)) for e in v] for k, v in d.items()}


def _random_traffic(kvb, lib, seed, size, ppk, n_keys, steps, max_batch, lookup_frac=0.35, evict_frac=0.2):
    K = kvb.kvblock
    rng = np.random.default_rng(seed)
    idx = K.Index(size=size, pod_cache_size=ppk, expected_keys=16, lib=lib)
    oidx = o.InMemoryIndex(size=size, pod_cache_size=ppk)
    pods = ["pod-%d" % i for i in range(12)]
    tiers = ["gpu", "cpu", "GPU", "disk"]
    keyspace = [int(x) for x in rng.integers(1, 1 << 63, n_keys)]
    for step in range(steps):
        op = rng.random()
        if op < 1.0 - lookup_frac - evict_frac:
            n = int(rng.integers(1, max_batch + 1))
            rks = [keyspace[int(i)] for i in rng.integers(0, len(keyspace), n)]
            mode = rng.integers(0, 3)
            eks = None if mode == 0 else [int(x) for x in rng.integers(1, 200, n if mode == 1 else 1)]
            ents = [(pods[int(rng.integers(0, 12))], tiers[int(rng.integers(0, 4))], bool(rng.integers(0, 2)))
                    for _ in range(int(rng.integers(1, 4)))]
            idx.add(eks, rks, [K.PodEntry(*e) for e in ents])
            oidx.add(eks, rks, [o.PodEntry(*e) for e in ents])
        elif op < 1.0 - lookup_frac:
            ents = [(pods[int(rng.integers(0, 12))], tiers[int(rng.integers(0, 4))], bool(rng.integers(0, 2)))
                    for _ in range(int(rng.integers(1, 3)))]
            if rng.random() < 0.5:
                k, kt = int(rng.integers(1, 200)), 0
            else:
                k, kt = keyspace[int(rng.integers(0, len(keyspace)))], 1
            idx.evict(k, kt, [K.PodEntry(*e) for e in ents])
            oidx.evict(k, kt, [o.PodEntry(*e) for e in ents])
        else:
            ks = [keyspace[int(i)] for i in rng.integers(0, len(keyspace), int(rng.integers(1, 40)))]
            flt = [] if rng.random() < 0.5 else [pods[int(i)] for i in rng.integers(0, 12, 3)] + ["unknown-pod"]
            assert _as_tuples(idx.lookup(ks, flt)) == _as_tuples(oidx.lookup(ks, flt)), step
        if step % 97 == 0:
            assert len(idx) == len(oidx.data), step
            for ek in range(1, 200, 17):
                try:
                    want = oidx.get_request_key(ek)
                except KeyError:
                    with pytest.raises(KeyError):
                        idx.get_request_key(ek)
                else:
                    assert idx.get_request_key(ek) == want
    # final state: every key, entry order included
    assert _as_tuples(idx.lookup(keyspace)) == _as_tuples(oidx.lookup(keyspace))
    st = idx.stats()
    idx.close()
    return st


def test_at_capacity_sequential_path_is_exact_lru(sim):
    """Size 300, 500 distinct keys: the outer LRU evicts all the time; lookups refresh recency in between (the
    reference's data.Get), so WHICH key goes is decided by adds, evicts and reads together."""
    kvb, lib = sim
    st = _random_traffic(kvb, lib, seed=123, size=300, ppk=4, n_keys=500, steps=2500, max_batch=5)
    assert st["lru_evictions"] > 100 and st["flushes_sequential"] > 0 and st["order_builds"] >= 1


def test_tiny_capacity_exhausts_the_order_array(sim):
    """Size 3 with batches of up to 40 keys: one Add inserts more keys than the index holds, so the order array runs out
    inside a batch and the oldest key is found by the scan; evicted keys reappear later in the same call."""
    kvb, lib = sim
    st = _random_traffic(kvb, lib, seed=5, size=3, ppk=2, n_keys=60, steps=600, max_batch=40)
    assert st["order_scans"] > 0


def test_sequential_replay_stops_and_resumes_instead_of_scanning(sim):
    """With KVB_INDEX_SCAN_MAX_SLOTS=0 every table counts as too large to scan: when the order array runs out inside a
    one-thread replay (KVB_INDEX_PLAN=0 sends every at-capacity batch there) the kernel stops, the host rebuilds the
    order array and the replay resumes at the next op — same reads as the oracle, no scan.  Own process: both switches
    are read once."""
    import subprocess
    code = (
        "import sys, importlib, ctypes as C\n"
        "sys.path.insert(0, %r)\n"
        "import tests.test_index_sim as T\n"
        "spec = importlib.util.spec_from_file_location('b', %r)\n"
        "mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)\n"
        "lib = C.CDLL(mod.build())\n"
        "kvb = importlib.import_module('llm-d-kv-cache_b200')\n"
        "kvb._lib.bind(lib, T.SIM_NAMES)\n"
        "lib.kvb_last_error = lambda: b'(sim)'\n"
        "tot = 0\n"
        "for seed, size, nk, mb in ((5, 3, 60, 40), (123, 300, 500, 5), (11, 2000, 6000, 300)):\n"
        "    st = T._random_traffic(kvb, lib, seed=seed, size=size, ppk=3, n_keys=nk, steps=400, max_batch=mb)\n"
        "    assert st['order_scans'] == 0, st\n"
        "    tot += st['replay_resumes']\n"
        "assert tot > 10, tot\n"
        "print('resumes', tot)\n") % (ROOT, os.path.join(ROOT, "tests", "cpp", "build_index_sim.py"))
    env = dict(os.environ, KVB_INDEX_SCAN_MAX_SLOTS="0", KVB_INDEX_PLAN="0")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "resumes" in r.stdout, (r.stdout[-500:], r.stderr[-1500:])


def test_unknown_only_filter_with_every_pod_id_taken(sim):
    """Pod ids 0..65534 are assignable, 65535 is reserved and refused by kvb_index_add.  With all of them taken, a lookup
    whose filter names only unknown pods returns {} (the reference returns an empty map) and still refreshes the keys
    it finds."""
    kvb, lib = sim
    K = kvb.kvblock
    idx = K.Index(size=3, pod_cache_size=2, expected_keys=16, lib=lib)
    for i in range(65535):
        assert idx.pods.get("p%d" % i) == i
    with pytest.raises(OverflowError):
        idx.pods.get("one-too-many")
    e = [K.PodEntry("p65534", "gpu")]
    for k in (1, 2, 3):
        idx.add(None, [k], e)
    assert idx.lookup([1, 99], ["nobody"]) == {}          # 1 is now the newest
    assert len(idx.pods.names) == 65535
    idx.add(None, [4], e)                                 # evicts 2
    assert idx.lookup([1], ["p65534", "nobody"]) == {1: e}
    assert set(idx.lookup([1, 2, 3, 4])) == {1, 3, 4}
    reserved = (kvb._lib.PodEntryC * 1)()
    reserved[0].pod = kvb._lib.NO_SUCH_POD                # no entry may carry the reserved id
    k = np.asarray([5], dtype=np.uint64)
    assert lib.kvb_index_add(idx._h, None, 0, 0, k.ctypes.data, 1, reserved, 1) == -1
    assert set(idx.lookup([1, 2, 3, 4, 5])) == {1, 3, 4}
    idx.close()


def test_parallel_path_big_batches_growth_and_tombstones(sim):
    """No capacity pressure, batches of up to 400 keys with many repeats: sorted per-key replay, device-side rehash
    (the table starts at 2048 slots) and tombstone reuse."""
    kvb, lib = sim
    st = _random_traffic(kvb, lib, seed=9, size=10 ** 8, ppk=10, n_keys=6000, steps=400, max_batch=400, lookup_frac=0.2)
    assert st["flushes_parallel"] > 50 and st["rehashes"] >= 1 and st["lru_evictions"] == 0


def test_capacity_crossing_mixed_paths(sim):
    """Size 2000 with 6000 keys and big batches: the index fills through the parallel path, then runs at capacity."""
    kvb, lib = sim
    st = _random_traffic(kvb, lib, seed=11, size=2000, ppk=3, n_keys=6000, steps=300, max_batch=300, lookup_frac=0.3)
    assert st["flushes_parallel"] > 0 and st["flushes_sequential"] > 0 and st["lru_evictions"] > 0


def test_at_capacity_add_only_batches_are_planned_in_parallel(sim):
    """Add-only batches of up to 400 keys into a full index: the victims are planned before the parallel apply and the
    result is the reference's one-at-a-time LRU, lookups (which re-stamp keys and leave stale order records) included."""
    kvb, lib = sim
    st = _random_traffic(kvb, lib, seed=21, size=1500, ppk=3, n_keys=5000, steps=400, max_batch=400, lookup_frac=0.4,
                         evict_frac=0.0)
    assert st["flushes_planned"] > 20 and st["lru_evictions"] > 1000
    st = _random_traffic(kvb, lib, seed=22, size=700, ppk=2, n_keys=900, steps=500, max_batch=120, lookup_frac=0.5,
                         evict_frac=0.02)   # small key space: old keys are re-announced all the time
    assert st["flushes_planned"] > 20


def test_at_capacity_mixed_add_evict_batches_are_planned_too(sim):
    """A quarter of the ops remove pods (keys disappear when their last pod leaves), so `live` moves both ways inside a
    batch: eviction times come from the running maximum of live, not from the insertion count."""
    kvb, lib = sim
    for seed, size, n_keys, mb in ((50, 1750, 3050, 380), (57, 1967, 3421, 429), (61, 2091, 3633, 457)):
        st = _random_traffic(kvb, lib, seed=seed, size=size, ppk=3, n_keys=n_keys, steps=300, max_batch=mb, lookup_frac=0.25,
                             evict_frac=0.25)
        assert st["flushes_planned"] > 30 and st["plan_fallbacks"] == 0 and st["lru_evictions"] > 5000, st


def test_planned_eviction_conflicts_and_survivors(sim):
    """The two cases the plan must tell apart (in_memory.go:186-199): an old key announced BEFORE the insertion that
    would have evicted it moves to the newest end and survives; announced AFTER, the reference evicts it and then
    re-creates it with only the new entry (one more insertion, so one more eviction) — the plan absorbs it."""
    kvb, lib = sim
    K = kvb.kvblock
    for late in (False, True):
        idx, oidx = K.Index(size=100, pod_cache_size=4, expected_keys=16, lib=lib), o.InMemoryIndex(size=100, pod_cache_size=4)
        for i in range(100):
            idx.add(None, [1000 + i], [K.PodEntry("old", "gpu")])
            oidx.add(None, [1000 + i], [o.PodEntry("old", "gpu")])
        idx.flush()
        new = list(range(5000, 5050))
        batch = new + [1010] if late else [1040] + new
        idx.add(None, batch, [K.PodEntry("new", "cpu")])
        oidx.add(None, batch, [o.PodEntry("new", "cpu")])
        probe = list(range(1000, 1100)) + new
        assert _as_tuples(idx.lookup(probe)) == _as_tuples(oidx.lookup(probe))
        st = idx.stats()
        assert st["plan_fallbacks"] == 0 and st["flushes_planned"] == 1 and st["lru_evictions"] == (51 if late else 50)
        if late:
            assert _as_tuples(idx.lookup([1010])) == {1010: [("new", "cpu", False)]}
        else:
            assert len(idx.lookup([1040])[1040]) == 2 and idx.lookup([1050]) == {}
        idx.close()


def test_planned_eviction_rebuilds_a_used_up_order(sim):
    """Lookups re-stamp most keys after the order array was built: its records go stale, the plan runs out of
    untouched records, rebuilds the order once and finishes in parallel."""
    kvb, lib = sim
    K = kvb.kvblock
    idx, oidx = K.Index(size=400, pod_cache_size=2, expected_keys=16, lib=lib), o.InMemoryIndex(size=400, pod_cache_size=2)
    keys = list(range(1, 401))
    for blk in (keys[:200], keys[200:]):
        idx.add(None, blk, [K.PodEntry("a", "gpu")])
        oidx.add(None, blk, [o.PodEntry("a", "gpu")])
    idx.flush()
    idx.add(None, list(range(1000, 1020)), [K.PodEntry("b", "gpu")])       # first eviction: builds the order array
    oidx.add(None, list(range(1000, 1020)), [o.PodEntry("b", "gpu")])
    assert _as_tuples(idx.lookup(keys[20:390])) == _as_tuples(oidx.lookup(keys[20:390]))   # ... and makes it stale
    idx.add(None, list(range(2000, 2100)), [K.PodEntry("c", "gpu")])
    oidx.add(None, list(range(2000, 2100)), [o.PodEntry("c", "gpu")])
    probe = keys + list(range(1000, 1020)) + list(range(2000, 2100))
    assert _as_tuples(idx.lookup(probe)) == _as_tuples(oidx.lookup(probe))
    st = idx.stats()
    assert (st["flushes_planned"], st["plan_fallbacks"]) == (2, 0) and st["order_builds"] >= 2, st
    idx.close()


def test_contract_scenarios_on_the_sim(sim):
    """index_test.go:119-264,589-735; in_memory_test.go:45-236 (the assertions of tests/test_gpu_index.py::test_index_contract)."""
    kvb, lib = sim
    K = kvb.kvblock
    P = lambda p, t, s=False: K.PodEntry(p, t, s)
    idx = K.Index(lib=lib)
    idx.add([1, 2], [11, 12], [P("p1", "gpu"), P("p2", "gpu")])
    assert idx.lookup([11, 12]) == {11: [P("p1", "gpu"), P("p2", "gpu")], 12: [P("p1", "gpu"), P("p2", "gpu")]}
    idx.add([1], [11], [P("p1", "gpu")])
    assert idx.lookup([11])[11] == [P("p2", "gpu"), P("p1", "gpu")]          # re-added entry becomes the newest
    assert idx.lookup([11, 12], {"p1"}) == {11: [P("p1", "gpu")], 12: [P("p1", "gpu")]}
    assert idx.lookup([11], {"nobody"}) == {}
    assert idx.lookup([999, 11]).keys() == {11}
    idx.add([3], [13], [P("p3", "gpu"), P("p3", "cpu")])
    idx.evict(3, K.ENGINE_KEY, [P("p3", "cpu")])
    assert idx.lookup([13]) == {13: [P("p3", "gpu")]}
    idx.add([20, 21, 22, 23], [30], [P("p", "gpu")])
    assert idx.get_request_key(20) == 30 and idx.get_request_key(23) == 30
    idx.evict(21, K.ENGINE_KEY, [P("p", "gpu")])
    assert idx.lookup([30]) == {}
    idx.add([40], [50, 51, 52, 53], [P("p", "gpu")])
    assert idx.get_request_key(40) == 53
    with pytest.raises(KeyError):
        idx.get_request_key(12345)
    idx.evict(777, K.ENGINE_KEY, [P("p", "gpu")])
    idx.add(None, [60], [P("p", "gpu", True)])
    idx.add([61], [60], [P("p", "gpu", False)])
    assert idx.lookup([60])[60] == [P("p", "gpu", True), P("p", "gpu", False)]
    idx.evict(60, K.REQUEST_KEY, [P("p", "gpu", True)])
    assert idx.lookup([60])[60] == [P("p", "gpu", False)]
    assert idx.host_peek(60) == [P("p", "gpu", False)] and idx.host_peek(4242) is None
    small = K.Index(size=2, pod_cache_size=2, lib=lib)
    for k in (1, 2, 3):
        small.add([k], [k], [P("p", "gpu")])
    assert small.lookup([1, 2, 3]).keys() == {2, 3}
    small.add([2], [2], [P("a", "gpu"), P("b", "gpu"), P("c", "gpu")])
    assert small.lookup([2])[2] == [P("b", "gpu"), P("c", "gpu")]


def test_reads_decide_which_key_is_evicted(sim):
    """Capacity pressure with reads between adds: a key that was only LOOKED UP must survive the next eviction
    (Lookup's data.Get, in_memory.go:120) — the default, no flag."""
    kvb, lib = sim
    K = kvb.kvblock
    e = [K.PodEntry("p", "gpu")]
    idx = K.Index(size=4, pod_cache_size=2, lib=lib)
    for k in (1, 2, 3, 4):
        idx.add(None, [k], e)
    assert set(idx.lookup([1])) == {1}            # 1 becomes the newest
    idx.add(None, [5], e)                         # evicts 2, not 1
    assert set(idx.lookup([1, 2, 3, 4, 5])) == {1, 3, 4, 5}
    idx.add(None, [6, 7], e)                      # the lookup above refreshed 1,3,4,5 in that order -> 1 and 3 go
    assert set(idx.lookup([1, 2, 3, 4, 5, 6, 7])) == {4, 5, 6, 7}
