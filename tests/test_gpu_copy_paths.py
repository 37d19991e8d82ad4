"""The paged-block movers of copy_kernels.cu (gather, scatter, migrate) under every configuration the flags word can
select, byte-exact against a numpy reference, inside guard bands, with a check of which kernel ran.

Guard bands: every buffer (each pool tensor, the packed buffer, pinned host buffers) is carved out of a larger
allocation whose margins (64 KiB or more: larger than any piece a mover uses) hold seeded random bytes.  After every
call the whole allocation is compared with what it must hold: the result region, every margin, every row that was not
listed and the [frag, stride) tail of every row.

Selection model: expected_launch() restates the launch logic of copy_kernels.cu and the vector width kvb_pool_create
picks.  The unmarked tests pin it to hand-worked cases.  On the GPU, each block of calls runs under torch.profiler with
CUDA activity, and the mover kernels in the trace must be, one per call and in order, the ones the model predicts:
demangled name, and grid, block and shared memory where the trace records them.  When the profiler returns no kernel
activity at all, those tests check every byte and then skip, saying that the kernel identity was not asserted.

flags layout (copy_kernels.cu): bits 0-7 variant (0 = KVB_COPY_VARIANT, default BULK), bits 8-11 LDG unroll or BULK
depth code + 1, bits 12-19 CTAs per SM, bits 20-23 BULK piece = 1 KiB << code."""
from __future__ import annotations

import importlib
import json
import os
import subprocess
import sys
import tempfile
import threading
from typing import NamedTuple

import numpy as np
import pytest

from oracle import offload_oracle as oo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LDG, BULK = 1, 2
GATHER, SCATTER, MIGRATE = 0, 1, 2            # the kernels' MODE template argument
LDG_THREADS, BULK_THREADS = 256, 32
RING_BUDGET = 224 << 10                        # launch_bulk: rings of all CTAs of an SM fit 224 KiB
PEER_DEFAULT = LDG | 4 << 8 | 8 << 12          # launch_migrate: default mover for a peer destination
VEC_TYPE = {16: "int4", 8: "uint2", 4: "unsigned int", 2: "unsigned char", 1: "unsigned char"}
MARGIN = 64 << 10
SM_COUNT_FALLBACK = 132


# ------------------------------------------------------------------------------------------------- selection model
class Tuning(NamedTuple):
    """The library defaults (copy_kernels.cu tuning()), each overridable by its environment variable."""
    variant: int = BULK        # KVB_COPY_VARIANT
    ldg_unroll: int = 4        # KVB_LDG_UNROLL
    ldg_ctas: int = 8          # KVB_LDG_CTAS_PER_SM
    bulk_piece: int = 8192     # KVB_BULK_PIECE
    bulk_ctas: int = 2         # KVB_BULK_CTAS_PER_SM
    bulk_deep: int = 0         # KVB_BULK_DEEP


DEFAULT_TUNING = Tuning()


class Launch(NamedTuple):
    family: str      # "ldg" or "bulk"
    mode: int        # GATHER / SCATTER / MIGRATE
    vec: int         # bytes per vector access (bulk: 16)
    unroll: int      # ldg only
    stages: int      # bulk only
    lookahead: int   # bulk only
    piece: int       # bytes per work item (the last piece of a fragment may be shorter)
    grid: int
    block: int
    smem: int        # dynamic shared memory

    @property
    def kernel(self) -> str:
        if self.family == "ldg":
            return f"paged_copy_ldg_kernel<{self.mode}, {VEC_TYPE[self.vec]}, {self.unroll}>"
        return f"paged_copy_bulk_kernel<{self.mode}, {self.stages}, {self.lookahead}>"


def pool_vec(frag: int, stride: int, bases) -> int:
    """kvb_pool_create: the widest of 16/8/4/2/1 B dividing the fragment, the row stride and every tensor base."""
    vec = 16
    while vec > 1 and (frag % vec or stride % vec):
        vec >>= 1
    for b in bases:
        while vec > 1 and b % vec:
            vec >>= 1
    return vec


def expected_launch(mode: int, n: int, T: int, frag: int, vec: int, flags: int, sms: int,
                    tuning: Tuning = DEFAULT_TUNING, packed_addr: int = 0, peer: bool = False):
    """The kernel one gather / scatter / migrate call launches, or None when it launches nothing.

    vec: the pool's width (migrate: the smaller of the two pools'); gather and scatter narrow it to the packed address.
    peer: migrate only, the destination pool is marked peer."""
    if mode == MIGRATE:
        if flags & 0xFF == 0 and peer and vec == 16:
            flags = PEER_DEFAULT
    else:
        while vec > 1 and packed_addr % vec:
            vec >>= 1
    frags = n * T
    if frags == 0:
        return None
    variant = flags & 0xFF or tuning.variant
    if variant == BULK and vec != 16:  # TMA bulk copies need 16 B aligned addresses and sizes
        variant = LDG
    code8, ctas_code, piece_code = (flags >> 8) & 0xF, (flags >> 12) & 0xFF, (flags >> 20) & 0xF
    if variant == BULK:
        deep = code8 - 1 if code8 else tuning.bulk_deep
        ctas = max(1, ctas_code or tuning.bulk_ctas)
        piece = 1024 << piece_code if piece_code else tuning.bulk_piece
        if piece < 1024 or piece % 16:
            piece = 16384
        stages = {1: 8, 2: 12}.get(deep, 6)
        while piece > 1024 and piece * stages * ctas > RING_BUDGET:
            piece >>= 1
        piece = min(piece, frag)
        items = frags * -(-frag // piece)
        return Launch("bulk", mode, 16, 0, stages, stages // 2, piece, max(1, min(items, sms * ctas)), BULK_THREADS,
                      stages * piece)
    unroll = code8 or tuning.ldg_unroll
    unroll = unroll if unroll in (2, 8) else 4
    ctas = max(1, ctas_code or tuning.ldg_ctas)
    piece = LDG_THREADS * unroll * vec
    items = frags * -(-frag // piece)
    return Launch("ldg", mode, vec, unroll, 0, 0, piece, max(1, min(items, sms * ctas)), LDG_THREADS, 0)


# ------------------------------------------------------------------------------------------------ flag matrix
LDG_FLAGS = [LDG | u << 8 | c << 12 for u in (2, 4, 8) for c in (1, 8, 32)]
BULK_FLAGS = [BULK | (d + 1) << 8 | c << 12 | p << 20 for d in (0, 1, 2) for c in (1, 2, 4, 64) for p in range(1, 7)]
PLAIN_FLAGS = [0, LDG, BULK]
# out-of-range codes: unroll 3 runs unroll 4, depth code 5 runs the 6-stage ring, piece code 9 (512 KiB) is halved
ODD_FLAGS = [LDG | 3 << 8, BULK | 5 << 8, BULK | 9 << 20]
FULL_FLAGS = PLAIN_FLAGS + LDG_FLAGS + BULK_FLAGS + ODD_FLAGS
SHORT_FLAGS = PLAIN_FLAGS + [LDG | 2 << 8 | 32 << 12, LDG | 8 << 8 | 1 << 12, BULK | 2 << 8 | 1 << 12 | 1 << 20,
                             BULK | 3 << 8 | 4 << 12 | 6 << 20, BULK | 2 << 8 | 64 << 12]


def flag_name(f: int) -> str:
    return (f"flags={f:#x} (variant {f & 0xFF}, bits 8-11 {(f >> 8) & 0xF}, CTAs/SM {(f >> 12) & 0xFF}, "
            f"piece code {(f >> 20) & 0xF})")


# ------------------------------------------------------------------------------------------------ numpy reference
def ref_gather(rows, frag: int, ids) -> np.ndarray:
    """Packed [block][tensor][fragment] bytes of the listed rows; rows: T arrays (num_blocks, stride)."""
    ids = np.asarray(ids, dtype=np.int64)
    out = np.empty((ids.size, len(rows), frag), dtype=np.uint8)
    for t, r in enumerate(rows):
        out[:, t, :] = r[ids, :frag]
    return out.reshape(-1)


def ref_scatter(rows, frag: int, ids, packed: np.ndarray) -> None:
    """In place: row ids[b] of tensor t gets packed block (b, t) in its first frag bytes; nothing else changes."""
    ids = np.asarray(ids, dtype=np.int64)
    src = packed.reshape(ids.size, len(rows), frag)
    for t, r in enumerate(rows):
        r[ids, :frag] = src[:, t, :]


def ref_migrate(src_rows, dst_rows, frag: int, src_ids, dst_ids) -> None:
    """In place: dst[dst_ids[i]][:frag] = src[src_ids[i]][:frag] in every tensor; nothing else changes."""
    s, d = np.asarray(src_ids, dtype=np.int64), np.asarray(dst_ids, dtype=np.int64)
    for sr, dr in zip(src_rows, dst_rows):
        dr[d, :frag] = sr[s, :frag]


def id_lists(N: int, n: int, rng, dup: bool):
    """(name, ids) lists of min(n, N) ids: a random permutation, reversed order, two contiguous runs (N-k..N-1, 0..),
    both ends first and last, and, when dup, random ids with repeats (gather only: repeated scatter targets race)."""
    n = min(n, N)
    out = [("permutation", rng.permutation(N)[:n]),
           ("reversed", np.arange(N)[::-1][:n]),
           ("runs", np.roll(np.arange(N), N // 3)[:n]),
           ("ends", np.r_[N - 1, rng.permutation(np.arange(1, N - 1))[:max(0, n - 2)], 0][:n] if n > 1
            else np.array([N - 1]))]
    if dup:
        d = rng.integers(0, N, n)
        if n > 1:
            d[-1] = d[0]
        out.append(("duplicates", d))
    return [(name, np.ascontiguousarray(ids, dtype=np.int64)) for name, ids in out]


# ------------------------------------------------------------------------------------------------ guarded memory
class Ptr(int):
    """A raw address passed where KVPool expects a tensor."""

    def data_ptr(self) -> int:
        return int(self)


def _round_up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


class Slab:
    """One allocation holding named regions, each placed at a chosen address mod 16 with MARGIN or more of seeded random
    guard bytes around it.  ``want`` holds what every byte of the allocation must be; check() compares all of it.

    pinned: None for device memory, else a callable returning a PinnedBuffer of the given size."""

    def __init__(self, torch, regions, seed: int, pinned=None):
        self.torch = torch
        self.rng = np.random.default_rng(seed)
        self.names, self.sizes, self.strides, offs = [], [], [], []
        pos = MARGIN
        for name, nbytes, mis, stride in regions:
            pos = _round_up(pos, 256) + mis
            offs.append(pos)
            self.names.append(name)
            self.sizes.append(nbytes)
            self.strides.append(stride)
            pos += nbytes + MARGIN
        total = pos + 256
        if pinned is None:
            self.dev = torch.empty(total, dtype=torch.uint8, device="cuda")
            self.host = None
            base = self.dev.data_ptr()
        else:
            self.host = pinned(total)
            self.dev = None
            base = self.host.ptr
        self.base = base
        shift = (-base) % 256
        self.start = [shift + o for o in offs]
        self.want = self.rng.integers(0, 256, total, dtype=np.uint8)
        self.upload()

    def addr(self, i: int) -> int:
        return self.base + self.start[i]

    def view(self, i: int) -> np.ndarray:
        return self.want[self.start[i]:self.start[i] + self.sizes[i]]

    def rows(self, i: int, stride: int) -> np.ndarray:
        return self.view(i)[: self.sizes[i] // stride * stride].reshape(-1, stride)

    def upload(self, i: int | None = None) -> None:
        lo, hi = (0, self.want.size) if i is None else (self.start[i], self.start[i] + self.sizes[i])
        if self.dev is not None:
            self.dev[lo:hi].copy_(self.torch.from_numpy(self.want[lo:hi]))
        else:
            np.copyto(self.host.numpy()[lo:hi], self.want[lo:hi])

    def refill(self, i: int) -> None:
        """New random bytes in region i (device and mirror)."""
        self.view(i)[:] = self.rng.integers(0, 256, self.sizes[i], dtype=np.uint8)
        self.upload(i)

    def check(self):
        """None when every byte is as expected, else where the first and last wrong bytes are."""
        got = self.dev.cpu().numpy() if self.dev is not None else self.host.numpy().copy()
        if np.array_equal(got, self.want):
            return None
        bad = np.flatnonzero(got != self.want)
        self.upload()  # start the next call from the expected state
        return f"{bad.size} wrong bytes, first at {self._where(bad[0])}, last at {self._where(bad[-1])}"

    def _where(self, k: int) -> str:
        for i, s in enumerate(self.start):
            if k < s:
                return f"guard band {s - k} B before {self.names[i]}"
            if k < s + self.sizes[i]:
                o = k - s
                if self.strides[i]:
                    return f"{self.names[i]} row {o // self.strides[i]} byte {o % self.strides[i]}"
                return f"{self.names[i]} byte {o}"
        end = self.start[-1] + self.sizes[-1]
        return f"guard band {k - end} B after {self.names[-1]}"


class PoolUT(NamedTuple):
    pool: object
    rows: list       # T views (N, stride) into the slab's expected bytes
    T: int
    N: int
    frag: int
    stride: int
    vec: int


def make_pool(kvb, slab: Slab, regions, N: int, frag: int, stride: int) -> PoolUT:
    ptrs = [slab.addr(i) for i in regions]
    pool = kvb.pool.KVPool(None, 0, ptrs=ptrs, num_blocks=N, frag_bytes=frag, stride_bytes=stride)
    pool._slab = slab  # the pool borrows the slab's memory
    return PoolUT(pool, [slab.rows(i, stride) for i in regions], len(ptrs), N, frag, stride,
                  pool_vec(frag, stride, ptrs))


def tensor_regions(prefix: str, T: int, N: int, stride: int, bases=(0,)):
    return [(f"{prefix}{t}", N * stride, bases[t % len(bases)], stride) for t in range(T)]


# ------------------------------------------------------------------------------------------------ kernel identity
class KernelLog:
    """torch.profiler with CUDA activity around a block of calls.  Afterwards ``kernels`` holds the mover kernels of the
    trace in launch order (name and the trace's args), and ``any_kernels`` says whether the trace had kernels at all."""

    def __init__(self, torch):
        self.torch = torch
        self.kernels, self.any_kernels = [], False

    def __enter__(self):
        from torch.profiler import ProfilerActivity, profile
        try:
            self.prof = profile(activities=[ProfilerActivity.CUDA])
            self.prof.__enter__()
        except Exception:  # noqa: BLE001 - no profiler: the calls still run and every byte is still checked
            self.prof = None
        # the first kernel after the profiler starts is sometimes missing from the trace (seen on H100 with torch
        # 2.11): let a kernel that is not a mover take that place
        self.torch.cuda._sleep(1000)
        self.torch.cuda.synchronize()
        return self

    def __exit__(self, *exc):
        self.torch.cuda.synchronize()
        if self.prof is None:
            return False
        self.prof.__exit__(*exc)
        if exc[0] is not None:
            return False
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            self.prof.export_chrome_trace(path)
            with open(path) as f:
                events = json.load(f).get("traceEvents", [])
        ks = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e.get("ts", 0))
        self.any_kernels = bool(ks)
        self.kernels = [{"name": _mover_name(e.get("name", "")), "args": e.get("args", {})}
                        for e in ks if "paged_copy_" in e.get("name", "")]
        return False


def _mover_name(demangled: str) -> str:
    """'void kvb::paged_copy_bulk_kernel<1, 12, 6>(kvb::CopyArgs)' -> 'paged_copy_bulk_kernel<1, 12, 6>'."""
    i = demangled.find("paged_copy_")
    j = demangled.find(">", i)
    return demangled[i:j + 1] if i >= 0 and j > i else demangled


def identity_failures(kernels, expected) -> list:
    """Mover kernels of a trace against [(label, Launch)] in call order.  Shared memory in the trace is static plus
    dynamic: what is left after the predicted dynamic size must be one small constant per kernel."""
    out = []
    if len(kernels) != len(expected):
        out.append(f"{len(kernels)} mover kernels in the trace, {len(expected)} launches expected")
    static = {}
    for (label, want), k in zip(expected, kernels):
        args, msg = k["args"], []
        if k["name"] != want.kernel:
            msg.append(f"ran {k['name']}, the model says {want.kernel}")
        if "grid" in args and list(args["grid"]) != [want.grid, 1, 1]:
            msg.append(f"grid {args['grid']}, the model says {want.grid}")
        if "block" in args and list(args["block"]) != [want.block, 1, 1]:
            msg.append(f"block {args['block']}, the model says {want.block}")
        if "shared memory" in args:
            rest = int(args["shared memory"]) - want.smem
            static.setdefault(want.kernel, {}).setdefault(rest, label)
            if not 0 <= rest <= 2048:
                msg.append(f"shared memory {args['shared memory']} B, the model's dynamic size is {want.smem} B")
        if msg:
            out.append(f"{label}: " + "; ".join(msg))
    for name, rests in static.items():
        if len(rests) > 1:
            out.append(f"{name}: trace shared memory minus the model's dynamic size differs between launches: "
                       + "; ".join(f"{r} B at {lab}" for r, lab in sorted(rests.items())))
    return out


class Run:
    """Calls movers one at a time; after each it checks the launch count and every byte of every slab, and records the
    launch the model predicts."""

    def __init__(self, kvb, torch, slabs):
        self.lib = kvb._lib.load()
        self.torch = torch
        self.slabs = slabs
        self.sms = sm_count(torch)
        self.expected, self.failures = [], []

    def call(self, label: str, fn, launch) -> None:
        before = self.lib.kvb_launch_count()
        try:
            fn()
        except Exception as e:  # noqa: BLE001 - a refused call is a finding for this configuration
            self.failures.append(f"{label}: {e}")
            return
        self.torch.cuda.synchronize()
        ran = self.lib.kvb_launch_count() - before
        want = 0 if launch is None else 1
        if ran != want:
            self.failures.append(f"{label}: {ran} launches counted, {want} expected")
        if launch is not None:
            self.expected.append((label, launch))
        for s in self.slabs:
            err = s.check()
            if err:
                self.failures.append(f"{label}: {err}")

    def finish(self, log: KernelLog) -> None:
        assert not self.failures, f"{len(self.failures)} failing calls:\n" + "\n".join(self.failures[:20])
        if self.expected and not log.any_kernels:
            pytest.skip(f"every byte of {len(self.expected)} launches checked; torch.profiler returned no CUDA kernel "
                        f"activity, so which kernel ran was not asserted")
        fails = identity_failures(log.kernels, self.expected)
        assert not fails, f"{len(fails)} kernel-identity mismatches:\n" + "\n".join(fails[:20])


def sm_count(torch) -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count or SM_COUNT_FALLBACK


# ------------------------------------------------------------------------------------------------ the three moves
def do_gather(run: Run, p: PoolUT, slab: Slab, preg: int, ids, flags: int, label: str) -> None:
    slab.refill(preg)
    want = ref_gather(p.rows, p.frag, ids)
    slab.view(preg)[:want.size] = want
    launch = expected_launch(GATHER, ids.size, p.T, p.frag, p.vec, flags, run.sms, packed_addr=slab.addr(preg))
    run.call(f"gather {label}", lambda: p.pool.gather(ids, Ptr(slab.addr(preg)), flags=flags), launch)


def do_scatter(run: Run, p: PoolUT, slab: Slab, preg: int, ids, flags: int, label: str) -> None:
    slab.refill(preg)
    ref_scatter(p.rows, p.frag, ids, slab.view(preg)[:ids.size * p.T * p.frag])
    launch = expected_launch(SCATTER, ids.size, p.T, p.frag, p.vec, flags, run.sms, packed_addr=slab.addr(preg))
    run.call(f"scatter {label}", lambda: p.pool.scatter(ids, Ptr(slab.addr(preg)), flags=flags), launch)


def do_roundtrip(run: Run, p: PoolUT, slab: Slab, preg: int, ids, flags: int, label: str) -> None:
    """gather -> zero the listed rows' fragments -> scatter: the pool ends as it began."""
    do_gather(run, p, slab, preg, ids, flags, f"(round trip) {label}")
    before = [r.copy() for r in p.rows]
    for r in p.rows:
        r[ids, :p.frag] = 0
    slab.upload()
    for r, b in zip(p.rows, before):
        r[:] = b
    launch = expected_launch(SCATTER, ids.size, p.T, p.frag, p.vec, flags, run.sms, packed_addr=slab.addr(preg))
    run.call(f"scatter (round trip) {label}", lambda: p.pool.scatter(ids, Ptr(slab.addr(preg)), flags=flags), launch)


def do_migrate(kvb, run: Run, src: PoolUT, dst: PoolUT, sids, dids, flags: int, peer: bool, label: str) -> None:
    ref_migrate(src.rows, dst.rows, src.frag, sids, dids)
    launch = expected_launch(MIGRATE, sids.size, src.T, src.frag, min(src.vec, dst.vec), flags, run.sms, peer=peer)
    run.call(f"migrate {label}", lambda: kvb.migrate.migrate_blocks(src.pool, dst.pool, sids, dids, flags=flags),
             launch)


# ================================================================================================ CPU: the model
def _L(family, mode, vec, unroll, stages, piece, grid, smem):
    return Launch(family, mode, vec, unroll, stages, stages // 2, piece, grid,
                  LDG_THREADS if family == "ldg" else BULK_THREADS, smem)


# (id, model arguments, expected launch), worked by hand from copy_kernels.cu on a 132-SM part
HAND_CASES = [
    # piece code 6 (64 KiB) x 6 stages x 2 CTAs = 768 KiB > 224 KiB: halved twice to 16 KiB (192 KiB)
    ("piece6-6stages-2ctas", dict(mode=GATHER, n=10, T=4, frag=65536, vec=16, flags=BULK | 1 << 8 | 2 << 12 | 6 << 20),
     _L("bulk", GATHER, 16, 0, 6, 16384, 160, 6 * 16384)),
    # 48 B fragment under BULK: the 8 KiB piece is clamped to 48 B, 6 x 48 = 288 B of ring; 2 x 3 items < grid
    ("bulk-48B-fragment", dict(mode=GATHER, n=2, T=3, frag=48, vec=16, flags=BULK),
     _L("bulk", GATHER, 16, 0, 6, 48, 6, 288)),
    # flag 0 = library default BULK, 8 KiB pieces, 2 CTAs/SM: config #2's 10 000 x 64 x 32 KiB
    ("default-config2", dict(mode=GATHER, n=10000, T=64, frag=32768, vec=16, flags=0),
     _L("bulk", GATHER, 16, 0, 6, 8192, 264, 6 * 8192)),
    # LDG defaults: unroll 4 x 256 threads x 16 B = 16 KiB pieces, 8 CTAs/SM
    ("ldg-default", dict(mode=SCATTER, n=3, T=2, frag=32768, vec=16, flags=LDG),
     _L("ldg", SCATTER, 16, 4, 0, 16384, 12, 0)),
    # packed address 8 mod 16: BULK demoted to LDG with uint2; its depth code 2 read as LDG unroll 2, 64 CTAs/SM kept
    ("bulk-demoted-by-packed", dict(mode=GATHER, n=50, T=3, frag=4096, vec=16, flags=BULK | 2 << 8 | 64 << 12,
                                    packed_addr=0x10008),
     _L("ldg", GATHER, 8, 2, 0, 4096, 150, 0)),
    # packed address odd: byte mover; pool width 2 (not a kernel type) keeps a 2 KiB piece for the byte kernel
    ("vec2-byte-kernel", dict(mode=GATHER, n=4, T=1, frag=1000, vec=2, flags=LDG), _L("ldg", GATHER, 2, 4, 0, 2048, 4, 0)),
    ("odd-packed", dict(mode=SCATTER, n=4, T=1, frag=4096, vec=16, flags=LDG | 8 << 8, packed_addr=3),
     _L("ldg", SCATTER, 1, 8, 0, 2048, 8, 0)),
    # peer destination, flag 0, width 16: LDG unroll 4, 8 CTAs/SM
    ("peer-default", dict(mode=MIGRATE, n=100, T=8, frag=16384, vec=16, flags=0, peer=True),
     _L("ldg", MIGRATE, 16, 4, 0, 16384, 800, 0)),
    # explicit flags win over the peer default
    ("peer-explicit", dict(mode=MIGRATE, n=100, T=8, frag=16384, vec=16, flags=BULK | 3 << 8, peer=True),
     _L("bulk", MIGRATE, 16, 0, 12, 8192, 264, 12 * 8192)),
    # peer with width 8: no peer default; the library default BULK is demoted to LDG with its own tuning
    ("peer-narrow", dict(mode=MIGRATE, n=100, T=8, frag=16384, vec=8, flags=0, peer=True),
     _L("ldg", MIGRATE, 8, 4, 0, 8192, 1056, 0)),
    # not peer, flag 0: BULK
    ("local-migrate", dict(mode=MIGRATE, n=1, T=1, frag=16400, vec=16, flags=0),
     _L("bulk", MIGRATE, 16, 0, 6, 8192, 3, 6 * 8192)),
    # piece code 9 = 512 KiB, halved to 16 KiB for 6 stages x 2 CTAs
    ("piece-code-9", dict(mode=GATHER, n=1, T=1, frag=1 << 20, vec=16, flags=BULK | 9 << 20),
     _L("bulk", GATHER, 16, 0, 6, 16384, 64, 6 * 16384)),
    # 12 stages x 64 CTAs: halving stops at 1 KiB even though the rings exceed 224 KiB
    ("piece-floor-1KiB", dict(mode=GATHER, n=7, T=64, frag=4096, vec=16, flags=BULK | 3 << 8 | 64 << 12 | 1 << 20),
     _L("bulk", GATHER, 16, 0, 12, 1024, 1792, 12 * 1024)),
    # fragment below 1 KiB: piece = fragment
    ("frag-1008", dict(mode=SCATTER, n=5, T=64, frag=1008, vec=16, flags=BULK | 2 << 8 | 1 << 12 | 3 << 20),
     _L("bulk", SCATTER, 16, 0, 8, 1008, 132, 8 * 1008)),
    # out-of-range codes: unroll 3 -> 4, depth code 5 -> 6 stages
    ("unroll-3", dict(mode=GATHER, n=1, T=1, frag=16, vec=16, flags=LDG | 3 << 8), _L("ldg", GATHER, 16, 4, 0, 16384, 1, 0)),
    ("depth-code-5", dict(mode=GATHER, n=1, T=3, frag=16400, vec=16, flags=BULK | 5 << 8),
     _L("bulk", GATHER, 16, 0, 6, 8192, 9, 6 * 8192)),
    # short last piece: 16400 = 2 x 8 KiB + 16 B, 3 pieces per fragment
    ("short-last-piece", dict(mode=GATHER, n=96, T=3, frag=16400, vec=16, flags=BULK | 1 << 8 | 1 << 12),
     _L("bulk", GATHER, 16, 0, 6, 8192, 132, 6 * 8192)),
    ("nothing", dict(mode=GATHER, n=0, T=3, frag=4096, vec=16, flags=BULK), None),
    ("nothing-migrate", dict(mode=MIGRATE, n=0, T=3, frag=4096, vec=16, flags=0, peer=True), None),
]

# KVB_COPY_VARIANT=1 KVB_LDG_UNROLL=8 KVB_BULK_PIECE=100 KVB_BULK_DEEP=2
ENV_TUNING = Tuning(variant=LDG, ldg_unroll=8, bulk_piece=100, bulk_deep=2)
ENV_VARS = {"KVB_COPY_VARIANT": "1", "KVB_LDG_UNROLL": "8", "KVB_BULK_PIECE": "100", "KVB_BULK_DEEP": "2"}
ENV_CASES = [
    # flag 0 now means LDG, unroll 8: 256 x 8 x 16 B = 32 KiB pieces
    ("env-flag0", dict(mode=GATHER, n=5, T=3, frag=32768, vec=16, flags=0, tuning=ENV_TUNING),
     _L("ldg", GATHER, 16, 8, 0, 32768, 15, 0)),
    # plain BULK: invalid piece 100 -> 16 KiB, 12 stages x 2 CTAs -> halved to 8 KiB
    ("env-bulk", dict(mode=GATHER, n=5, T=3, frag=32768, vec=16, flags=BULK, tuning=ENV_TUNING),
     _L("bulk", GATHER, 16, 0, 12, 8192, 60, 12 * 8192)),
]


@pytest.mark.parametrize("case", HAND_CASES + ENV_CASES, ids=[c[0] for c in HAND_CASES + ENV_CASES])
def test_model_hand_worked(case):
    _, kw, want = case
    kw = dict(kw)
    assert expected_launch(sms=132, **kw) == want


def test_model_names_and_widths():
    assert _L("bulk", SCATTER, 16, 0, 12, 1024, 1, 0).kernel == "paged_copy_bulk_kernel<1, 12, 6>"
    assert _L("ldg", GATHER, 8, 8, 0, 0, 1, 0).kernel == "paged_copy_ldg_kernel<0, uint2, 8>"
    assert pool_vec(4096, 4096, [0x1000, 0x2004]) == 4
    assert pool_vec(4096, 4097, [0]) == 1 and pool_vec(1000, 1002, [0]) == 2 and pool_vec(4096, 4104, [8]) == 8
    assert len(FULL_FLAGS) == len(set(FULL_FLAGS)) == 87


def test_reference_matches_oracle():
    """The strided numpy reference equals offload_oracle.pack_blocks / unpack_blocks on the first frag bytes of every
    row, and leaves each row's tail alone; migrate equals a gather from the source then a scatter into the
    destination."""
    rng = np.random.default_rng(7)
    for T, N, frag, extra in ((3, 20, 48, 0), (2, 9, 1000, 8), (4, 16, 16, 1), (1, 5, 4096, 0)):
        stride = frag + extra
        rows = [rng.integers(0, 256, (N, stride), dtype=np.uint8) for _ in range(T)]
        for name, ids in id_lists(N, 7, rng, dup=True):
            want = oo.pack_blocks([np.ascontiguousarray(r[:, :frag]) for r in rows], ids)
            assert np.array_equal(ref_gather(rows, frag, ids), want), name
        for name, ids in id_lists(N, 7, rng, dup=False):
            assert np.unique(ids).size == ids.size, name
            packed = rng.integers(0, 256, ids.size * T * frag, dtype=np.uint8)
            mine = [r.copy() for r in rows]
            ref_scatter(mine, frag, ids, packed)
            theirs = [np.ascontiguousarray(r[:, :frag]) for r in rows]
            oo.unpack_blocks(theirs, ids, packed)
            for m, th, r in zip(mine, theirs, rows):
                assert np.array_equal(m[:, :frag], th), name
                assert np.array_equal(m[:, frag:], r[:, frag:]), name
        sids, dids = rng.permutation(N)[:5], rng.permutation(N)[:5]
        dst = [rng.integers(0, 256, (N, stride + 16), dtype=np.uint8) for _ in range(T)]
        via_packed = [d.copy() for d in dst]
        ref_migrate(rows, dst, frag, sids, dids)
        ref_scatter(via_packed, frag, dids, ref_gather(rows, frag, sids))
        for a, b in zip(dst, via_packed):
            assert np.array_equal(a, b)


# ================================================================================================ GPU: the matrix
# (T, N, frag, n): stride = frag, 16 B aligned bases and packed buffer
FULL_SHAPES = [
    (1, 8, 16, 1),             # a single 16 B item: below every grid
    (3, 40, 48, 17),           # BULK piece = 48 B
    (64, 12, 1008, 5),         # fragment below 1 KiB: BULK piece clamped to it
    (3, 64, 1040, 33),
    (3, 96, 16400, 64),        # 16 B last piece at every piece size
    (3, 24, 65552, 24),        # 4680 items at 1 KiB pieces: each BULK CTA wraps its ring several times
    (64, 10, 4096, 7),
    (3, 10, 32768, 6),
    (1, 6, 1 << 20, 4),
]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", FULL_SHAPES, ids=[f"T{s[0]}-N{s[1]}-frag{s[2]}-n{s[3]}" for s in FULL_SHAPES])
def test_flag_matrix(kvb, torch_cuda, shape):
    """Every flag configuration, gather and scatter, on one pool; the round trip under a shorter list."""
    torch = torch_cuda
    T, N, frag, n = shape
    slab = Slab(torch, tensor_regions("tensor", T, N, frag) + [("packed", n * T * frag, 0, 0)], seed=frag + T)
    p = make_pool(kvb, slab, range(T), N, frag, frag)
    preg = T
    rng = np.random.default_rng(N)
    g_ids, s_ids = id_lists(N, n, rng, dup=True), id_lists(N, n, rng, dup=False)
    run = Run(kvb, torch, [slab])
    with KernelLog(torch) as log:
        for i, flags in enumerate(FULL_FLAGS):
            name, ids = g_ids[i % len(g_ids)]
            do_gather(run, p, slab, preg, ids, flags, f"{flag_name(flags)} ids={name}")
            name, ids = s_ids[i % len(s_ids)]
            do_scatter(run, p, slab, preg, ids, flags, f"{flag_name(flags)} ids={name}")
        for i, flags in enumerate(SHORT_FLAGS):
            name, ids = s_ids[i % len(s_ids)]
            do_roundtrip(run, p, slab, preg, ids, flags, f"{flag_name(flags)} ids={name}")
    run.finish(log)


# (T, N, frag, stride - frag, tensor bases mod 16, n)
ALIGN_SHAPES = [
    (4, 24, 4096, 0, (0,), 9),
    (4, 24, 4096, 8, (0,), 9),
    (4, 24, 4096, 4, (0,), 9),
    (4, 24, 4096, 1, (0,), 9),
    (4, 24, 4096, 0, (0, 4, 8, 12), 9),
    (4, 24, 4096, 0, (8,), 9),
    (3, 30, 1040, 8, (12,), 11),
    (3, 20, 1000, 2, (0,), 7),       # width 2: the byte kernel with 2 KiB pieces
]
PACKED_OFFSETS = (0, 1, 2, 4, 8, 12, 16)
ALIGN_FLAGS = [0, LDG, BULK, LDG | 8 << 8 | 1 << 12, BULK | 3 << 8 | 4 << 12 | 2 << 20, BULK | 2 << 8 | 64 << 12]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ALIGN_SHAPES,
                         ids=[f"frag{s[2]}-stride+{s[3]}-bases{'.'.join(map(str, s[4]))}" for s in ALIGN_SHAPES])
def test_alignment(kvb, torch_cuda, shape):
    """Misaligned tensor bases, strides of frag + 8 / 4 / 2 / 1 and packed offsets 0..16: the width the pool and the
    packed address allow, and BULK demoted to LDG whenever that width is not 16."""
    torch = torch_cuda
    T, N, frag, extra, bases, n = shape
    stride = frag + extra
    regions = tensor_regions("tensor", T, N, stride, bases)
    regions += [(f"packed@{o}", n * T * frag, o, 0) for o in PACKED_OFFSETS]
    slab = Slab(torch, regions, seed=stride)
    p = make_pool(kvb, slab, range(T), N, frag, stride)
    assert p.vec == pool_vec(frag, stride, bases)
    rng = np.random.default_rng(stride)
    g_ids, s_ids = id_lists(N, n, rng, dup=True), id_lists(N, n, rng, dup=False)
    run = Run(kvb, torch, [slab])
    with KernelLog(torch) as log:
        k = 0
        for j, off in enumerate(PACKED_OFFSETS):
            preg = T + j
            for flags in ALIGN_FLAGS:
                label = f"{flag_name(flags)} packed+{off}"
                name, ids = g_ids[k % len(g_ids)]
                do_gather(run, p, slab, preg, ids, flags, f"{label} ids={name}")
                name, ids = s_ids[k % len(s_ids)]
                do_scatter(run, p, slab, preg, ids, flags, f"{label} ids={name}")
                k += 1
    run.finish(log)


# (T, N, frag, src stride - frag, dst stride - frag, flag list)
MIGRATE_SHAPES = [
    (3, 40, 16400, 0, 0, FULL_FLAGS),
    (3, 40, 4096, 32, 16, FULL_FLAGS),      # unequal strides, both 16 B multiples: BULK with two strides
    (2, 30, 4096, 16, 8, SHORT_FLAGS),      # width min(16, 8) = 8
    (2, 30, 4096, 0, 4, SHORT_FLAGS),       # width 4
    (4, 25, 1040, 0, 0, SHORT_FLAGS),
]
PEER_FLAGS = [0, LDG, BULK, LDG | 2 << 8 | 1 << 12, BULK | 3 << 8 | 1 << 12 | 3 << 20]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", MIGRATE_SHAPES,
                         ids=[f"T{s[0]}-frag{s[2]}-src+{s[3]}-dst+{s[4]}" for s in MIGRATE_SHAPES])
def test_migrate(kvb, torch_cuda, shape):
    """Page -> page within one GPU, source and destination pools of equal size; then the same destination marked peer,
    under the default flags (peer default) and under explicit flags (which win)."""
    torch = torch_cuda
    T, N, frag, se, de, flag_list = shape
    sstride, dstride = frag + se, frag + de
    slab = Slab(torch, tensor_regions("src", T, N, sstride) + tensor_regions("dst", T, N, dstride), seed=frag + se)
    src = make_pool(kvb, slab, range(T), N, frag, sstride)
    dst = make_pool(kvb, slab, range(T, 2 * T), N, frag, dstride)
    lib = kvb._lib.load()
    rng = np.random.default_rng(frag)
    n = N * 2 // 3
    sl, dl = id_lists(N, n, rng, dup=False), id_lists(N, n, rng, dup=False)
    pairs = [(f"src ids={a} -> dst ids={b}", sa, db) for (a, sa), (b, db) in zip(sl, dl[1:] + dl[:1])]
    run = Run(kvb, torch, [slab])
    with KernelLog(torch) as log:
        for i, flags in enumerate(flag_list):
            name, sids, dids = pairs[i % len(pairs)]
            do_migrate(kvb, run, src, dst, sids, dids, flags, False, f"{flag_name(flags)} {name}")
        kvb._lib.check(lib.kvb_pool_mark_peer(dst.pool.handle, 1))
        try:
            for i, flags in enumerate(PEER_FLAGS):
                name, sids, dids = pairs[i % len(pairs)]
                do_migrate(kvb, run, src, dst, sids, dids, flags, True, f"peer destination {flag_name(flags)} {name}")
        finally:
            kvb._lib.check(lib.kvb_pool_mark_peer(dst.pool.handle, 0))
    run.finish(log)


@pytest.mark.gpu
@pytest.mark.parametrize("huge_pages", [False, True], ids=["pinned", "pinned-huge-pages"])
def test_pinned_host_packed(kvb, torch_cuda, huge_pages):
    """The packed side in pinned host memory (device-mapped), as the engine's direct host I/O uses it: gather writes
    and scatter reads it across PCIe, at offsets +0 / +4 / +8 and under LDG, BULK and the default."""
    torch = torch_cuda
    T, N, frag, n = 3, 20, 16400, 12
    dslab = Slab(torch, tensor_regions("tensor", T, N, frag), seed=21)
    offsets = (0, 4, 8)
    hslab = Slab(torch, [(f"pinned packed@{o}", n * T * frag, o, 0) for o in offsets], seed=22,
                 pinned=lambda nb: kvb.pool.PinnedBuffer(nb, huge_pages=huge_pages))
    p = make_pool(kvb, dslab, range(T), N, frag, frag)
    rng = np.random.default_rng(23)
    g_ids, s_ids = id_lists(N, n, rng, dup=True), id_lists(N, n, rng, dup=False)
    run = Run(kvb, torch, [dslab, hslab])
    try:
        with KernelLog(torch) as log:
            k = 0
            for j, off in enumerate(offsets):
                for flags in (LDG, BULK, 0, BULK | 2 << 8 | 1 << 12 | 1 << 20):
                    label = f"{flag_name(flags)} pinned+{off}"
                    name, ids = g_ids[k % len(g_ids)]
                    do_gather(run, p, hslab, j, ids, flags, f"{label} ids={name}")
                    name, ids = s_ids[k % len(s_ids)]
                    do_scatter(run, p, hslab, j, ids, flags, f"{label} ids={name}")
                    k += 1
        run.finish(log)
    finally:
        p.pool.close()
        hslab.host.free()


@pytest.mark.gpu
def test_empty_calls_launch_nothing(kvb, torch_cuda):
    """n = 0 under every variant, on the host-id, device-id and migrate entry points: no launch, no byte changes."""
    torch = torch_cuda
    T, N, frag = 3, 8, 4096
    slab = Slab(torch, tensor_regions("a", T, N, frag) + tensor_regions("b", T, N, frag)
                + [("packed", T * frag, 0, 0)], seed=31)
    a = make_pool(kvb, slab, range(T), N, frag, frag)
    b = make_pool(kvb, slab, range(T, 2 * T), N, frag, frag)
    packed = Ptr(slab.addr(2 * T))
    none = np.zeros(0, dtype=np.int64)
    none_dev = torch.zeros(0, dtype=torch.int64, device="cuda")
    run = Run(kvb, torch, [slab])
    with KernelLog(torch) as log:
        for flags in PLAIN_FLAGS + [LDG | 8 << 8 | 32 << 12, BULK | 3 << 8 | 64 << 12 | 6 << 20, BULK | 9 << 20]:
            f = flag_name(flags)
            run.call(f"gather n=0 {f}", lambda: a.pool.gather(none, packed, flags=flags), None)
            run.call(f"scatter n=0 {f}", lambda: a.pool.scatter(none, packed, flags=flags), None)
            run.call(f"gather_dev n=0 {f}", lambda: a.pool.gather_dev(none_dev, packed, flags=flags), None)
            run.call(f"scatter_dev n=0 {f}", lambda: a.pool.scatter_dev(none_dev, packed, flags=flags), None)
            run.call(f"migrate n=0 {f}", lambda: kvb.migrate.migrate_blocks(a.pool, b.pool, none, none, flags=flags),
                     None)
    run.finish(log)
    assert log.kernels == []


def hold_streams(torch, streams, cycles: int = 100_000_000) -> None:
    """Queue a ~50 ms spin kernel on each stream, so that the id copies and movers enqueued next are still pending
    when the 8-slot id ring comes round to their slots again."""
    for s in streams:
        with torch.cuda.stream(s):
            torch.cuda._sleep(cycles)


@pytest.mark.gpu
def test_id_ring_many_calls_across_streams(kvb, torch_cuda):
    """40 host-id calls (20 gathers, 20 scatters) round-robin over 3 streams with no sync in between: the 8-slot id ring
    is reused many times, and slots regrow (n from 1 to 5000) while earlier users of the ring are still queued."""
    torch = torch_cuda
    T, frag, NA, NB = 2, 64, 6000, 40000
    g = torch.Generator(device="cuda").manual_seed(41)
    A = [torch.randint(0, 256, (NA, frag), dtype=torch.uint8, device="cuda", generator=g) for _ in range(T)]
    B = [torch.randint(0, 256, (NB, frag), dtype=torch.uint8, device="cuda", generator=g) for _ in range(T)]
    pa, pb = kvb.pool.KVPool(A), kvb.pool.KVPool(B)
    ns = [1, 1500, 5000, 3, 1025, 4096, 2, 2049, 700, 5000, 17, 3000, 4999, 1, 2500, 1024, 4097, 9, 2048, 333]
    rng = np.random.default_rng(42)
    g_ids = [rng.integers(0, NA, n).astype(np.int64) for n in ns]
    targets = rng.permutation(NB)
    assert sum(ns) <= NB
    cut = np.cumsum([0] + ns)
    s_ids = [targets[cut[i]:cut[i + 1]].astype(np.int64) for i in range(len(ns))]
    outs = [torch.empty(n * T * frag, dtype=torch.uint8, device="cuda") for n in ns]
    srcs = [torch.randint(0, 256, (n * T * frag,), dtype=torch.uint8, device="cuda", generator=g) for n in ns]
    want_b = [b.clone() for b in B]
    for ids, src in zip(s_ids, srcs):
        ids_d = torch.from_numpy(ids).cuda()
        for t in range(T):
            want_b[t][ids_d] = src.view(-1, T, frag)[:, t]
    streams = [torch.cuda.Stream() for _ in range(3)]
    torch.cuda.synchronize()
    hold_streams(torch, streams)
    for i in range(len(ns)):
        s = streams[i % 3]
        pa.gather(g_ids[i], outs[i], stream=s)
        pb.scatter(s_ids[i], srcs[i], stream=s)
    torch.cuda.synchronize()
    for i, ids in enumerate(g_ids):
        ids_d = torch.from_numpy(ids).cuda()
        want = torch.stack([a[ids_d] for a in A], 1).reshape(-1)
        assert torch.equal(outs[i], want), f"gather {i} (n={ns[i]}, stream {i % 3})"
    for t in range(T):
        assert torch.equal(B[t], want_b[t]), f"scatter target tensor {t}"


@pytest.mark.gpu
def test_threads_share_one_pool(kvb, torch_cuda):
    """4 host threads gather from one pool at once, each on its own stream into its own buffers, with different valid
    ids of one length (every id slot already large enough: a wrong slot hand-off can only produce wrong bytes)."""
    torch = torch_cuda
    T, N, frag, n, iters, nthreads = 2, 4096, 256, 1000, 50, 4
    g = torch.Generator(device="cuda").manual_seed(51)
    tensors = [torch.randint(0, 256, (N, frag), dtype=torch.uint8, device="cuda", generator=g) for _ in range(T)]
    pool = kvb.pool.KVPool(tensors)
    scratch = torch.empty(n * T * frag, dtype=torch.uint8, device="cuda")
    for _ in range(8):  # size every slot of the ring for n ids
        pool.gather(np.zeros(n, dtype=np.int64), scratch)
    rng = np.random.default_rng(52)
    ids = [[rng.integers(0, N, n).astype(np.int64) for _ in range(iters)] for _ in range(nthreads)]
    outs = [torch.empty((iters, n * T * frag), dtype=torch.uint8, device="cuda") for _ in range(nthreads)]
    streams = [torch.cuda.Stream() for _ in range(nthreads)]
    torch.cuda.synchronize()
    start, errors = threading.Barrier(nthreads), []

    def worker(j):
        try:
            torch.cuda.set_device(0)
            start.wait()
            for k in range(iters):
                pool.gather(ids[j][k], outs[j][k], stream=streams[j])
        except Exception as e:  # noqa: BLE001 - reported by the main thread
            errors.append(f"thread {j}: {e!r}")

    threads = [threading.Thread(target=worker, args=(j,)) for j in range(nthreads)]
    hold_streams(torch, streams)
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    assert not errors, errors
    bad = []
    for j in range(nthreads):
        for k in range(iters):
            ids_d = torch.from_numpy(ids[j][k]).cuda()
            if not torch.equal(outs[j][k], torch.stack([t[ids_d] for t in tensors], 1).reshape(-1)):
                bad.append((j, k))
    assert not bad, f"{len(bad)} of {nthreads * iters} gathers wrong, first (thread, call): {bad[:8]}"


@pytest.mark.gpu
def test_offsets_above_4GiB(kvb, torch_cuda):
    """One 16 MiB-fragment tensor of 280 rows (id * stride past 2^32) and a packed buffer past 4 GiB: 270 gathered ids
    with repeats under LDG and BULK, then gather -> zero -> scatter of 260 distinct ids; compared block by block on the
    device, with guard bands around the packed buffer and per-row sums of the rows not listed."""
    torch = torch_cuda
    free, _ = torch.cuda.mem_get_info()
    if free < 20 << 30:
        pytest.skip(f"needs 20 GB of free HBM for a 4.4 GiB pool and a 4.2 GiB packed buffer; {free >> 30} GiB free")
    frag, N, n = 16 << 20, 280, 270
    g = torch.Generator(device="cuda").manual_seed(61)
    tensor = torch.empty((N, frag), dtype=torch.uint8, device="cuda")
    tensor.random_(0, 256, generator=g)
    pool = kvb.pool.KVPool([tensor])
    buf = torch.empty(n * frag + 2 * MARGIN, dtype=torch.uint8, device="cuda")
    guard = torch.randint(0, 256, (2, MARGIN), dtype=torch.uint8, device="cuda", generator=g)
    buf[:MARGIN] = guard[0]
    buf[-MARGIN:] = guard[1]
    packed = buf[MARGIN:MARGIN + n * frag]
    rng = np.random.default_rng(62)
    dup = rng.integers(0, N, n).astype(np.int64)
    dup[:3] = [N - 1, N - 1, 0]
    dup[-1] = N - 2
    words = tensor.view(torch.int64)
    row_sums = words.sum(1)

    def check_packed(ids, what):
        for b, i in enumerate(ids):
            assert torch.equal(packed[b * frag:(b + 1) * frag], tensor[int(i)]), f"{what}: block {b} (row {i})"
        assert torch.equal(buf[:MARGIN], guard[0]) and torch.equal(buf[-MARGIN:], guard[1]), f"{what}: guard band"

    for flags in (LDG, BULK):
        packed.fill_(0xA5)
        pool.gather(dup, packed, flags=flags)
        torch.cuda.synchronize()
        check_packed(dup, f"gather {flag_name(flags)}")
        assert torch.equal(words.sum(1), row_sums), "gather changed the pool"
    uniq = rng.permutation(N)[:260].astype(np.int64)
    uniq[:2] = [N - 1, 0]
    uniq = np.r_[uniq[2:], uniq[:2]]
    rest = torch.from_numpy(np.setdiff1d(np.arange(N), uniq)).cuda()
    for flags in (BULK, LDG):
        packed.fill_(0x5A)
        pool.gather(uniq, packed, flags=flags)
        torch.cuda.synchronize()
        check_packed(uniq, f"gather of distinct ids {flag_name(flags)}")
        for i in uniq:
            tensor[int(i)].zero_()
        pool.scatter(uniq, packed, flags=flags)
        torch.cuda.synchronize()
        check_packed(uniq, f"scatter {flag_name(flags)}")
        assert torch.equal(words[rest].sum(1), row_sums[rest]), f"scatter {flag_name(flags)} wrote rows not listed"


def _env_child() -> None:
    """Run in a subprocess with ENV_VARS set (tuning() reads them once per process): flag 0, LDG and BULK gathers on
    one pool under the profiler; prints one JSON line for the parent test."""
    import torch
    kvb = importlib.import_module("llm-d-kv-cache_b200")
    torch.cuda.set_device(0)
    T, N, frag, n = 3, 16, 32768, 5
    slab = Slab(torch, tensor_regions("tensor", T, N, frag) + [("packed", n * T * frag, 0, 0)], seed=71)
    p = make_pool(kvb, slab, range(T), N, frag, frag)
    ids = np.array([15, 0, 7, 7, 3], dtype=np.int64)
    run = Run(kvb, torch, [slab])
    with KernelLog(torch) as log:
        for flags in (0, LDG, BULK):
            do_gather(run, p, slab, T, ids, flags, flag_name(flags))
    print(json.dumps({"failures": run.failures, "any_kernels": log.any_kernels, "kernels": log.kernels,
                      "sms": run.sms, "packed": slab.addr(T), "vec": p.vec}), flush=True)


@pytest.mark.gpu
def test_environment_defaults(kvb, torch_cuda):
    """KVB_COPY_VARIANT=1, KVB_LDG_UNROLL=8, KVB_BULK_PIECE=100 (invalid: 16 KiB) and KVB_BULK_DEEP=2 in a fresh
    process: flag 0 resolves to LDG unroll 8, plain LDG takes unroll 8 and plain BULK the 12-stage ring with the
    fallback piece halved to fit; every byte checked."""
    env = dict(os.environ, **ENV_VARS)
    code = f"import sys; sys.path.insert(0, {ROOT!r}); from tests.test_gpu_copy_paths import _env_child; _env_child()"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert not out["failures"], out["failures"]
    T, frag, n = 3, 32768, 5
    expected = [(flag_name(f), expected_launch(GATHER, n, T, frag, out["vec"], f, out["sms"], tuning=ENV_TUNING,
                                               packed_addr=out["packed"])) for f in (0, LDG, BULK)]
    assert [e.kernel for _, e in expected] == ["paged_copy_ldg_kernel<0, int4, 8>"] * 2 + \
        ["paged_copy_bulk_kernel<0, 12, 6>"]
    assert expected[2][1].piece == 8192
    if not out["any_kernels"]:
        pytest.skip("every byte checked; torch.profiler returned no CUDA kernel activity in the subprocess, so which "
                    "kernel ran was not asserted")
    fails = identity_failures(out["kernels"], expected)
    assert not fails, fails
