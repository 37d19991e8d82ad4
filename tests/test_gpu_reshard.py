"""Head-slice migration between pools of different tensor-parallel size and KV layout (kvb_migrate_heads, kvb.h
section 5): the TP planning rule, a numpy statement of the semantics, the kernel's run / offset formulas against it,
and, on the GPU, every layout pair, head width, vector width and tuning knob byte-exact inside guard bands, with a
check of which kernel ran.

reshard_heads() below states the semantics through [P, B, H, E] / [P, H, B, E] array views; kernel_offsets() restates
the byte arithmetic paged_copy_heads_kernel uses.  The unmarked tests pin one to the other; the GPU tests compare every
byte of every slab (pools, untouched heads, rows not listed, row tails and guard bands) with reshard_heads()."""
from __future__ import annotations

import importlib
import os
import sys
import threading
from typing import NamedTuple

import numpy as np
import pytest

from tests.test_gpu_copy_paths import (LDG, MIGRATE, VEC_TYPE, KernelLog, Run, Slab, expected_launch, hold_streams,
                                       pool_vec)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LDG_THREADS = 256
INVALID = -1  # KVB_ERR_INVALID


# ------------------------------------------------------------------------------------------------- the semantics
def _heads_view(frags: np.ndarray, geom) -> np.ndarray:
    """(n, frag) bytes -> (n, planes, tokens, heads, head_bytes), a view in either layout."""
    P, B, H, E, layout = geom
    if layout == "NHD":
        return frags.reshape(-1, P, B, H, E)
    return frags.reshape(-1, P, H, B, E).transpose(0, 1, 3, 2, 4)


def reshard_heads(src_rows, dst_rows, geom_src, geom_dst, src_ids, dst_ids, src_head0, dst_head0, n_heads) -> None:
    """In place on dst_rows: heads [src_head0, +n_heads) of source blocks src_ids[i] become heads [dst_head0, +n_heads)
    of destination blocks dst_ids[i], in every tensor; nothing else changes.  rows: T arrays (num_blocks, stride) whose
    first planes*tokens*heads*head_bytes bytes are the fragment; geom: (planes, tokens, heads, head_bytes, layout)."""
    s, d = np.asarray(src_ids, dtype=np.int64), np.asarray(dst_ids, dtype=np.int64)
    fs, fd = int(np.prod(geom_src[:4])), int(np.prod(geom_dst[:4]))
    for sr, dr in zip(src_rows, dst_rows):
        src = _heads_view(np.ascontiguousarray(sr[s, :fs]), geom_src)
        out = np.ascontiguousarray(dr[d, :fd])
        _heads_view(out, geom_dst)[:, :, :, dst_head0:dst_head0 + n_heads] = src[:, :, :, src_head0:src_head0 + n_heads]
        dr[d, :fd] = out


# ------------------------------------------------------------------------------------------------- the kernel's math
def kernel_offsets(gs, gd, hs0: int, hd0: int, nh: int):
    """Byte q of one (block, tensor) pair -> (source offset, destination offset), as paged_copy_heads_kernel computes
    them: q -> (run, offset in run) -> (plane, token, slice head) -> both layouts' offset formulas."""
    P, B, Hs, E, ls = gs
    Hd, ld = gd[2], gd[4]
    q = np.arange(P * B * nh * E, dtype=np.int64)
    if ls == ld == "NHD":
        R = nh * E
        r, o = q // R, q % R
        p, t, j = r // B, r % B, 0 * r
    elif ls == ld == "HND":
        R = nh * B * E
        r, o = q // R, q % R
        p, t, j = r, 0 * r, 0 * r
    else:
        R = E
        r, o = q // R, q % R
        if ld == "HND":   # runs (p, j, t), t fastest
            t, p, j = r % B, (r // B) // nh, (r // B) % nh
        else:             # runs (p, t, j), j fastest
            j, t, p = r % nh, (r // nh) % B, (r // nh) // B

    def off(layout, H, h):
        return ((p * H + h) * B + t) * E if layout == "HND" else ((p * B + t) * H + h) * E

    return off(ls, Hs, hs0 + j) + o, off(ld, Hd, hd0 + j) + o, R


def kernel_apply(src_rows, dst_rows, gs, gd, src_ids, dst_ids, hs0, hd0, nh) -> None:
    soff, doff, _ = kernel_offsets(gs, gd, hs0, hd0, nh)
    for sr, dr in zip(src_rows, dst_rows):
        for a, b in zip(src_ids, dst_ids):
            dr[b, doff] = sr[a, soff]


# ------------------------------------------------------------------------------------------------- launch model
class HeadsLaunch(NamedTuple):
    vec: int
    unroll: int
    piece: int
    grid: int
    block: int = LDG_THREADS
    smem: int = 0

    @property
    def kernel(self) -> str:
        return f"paged_copy_heads_kernel<{VEC_TYPE[self.vec]}, {self.unroll}>"


def whole_fragment(gs, gd, hs0, hd0, nh) -> bool:
    """launch_migrate_heads hands the whole fragment in the same layout to the plain migrate mover."""
    return nh == gs[2] == gd[2] and hs0 == hd0 == 0 and gs[4] == gd[4]


def heads_vec(pool_vecs: int, E: int) -> int:
    vec = pool_vecs
    while vec > 1 and E % vec:
        vec >>= 1
    return vec if vec >= 4 else 1


def expected_heads_launch(n, T, gs, gd, hs0, hd0, nh, pool_vecs, flags, sms):
    """The kernel one kvb_migrate_heads call launches (None: nothing).  pool_vecs: min of the two pools' widths."""
    if n == 0:
        return None
    P, B, _, E, _ = gs
    if whole_fragment(gs, gd, hs0, hd0, nh):
        return expected_launch(MIGRATE, n, T, P * B * nh * E, pool_vecs, flags, sms)
    vec = heads_vec(pool_vecs, E)
    unroll = (flags >> 8) & 0xF or 4
    unroll = unroll if unroll in (2, 8) else 4
    ctas = (flags >> 12) & 0xFF or 8
    piece = LDG_THREADS * unroll * vec
    items = n * T * -(-(P * B * nh * E) // piece)
    return HeadsLaunch(vec, unroll, piece, max(1, min(items, sms * ctas)))


# ================================================================================================ CPU: TP planning
def owned(rank, tp, H, mla=False):
    """Global heads of a TP rank, restated: contiguous share, or one replicated head, or the MLA latent."""
    if mla:
        return [0]
    return list(range(rank * H // tp, (rank + 1) * H // tp)) if tp <= H else [rank // (tp // H)]


PLAN_CASES = [
    ((8, 1, 2), [(0, 0, 0, 0, 4), (0, 1, 4, 0, 4)]),
    ((8, 2, 1), [(0, 0, 0, 0, 4), (1, 0, 0, 4, 4)]),
    ((8, 1, 8), [(0, d, d, 0, 1) for d in range(8)]),
    ((8, 4, 16), [(d // 4, d, (d // 2) % 2, 0, 1) for d in range(16)]),
    ((2, 8, 1), [(0, 0, 0, 0, 1), (4, 0, 0, 1, 1)]),
    ((8, 8, 2), [(s, s // 4, 0, s % 4, 1) for s in range(8)]),
    ((8, 4, 4), [(r, r, 0, 0, 2) for r in range(4)]),
    # source rank r holds head r // 2, destination rank d head d // 4: holders [2h, 2h+1], d % 2 picks
    ((2, 4, 8), [(2 * (d // 4) + d % 2, d, 0, 0, 1) for d in range(8)]),
]


@pytest.mark.parametrize("case", PLAN_CASES, ids=[f"H{c[0][0]}-tp{c[0][1]}to{c[0][2]}" for c in PLAN_CASES])
def test_tp_head_transfers_hand_worked(kvb, case):
    (H, s, d), want = case
    assert kvb.partition.tp_head_transfers(H, s, d) == want


def test_tp_head_transfers_mla_and_refusals(kvb):
    plan = kvb.partition.tp_head_transfers
    assert plan(1, 2, 4, mla=True) == [(d % 2, d, 0, 0, 1) for d in range(4)]
    assert plan(8, 4, 1, mla=True) == [(0, 0, 0, 0, 1)]
    for bad in ((8, 3, 1), (8, 1, 12), (0, 1, 1), (8, 0, 2)):
        with pytest.raises(ValueError):
            plan(*bad)


def test_tp_head_transfers_sweep(kvb):
    """Every destination head written exactly once, from a source rank that holds it, local indices in range, and no
    two transfers that could have been one."""
    n_cases = 0
    for H in (1, 2, 4, 8, 16):
        tps = [t for t in (1, 2, 4, 8, 16, 32) if H % t == 0 or t % H == 0]
        for s in tps:
            for d in tps:
                for mla in (False, True):
                    plan = kvb.partition.tp_head_transfers(H, s, d, mla=mla)
                    Hg = 1 if mla else H
                    written = {}
                    for (sr, dr, sh, dh, nh) in plan:
                        assert 0 <= sr < s and 0 <= dr < d and nh >= 1
                        src_heads, dst_heads = owned(sr, s, Hg, mla), owned(dr, d, Hg, mla)
                        assert 0 <= sh and sh + nh <= len(src_heads) and 0 <= dh and dh + nh <= len(dst_heads)
                        for k in range(nh):
                            assert src_heads[sh + k] == dst_heads[dh + k], (H, s, d, mla)
                            written[(dr, dh + k)] = written.get((dr, dh + k), 0) + 1
                    want = {(r, j) for r in range(d) for j in range(len(owned(r, d, Hg, mla)))}
                    assert set(written) == want and set(written.values()) == {1}, (H, s, d, mla)
                    for a, b in zip(plan, plan[1:]):
                        assert not (a[0] == b[0] and a[1] == b[1] and a[2] + a[4] == b[2] and a[3] + a[4] == b[3])
                    n_cases += 1
    assert n_cases > 100


# ================================================================================================ CPU: oracle, formulas
def test_oracle_hand_written():
    """Two heads, two tokens, 2-byte heads, one plane: NHD bytes [t0h0 t0h1 t1h0 t1h1], HND [h0t0 h0t1 h1t0 h1t1]."""
    src = [np.array([[10, 11, 20, 21, 30, 31, 40, 41]], dtype=np.uint8)]   # NHD: t0h0=10 11, t0h1=20 21, ...
    dst = [np.zeros((2, 9), dtype=np.uint8)]
    reshard_heads(src, dst, (1, 2, 2, 2, "NHD"), (1, 2, 2, 2, "HND"), [0], [1], 0, 0, 2)
    assert dst[0][1].tolist() == [10, 11, 30, 31, 20, 21, 40, 41, 0]      # HND: h0t0 h0t1 h1t0 h1t1; tail untouched
    assert dst[0][0].tolist() == [0] * 9
    # head 1 of the source into head 0 of a one-head pool (layouts agree for H = 1)
    one = [np.full((1, 4), 7, dtype=np.uint8)]
    reshard_heads(src, one, (1, 2, 2, 2, "NHD"), (1, 2, 1, 2, "HND"), [0], [0], 1, 0, 1)
    assert one[0][0].tolist() == [20, 21, 40, 41]
    # K and V planes sharing a fragment, HND source, one head merged into slot 1 of a 2-head NHD destination
    src2 = [np.arange(16, dtype=np.uint8).reshape(1, 16)]                   # P=2, H=2, B=2, E=2 in HND
    dst2 = [np.full((1, 16), 255, dtype=np.uint8)]
    reshard_heads(src2, dst2, (2, 2, 2, 2, "HND"), (2, 2, 2, 2, "NHD"), [0], [0], 0, 1, 1)
    # source (p, h=0, t): plane 0 bytes 0-3, plane 1 bytes 8-11; destination head 1 of (p, t) at ((p*2 + t)*2 + 1)*2
    assert dst2[0][0].tolist() == [255, 255, 0, 1, 255, 255, 2, 3, 255, 255, 8, 9, 255, 255, 10, 11]


GEOMS = [  # (P, B, E, Hs, Hd, hs0, hd0, nh)
    (1, 4, 4, 8, 4, 4, 0, 4), (2, 3, 8, 4, 8, 1, 5, 3), (2, 4, 6, 8, 1, 6, 0, 1), (1, 2, 16, 1, 1, 0, 0, 1),
    (2, 5, 4, 8, 8, 2, 5, 3), (1, 3, 12, 8, 8, 0, 0, 8), (2, 2, 2, 2, 4, 0, 2, 2),
]
LAYOUT_PAIRS = [(a, b) for a in ("NHD", "HND") for b in ("NHD", "HND")]


@pytest.mark.parametrize("layouts", LAYOUT_PAIRS, ids=[f"{a}-{b}" for a, b in LAYOUT_PAIRS])
def test_kernel_formulas_match_oracle(layouts):
    """The kernel's run / offset arithmetic writes what the view-based statement writes, every run starts at a
    multiple of E on both sides (so every vector width dividing E is aligned), no destination byte is written twice,
    and the run length is the one each layout pair promises."""
    ls, ld = layouts
    rng = np.random.default_rng(3)
    for (P, B, E, Hs, Hd, hs0, hd0, nh) in GEOMS:
        gs, gd = (P, B, Hs, E, ls), (P, B, Hd, E, ld)
        N, T = 5, 2
        src = [rng.integers(0, 256, (N, P * B * Hs * E + 3), dtype=np.uint8) for _ in range(T)]
        dst = [rng.integers(0, 256, (N, P * B * Hd * E + 5), dtype=np.uint8) for _ in range(T)]
        sids, dids = rng.permutation(N)[:3], rng.permutation(N)[:3]
        a, b = [d.copy() for d in dst], [d.copy() for d in dst]
        reshard_heads(src, a, gs, gd, sids, dids, hs0, hd0, nh)
        kernel_apply(src, b, gs, gd, sids, dids, hs0, hd0, nh)
        for x, y in zip(a, b):
            assert np.array_equal(x, y), (gs, gd)
        soff, doff, R = kernel_offsets(gs, gd, hs0, hd0, nh)
        assert R == {("NHD", "NHD"): nh * E, ("HND", "HND"): nh * B * E}.get(layouts, E)
        assert np.all(soff[::E] % E == 0) and np.all(doff[::E] % E == 0)
        assert np.unique(doff).size == doff.size
        assert soff.max() < P * B * Hs * E and doff.max() < P * B * Hd * E


# (id, expected_heads_launch arguments, launch), worked by hand from launch_migrate_heads on a 132-SM part
NHD8 = (1, 16, 8, 256, "NHD")
MODEL_CASES = [
    # Llama-3-8B split: pair = 16 x 4 x 256 = 16 KiB = one 16 KiB piece (256 threads x 4 x 16 B); 2048 x 64 pairs
    ("8b-split", dict(n=2048, T=64, gs=NHD8, gd=(1, 16, 4, 256, "NHD"), hs0=4, hd0=0, nh=4, pool_vecs=16, flags=0),
     HeadsLaunch(16, 4, 16384, 1056)),
    # E = 36: width 4; unroll 8, 1 CTA/SM: 8 KiB pieces, pair 2 x 16 x 1 x 36 = 1152 B, 5 x 2 items
    ("e36-unroll8", dict(n=5, T=2, gs=(2, 16, 8, 36, "HND"), gd=(2, 16, 1, 36, "NHD"), hs0=6, hd0=0, nh=1,
                         pool_vecs=16, flags=LDG | 8 << 8 | 1 << 12), HeadsLaunch(4, 8, 8192, 10)),
    # E = 24: width 8; unroll 2, 32 CTAs/SM: 4 KiB pieces, pair 32 x 8 x 24 = 6 KiB -> 2 pieces, 3 blocks x 1 tensor
    ("e24-unroll2", dict(n=3, T=1, gs=(1, 32, 8, 24, "NHD"), gd=(1, 32, 8, 24, "HND"), hs0=0, hd0=0, nh=8,
                         pool_vecs=16, flags=2 << 8 | 32 << 12), HeadsLaunch(8, 2, 4096, 6)),
    # a pool of width 2 (stride frag + 2): the byte kernel
    ("width2", dict(n=1, T=1, gs=(1, 16, 8, 128, "NHD"), gd=(1, 16, 4, 128, "NHD"), hs0=1, hd0=0, nh=4, pool_vecs=2,
                    flags=0), HeadsLaunch(1, 4, 1024, 8)),
    # whole fragment, same layout: the migrate mover (library default BULK, 8 KiB pieces, 2 CTAs/SM)
    ("whole-nhd", dict(n=10, T=4, gs=NHD8, gd=NHD8, hs0=0, hd0=0, nh=8, pool_vecs=16, flags=0),
     expected_launch(MIGRATE, 10, 4, 32768, 16, 0, 132)),
    # whole fragment, layout change: the head mover
    ("whole-relayout", dict(n=10, T=4, gs=NHD8, gd=(1, 16, 8, 256, "HND"), hs0=0, hd0=0, nh=8, pool_vecs=16, flags=0),
     HeadsLaunch(16, 4, 16384, 80)),
    ("nothing", dict(n=0, T=4, gs=NHD8, gd=NHD8, hs0=0, hd0=0, nh=2, pool_vecs=16, flags=0), None),
]


@pytest.mark.parametrize("case", MODEL_CASES, ids=[c[0] for c in MODEL_CASES])
def test_launch_model_hand_worked(case):
    _, kw, want = case
    assert expected_heads_launch(sms=132, **kw) == want


def test_launch_model_names():
    assert HeadsLaunch(16, 4, 0, 1).kernel == "paged_copy_heads_kernel<int4, 4>"
    assert HeadsLaunch(4, 2, 0, 1).kernel == "paged_copy_heads_kernel<unsigned int, 2>"
    assert expected_launch(MIGRATE, 10, 4, 32768, 16, 0, 132).kernel == "paged_copy_bulk_kernel<2, 6, 3>"
    assert [heads_vec(16, E) for E in (16, 24, 36, 128, 256, 1152, 18)] == [16, 8, 4, 16, 16, 16, 1]


# ================================================================================================ GPU helpers
class HPool(NamedTuple):
    pool: object
    rows: list
    geom: tuple
    N: int
    vec: int


def make_hpool(kvb, slab, regions, N, geom, stride) -> HPool:
    ptrs = [slab.addr(i) for i in regions]
    frag = int(np.prod(geom[:4]))
    pool = kvb.pool.KVPool(None, 0, ptrs=ptrs, num_blocks=N, frag_bytes=frag, stride_bytes=stride, geometry=geom)
    pool._slab = slab
    return HPool(pool, [slab.rows(i, stride) for i in regions], tuple(geom), N, pool_vec(frag, stride, ptrs))


def do_heads(kvb, run, src: HPool, dst: HPool, sids, dids, hs0, hd0, nh, flags, label) -> None:
    reshard_heads(src.rows, dst.rows, src.geom, dst.geom, sids, dids, hs0, hd0, nh)
    launch = expected_heads_launch(len(sids), len(src.rows), src.geom, dst.geom, hs0, hd0, nh, min(src.vec, dst.vec),
                                   flags, run.sms)
    run.call(label, lambda: kvb.migrate.migrate_heads(src.pool, dst.pool, sids, dids, hs0, hd0, nh, flags=flags),
             launch)


def heads_slab(torch, T, Ns, Nd, sframe, dframe, sbase, dbase, seed):
    """Slab with T source tensors then T destination tensors; frame = (fragment, stride)."""
    regions = [(f"src{t}", Ns * sframe[1], sbase, sframe[1]) for t in range(T)]
    regions += [(f"dst{t}", Nd * dframe[1], dbase, dframe[1]) for t in range(T)]
    return Slab(torch, regions, seed=seed)


# ================================================================================================ GPU: the matrix
# (E, Hs, Hd, hs0, hd0, nh, B, src stride - frag, dst stride - frag, src base mod 16, dst base mod 16, flags)
MATRIX = [
    (16, 8, 4, 4, 0, 4, 16, 0, 0, 0, 0, 0),
    (24, 4, 8, 1, 5, 3, 32, 8, 0, 0, 8, LDG | 2 << 8 | 32 << 12),
    (36, 8, 1, 6, 0, 1, 16, 4, 4, 4, 0, 0),
    (128, 8, 4, 0, 0, 4, 32, 16, 0, 0, 0, LDG | 8 << 8 | 1 << 12),
    (128, 4, 8, 0, 4, 4, 16, 0, 8, 0, 0, 2 << 8 | 8 << 12),
    (256, 8, 8, 2, 5, 3, 16, 0, 16, 0, 0, 0),
    (256, 8, 8, 1, 0, 7, 16, 0, 0, 0, 0, 0),              # offset head range over all but one head
    (1152, 8, 4, 3, 1, 3, 16, 0, 0, 12, 0, 4 << 8),
    (128, 1, 1, 0, 0, 1, 16, 0, 8, 0, 0, 0),              # whole fragment: migrate mover in one layout
    (256, 8, 8, 0, 0, 8, 32, 16, 16, 0, 0, LDG),          # whole fragment
]
COMBOS = [(ls, ld, P) for ls, ld in LAYOUT_PAIRS for P in (1, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("combo", COMBOS, ids=[f"{a}-{b}-P{p}" for a, b, p in COMBOS])
def test_matrix(kvb, torch_cuda, combo):
    """Every MATRIX row under one layout pair and plane count: two calls each (different id lists), every byte of the
    slab checked after each, and the kernels in the trace against the launch model."""
    torch = torch_cuda
    ls, ld, P = combo
    T, Ns, Nd, n = 2, 7, 6, 4
    run = Run(kvb, torch, [])
    with KernelLog(torch) as log:
        for k, (E, Hs, Hd, hs0, hd0, nh, B, se, de, sb, db, flags) in enumerate(MATRIX):
            gs, gd = (P, B, Hs, E, ls), (P, B, Hd, E, ld)
            fs, fd = P * B * Hs * E, P * B * Hd * E
            slab = heads_slab(torch, T, Ns, Nd, (fs, fs + se), (fd, fd + de), sb, db, seed=100 * COMBOS.index(combo) + k)
            run.slabs = [slab]
            src = make_hpool(kvb, slab, range(T), Ns, gs, fs + se)
            dst = make_hpool(kvb, slab, range(T, 2 * T), Nd, gd, fd + de)
            rng = np.random.default_rng(k)
            for c in range(2):
                sids = rng.permutation(Ns)[:n].astype(np.int64)
                dids = (rng.permutation(Nd)[:n] if c == 0 else np.array([Nd - 1, 0, 3, 2])).astype(np.int64)
                label = (f"E={E} H {Hs}->{Hd} heads [{hs0},+{nh})->[{hd0},+{nh}) B={B} strides +{se}/+{de} "
                         f"bases {sb}/{db} flags={flags:#x} call {c}")
                do_heads(kvb, run, src, dst, sids, dids, hs0, hd0, nh, flags, label)
            src.pool.close()
            dst.pool.close()
    run.finish(log)


# ================================================================================================ GPU: other checks
@pytest.mark.gpu
@pytest.mark.parametrize("r", [2, 4, 8])
def test_round_trip_split_merge(kvb, torch_cuda, r):
    """TP1 -> TPr split (odd ranks in HND) by the plan of tp_head_transfers, then TPr -> TP1 merge into a poisoned pool:
    the pool comes back equal to the original."""
    torch = torch_cuda
    H, P, B, E, T, N = 8, 2, 16, 128, 3, 12
    g = torch.Generator(device="cuda").manual_seed(r)
    frag = P * B * H * E
    orig = [torch.randint(0, 256, (N, frag), dtype=torch.uint8, device="cuda", generator=g) for _ in range(T)]
    src = kvb.pool.KVPool(orig, geometry=(P, B, H, E, "NHD"))
    parts_t = [[torch.full((N, frag // r), 0x5A, dtype=torch.uint8, device="cuda") for _ in range(T)] for _ in range(r)]
    parts = [kvb.pool.KVPool(pt, geometry=(P, B, H // r, E, "HND" if d % 2 else "NHD")) for d, pt in enumerate(parts_t)]
    rng = np.random.default_rng(r)
    ids = np.arange(N, dtype=np.int64)
    perm = rng.permutation(N).astype(np.int64)
    for (s, d, sh, dh, nh) in kvb.partition.tp_head_transfers(H, 1, r):
        kvb.migrate.migrate_heads(src, parts[d], ids, perm, sh, dh, nh)
    back_t = [torch.full((N, frag), 0xA5, dtype=torch.uint8, device="cuda") for _ in range(T)]
    back = kvb.pool.KVPool(back_t, geometry=(P, B, H, E, "NHD"))
    for (s, d, sh, dh, nh) in kvb.partition.tp_head_transfers(H, r, 1):
        kvb.migrate.migrate_heads(parts[s], back, perm, ids, sh, dh, nh)
    torch.cuda.synchronize()
    for t in range(T):
        assert torch.equal(back_t[t], orig[t]), f"tensor {t}"
    # one part checked against the view statement: its heads in its own layout
    half = orig[0].view(N, P, B, H, E)[:, :, :, H // r:2 * H // r]
    want = half.permute(0, 1, 3, 2, 4).contiguous().view(N, -1)          # part 1 is HND
    assert torch.equal(parts_t[1][0][torch.from_numpy(perm).cuda()], want)


@pytest.mark.gpu
def test_whole_fragment_routing(kvb, torch_cuda):
    """The same-layout whole-fragment call takes the existing migrate mover; a layout-only change and an offset head
    range take the head mover."""
    torch = torch_cuda
    T, N, P, B, H, E = 2, 6, 1, 16, 4, 64
    frag = P * B * H * E
    ids = np.array([5, 0, 2], dtype=np.int64)
    run = Run(kvb, torch, [])
    with KernelLog(torch) as log:
        for ls, ld, hs0, hd0, nh, want in (("NHD", "NHD", 0, 0, 4, "paged_copy_bulk_kernel"),
                                           ("HND", "HND", 0, 0, 4, "paged_copy_bulk_kernel"),
                                           ("NHD", "HND", 0, 0, 4, "paged_copy_heads_kernel"),
                                           ("HND", "NHD", 0, 0, 4, "paged_copy_heads_kernel"),
                                           ("NHD", "NHD", 1, 1, 3, "paged_copy_heads_kernel"),
                                           ("HND", "HND", 0, 1, 3, "paged_copy_heads_kernel")):
            slab = heads_slab(torch, T, N, N, (frag, frag), (frag, frag), 0, 0, seed=hs0 * 3 + hd0 + len(ls + ld))
            run.slabs = [slab]
            src = make_hpool(kvb, slab, range(T), N, (P, B, H, E, ls), frag)
            dst = make_hpool(kvb, slab, range(T, 2 * T), N, (P, B, H, E, ld), frag)
            launch = expected_heads_launch(3, T, src.geom, dst.geom, hs0, hd0, nh, 16, 0, run.sms)
            assert launch.kernel.startswith(want)
            do_heads(kvb, run, src, dst, ids, ids[::-1].copy(), hs0, hd0, nh, 0, f"{ls}->{ld} [{hs0},+{nh})->[{hd0},+{nh})")
    run.finish(log)


def _refused(kvb, fn, needle: str):
    lib = kvb._lib.load()
    before = lib.kvb_launch_count()
    with pytest.raises(kvb._lib.KvbError) as e:
        fn()
    assert e.value.code == INVALID, e.value
    assert needle in e.value.msg, e.value.msg
    assert lib.kvb_launch_count() == before
    return e.value.msg


@pytest.mark.gpu
def test_refusals(kvb, torch_cuda):
    """Each malformed call returns KVB_ERR_INVALID with a message, launches nothing and writes nothing; n = 0 launches
    nothing; kvb_migrate_blocks still refuses pools that differ only in heads, with its old message."""
    torch = torch_cuda
    N = 4

    def pool(P=1, B=16, H=8, E=64, layout="NHD", T=2, geometry=True):
        ts = [torch.randint(0, 256, (N, P * B * H * E), dtype=torch.uint8, device="cuda") for _ in range(T)]
        return kvb.pool.KVPool(ts, geometry=(P, B, H, E, layout) if geometry else None), ts

    (src, st), (dst, dt) = pool(), pool(H=4)
    snap = [t.clone() for t in st + dt]
    mh = kvb.migrate.migrate_heads
    ids = [0, 1]
    bare, _ = pool(geometry=False)
    _refused(kvb, lambda: mh(bare, dst, ids, ids, 0, 0, 1), "source pool has no KV geometry")
    _refused(kvb, lambda: mh(src, bare, ids, ids, 0, 0, 1), "destination pool has no KV geometry")
    for kw in (dict(T=3), dict(P=2, H=2), dict(B=32, H=2), dict(E=128, H=2)):
        other, _ = pool(**kw)
        _refused(kvb, lambda: mh(src, other, ids, ids, 0, 0, 1), "pools differ in shape")
    for hs0, hd0, nh in ((0, 0, 0), (0, 0, -1), (5, 0, 4), (0, 1, 4), (-1, 0, 1), (0, -1, 1), (8, 0, 1), (0, 4, 1)):
        _refused(kvb, lambda: mh(src, dst, ids, ids, hs0, hd0, nh), "out of range")
    _refused(kvb, lambda: mh(src, dst, [0, N], ids, 0, 0, 1), "out of range")
    _refused(kvb, lambda: mh(src, dst, ids, [-1, 0], 0, 0, 1), "out of range")
    # argument errors are reported even when there is nothing to move
    _refused(kvb, lambda: mh(src, dst, [], [], 0, 0, 9), "out of range")
    lib = kvb._lib.load()
    before = lib.kvb_launch_count()
    mh(src, dst, [], [], 0, 0, 4)
    mh(src, src, np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64), 0, 0, 8)
    torch.cuda.synchronize()
    assert lib.kvb_launch_count() == before
    # a geometry must describe the fragment
    with pytest.raises(kvb._lib.KvbError) as e:
        bare.set_geometry((1, 16, 8, 32, "NHD"))
    assert e.value.code == INVALID and "fragment is" in e.value.msg
    with pytest.raises(kvb._lib.KvbError):
        bare.set_geometry((0, 16, 8, 64, "NHD"))
    with pytest.raises(ValueError):
        bare.set_geometry((1, 16, 8, 64, "THD"))
    assert bare.geometry is None
    # the whole-page mover keeps its shape rule: pools differing only in heads differ in fragment size
    _refused(kvb, lambda: kvb.migrate.migrate_blocks(src, dst, ids, ids), "migrate: pools differ in shape")
    torch.cuda.synchronize()
    for a, b in zip(st + dt, snap):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_refuses_device_mismatch(kvb, torch_cuda):
    """A destination described on another device than the source is refused (needs 2 GPUs to build such a pool)."""
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs to describe a pool on a second device")
    geom = (1, 16, 8, 64, "NHD")
    a = [torch.zeros((4, 8192), dtype=torch.uint8, device="cuda:0")]
    b = [torch.zeros((4, 8192), dtype=torch.uint8, device="cuda:1")]
    pa, pb = kvb.pool.KVPool(a, geometry=geom), kvb.pool.KVPool(b, geometry=geom)
    _refused(kvb, lambda: kvb.migrate.migrate_heads(pa, pb, [0], [0], 0, 0, 2), "describe the destination pool")


@pytest.mark.gpu
def test_threads_share_one_source_pool(kvb, torch_cuda):
    """4 host threads split one 8-head source pool at once, each into its own 2-head HND pool on its own stream, 30
    calls each to distinct destination rows; every destination row checked afterwards."""
    torch = torch_cuda
    T, N, P, B, H, E, n, iters, nthreads = 2, 512, 2, 16, 8, 64, 16, 30, 4
    g = torch.Generator(device="cuda").manual_seed(81)
    frag = P * B * H * E
    st = [torch.randint(0, 256, (N, frag), dtype=torch.uint8, device="cuda", generator=g) for _ in range(T)]
    src = kvb.pool.KVPool(st, geometry=(P, B, H, E, "NHD"))
    dts = [[torch.zeros((n * iters, frag // 4), dtype=torch.uint8, device="cuda") for _ in range(T)]
           for _ in range(nthreads)]
    dsts = [kvb.pool.KVPool(d, geometry=(P, B, 2, E, "HND")) for d in dts]
    rng = np.random.default_rng(82)
    ids = [[rng.integers(0, N, n).astype(np.int64) for _ in range(iters)] for _ in range(nthreads)]
    streams = [torch.cuda.Stream() for _ in range(nthreads)]
    torch.cuda.synchronize()
    start, errors = threading.Barrier(nthreads), []

    def worker(j):
        try:
            torch.cuda.set_device(0)
            start.wait()
            for k in range(iters):
                kvb.migrate.migrate_heads(src, dsts[j], ids[j][k], np.arange(k * n, (k + 1) * n), 2 * j, 0, 2,
                                          stream=streams[j])
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
    for j in range(nthreads):
        all_ids = torch.from_numpy(np.concatenate(ids[j])).cuda()
        for t in range(T):
            want = st[t][all_ids].view(-1, P, B, H, E)[:, :, :, 2 * j:2 * j + 2].permute(0, 1, 3, 2, 4)
            assert torch.equal(dts[j][t], want.reshape(n * iters, -1)), f"thread {j} tensor {t}"


# ================================================================================================ GPU: two processes
def _ipc_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        kvb = importlib.import_module("llm-d-kv-cache_b200")
        part, mig = kvb.partition, kvb.migrate
        T, N, P, B, E, n = 4, 64, 2, 16, 128, 40
        H = 8 if rank == 0 else 4
        geom = (P, B, H, E, "NHD" if rank == 0 else "HND")
        g = torch.Generator(device="cuda").manual_seed(11 + rank)
        tensors = [torch.randint(0, 256, (N, P * B * H * E), dtype=torch.uint8, device="cuda", generator=g)
                   for _ in range(T)]
        pool = kvb.pool.KVPool(tensors, geometry=geom)
        descs = part.exchange_objects(mig.export_pool(pool), dist)
        src_ids = np.random.default_rng(1).permutation(N)[:n].astype(np.int64)
        dst_ids = np.random.default_rng(2).permutation(N)[:n].astype(np.int64)
        before = [t.clone() for t in tensors]
        remote = None
        # 1. rank 0 writes its heads 4..7 into rank 1's 4-head HND pool
        if rank == 0:
            remote = mig.RemotePool(descs[1], 0)
            assert remote.geometry == kvb.pool.KVGeometry(P, B, 4, E, "HND")
            mig.migrate_heads(pool, remote, src_ids, dst_ids, 4, 0, 4)
            torch.cuda.synchronize()
        dist.barrier()
        sent = part.exchange_objects([t[torch.from_numpy(src_ids).cuda()].cpu().numpy() for t in tensors], dist)[0]
        if rank == 1:
            d = torch.from_numpy(dst_ids).cuda()
            rest = torch.from_numpy(np.setdiff1d(np.arange(N), dst_ids)).cuda()
            for t, b, s in zip(tensors, before, sent):
                want = torch.from_numpy(s).cuda().view(n, P, B, 8, E)[:, :, :, 4:].permute(0, 1, 3, 2, 4)
                assert torch.equal(t[d], want.reshape(n, -1))
                assert torch.equal(t[rest], b[rest])
            # 2. rank 1 merges its heads back into heads 0..3 of rank 0's pool
            remote = mig.RemotePool(descs[0], 1)
            mig.migrate_heads(pool, remote, dst_ids, src_ids, 0, 0, 4)
            torch.cuda.synchronize()
        dist.barrier()
        if rank == 0:
            s = torch.from_numpy(src_ids).cuda()
            for t, b in zip(tensors, before):
                got, old = t[s].view(n, P, B, 8, E), b[s].view(n, P, B, 8, E)
                assert torch.equal(got[:, :, :, :4], old[:, :, :, 4:]), "merged heads"
                assert torch.equal(got[:, :, :, 4:], old[:, :, :, 4:]), "heads not listed"
        dist.barrier()
        remote.close()
        q.put((rank, "ok"))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_split_and_merge_over_ipc_two_gpus(torch_cuda):
    """Rank 0 (8 heads, NHD) splits heads 4..7 into rank 1's 4-head HND pool over CUDA IPC, the geometry travelling in
    the exported descriptor; rank 1 checks the bytes, then merges them back into heads 0..3 of rank 0's pool."""
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31600 + os.getpid() % 2000
    procs = [ctx.Process(target=_ipc_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert res == {0: "ok", 1: "ok"}, res
