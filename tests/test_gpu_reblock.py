"""Token-segment migration between pools of different block sizes (kvb_migrate_tokens, kvb.h section 5): the segment
planner, a numpy statement of the semantics, the kernel's run / offset formulas against it, the launch model, and, on
the GPU, every layout pair, block-size pair, head width, vector width and tuning knob byte-exact inside guard bands,
with a check of which kernel ran.

reblock_tokens() states the semantics through [P, B, H, E] / [P, H, B, E] array views, each side with its own B;
kernel_offsets_tokens() restates the byte arithmetic paged_copy_tokens_kernel uses.  The unmarked tests pin one to the
other; the GPU tests compare every byte of every slab (pools, untouched tokens and heads, rows not listed, row tails and
guard bands) with reblock_tokens()."""
from __future__ import annotations

import importlib
import os
import sys
import threading
import time
from typing import NamedTuple

import numpy as np
import pytest

from tests.test_gpu_copy_paths import LDG, MIGRATE, VEC_TYPE, KernelLog, Run, expected_launch, hold_streams
from tests.test_gpu_reshard import (HeadsLaunch, _heads_view, expected_heads_launch, heads_slab, heads_vec,
                                    make_hpool, reshard_heads)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LDG_THREADS = 256
INVALID = -1  # KVB_ERR_INVALID
LAYOUT_PAIRS = [(a, b) for a in ("NHD", "HND") for b in ("NHD", "HND")]


class TraceLog(KernelLog):
    """KernelLog with more non-mover kernels ahead of the first mover: after other GPU tests in the same process the
    trace was seen to miss the first mover kernel as well as the one KernelLog puts first."""

    def __enter__(self):
        super().__enter__()
        for _ in range(8):
            self.torch.cuda._sleep(1000)
        self.torch.cuda.synchronize()
        time.sleep(0.05)
        return self


# ------------------------------------------------------------------------------------------------- the semantics
def reblock_tokens(src_rows, dst_rows, geom_src, geom_dst, segs, src_head0, dst_head0, n_heads) -> None:
    """In place on dst_rows: for every segment [src_block, src_tok0, dst_block, dst_tok0, n], tokens [src_tok0, +n) x
    heads [src_head0, +n_heads) of the source block become tokens [dst_tok0, +n) x heads [dst_head0, +n_heads) of the
    destination block, in every tensor and plane; nothing else changes.  rows: T arrays (num_blocks, stride) whose first
    planes*tokens*heads*head_bytes bytes are the fragment; geom: (planes, tokens, heads, head_bytes, layout)."""
    fs, fd = int(np.prod(geom_src[:4])), int(np.prod(geom_dst[:4]))
    hs, hd = slice(src_head0, src_head0 + n_heads), slice(dst_head0, dst_head0 + n_heads)
    for sr, dr in zip(src_rows, dst_rows):
        for sb, st, db, dt, n in np.asarray(segs, dtype=np.int64).reshape(-1, 5):
            s = _heads_view(sr[sb, :fs], geom_src)[0]           # (P, B, H, E) views of one block
            d = _heads_view(dr[db, :fd], geom_dst)[0]
            d[:, dt:dt + n, hd] = s[:, st:st + n, hs]


# ------------------------------------------------------------------------------------------------- the kernel's math
def kernel_offsets_tokens(gs, gd, seg, hs0: int, hd0: int, nh: int):
    """Byte q of one (segment, tensor) pair -> (source offset, destination offset) in their blocks, as
    paged_copy_tokens_kernel computes them: q -> (run, offset in run) -> (plane, token i, slice head j) -> both layouts'
    offset formulas, each with its own block size.  Also returns the run length."""
    P, Bs, Hs, E, ls = gs
    Bd, Hd, ld = gd[1], gd[2], gd[4]
    _, st, _, dt, n = (int(x) for x in seg)
    q = np.arange(P * n * nh * E, dtype=np.int64)
    if ls == ld == "NHD":
        R = nh * E
        r = q // R
        p, i, j = r // n, r % n, 0 * r
    elif ls == ld == "HND":
        R = n * E
        r = q // R
        p, i, j = r // nh, 0 * r, r % nh
    else:
        R = E
        r = q // R
        if ld == "HND":   # runs (p, j, i), i fastest
            i, j, p = r % n, (r // n) % nh, (r // n) // nh
        else:             # runs (p, i, j), j fastest
            j, i, p = r % nh, (r // nh) % n, (r // nh) // n
    o = q % R

    def off(layout, B, H, t, h):
        return ((p * H + h) * B + t) * E if layout == "HND" else ((p * B + t) * H + h) * E

    return off(ls, Bs, Hs, st + i, hs0 + j) + o, off(ld, Bd, Hd, dt + i, hd0 + j) + o, R


def kernel_apply_tokens(src_rows, dst_rows, gs, gd, segs, hs0, hd0, nh) -> None:
    for seg in np.asarray(segs).reshape(-1, 5):
        soff, doff, _ = kernel_offsets_tokens(gs, gd, seg, hs0, hd0, nh)
        for sr, dr in zip(src_rows, dst_rows):
            dr[seg[2], doff] = sr[seg[0], soff]


# ------------------------------------------------------------------------------------------------- launch model
class TokensLaunch(NamedTuple):
    vec: int
    unroll: int
    piece: int
    grid: int
    block: int = LDG_THREADS
    smem: int = 0

    @property
    def kernel(self) -> str:
        return f"paged_copy_tokens_kernel<{VEC_TYPE[self.vec]}, {self.unroll}>"


def whole_blocks(segs, gs, gd) -> bool:
    """kvb_migrate_tokens hands a call whose every segment covers whole blocks on both sides to kvb_migrate_heads."""
    segs = np.asarray(segs).reshape(-1, 5)
    return bool(np.all(segs[:, 1] == 0) and np.all(segs[:, 3] == 0) and np.all(segs[:, 4] == gs[1])
                and np.all(segs[:, 4] == gd[1]))


def expected_tokens_launch(segs, T, gs, gd, hs0, hd0, nh, pool_vecs, flags, sms):
    """The kernel one kvb_migrate_tokens call launches (None: nothing).  pool_vecs: min of the two pools' widths."""
    segs = np.asarray(segs, dtype=np.int64).reshape(-1, 5)
    if len(segs) == 0:
        return None
    if whole_blocks(segs, gs, gd):
        return expected_heads_launch(len(segs), T, gs, gd, hs0, hd0, nh, pool_vecs, flags, sms)
    P, E = gs[0], gs[3]
    vec = heads_vec(pool_vecs, E)
    unroll = (flags >> 8) & 0xF or 4
    unroll = unroll if unroll in (2, 8) else 4
    ctas = (flags >> 12) & 0xFF or 8
    piece = LDG_THREADS * unroll * vec
    items = len(segs) * T * -(-(P * int(segs[:, 4].max()) * nh * E) // piece)
    return TokensLaunch(vec, unroll, piece, max(1, min(items, sms * ctas)))


# ================================================================================================ CPU: the planner
def test_token_segments_hand_worked(kvb):
    plan = kvb.partition.token_segments
    # 16 -> 64 over 100 tokens: seven source blocks, the last one partial, into two destination blocks
    assert plan(range(10, 17), 16, [20, 21], 64, 100).tolist() == [
        [10, 0, 20, 0, 16], [11, 0, 20, 16, 16], [12, 0, 20, 32, 16], [13, 0, 20, 48, 16],
        [14, 0, 21, 0, 16], [15, 0, 21, 16, 16], [16, 0, 21, 32, 4]]
    # 64 -> 16 over 100 tokens
    assert plan([1, 2], 64, range(5, 12), 16, 100).tolist() == [
        [1, 0, 5, 0, 16], [1, 16, 6, 0, 16], [1, 32, 7, 0, 16], [1, 48, 8, 0, 16],
        [2, 0, 9, 0, 16], [2, 16, 10, 0, 16], [2, 32, 11, 0, 4]]
    # 32 -> 48: cut at the destination's boundary (token 48) and the source's (tokens 32 and 96)
    assert plan([0, 1, 2, 3], 32, [7, 8, 9], 48, 100).tolist() == [
        [0, 0, 7, 0, 32], [1, 0, 7, 32, 16], [1, 16, 8, 0, 16], [2, 0, 8, 16, 32], [3, 0, 9, 0, 4]]
    # the transfer starts 8 tokens into the source request: 64 -> 16
    assert plan([3, 4], 64, [0, 1, 2, 5], 16, 64, src_start=8).tolist() == [
        [3, 8, 0, 0, 16], [3, 24, 1, 0, 16], [3, 40, 2, 0, 16], [3, 56, 5, 0, 8], [4, 0, 5, 8, 8]]
    # equal block sizes and equal starts: whole blocks, also from a block-aligned start
    assert plan([4, 5, 6, 7], 16, [9, 8, 7, 6], 16, 64).tolist() == [
        [4, 0, 9, 0, 16], [5, 0, 8, 0, 16], [6, 0, 7, 0, 16], [7, 0, 6, 0, 16]]
    assert plan([4, 5, 6], 16, [9, 8, 7], 16, 32, src_start=16, dst_start=16).tolist() == [
        [5, 0, 8, 0, 16], [6, 0, 7, 0, 16]]
    # a prefix hit: equal block sizes, different starts
    assert plan([0, 1], 16, [2, 3], 16, 20, src_start=5, dst_start=9).tolist() == [
        [0, 5, 2, 9, 7], [0, 12, 3, 0, 4], [1, 0, 3, 4, 9]]
    assert plan([0], 16, [1], 16, 0).shape == (0, 5)


def test_token_segments_refusals(kvb):
    plan = kvb.partition.token_segments
    for args, kw in (((range(6), 16, [0, 1], 64, 100), {}),               # 96 source tokens for 100
                     ((range(7), 16, [0], 64, 100), {}),                   # 64 destination tokens for 100
                     (([0, 1], 64, range(7), 16, 100), dict(src_start=30)),
                     (([0, 1], 64, range(7), 16, 100), dict(dst_start=13)),
                     (([0], 0, [0], 16, 1), {}), (([0], 16, [0], 0, 1), {}),
                     (([0], 16, [0], 16, -1), {}), (([0], 16, [0], 16, 1), dict(src_start=-1))):
        with pytest.raises(ValueError):
            plan(*args, **kw)


def check_plan(segs, src_ids, Bs, dst_ids, Bd, n, s0, d0) -> None:
    """Every token moved exactly once to its place, every segment inside one block on each side, no two adjacent
    segments that could have been one."""
    spos = {int(b): k for k, b in enumerate(src_ids)}
    dpos = {int(b): k for k, b in enumerate(dst_ids)}
    moved = np.zeros(n, dtype=np.int64)
    for sb, st, db, dt, m in segs:
        assert m >= 1 and 0 <= st and st + m <= Bs and 0 <= dt and dt + m <= Bd
        u0 = spos[sb] * Bs + st - s0
        assert dpos[db] * Bd + dt - d0 == u0, "token lands at the wrong position"
        moved[u0:u0 + m] += 1
    assert np.all(moved == 1)
    for a, b in zip(segs, segs[1:]):
        assert not (a[0] == b[0] and a[2] == b[2] and a[1] + a[4] == b[1] and a[3] + a[4] == b[3]), (a, b)


def test_token_segments_sweep(kvb):
    rng = np.random.default_rng(5)
    sizes = (1, 2, 16, 32, 48, 64, 128)
    n_cases = 0
    for Bs in sizes:
        for Bd in sizes:
            for _ in range(4):
                n = int(rng.integers(0, 700))
                s0, d0 = int(rng.integers(0, 3 * Bs)), int(rng.integers(0, 3 * Bd))
                ns, nd = -(-(s0 + n) // Bs) + int(rng.integers(0, 3)), -(-(d0 + n) // Bd) + int(rng.integers(0, 3))
                sids, dids = rng.permutation(4 * ns + 4)[:ns], rng.permutation(4 * nd + 4)[:nd]
                segs = kvb.partition.token_segments(sids, Bs, dids, Bd, n, src_start=s0, dst_start=d0)
                assert segs.dtype == np.int64 and segs.shape[1] == 5
                check_plan(segs.tolist(), sids, Bs, dids, Bd, n, s0, d0)
                n_cases += 1
    assert n_cases == 4 * len(sizes) ** 2


# ================================================================================================ CPU: oracle, formulas
def test_oracle_hand_written():
    # a 2-token source block (one head of 2 bytes) into a 4-token destination block at dst_tok0 = 1; tail untouched
    src = [np.array([[10, 11, 20, 21]], dtype=np.uint8)]
    dst = [np.full((2, 9), 0, dtype=np.uint8)]
    reblock_tokens(src, dst, (1, 2, 1, 2, "NHD"), (1, 4, 1, 2, "NHD"), [[0, 0, 1, 1, 2]], 0, 0, 1)
    assert dst[0][1].tolist() == [0, 0, 10, 11, 20, 21, 0, 0, 0]
    assert dst[0][0].tolist() == [0] * 9
    # HND (P = 2, H = 2, B = 2, E = 1) -> NHD (P = 2, H = 2, B = 4): source token 1 to destination token 2
    src2 = [np.arange(8, dtype=np.uint8).reshape(1, 8)]                  # (p, h, t) at (p*2 + h)*2 + t
    dst2 = [np.full((1, 17), 255, dtype=np.uint8)]
    reblock_tokens(src2, dst2, (2, 2, 2, 1, "HND"), (2, 4, 2, 1, "NHD"), [[0, 1, 0, 2, 1]], 0, 0, 2)
    # destination (p, t=2, h) at (p*4 + 2)*2 + h: plane 0 bytes 4, 5 <- (0, h, 1) = 1, 3; plane 1 bytes 12, 13 <- 5, 7
    want = [255] * 17
    want[4], want[5], want[12], want[13] = 1, 3, 5, 7
    assert dst2[0][0].tolist() == want
    # NHD -> HND with a head slice: head 1 of source tokens 0-1 into head 0 of destination tokens 2-3
    dst3 = [np.full((1, 8), 9, dtype=np.uint8)]                          # P=1, H=2, B=4, E=1, HND: (h, t) at h*4 + t
    reblock_tokens([np.array([[1, 2, 3, 4]], dtype=np.uint8)], dst3, (1, 2, 2, 1, "NHD"), (1, 4, 2, 1, "HND"),
                   [[0, 0, 0, 2, 2]], 1, 0, 1)
    assert dst3[0][0].tolist() == [9, 9, 2, 4, 9, 9, 9, 9]
    # with equal block sizes and whole blocks it is the head-slice statement
    rng = np.random.default_rng(1)
    s = [rng.integers(0, 256, (3, 2 * 4 * 3 * 2 + 1), dtype=np.uint8)]
    a, b = [np.zeros((3, 2 * 4 * 2 * 2), dtype=np.uint8)], [np.zeros((3, 2 * 4 * 2 * 2), dtype=np.uint8)]
    gs, gd = (2, 4, 3, 2, "NHD"), (2, 4, 2, 2, "HND")
    reblock_tokens(s, a, gs, gd, [[2, 0, 0, 0, 4], [0, 0, 1, 0, 4]], 1, 0, 2)
    reshard_heads(s, b, gs, gd, [2, 0], [0, 1], 1, 0, 2)
    assert np.array_equal(a[0], b[0])


GEOMS = [  # (P, Bs, Bd, E, Hs, Hd, hs0, hd0, nh, src_start, dst_start, n_tokens)
    (1, 4, 8, 4, 8, 4, 4, 0, 4, 0, 0, 21), (2, 8, 4, 8, 4, 8, 1, 5, 3, 3, 0, 17), (2, 3, 5, 6, 8, 1, 6, 0, 1, 1, 2, 13),
    (1, 2, 2, 16, 1, 1, 0, 0, 1, 1, 0, 7), (2, 5, 4, 4, 8, 8, 2, 5, 3, 0, 3, 11), (1, 3, 6, 12, 8, 8, 0, 0, 8, 0, 0, 12),
    (2, 1, 4, 2, 2, 4, 0, 2, 2, 0, 1, 9), (1, 4, 4, 4, 2, 2, 0, 0, 2, 0, 0, 8),
]


@pytest.mark.parametrize("layouts", LAYOUT_PAIRS, ids=[f"{a}-{b}" for a, b in LAYOUT_PAIRS])
def test_kernel_formulas_match_oracle(kvb, layouts):
    """The kernel's run / offset arithmetic writes what the view-based statement writes; every run starts at a
    multiple of E on both sides; no destination byte is written twice; each layout pair's run has the promised length."""
    ls, ld = layouts
    rng = np.random.default_rng(4)
    for (P, Bs, Bd, E, Hs, Hd, hs0, hd0, nh, s0, d0, n) in GEOMS:
        gs, gd = (P, Bs, Hs, E, ls), (P, Bd, Hd, E, ld)
        ns, nd, T = -(-(s0 + n) // Bs), -(-(d0 + n) // Bd), 2
        src = [rng.integers(0, 256, (ns + 2, P * Bs * Hs * E + 3), dtype=np.uint8) for _ in range(T)]
        dst = [rng.integers(0, 256, (nd + 2, P * Bd * Hd * E + 5), dtype=np.uint8) for _ in range(T)]
        segs = kvb.partition.token_segments(rng.permutation(ns + 2)[:ns], Bs, rng.permutation(nd + 2)[:nd], Bd, n,
                                            src_start=s0, dst_start=d0)
        a, b = [d.copy() for d in dst], [d.copy() for d in dst]
        reblock_tokens(src, a, gs, gd, segs, hs0, hd0, nh)
        kernel_apply_tokens(src, b, gs, gd, segs, hs0, hd0, nh)
        for x, y in zip(a, b):
            assert np.array_equal(x, y), (gs, gd)
        written = []
        for seg in segs:
            soff, doff, R = kernel_offsets_tokens(gs, gd, seg, hs0, hd0, nh)
            assert R == {("NHD", "NHD"): nh * E, ("HND", "HND"): seg[4] * E}.get(layouts, E)
            assert np.all(soff[::E] % E == 0) and np.all(doff[::E] % E == 0)
            assert soff.max() < P * Bs * Hs * E and doff.max() < P * Bd * Hd * E
            written.append(seg[2] * (1 << 32) + doff)
        written = np.concatenate(written)
        assert np.unique(written).size == written.size


def test_full_heads_nhd_runs_are_one_stretch():
    """With all heads on both sides, NHD -> NHD runs of consecutive tokens are adjacent: a segment is one n*H*E byte
    stretch per plane on both sides."""
    gs, gd = (2, 16, 8, 128, "NHD"), (2, 64, 8, 128, "NHD")
    soff, doff, _ = kernel_offsets_tokens(gs, gd, (0, 3, 0, 40, 13), 0, 0, 8)
    half = 13 * 8 * 128
    for off, B, t0 in ((soff, 16, 3), (doff, 64, 40)):
        for p in (0, 1):
            start = (p * B + t0) * 8 * 128
            assert np.array_equal(off[p * half:(p + 1) * half], np.arange(start, start + half))


# (id, expected_tokens_launch arguments, launch), worked by hand from launch_migrate_tokens on a 132-SM part
NHD8 = (1, 16, 8, 256, "NHD")
NHD8_64 = (1, 64, 8, 256, "NHD")
SEG16_64 = [[b, 0, b // 4, 16 * (b % 4), 16] for b in range(2048)]     # a 32k-token request, 16 -> 64
MODEL_CASES = [
    # Llama-3-8B 16 -> 64: a segment is 16 x 8 x 256 = 32 KiB = two 16 KiB pieces; 2048 x 64 x 2 items, 1056 CTAs
    ("8b-16to64", dict(segs=SEG16_64, T=64, gs=NHD8, gd=NHD8_64, hs0=0, hd0=0, nh=8, pool_vecs=16, flags=0),
     TokensLaunch(16, 4, 16384, 1056)),
    # E = 36: width 4; unroll 8, 1 CTA/SM: 8 KiB pieces, segment 2 x 16 x 1 x 36 = 1152 B, 5 x 2 items
    ("e36-unroll8", dict(segs=[[k, 0, k // 4, 16 * (k % 4), 16] for k in range(5)], T=2, gs=(2, 16, 8, 36, "HND"),
                         gd=(2, 64, 1, 36, "NHD"), hs0=6, hd0=0, nh=1, pool_vecs=16, flags=LDG | 8 << 8 | 1 << 12),
     TokensLaunch(4, 8, 8192, 10)),
    # E = 24: width 8; unroll 2, 32 CTAs/SM: 4 KiB pieces; the longest segment (20 tokens) is 2 x 20 x 8 x 24 = 7680 B,
    # 2 pieces for each of the 3 segments, however short
    ("e24-unroll2-ctas32", dict(segs=[[0, 0, 0, 0, 5], [1, 3, 0, 5, 20], [2, 0, 1, 0, 7]], T=1,
                                gs=(2, 32, 8, 24, "NHD"), gd=(2, 48, 8, 24, "HND"), hs0=0, hd0=0, nh=8, pool_vecs=16,
                                flags=2 << 8 | 32 << 12), TokensLaunch(8, 2, 4096, 6)),
    # a pool of width 2 (stride frag + 2): the byte kernel, 1 KiB pieces, segment 16 x 4 x 128 = 8 KiB -> 8 pieces
    ("width2", dict(segs=[[0, 16 * k, k, 0, 16] for k in range(3)], T=1, gs=(1, 64, 8, 128, "NHD"),
                    gd=(1, 16, 4, 128, "NHD"), hs0=1, hd0=0, nh=4, pool_vecs=2, flags=0), TokensLaunch(1, 4, 1024, 24)),
    # whole blocks, layout change: exactly kvb_migrate_heads' head mover
    ("whole-relayout", dict(segs=[[k, 0, 9 - k, 0, 16] for k in range(10)], T=4, gs=NHD8, gd=(1, 16, 8, 256, "HND"),
                            hs0=0, hd0=0, nh=8, pool_vecs=16, flags=0), HeadsLaunch(16, 4, 16384, 80)),
    # whole blocks, a head slice: the head mover
    ("whole-slice", dict(segs=[[k, 0, k, 0, 16] for k in range(3)], T=2, gs=NHD8, gd=(1, 16, 4, 256, "NHD"), hs0=4,
                         hd0=0, nh=4, pool_vecs=16, flags=0), HeadsLaunch(16, 4, 16384, 6)),
    # whole blocks, whole fragment in one layout: the page mover (library default BULK, 8 KiB pieces, 2 CTAs/SM)
    ("whole-page", dict(segs=[[k, 0, k, 0, 16] for k in range(10)], T=4, gs=NHD8, gd=NHD8, hs0=0, hd0=0, nh=8,
                        pool_vecs=16, flags=0), expected_launch(MIGRATE, 10, 4, 32768, 16, 0, 132)),
    # equal block sizes, one segment off a block start: the token mover, 2 x 16 KiB per segment
    ("equal-b-offset", dict(segs=[[0, 0, 0, 0, 16], [1, 0, 1, 1, 15]], T=4, gs=NHD8, gd=NHD8, hs0=0, hd0=0, nh=8,
                            pool_vecs=16, flags=0), TokensLaunch(16, 4, 16384, 16)),
    ("nothing", dict(segs=np.zeros((0, 5)), T=4, gs=NHD8, gd=NHD8_64, hs0=0, hd0=0, nh=8, pool_vecs=16, flags=0), None),
]


@pytest.mark.parametrize("case", MODEL_CASES, ids=[c[0] for c in MODEL_CASES])
def test_launch_model_hand_worked(case):
    _, kw, want = case
    assert expected_tokens_launch(sms=132, **kw) == want


def test_launch_model_names():
    assert TokensLaunch(16, 4, 0, 1).kernel == "paged_copy_tokens_kernel<int4, 4>"
    assert TokensLaunch(1, 8, 0, 1).kernel == "paged_copy_tokens_kernel<unsigned char, 8>"
    assert expected_launch(MIGRATE, 10, 4, 32768, 16, 0, 132).kernel == "paged_copy_bulk_kernel<2, 6, 3>"


# ================================================================================================ GPU helpers
def do_tokens(kvb, run, src, dst, segs, hs0, hd0, nh, flags, label) -> None:
    reblock_tokens(src.rows, dst.rows, src.geom, dst.geom, segs, hs0, hd0, nh)
    launch = expected_tokens_launch(segs, len(src.rows), src.geom, dst.geom, hs0, hd0, nh, min(src.vec, dst.vec),
                                    flags, run.sms)
    run.call(label, lambda: kvb.migrate.migrate_tokens(src.pool, dst.pool, segs, hs0, hd0, nh, flags=flags), launch)


# ================================================================================================ GPU: the matrix
# (Bs, Bd, E, Hs, Hd, hs0, hd0, nh, src start, dst start, tokens, src stride - frag, dst stride - frag,
#  src base mod 16, dst base mod 16, flags)
MATRIX = [
    (16, 64, 16, 8, 4, 4, 0, 4, 0, 0, 100, 0, 0, 0, 0, 0),
    (64, 16, 24, 4, 8, 1, 5, 3, 8, 0, 90, 8, 0, 0, 8, LDG | 2 << 8 | 32 << 12),
    (32, 48, 36, 8, 1, 6, 0, 1, 5, 17, 80, 4, 4, 4, 0, 0),
    (16, 16, 128, 8, 4, 0, 0, 4, 3, 9, 40, 16, 0, 0, 0, LDG | 8 << 8 | 1 << 12),   # equal sizes, offsets
    (1, 16, 256, 8, 8, 2, 5, 3, 0, 7, 30, 0, 16, 0, 0, 0),
    (16, 64, 576, 1, 1, 0, 0, 1, 0, 0, 70, 0, 8, 0, 0, 2 << 8 | 8 << 12),         # one MLA-like latent head
    (64, 16, 1152, 8, 4, 3, 1, 3, 8, 0, 70, 0, 0, 12, 0, 4 << 8),
    (32, 48, 128, 4, 4, 0, 0, 4, 0, 0, 96, 0, 0, 0, 0, 0),                        # all heads on both sides
    (16, 64, 256, 8, 8, 0, 0, 8, 0, 16, 64, 16, 16, 0, 0, LDG),                  # all heads, offset destination
]
COMBOS = [(ls, ld, P) for ls, ld in LAYOUT_PAIRS for P in (1, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("combo", COMBOS, ids=[f"{a}-{b}-P{p}" for a, b, p in COMBOS])
def test_matrix(kvb, torch_cuda, combo):
    """Every MATRIX row under one layout pair and plane count: two calls each (different block tables), every byte of
    the slab checked after each, and the kernels in the trace against the launch model."""
    torch = torch_cuda
    ls, ld, P = combo
    T = 2
    run = Run(kvb, torch, [])
    with TraceLog(torch) as log:
        for k, (Bs, Bd, E, Hs, Hd, hs0, hd0, nh, s0, d0, n, se, de, sb, db, flags) in enumerate(MATRIX):
            gs, gd = (P, Bs, Hs, E, ls), (P, Bd, Hd, E, ld)
            fs, fd = P * Bs * Hs * E, P * Bd * Hd * E
            ns, nd = -(-(s0 + n) // Bs), -(-(d0 + n) // Bd)
            Ns, Nd = ns + 3, nd + 2
            slab = heads_slab(torch, T, Ns, Nd, (fs, fs + se), (fd, fd + de), sb, db, seed=100 * COMBOS.index(combo) + k)
            run.slabs = [slab]
            src = make_hpool(kvb, slab, range(T), Ns, gs, fs + se)
            dst = make_hpool(kvb, slab, range(T, 2 * T), Nd, gd, fd + de)
            rng = np.random.default_rng(k)
            for c in range(2):
                sids, dids = rng.permutation(Ns)[:ns], rng.permutation(Nd)[:nd]
                segs = kvb.partition.token_segments(sids, Bs, dids, Bd, n, src_start=s0, dst_start=d0)
                label = (f"B {Bs}->{Bd} E={E} H {Hs}->{Hd} heads [{hs0},+{nh})->[{hd0},+{nh}) tokens [{s0},+{n})->"
                         f"[{d0},+{n}) strides +{se}/+{de} bases {sb}/{db} flags={flags:#x} call {c}")
                do_tokens(kvb, run, src, dst, segs, hs0, hd0, nh, flags, label)
            src.pool.close()
            dst.pool.close()
    run.finish(log)


# ================================================================================================ GPU: other checks
@pytest.mark.gpu
@pytest.mark.parametrize("ld", ["NHD", "HND"])
def test_mixed_segment_lengths(kvb, torch_cuda, ld):
    """One call whose segments differ in length (16, 5, 9, 2 tokens; the grid is sized for the longest): each moves its
    own tokens only.  16 -> 64 blocks, every segment from a source block start, so each byte lands inside its blocks."""
    torch = torch_cuda
    T, Ns, Nd, H, E = 2, 6, 3, 4, 64
    segs = [[4, 0, 2, 0, 16], [1, 0, 2, 16, 5], [0, 0, 0, 40, 9], [5, 0, 0, 3, 2]]
    fs, fd = 16 * H * E, 64 * H * E
    run = Run(kvb, torch, [])
    with TraceLog(torch) as log:
        slab = heads_slab(torch, T, Ns, Nd, (fs, fs), (fd, fd), 0, 0, seed=60)
        run.slabs = [slab]
        src = make_hpool(kvb, slab, range(T), Ns, (1, 16, H, E, "NHD"), fs)
        dst = make_hpool(kvb, slab, range(T, 2 * T), Nd, (1, 64, H, E, ld), fd)
        do_tokens(kvb, run, src, dst, segs, 0, 0, H, 0, f"NHD->{ld} segments of 16, 5, 9, 2 tokens")
        do_tokens(kvb, run, src, dst, segs[1:], 1, 2, 2, 0, f"NHD->{ld} heads [1,+2)->[2,+2), 5, 9, 2 tokens")
        src.pool.close()
        dst.pool.close()
    run.finish(log)


@pytest.mark.gpu
def test_whole_block_routing(kvb, torch_cuda):
    """Segments covering whole blocks run exactly the kernel kvb_migrate_heads runs on the same id lists; equal block
    sizes with one segment off a block start run the token kernel."""
    torch = torch_cuda
    T, N, P, B, H, E = 2, 6, 1, 16, 4, 64
    frag = P * B * H * E
    ids = np.array([5, 0, 2], dtype=np.int64)
    whole = [[s, 0, d, 0, B] for s, d in zip(ids, ids[::-1])]
    offset = [[5, 0, 2, 0, B], [0, 0, 0, 1, B - 1], [2, 3, 5, 0, 4]]
    run = Run(kvb, torch, [])
    with TraceLog(torch) as log:
        for k, (ls, ld, hs0, hd0, nh, segs, want) in enumerate((
                ("NHD", "NHD", 0, 0, 4, whole, "paged_copy_bulk_kernel"),
                ("HND", "HND", 0, 0, 4, whole, "paged_copy_bulk_kernel"),
                ("NHD", "HND", 0, 0, 4, whole, "paged_copy_heads_kernel"),
                ("HND", "HND", 0, 1, 3, whole, "paged_copy_heads_kernel"),
                ("NHD", "NHD", 0, 0, 4, offset, "paged_copy_tokens_kernel"),
                ("HND", "NHD", 1, 0, 2, offset, "paged_copy_tokens_kernel"))):
            slab = heads_slab(torch, T, N, N, (frag, frag), (frag, frag), 0, 0, seed=40 + k)
            run.slabs = [slab]
            src = make_hpool(kvb, slab, range(T), N, (P, B, H, E, ls), frag)
            dst = make_hpool(kvb, slab, range(T, 2 * T), N, (P, B, H, E, ld), frag)
            launch = expected_tokens_launch(segs, T, src.geom, dst.geom, hs0, hd0, nh, 16, 0, run.sms)
            assert launch.kernel.startswith(want)
            if segs is whole:
                assert launch == expected_heads_launch(3, T, src.geom, dst.geom, hs0, hd0, nh, 16, 0, run.sms)
            do_tokens(kvb, run, src, dst, segs, hs0, hd0, nh, 0, f"{ls}->{ld} [{hs0},+{nh})->[{hd0},+{nh}) {want}")
            src.pool.close()
            dst.pool.close()
        # the same whole-block move through kvb_migrate_heads: same kernel, same bytes
        slab = heads_slab(torch, T, N, N, (frag, frag), (frag, frag), 0, 0, seed=50)
        run.slabs = [slab]
        src = make_hpool(kvb, slab, range(T), N, (P, B, H, E, "NHD"), frag)
        dst = make_hpool(kvb, slab, range(T, 2 * T), N, (P, B, H, E, "HND"), frag)
        reshard_heads(src.rows, dst.rows, src.geom, dst.geom, ids, ids[::-1], 0, 0, 4)
        run.call("migrate_heads, whole blocks", lambda: kvb.migrate.migrate_heads(src.pool, dst.pool, ids,
                                                                                   ids[::-1].copy(), 0, 0, 4),
                 expected_heads_launch(3, T, src.geom, dst.geom, 0, 0, 4, 16, 0, run.sms))
    run.finish(log)


def _tokens(t, n_blocks, P, B, H, E, layout):
    """(n_blocks, frag) torch rows -> (P, n_blocks * B, H, E): the request's token sequence."""
    v = t.view(n_blocks, P, B, H, E) if layout == "NHD" else t.view(n_blocks, P, H, B, E).transpose(2, 3)
    return v.permute(1, 0, 2, 3, 4).reshape(P, n_blocks * B, H, E)


@pytest.mark.gpu
def test_round_trip_tp1_b16_to_tp2_b64(kvb, torch_cuda):
    """TP1 B16 NHD -> two TP2 B64 HND pools through tp_head_transfers x token_segments, then back into a poisoned
    pool: the request's tokens come back equal and nothing past them is written."""
    torch = torch_cuda
    H, P, E, T, Bs, Bd, n_tok = 8, 2, 128, 3, 16, 64, 300
    ns, nd, Ns, Nd = -(-n_tok // Bs), -(-n_tok // Bd), 24, 7
    g = torch.Generator(device="cuda").manual_seed(7)
    fs, fd = P * Bs * H * E, P * Bd * (H // 2) * E
    orig = [torch.randint(0, 256, (Ns, fs), dtype=torch.uint8, device="cuda", generator=g) for _ in range(T)]
    src = kvb.pool.KVPool(orig, geometry=(P, Bs, H, E, "NHD"))
    parts_t = [[torch.full((Nd, fd), 0x5A, dtype=torch.uint8, device="cuda") for _ in range(T)] for _ in range(2)]
    parts = [kvb.pool.KVPool(pt, geometry=(P, Bd, H // 2, E, "HND")) for pt in parts_t]
    rng = np.random.default_rng(7)
    sids, dids, bids = rng.permutation(Ns)[:ns], rng.permutation(Nd)[:nd], rng.permutation(Ns)[:ns]
    fwd = kvb.partition.token_segments(sids, Bs, dids, Bd, n_tok)
    for (s, d, sh, dh, nh) in kvb.partition.tp_head_transfers(H, 1, 2):
        kvb.migrate.migrate_tokens(src, parts[d], fwd, sh, dh, nh)
    back_t = [torch.full((Ns, fs), 0xA5, dtype=torch.uint8, device="cuda") for _ in range(T)]
    back = kvb.pool.KVPool(back_t, geometry=(P, Bs, H, E, "NHD"))
    bwd = kvb.partition.token_segments(dids, Bd, bids, Bs, n_tok)
    for (s, d, sh, dh, nh) in kvb.partition.tp_head_transfers(H, 2, 1):
        kvb.migrate.migrate_tokens(parts[s], back, bwd, sh, dh, nh)
    torch.cuda.synchronize()
    cu = lambda a: torch.from_numpy(np.asarray(a, dtype=np.int64)).cuda()  # noqa: E731
    for t in range(T):
        want = _tokens(orig[t][cu(sids)], ns, P, Bs, H, E, "NHD")[:, :n_tok]
        got = _tokens(back_t[t][cu(bids)], ns, P, Bs, H, E, "NHD")
        assert torch.equal(got[:, :n_tok], want), f"tensor {t}"
        assert bool((got[:, n_tok:] == 0xA5).all()), "tokens past the request were written"
        rest = np.setdiff1d(np.arange(Ns), bids)
        assert bool((back_t[t][cu(rest)] == 0xA5).all())
        # part 1 holds heads 4..7 as HND 64-token blocks
        half = _tokens(parts_t[1][t][cu(dids)], nd, P, Bd, H // 2, E, "HND")
        assert torch.equal(half[:, :n_tok], want[:, :, H // 2:])
        assert bool((half[:, n_tok:] == 0x5A).all())


@pytest.mark.gpu
def test_prefix_hit_mid_block(kvb, torch_cuda):
    """The decode side already holds 37 tokens: tokens 21.. of the prefill request (48-token blocks, HND) go to positions
    37.. of the decode request (16-token blocks, NHD); every other byte of the destination stays."""
    torch = torch_cuda
    H, P, E, T, Bs, Bd, s0, d0, n_tok = 4, 2, 64, 2, 48, 16, 21, 37, 150
    ns, nd, Ns, Nd = -(-(s0 + n_tok) // Bs), -(-(d0 + n_tok) // Bd), 6, 16
    g = torch.Generator(device="cuda").manual_seed(9)
    st = [torch.randint(0, 256, (Ns, P * Bs * H * E), dtype=torch.uint8, device="cuda", generator=g) for _ in range(T)]
    dt = [torch.randint(0, 256, (Nd, P * Bd * H * E), dtype=torch.uint8, device="cuda", generator=g) for _ in range(T)]
    before = [d.clone() for d in dt]
    src = kvb.pool.KVPool(st, geometry=(P, Bs, H, E, "HND"))
    dst = kvb.pool.KVPool(dt, geometry=(P, Bd, H, E, "NHD"))
    rng = np.random.default_rng(9)
    sids, dids = rng.permutation(Ns)[:ns], rng.permutation(Nd)[:nd]
    segs = kvb.partition.token_segments(sids, Bs, dids, Bd, n_tok, src_start=s0, dst_start=d0)
    assert segs[0, 1] == s0 % Bs and segs[0, 3] == d0 % Bd
    kvb.migrate.migrate_tokens(src, dst, segs)
    torch.cuda.synchronize()
    cu = lambda a: torch.from_numpy(np.asarray(a, dtype=np.int64)).cuda()  # noqa: E731
    for t in range(T):
        want = _tokens(st[t][cu(sids)], ns, P, Bs, H, E, "HND")[:, s0:s0 + n_tok]
        got = _tokens(dt[t][cu(dids)], nd, P, Bd, H, E, "NHD")
        old = _tokens(before[t][cu(dids)], nd, P, Bd, H, E, "NHD")
        assert torch.equal(got[:, d0:d0 + n_tok], want)
        assert torch.equal(got[:, :d0], old[:, :d0]) and torch.equal(got[:, d0 + n_tok:], old[:, d0 + n_tok:])
        rest = cu(np.setdiff1d(np.arange(Nd), dids))
        assert torch.equal(dt[t][rest], before[t][rest])


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
    """Each malformed call returns KVB_ERR_INVALID with a message, launches nothing and writes nothing; n_segs = 0
    launches nothing; kvb_migrate_heads still refuses pools of different block sizes."""
    torch = torch_cuda
    import ctypes as C
    N = 4

    def pool(P=1, B=16, H=8, E=64, layout="NHD", T=2, geometry=True):
        ts = [torch.randint(0, 256, (N, P * B * H * E), dtype=torch.uint8, device="cuda") for _ in range(T)]
        return kvb.pool.KVPool(ts, geometry=(P, B, H, E, layout) if geometry else None), ts

    (src, st), (dst, dt) = pool(), pool(B=64, H=4, layout="HND")
    snap = [t.clone() for t in st + dt]
    mt = kvb.migrate.migrate_tokens
    ok = [[0, 0, 1, 16, 16]]
    bare, _ = pool(geometry=False)
    _refused(kvb, lambda: mt(bare, dst, ok, 0, 0, 1), "source pool has no KV geometry")
    _refused(kvb, lambda: mt(src, bare, ok, 0, 0, 1), "destination pool has no KV geometry")
    for kw in (dict(T=3), dict(P=2, H=2), dict(E=128, H=2)):
        other, _ = pool(**kw)
        _refused(kvb, lambda: mt(src, other, ok, 0, 0, 1), "pools differ in shape")
    for hs0, hd0, nh in ((0, 0, 0), (0, 0, -1), (5, 0, 4), (0, 1, 4), (-1, 0, 1), (0, -1, 1), (8, 0, 1), (0, 4, 1)):
        _refused(kvb, lambda: mt(src, dst, ok, hs0, hd0, nh), "out of range")
    for seg in ([0, 0, 1, 0, 0], [0, 0, 1, 0, -1], [0, -1, 1, 0, 4], [0, 0, 1, -1, 4], [0, 10, 1, 0, 7],
                [0, 0, 1, 60, 5], [0, 0, 1, 0, 17], [0, 16, 1, 0, 1], [0, 0, 1, 64, 1]):
        _refused(kvb, lambda: mt(src, dst, [[1, 0, 0, 0, 4], seg], 0, 0, 4), "segment 1 tokens")
    for seg in ([N, 0, 0, 0, 4], [-1, 0, 0, 0, 4], [0, 0, N, 0, 4], [0, 0, -1, 0, 4]):
        _refused(kvb, lambda: mt(src, dst, [seg], 0, 0, 4), "out of range")
    for segs in ([[0, 0, 1, 10, 8], [1, 0, 1, 17, 4]], [[2, 0, 3, 0, 16], [0, 0, 1, 0, 4], [3, 0, 3, 15, 1]],
                 [[0, 0, 2, 5, 1], [1, 0, 2, 5, 1]]):
        _refused(kvb, lambda: mt(src, dst, segs, 0, 0, 4), "overlap")
    # argument errors are reported even when there is nothing to move
    _refused(kvb, lambda: mt(src, dst, np.zeros((0, 5)), 0, 0, 9), "out of range")
    lib = kvb._lib.load()
    empty = (kvb._lib.TokenSegment * 1)()
    assert lib.kvb_migrate_tokens(None, dst.handle, empty, 0, 0, 0, 1, None, 0) == INVALID
    assert lib.kvb_migrate_tokens(src.handle, None, empty, 0, 0, 0, 1, None, 0) == INVALID
    assert lib.kvb_migrate_tokens(src.handle, dst.handle, empty, -1, 0, 0, 1, None, 0) == INVALID
    assert lib.kvb_migrate_tokens(src.handle, dst.handle, C.cast(None, C.POINTER(kvb._lib.TokenSegment)), 1, 0, 0, 1,
                                  None, 0) == INVALID
    with pytest.raises(ValueError):
        mt(src, dst, ok)                       # n_heads=None with 8 vs 4 heads
    with pytest.raises(ValueError):
        mt(src, dst, [[0, 0, 1, 0]], 0, 0, 4)  # rows of 4
    with pytest.raises(ValueError):
        mt(src, dst, [[0, 0, 1, 0, 1 << 32]], 0, 0, 4)
    before = lib.kvb_launch_count()
    mt(src, dst, np.zeros((0, 5), dtype=np.int64), 0, 0, 4)
    mt(src, dst, [], 0, 0, 4)
    torch.cuda.synchronize()
    assert lib.kvb_launch_count() == before
    # kvb_migrate_heads keeps its rule: equal block sizes only
    _refused(kvb, lambda: kvb.migrate.migrate_heads(src, dst, [0], [0], 0, 0, 4), "migrate_heads: pools differ in shape")
    torch.cuda.synchronize()
    for a, b in zip(st + dt, snap):
        assert torch.equal(a, b)
    # segments that touch but do not overlap are accepted
    kvb.migrate.migrate_tokens(src, dst, [[0, 0, 1, 10, 8], [1, 0, 1, 18, 4], [2, 0, 1, 0, 10]], 0, 0, 4)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_refuses_device_mismatch(kvb, torch_cuda):
    """A destination described on another device than the source is refused (needs 2 GPUs to build such a pool)."""
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs to describe a pool on a second device")
    a = [torch.zeros((4, 8192), dtype=torch.uint8, device="cuda:0")]
    b = [torch.zeros((4, 32768), dtype=torch.uint8, device="cuda:1")]
    pa = kvb.pool.KVPool(a, geometry=(1, 16, 8, 64, "NHD"))
    pb = kvb.pool.KVPool(b, geometry=(1, 64, 8, 64, "NHD"))
    _refused(kvb, lambda: kvb.migrate.migrate_tokens(pa, pb, [[0, 0, 0, 0, 16]]), "describe the destination pool")


@pytest.mark.gpu
def test_threads_share_one_source_pool(kvb, torch_cuda):
    """4 host threads read one 16-token source pool at once, each into its own 64-token HND pool of 2 heads on its own
    stream, 30 calls each (segments through the id ring); every destination row checked afterwards."""
    torch = torch_cuda
    T, N, P, B, Bd, H, E, iters, nthreads, n_tok = 2, 256, 2, 16, 64, 8, 64, 30, 4, 64
    g = torch.Generator(device="cuda").manual_seed(83)
    frag = P * B * H * E
    st = [torch.randint(0, 256, (N, frag), dtype=torch.uint8, device="cuda", generator=g) for _ in range(T)]
    src = kvb.pool.KVPool(st, geometry=(P, B, H, E, "NHD"))
    dts = [[torch.zeros((iters, P * Bd * 2 * E), dtype=torch.uint8, device="cuda") for _ in range(T)]
           for _ in range(nthreads)]
    dsts = [kvb.pool.KVPool(d, geometry=(P, Bd, 2, E, "HND")) for d in dts]
    rng = np.random.default_rng(84)
    ids = [[rng.integers(0, N, n_tok // B).astype(np.int64) for _ in range(iters)] for _ in range(nthreads)]
    segs = [[kvb.partition.token_segments(ids[j][k], B, [k], Bd, n_tok) for k in range(iters)] for j in range(nthreads)]
    streams = [torch.cuda.Stream() for _ in range(nthreads)]
    torch.cuda.synchronize()
    start, errors = threading.Barrier(nthreads), []

    def worker(j):
        try:
            torch.cuda.set_device(0)
            start.wait()
            for k in range(iters):
                kvb.migrate.migrate_tokens(src, dsts[j], segs[j][k], 2 * j, 0, 2, stream=streams[j])
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
        for k in range(iters):
            for t in range(T):
                sel = torch.from_numpy(ids[j][k]).cuda()
                want = _tokens(st[t][sel], n_tok // B, P, B, H, E, "NHD")[:, :, 2 * j:2 * j + 2]
                got = _tokens(dts[j][t][k:k + 1], 1, P, Bd, 2, E, "HND")
                assert torch.equal(got, want), f"thread {j} call {k} tensor {t}"


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
        T, N, P, H, E, n_tok = 4, 32, 2, 8, 128, 200
        B = 16 if rank == 0 else 64
        geom = (P, B, H, E, "NHD" if rank == 0 else "HND")
        g = torch.Generator(device="cuda").manual_seed(21 + rank)
        tensors = [torch.randint(0, 256, (N, P * B * H * E), dtype=torch.uint8, device="cuda", generator=g)
                   for _ in range(T)]
        pool = kvb.pool.KVPool(tensors, geometry=geom)
        descs = part.exchange_objects(mig.export_pool(pool), dist)
        sids = np.random.default_rng(1).permutation(N)[:-(-n_tok // 16)].astype(np.int64)
        dids = np.random.default_rng(2).permutation(N)[:-(-n_tok // 64)].astype(np.int64)
        before = [t.clone() for t in tensors]
        remote = None
        if rank == 0:  # rank 0 writes its 16-token NHD blocks into rank 1's 64-token HND blocks
            remote = mig.RemotePool(descs[1], 0)
            assert remote.geometry == kvb.pool.KVGeometry(P, 64, H, E, "HND")
            mig.migrate_tokens(pool, remote, part.token_segments(sids, 16, dids, 64, n_tok))
            torch.cuda.synchronize()
        dist.barrier()
        sent = part.exchange_objects([t[torch.from_numpy(sids).cuda()].cpu().numpy() for t in tensors], dist)[0]
        if rank == 1:
            d = torch.from_numpy(dids).cuda()
            for t, b, s in zip(tensors, before, sent):
                want = _tokens(torch.from_numpy(s).cuda(), len(sids), P, 16, H, E, "NHD")[:, :n_tok]
                got, old = _tokens(t[d], len(dids), P, 64, H, E, "HND"), _tokens(b[d], len(dids), P, 64, H, E, "HND")
                assert torch.equal(got[:, :n_tok], want)
                assert torch.equal(got[:, n_tok:], old[:, n_tok:])
        dist.barrier()
        if remote is not None:
            remote.close()
        q.put((rank, "ok"))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_reblock_over_ipc_two_gpus(torch_cuda):
    """Rank 0 (16-token NHD blocks) writes a 200-token request into rank 1's 64-token HND blocks over CUDA IPC, the
    geometry travelling in the exported descriptor; rank 1 checks every token and the untouched tail."""
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33600 + os.getpid() % 2000
    procs = [ctx.Process(target=_ipc_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    assert res == {0: "ok", 1: "ok"}, res
