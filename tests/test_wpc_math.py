"""The arithmetic behind hash_chain_kernel_wpc, restated lane by lane in Python and checked against plain FNV-1a:
  (1) FNV-1a is a T-function, so the low byte of the running state resolves in 8 prefix-XOR rounds over the stream
      (one warp vote + popcount per round, 3 consecutive stream positions per lane);
  (2) h ^ b = h + e with e = z - l, so  h_m = P^m * (h_0 + sum_i e_i * Q^i),  Q = P^-1 mod 2^64, summed over the
      warp in four 16-bit limbs.
CPU-only: a change to the kernel's math can be tried here before it costs GPU time."""
import random

M = (1 << 64) - 1
P = 0x100000001B3
Q = pow(P, -1, 1 << 64)
H0 = 0xCBF29CE484222325


def fnv(stream):
    h = H0
    for b in stream:
        h = ((h ^ b) * P) & M
    return h


def wpc(stream):
    m = len(stream)
    assert m <= 96
    b = [[stream[3 * L + j] if 3 * L + j < m else 0 for j in range(3)] for L in range(32)]
    z = [row[:] for row in b]                      # z starts as b: bit k of z*0xb3 is then b_k ^ c_k
    for k in range(8):
        mask = 1 << k
        p = [[(z[L][j] * 0xB3) & 0xFFFFFFFF for j in range(3)] for L in range(32)]
        votes = sum((((p[L][0] ^ p[L][1] ^ p[L][2]) >> k) & 1) << L for L in range(32))      # __ballot_sync
        for L in range(32):
            before = bin(votes & ((1 << L) - 1)).count("1")                                   # popc(votes & lanemask_lt)
            m0 = mask if (H0 & 0xFF) & mask else 0
            zc = [z[L][0] ^ m0, z[L][1] ^ m0 ^ (p[L][0] & mask), z[L][2] ^ m0 ^ ((p[L][0] ^ p[L][1]) & mask)]
            sh = before << k
            z[L] = [zc[j] ^ (sh & mask) for j in range(3)]
    limbs = [0, 0, 0, 0]
    for L in range(32):
        acc, hi = 0, 0
        for j in range(3):
            q = pow(Q, 3 * L + j, 1 << 64)
            qlo = q & 0xFFFFFFFF
            qlo_s = qlo - (1 << 32) if qlo >= 1 << 31 else qlo          # q = (qhi + [qlo < 0]) * 2^32 + signed qlo
            qhi = ((q >> 32) + (1 if qlo_s < 0 else 0)) & 0xFFFFFFFF
            e = z[L][j] - (z[L][j] ^ b[L][j])                           # e = z - l, l = z ^ b
            acc += e * qlo_s
            hi = (hi + e * qhi) & 0xFFFFFFFF
        t = (acc + (hi << 32) + (H0 if L == 0 else 0)) & M             # lane 0 carries the offset basis
        for c in range(4):
            limbs[c] += (t >> (16 * c)) & 0xFFFF                        # redux.sync.add of 16-bit limbs
    total = sum(limbs[c] << (16 * c) for c in range(4)) & M
    return (pow(P, m, 1 << 64) * total) & M


def test_vote_round_formulation_equals_fnv1a():
    rng = random.Random(3)
    for _ in range(400):
        stream = [rng.randrange(256) for _ in range(rng.randrange(0, 97))]
        assert wpc(stream) == fnv(stream)


def test_block_streams_of_the_kernel_shape():
    """83 1b P7..P0 90 | 16 tokens in 1/2/3/5-byte CBOR forms | f6  — the streams the kernel folds (<= 92 bytes)."""
    rng = random.Random(4)
    for _ in range(200):
        parent = rng.getrandbits(64) | (1 << 32)
        stream = [0x83, 0x1B] + list(parent.to_bytes(8, "big")) + [0x90]
        for _ in range(16):
            t = rng.choice([rng.randrange(24), rng.randrange(24, 256), rng.randrange(256, 65536), rng.randrange(65536, 1 << 32)])
            if t < 24:
                stream += [t]
            elif t < 256:
                stream += [0x18, t]
            elif t < 65536:
                stream += [0x19] + list(t.to_bytes(2, "big"))
            else:
                stream += [0x1A] + list(t.to_bytes(4, "big"))
        stream += [0xF6]
        assert len(stream) <= 92 and wpc(stream) == fnv(stream)


def test_three_redux_limb_split_is_exact():
    """Variant tried in round 1 (correct, not faster): sum the 32 lanes' 64-bit terms with THREE redux.sync.add.u32 instead of
    four — 27-bit low limbs of both halves, and the two 5-bit tops packed into one word (10-bit fields: 32 * 31 < 1024)."""
    rng = random.Random(5)
    m27 = (1 << 27) - 1
    for _ in range(300):
        terms = [rng.getrandbits(64) if rng.random() < 0.9 else M for _ in range(32)]
        lo = [t & 0xFFFFFFFF for t in terms]
        hi = [t >> 32 for t in terms]
        a = sum(x & m27 for x in lo)                                   # redux 1 (< 2^32: no wrap)
        b = sum((x >> 27) | ((y >> 27) << 10) for x, y in zip(lo, hi))  # redux 2, two 10-bit fields
        c = sum(y & m27 for y in hi)                                   # redux 3
        assert a < 1 << 32 and b < 1 << 32 and c < 1 << 32
        total = (a + ((b & 0x3FF) << 27) + ((c + ((b >> 10) << 27)) << 32)) & M
        assert total == sum(terms) & M


def test_round_without_the_shift():
    """Variant tried in round 1 (correct, not faster): keep C_j = (resolved low bits of z_j) * 0xb3 as an accumulator and add
    zeta * (0xb3 << k) per round, zeta = the newly resolved bit taken from the popcount's bit 0 — the parity then needs no
    shift on the vote -> popc -> vote chain.  Must resolve the same z bytes as the shipped formulation."""
    rng = random.Random(6)
    for _ in range(300):
        m = rng.randrange(0, 97)
        stream = [rng.randrange(256) for _ in range(m)]
        b = [[stream[3 * L + j] if 3 * L + j < m else 0 for j in range(3)] for L in range(32)]
        C = [[0, 0, 0] for _ in range(32)]
        z = [[0, 0, 0] for _ in range(32)]
        for k in range(8):
            t = [[((C[L][j] >> k) ^ (b[L][j] >> k)) & 1 for j in range(3)] for L in range(32)]
            votes = sum((t[L][0] ^ t[L][1] ^ t[L][2]) << L for L in range(32))
            l0k = ((H0 & 0xFF) >> k) & 1
            for L in range(32):
                par = bin(votes & ((1 << L) - 1)).count("1")            # only bit 0 is used
                local = [0, t[L][0], t[L][0] ^ t[L][1]]
                for j in range(3):
                    pre = l0k ^ local[j] ^ ((b[L][j] >> k) & 1)         # prepared while the vote is in flight
                    zeta = (pre ^ par) & 1
                    C[L][j] += zeta * (0xB3 << k)
                    z[L][j] |= zeta << k
        # z must be the xor of the running low byte and the stream byte at every position
        h = H0
        for i, byte in enumerate(stream):
            assert z[i // 3][i % 3] == (h & 0xFF) ^ byte
            h = ((h ^ byte) * P) & M


# ---- round 2 formulation (chain_kernel): merged first round for bits 0 and 1, per-block table constants, 3 REDUX -------
def _ballot(preds):
    return sum((1 << L) for L in range(32) if preds[L])


def _par(x):
    return bin(x).count("1") & 1


def resolve_z_merged(b):
    """z bytes (running low byte xor stream byte) for all 96 positions; bits 0 and 1 come from SIX independent ballots
    (bit 0 / bit 1 of each lane's three bytes) — mod 4, x -> 0xb3 * x is the GF(2)-linear map (z1,z0) -> (z1^z0, z0), so the
    prefix is a plain XOR prefix with position-parity masks — bits 2..7 from the usual dependent vote rounds."""
    l00, l01 = H0 & 1, (H0 >> 1) & 1
    V0 = [_ballot([(b[L][j] >> 0) & 1 for L in range(32)]) for j in range(3)]
    V1 = [_ballot([(b[L][j] >> 1) & 1 for L in range(32)]) for j in range(3)]
    EVEN, ODD = 0x55555555, 0xAAAAAAAA
    z = [[0, 0, 0] for _ in range(32)]
    for L in range(32):
        lt = (1 << L) - 1
        for j in range(3):
            i = 3 * L + j
            # lanes whose slot-j' position is <= i (le) / < i (ls): all earlier lanes, plus my own lane when j' <= j / j' < j
            le = [lt | ((1 << L) if jp <= j else 0) for jp in range(3)]
            ls = [lt | ((1 << L) if jp < j else 0) for jp in range(3)]
            # positions of the OPPOSITE parity to i among slot j': lane parity must differ from (i + j') parity ...
            opp = [(EVEN if ((i + jp) & 1) else ODD) for jp in range(3)]      # position 3L'+j' has parity (L'+j')&1
            z0 = l00 ^ _par((V0[0] & le[0]) ^ (V0[1] & le[1]) ^ (V0[2] & le[2]))
            a = _par((V0[0] & ls[0] & opp[0]) ^ (V0[1] & ls[1] & opp[1]) ^ (V0[2] & ls[2] & opp[2]))
            z1 = l01 ^ _par((V1[0] & le[0]) ^ (V1[1] & le[1]) ^ (V1[2] & le[2])) ^ ((i & 1) * l00) ^ a
            z[L][j] = (b[L][j] & 0xFC) | (z1 << 1) | z0
    for k in range(2, 8):                       # the dependent rounds, unchanged
        mask = 1 << k
        p = [[(z[L][j] * 0xB3) & 0xFFFFFFFF for j in range(3)] for L in range(32)]
        votes = _ballot([((p[L][0] ^ p[L][1] ^ p[L][2]) >> k) & 1 for L in range(32)])
        for L in range(32):
            before = _par(votes & ((1 << L) - 1))
            m0 = mask if (H0 & 0xFF) & mask else 0
            zc = [z[L][0] ^ m0, z[L][1] ^ m0 ^ (p[L][0] & mask), z[L][2] ^ m0 ^ ((p[L][0] ^ p[L][1]) & mask)]
            z[L] = [zc[j] ^ ((before << k) & mask) for j in range(3)]
    return z


def chain2(stream):
    m = len(stream)
    assert m <= 96
    b = [[stream[3 * L + j] if 3 * L + j < m else 0 for j in range(3)] for L in range(32)]
    z = resolve_z_merged(b)
    # key = P^m * H0 + sum_i e_i * P^(m - i): the per-lane constants come from a table indexed by m - position, so no
    # multiply follows the reduction
    terms = []
    for L in range(32):
        t = (pow(P, m, 1 << 64) * H0) & M if L == 0 else 0
        for j in range(3):
            i = 3 * L + j
            c = pow(P, max(m - i, 0), 1 << 64)
            clo = c & 0xFFFFFFFF
            clo_s = clo - (1 << 32) if clo >= 1 << 31 else clo
            chi = ((c >> 32) + (1 if clo_s < 0 else 0)) & 0xFFFFFFFF
            e = z[L][j] - (z[L][j] ^ b[L][j])
            t = (t + e * clo_s + ((e * chi & 0xFFFFFFFF) << 32)) & M
        terms.append(t)
    # three REDUX: sum of low words mod 2^32, EXACT sum of their upper halves (21 bits), sum of high words mod 2^32
    r1 = sum(t & 0xFFFFFFFF for t in terms) & 0xFFFFFFFF
    r2 = sum((t & 0xFFFFFFFF) >> 16 for t in terms)
    r3 = sum(t >> 32 for t in terms) & 0xFFFFFFFF
    low_part = (r1 - (r2 << 16)) & 0xFFFFFFFF            # = exact sum of the lower halves (< 2^21)
    carry = ((r2 << 16) + low_part) >> 32
    return ((((r3 + carry) & 0xFFFFFFFF) << 32) | r1)


def test_merged_first_round_resolves_the_same_low_bytes():
    rng = random.Random(7)
    for _ in range(300):
        m = rng.randrange(0, 97)
        stream = [rng.randrange(256) for _ in range(m)]
        b = [[stream[3 * L + j] if 3 * L + j < m else 0 for j in range(3)] for L in range(32)]
        z = resolve_z_merged(b)
        h = H0
        for i, byte in enumerate(stream):
            assert z[i // 3][i % 3] == (h & 0xFF) ^ byte, (m, i)
            h = ((h ^ byte) * P) & M


def test_chain2_equals_fnv1a():
    rng = random.Random(8)
    for _ in range(400):
        stream = [rng.randrange(256) for _ in range(rng.randrange(0, 97))]
        assert chain2(stream) == fnv(stream)
    for _ in range(100):                                   # adversarial for the carry logic: all-ones bytes
        stream = [rng.choice([0xFF, 0x00, 0x80]) for _ in range(rng.randrange(60, 97))]
        assert chain2(stream) == fnv(stream)


def test_static_plus_parent_masks_decomposition():
    """What chain_kernel ships: the stager resolves bits 0/1 of z for the stream with the parent bytes ZEROED (six ballots,
    off the chain); the folder adds the parent's contribution with two 64-bit masks per position and a popcount each —
    no warp vote on the chain for the first two bits.  Stream = 83 1b P7..P0 (80+bs) tokens.. f6, parent at positions 2..9."""
    rng = random.Random(9)
    for _ in range(300):
        key = rng.getrandbits(64) | (1 << 32)
        body = [rng.randrange(256) for _ in range(rng.randrange(1, 83))]
        stream = [0x83, 0x1B] + list(key.to_bytes(8, "big")) + [0x90] + body
        m = len(stream)
        zeroed = stream[:2] + [0] * 8 + stream[10:]
        bz = [[zeroed[3 * L + j] if 3 * L + j < m else 0 for j in range(3)] for L in range(32)]
        bs = [[stream[3 * L + j] if 3 * L + j < m else 0 for j in range(3)] for L in range(32)]
        # static part: bits 0/1 of z with parent bytes zero (the merged round on the zeroed stream)
        l00, l01 = H0 & 1, (H0 >> 1) & 1
        V0 = [_ballot([(bz[L][j] >> 0) & 1 for L in range(32)]) for j in range(3)]
        V1 = [_ballot([(bz[L][j] >> 1) & 1 for L in range(32)]) for j in range(3)]
        EVEN, ODD = 0x55555555, 0xAAAAAAAA
        h = H0
        want = []
        for byte in stream:
            want.append((h & 0xFF) ^ byte)
            h = ((h ^ byte) * P) & M
        for L in range(32):
            lt = (1 << L) - 1
            for j in range(3):
                i = 3 * L + j
                if i >= m:
                    continue
                le = [lt | ((1 << L) if jp <= j else 0) for jp in range(3)]
                lso = [(lt | ((1 << L) if jp < j else 0)) & (EVEN if ((i + jp) & 1) else ODD) for jp in range(3)]
                st0 = l00 ^ _par((V0[0] & le[0]) ^ (V0[1] & le[1]) ^ (V0[2] & le[2]))
                st1 = (l01 ^ ((i & 1) * l00) ^ _par((V1[0] & le[0]) ^ (V1[1] & le[1]) ^ (V1[2] & le[2]))
                       ^ _par((V0[0] & lso[0]) ^ (V0[1] & lso[1]) ^ (V0[2] & lso[2])))
                # dynamic part: masks over the parent key; the parent byte at stream position p is byte (9 - p) of the key
                mle = sum(1 << (8 * (9 - p)) for p in range(2, min(i, 9) + 1))
                mopp = sum(1 << (8 * (9 - p)) for p in range(2, min(i - 1, 9) + 1) if (i - p) & 1)
                z0 = st0 ^ _par(key & mle)
                z1 = st1 ^ _par(key & ((mle << 1) | mopp))
                assert (z0, z1) == (want[i] & 1, (want[i] >> 1) & 1), (i, m)


def test_offset_basis_rides_on_position_zero():
    """Position 0 of every block stream is 0x83 and the running low byte there is the offset basis' (0x25), so
    e_0 = (0x25 ^ 0x83) - 0x25 = 129 is a constant: the term P^m * H0 is folded into position 0's table constant,
    c_0' = P^m * (1 + H0 * 129^-1), and nothing is added after the dot product."""
    inv129 = pow(129, -1, 1 << 64)
    g = (1 + H0 * inv129) & M
    rng = random.Random(10)
    for _ in range(200):
        body = [rng.randrange(256) for _ in range(rng.randrange(1, 95))]
        stream = [0x83] + body
        m = len(stream)
        h, es = H0, []
        for byte in stream:
            lo = h & 0xFF
            es.append((lo ^ byte) - lo)
            h = ((h ^ byte) * P) & M
        assert es[0] == 129
        total = (es[0] * ((pow(P, m, 1 << 64) * g) & M)) & M
        for i in range(1, m):
            total = (total + es[i] * pow(P, m - i, 1 << 64)) & M
        assert total == fnv(stream)


def test_table_kernel_identity_fnv_is_linear_above_the_low_byte():
    """hash_spec_kernel: with h = u + l (l = low byte of h),  fold(h, bytes) = u * P^m + fold(l, bytes)  exactly — the xor
    touches only the low byte, and the low byte of a product depends only on the factors' low bytes.  So a block's tail
    (array head | tokens | extra) is tabulated for the 256 values of l off the chain, and the chain folds only
    83 | U(parent), looks l up and multiplies by P^m.  Checked on the kernel's own stream layout, chained over blocks,
    against plain FNV-1a."""
    rng = random.Random(11)

    def fold(h, bs):
        for b in bs:
            h = ((h ^ b) * P) & M
        return h

    def cbor_uint(v):
        if v < 24:
            return [v]
        if v < 0x100:
            return [0x18, v]
        if v < 0x10000:
            return [0x19, v >> 8, v & 0xFF]
        if v < 0x100000000:
            return [0x1A] + [(v >> s) & 0xFF for s in (24, 16, 8, 0)]
        return [0x1B] + [(v >> s) & 0xFF for s in range(56, -8, -8)]

    for _ in range(40):
        bs = rng.choice([1, 4, 16, 17, 64])
        parent = rng.choice([0, 5, 70000, rng.getrandbits(33) | (1 << 32), rng.getrandbits(64)])
        for _blk in range(6):
            tokens = [rng.getrandbits(rng.choice([4, 8, 16, 17, 32])) for _ in range(bs)]
            head = [0x80 | bs] if bs < 24 else [0x98, bs]
            tail = head + [b for t in tokens for b in cbor_uint(t)] + [0xF6]
            table = [fold(v, tail) for v in range(256)]                  # phase A: 256 plain FNV runs from a bare low byte
            pm = pow(P, len(tail), 1 << 64)
            st = fold(H0, [0x83] + cbor_uint(parent)) if parent >= 24 else fold(H0, [0x83, parent])   # phase B prefix
            low = st & 0xFF
            key = ((st - low) * pm + table[low]) & M
            assert key == fnv([0x83] + cbor_uint(parent) + tail)
            parent = key
