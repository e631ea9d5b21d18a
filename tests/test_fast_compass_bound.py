"""The compass bound k_fast's phase A0 uses to drop work items (compass_x2 in frontend.cu), checked on the CPU against the FAST-9/16 arc
score's definition: the lattice identity behind its 3-operation form, that it never lies below the exact score, and that its u16x2
high-byte formulation (centre masked two ways, ring words unmasked) gives the plain-integer verdict whatever the low bytes hold."""
import itertools

import numpy as np

RUN = 9


def arc_bounds(R, c):
    """Exact A = max_k min(R[k..k+8]) and B = min_k max(R[k..k+8]) of rings R (n x 16) and the arc score s = max(0, A - c, c - B)."""
    RR = np.concatenate([R, R[:, :RUN - 1]], 1)
    win = np.stack([RR[:, k:k + RUN] for k in range(16)], 1)
    A, B = win.min(2).max(1), win.max(2).min(1)
    return A, B, np.maximum(0, np.maximum(A - c, c - B))


def compass(R):
    """The bound: upper of A, lower of B, from ring pixels 0, 4, 8, 12 (3 min/max each)."""
    r0, r4, r8, r12 = R[:, 0], R[:, 4], R[:, 8], R[:, 12]
    return np.minimum(np.maximum(r0, r8), np.maximum(r4, r12)), np.maximum(np.minimum(r0, r8), np.minimum(r4, r12))


def test_lattice_identity_and_dual():
    v = np.array(list(itertools.product(range(5), repeat=4)))   # every order pattern of 4 values, ties included
    v = np.concatenate([v, np.random.default_rng(0).integers(0, 256, (20000, 4))])
    a, b, c, d = v.T                                              # R0, R4, R8, R12
    pairs = [(a, b), (b, c), (c, d), (d, a)]                      # (R[4j], R[4j+4])
    assert np.array_equal(np.max([np.minimum(x, y) for x, y in pairs], 0), np.minimum(np.maximum(a, c), np.maximum(b, d)))
    assert np.array_equal(np.min([np.maximum(x, y) for x, y in pairs], 0), np.maximum(np.minimum(a, c), np.minimum(b, d)))


def _corner_rings(rng):
    """Every 9..16-pixel arc at every start, bright and dark, around random centres, the other ring pixels random."""
    R, C = [], []
    for start, n, bright in itertools.product(range(16), range(RUN, 17), (True, False)):
        c = rng.integers(1, 255, 64)
        r = rng.integers(0, 256, (64, 16))
        arc = rng.integers(c[:, None] + 1, 256, (64, n)) if bright else rng.integers(0, c[:, None], (64, n))
        r[:, (start + np.arange(n)) % 16] = arc
        R.append(r); C.append(c)
    return np.concatenate(R), np.concatenate(C)


def test_bound_never_below_the_arc_score():
    rng = np.random.default_rng(1)
    Rc, Cc = _corner_rings(rng)
    Rr, Cr = rng.integers(0, 256, (20000, 16)), rng.integers(0, 256, 20000)
    base = rng.integers(0, 256, 20000)                             # low-contrast rings: scores near the thresholds
    Rn, Cn = np.clip(base[:, None] + rng.integers(-12, 13, (20000, 16)), 0, 255), base
    R, C = np.concatenate([Rc, Rr, Rn]), np.concatenate([Cc, Cr, Cn])
    A, B, s = arc_bounds(R, C)
    UA, LB = compass(R)
    assert (A <= UA).all() and (B >= LB).all()
    assert (s[: len(Rc)] > 0).all()                                # the corner rings are corners
    for mt in range(1, 256):
        dropped = (UA - C <= mt) & (C - LB <= mt)
        assert (s[dropped] <= mt).all(), mt
    # the bound is not vacuous: at mt = 7 it drops some of the other rings
    assert ((UA - C <= 7) & (C - LB <= 7))[len(Rc):].any()


def _vmax(a, b):
    return ((np.maximum(a >> 16, b >> 16) << 16) | np.maximum(a & 0xffff, b & 0xffff)).astype(np.uint32)


def _vmin(a, b):
    return ((np.minimum(a >> 16, b >> 16) << 16) | np.minimum(a & 0xffff, b & 0xffff)).astype(np.uint32)


def compass_x2(r0, r4, r8, r12, c, T1):
    """frontend.cu's compass_x2 on u32 words of two u16 lanes (32-bit wrapping subtraction, as the device computes it)."""
    A = _vmin(_vmax(r0, r8), _vmax(r4, r12))
    Bm = _vmax(_vmin(r0, r8), _vmin(r4, r12))
    cl, ch = c & np.uint32(0xff00ff00), c | np.uint32(0x00ff00ff)
    t1 = (_vmax(A, cl) - cl).astype(np.uint32)
    t2 = (ch - _vmin(Bm, ch)).astype(np.uint32)
    return _vmax(_vmax(t1, t2), T1)


def test_u16x2_high_byte_verdict_matches_integers():
    rng = np.random.default_rng(2)
    n = 200000
    hi = rng.integers(0, 256, (5, 2, n)).astype(np.uint32)        # R0, R4, R8, R12, centre; two lanes
    hi[:4, :, : n // 2] = np.clip(hi[4, :, : n // 2] + rng.integers(-9, 10, (4, 2, n // 2)), 0, 255)   # margins near mt
    lo = rng.integers(0, 256, (5, 2, n)).astype(np.uint32)        # the neighbouring pixels in the low bytes
    lo[:, :, : n // 8] = rng.choice(np.array([0, 255], np.uint32), (5, 2, n // 8))
    words = (hi[:, 1] << 24) | (lo[:, 1] << 16) | (hi[:, 0] << 8) | lo[:, 0]
    r0, r4, r8, r12, c = words
    UA = np.minimum(np.maximum(hi[0], hi[2]), np.maximum(hi[1], hi[3])).astype(np.int64)
    LB = np.maximum(np.minimum(hi[0], hi[2]), np.minimum(hi[1], hi[3])).astype(np.int64)
    cc = hi[4].astype(np.int64)
    for mt in (1, 2, 7, 8, 20, 128, 254, 255):
        T1 = np.uint32(mt * 0x01000100 | 0x00ff00ff)
        got = compass_x2(r0, r4, r8, r12, c, T1)
        want = (UA - cc > mt) | (cc - LB > mt)                    # per lane: the bound can exceed mt
        lane = np.stack([(got & 0xffff) != (T1 & 0xffff), (got >> 16) != (T1 >> 16)])
        assert np.array_equal(lane, want), mt
