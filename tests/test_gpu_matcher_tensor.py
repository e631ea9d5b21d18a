"""GPU: the tensor-core (BMMA AND.POPC) all-pairs matcher against the CPU oracle, bit-exact on every output (match12, dist12, second12,
nmatches): the fragment layout on one 16 x 8 tile, ragged sizes around every tile / warp / CTA boundary, duplicate columns, popcount
extremes, first-column ties, the front end's strided layout with garbage past each frame's count, and pair counts of 1, 3 and 300."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 2, 7, 8, 9, 15, 16, 17, 127, 128, 129, 255, 257, 4095, 4096]


def make_pair(rng, nA, nB, match_frac=0.5, wrong_angle_frac=0.2):
    """Random descriptors; a share of B rows are A rows with ~5 % of their bits flipped (true matches) at a consistent rotation of ~30
    degrees, some of them at a random angle instead (the rotation histogram rejects those)."""
    A = rng.integers(0, 256, (nA, 32), dtype=np.uint8)
    B = rng.integers(0, 256, (nB, 32), dtype=np.uint8)
    angA = rng.uniform(0, 360, nA).astype(np.float32)
    angB = rng.uniform(0, 360, nB).astype(np.float32)
    if nA and nB:
        rows = np.nonzero(rng.random(nB) < match_frac)[0]
        src = rng.integers(0, nA, rows.size)
        B[rows] = A[src] ^ np.packbits(rng.random((rows.size, 256)) < 0.05, axis=1, bitorder="little")
        ang = np.mod(angA[src] + np.float32(30) + rng.uniform(-3, 3, rows.size).astype(np.float32), np.float32(360)).astype(np.float32)
        keep = rng.random(rows.size) >= wrong_angle_frac
        angB[rows[keep]] = ang[keep]
        angB[angB >= 360] = 0
    return A, angA, B, angB


def check_against_oracle(oracle, got, A, aA, B, aB, nnratio, check_ori, what):
    n, m, d, s = got
    rn, rm, rd, rs = oracle.match_bruteforce(A, aA, B, aB, nnratio, 50, check_ori)
    assert n == rn, "%s: nmatches %d vs %d" % (what, n, rn)
    assert np.array_equal(m, rm), "%s: match12 differs at %s" % (what, np.nonzero(m != rm)[0][:8])
    assert np.array_equal(d, rd), "%s: dist12 differs at %s" % (what, np.nonzero(d != rd)[0][:8])
    assert np.array_equal(s, rs), "%s: second12 differs at %s" % (what, np.nonzero(s != rs)[0][:8])


@pytest.fixture(scope="module")
def matchers():
    from cubemapslam_b200.matcher import ORBMatcher
    ms = {True: ORBMatcher(0.8, True, max_pairs=300, max_features=4096), False: ORBMatcher(0.8, False, max_pairs=300, max_features=4096)}
    yield ms
    for m in ms.values():
        m.close()


def test_one_tile_fragment_layout(oracle, matchers):
    """One 16 x 8 tile: dist12 / second12 of each row equal numpy's popcount of the XOR, and column c is the nearest of row c only (a
    row-specific distance, bits flipped in the c-th 32-bit word), so a row / column / bit-range mix-up of the BMMA fragments cannot go unnoticed."""
    rng = np.random.default_rng(7)
    A = rng.integers(0, 256, (16, 32), dtype=np.uint8)
    B = np.zeros((8, 32), np.uint8)
    for c in range(8):
        bits = rng.choice(np.arange(32 * c, 32 * c + 32), 1 + 3 * c, replace=False)
        B[c] = np.packbits(np.unpackbits(A[c], bitorder="little") ^ np.isin(np.arange(256), bits).astype(np.uint8), bitorder="little")
    D = np.unpackbits(A[:, None, :] ^ B[None, :, :], axis=2).sum(axis=2)
    aA = np.zeros(16, np.float32); aB = np.zeros(8, np.float32)
    n, m, d, s = matchers[False].match_bruteforce(A, aA, B, aB, th_low=256)
    Ds = np.sort(D, axis=1)
    assert np.array_equal(d, Ds[:, 0]) and np.array_equal(s, Ds[:, 1])
    assert np.array_equal(m[:8], np.arange(8)) and np.array_equal(d[:8], 1 + 3 * np.arange(8))
    check_against_oracle(oracle, (n, m, d, s), A, aA, B, aB, 0.8, False, "one tile")


@pytest.mark.parametrize("nA", SIZES)
def test_ragged_sizes(oracle, matchers, nA):
    rng = np.random.default_rng(1000 + nA)
    for nB in SIZES:
        A, aA, B, aB = make_pair(rng, nA, nB)
        for ori in (True, False):
            got = matchers[ori].match_bruteforce(A, aA, B, aB)
            check_against_oracle(oracle, got, A, aA, B, aB, 0.8, ori, "nA=%d nB=%d checkOri=%d" % (nA, nB, ori))


def test_duplicates_extremes_and_ties(oracle, matchers):
    rng = np.random.default_rng(3)
    nA, nB = 600, 700
    A, aA, B, aB = make_pair(rng, nA, nB)
    # exact duplicates of B columns across n8 tiles (7/8, 15/16), the 16-column ldmatrix group, the 128-column stage (127/128/300) and far
    # apart: a row whose nearest column is duplicated gets dist12 == second12 and the lowest column
    for group in ((7, 8), (15, 16), (127, 128, 300), (255, 256, 699), (31, 640)):
        B[list(group)] = B[group[0]]
        aB[list(group)] = aB[group[0]]
    # popcount extremes of the AND identity: all-zero and all-ones rows on both sides
    A[0] = 0; A[1] = 255; A[255] = 0; A[256] = 255; A[599] = 255
    B[3] = 0; B[4] = 255; B[129] = 255; B[698] = 0
    # rows whose best and second best are tied at different distances from the duplicated groups
    A[10] = B[127]; A[11] = B[15]; A[12] = B[31] ^ np.uint8(1)
    for ori in (True, False):
        got = matchers[ori].match_bruteforce(A, aA, B, aB)
        check_against_oracle(oracle, got, A, aA, B, aB, 0.8, ori, "duplicates checkOri=%d" % ori)
        n, m, d, s = got
        assert d[10] == 0 and s[10] == 0 and m[10] == -1          # tie at distance 0: ratio test 0 < 0.8 * 0 fails
        assert d[0] == s[0] == 0 and d[1] == s[1] == 0   # all-zero row: B[3] and B[698]; all-ones row: B[4] and B[129]
    # all-zero A against all-ones B: every distance is 256 -> no best column at all
    Z = np.zeros((20, 32), np.uint8); O = np.full((9, 32), 255, np.uint8)
    got = matchers[True].match_bruteforce(Z, np.zeros(20, np.float32), O, np.zeros(9, np.float32))
    check_against_oracle(oracle, got, Z, np.zeros(20, np.float32), O, np.zeros(9, np.float32), 0.8, True, "zeros vs ones")
    assert np.all(got[2] == 256) and np.all(got[3] == 256) and np.all(got[1] == -1)
    # everything identical: all keys tie, column 0 wins with distance 0 everywhere
    got = matchers[False].match_bruteforce(O[:5], np.zeros(5, np.float32), O, np.zeros(9, np.float32))
    assert np.all(got[2] == 0) and np.all(got[3] == 0)


@pytest.mark.parametrize("P", [1, 3, 300])
def test_pair_counts_device_entry(oracle, matchers, P):
    """cslam_match_bruteforce_dev on P pairs at once, dist12 and second12 included."""
    import torch
    rng = np.random.default_rng(50 + P)
    n = 1100 if P < 300 else 300
    data = [make_pair(rng, n, n) for _ in range(P)]
    dev = torch.device("cuda", 0)
    t = [torch.from_numpy(np.stack([d[k] for d in data])).to(dev) for k in range(4)]
    for ori in (True, False):
        mt = matchers[ori]
        m12 = torch.full((P, n), -7, dtype=torch.int32, device=dev); d12 = torch.zeros_like(m12); s12 = torch.zeros_like(m12)
        nm = torch.zeros(P, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        mt.match_bruteforce_dev(t[0].data_ptr(), t[1].data_ptr(), n, t[2].data_ptr(), t[3].data_ptr(), n, P, m12.data_ptr(), nm.data_ptr(),
                                d12.data_ptr(), s12.data_ptr())
        mt.sync()
        hm, hd, hs, hn = m12.cpu().numpy(), d12.cpu().numpy(), s12.cpu().numpy(), nm.cpu().numpy()
        for p in range(P):
            A, aA, B, aB = data[p]
            check_against_oracle(oracle, (hn[p], hm[p], hd[p], hs[p]), A, aA, B, aB, 0.8, ori, "P=%d pair %d checkOri=%d" % (P, p, ori))
        assert hn.sum() > 0


@pytest.mark.parametrize("P", [1, 3, 300])
def test_match_frames_dev_garbage_past_count(oracle, matchers, P):
    """cslam_match_frames_dev on the front end's layout (28-byte key-point records, angle at float 3) with rows past n[f] filled with
    0xA5: they must never be read as columns, and rows of match12 past n[f] are left alone."""
    import torch
    rng = np.random.default_rng(90 + P)
    F, stride = P + 1, 700 if P < 300 else 320
    n = rng.integers(0, stride + 1, F).astype(np.int32)
    n[0] = stride; n[-1] = max(int(n[-1]), 1)
    desc = np.full((F, stride, 32), 0xA5, np.uint8)
    kps = np.full((F, stride, 7), 0xA5A5A5A5, np.uint32).view(np.float32)
    for f in range(F):
        k = int(n[f])
        desc[f, :k] = rng.integers(0, 256, (k, 32), dtype=np.uint8)
        kps[f, :k, 3] = rng.uniform(0, 360, k).astype(np.float32)
        if f and k and n[f - 1]:   # true matches of the previous frame at a consistent rotation
            rows = np.nonzero(rng.random(k) < 0.5)[0]
            src = rng.integers(0, int(n[f - 1]), rows.size)
            desc[f, rows] = desc[f - 1, src] ^ np.packbits(rng.random((rows.size, 256)) < 0.05, axis=1, bitorder="little")
            a = np.mod(kps[f - 1, src, 3] + np.float32(20), np.float32(360)).astype(np.float32)
            a[a >= 360] = 0
            kps[f, rows, 3] = a
    dev = torch.device("cuda", 0)
    dk = torch.from_numpy(kps.view(np.uint8).reshape(F, stride, 28).copy()).to(dev)
    dd = torch.from_numpy(desc).to(dev); dn = torch.from_numpy(n).to(dev)
    for ori in (True, False):
        mt = matchers[ori]
        m12 = torch.full((P, stride), -7, dtype=torch.int32, device=dev); nm = torch.zeros(P, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        mt.match_frames_dev(dk.data_ptr(), dd.data_ptr(), dn.data_ptr(), stride, F, m12.data_ptr(), nm.data_ptr())
        mt.sync()
        hm, hn = m12.cpu().numpy(), nm.cpu().numpy()
        for f in range(P):
            a, b = int(n[f]), int(n[f + 1])
            rn, rm, _, _ = oracle.match_bruteforce(desc[f, :a], kps[f, :a, 3], desc[f + 1, :b], kps[f + 1, :b, 3], 0.8, 50, ori)
            assert hn[f] == rn and np.array_equal(hm[f, :a], rm), "P=%d pair %d checkOri=%d" % (P, f, ori)
            assert np.all(hm[f, a:] == -7), "rows past n[f] written"
        assert hn.sum() > 0
