"""The key-frame searches past 4096 features on the GPU: cslam_search_by_bow_fv, cslam_search_by_bow_kf_fv, cslam_search_for_triangulation_fv
and cslam_fuse_search_large against the oracle, exactly, and the four drop-ins on the reference's own objects at the initialisation
extractor's key-frame sizes (6024, 9024) against the reference's CPU bodies.

Batches are ragged: per-side counts 0, 1, 4095, 4096, 4097, 6024, 9024 and 16384 at stride 16384, rows past each count hold garbage, and one
count lies past the stride (it is clamped). Scenes (large_kf_scenes.bow_pair) put equal-distance copies 4096 and 8192 apart in one node, key-frame
copies 4096 apart (the second must skip the F feature the first took), and the rotation histogram then holds entries past 4095."""
import ctypes as C
import os

import numpy as np
import pytest

from cubemapslam_b200 import config
from cubemapslam_b200._capi import KP_DTYPE, CslamError
from cubemapslam_b200.mapper import Mapper
from cubemapslam_b200.matcher import ORBMatcher, pack_fv
from cubemapslam_b200.vocabulary import Vocabulary
from oracle.oracle import _p

from . import large_kf_scenes as S

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRIDE = Vocabulary.MAX_FV_FEATURES
COUNTS = (0, 1, 4095, 4096, 4097, 6024, 9024, 16384)
BADARG = r"error -2: "


def _garbage(rng, shape, dtype):
    return rng.integers(0, 256, shape).astype(dtype) if np.dtype(dtype).kind in "ui" else rng.uniform(-1e3, 1e3, shape).astype(dtype)


def _bow_batch(n1s, n2s, seed):
    """A ragged batch of bow_pair scenes at stride STRIDE, garbage past each count; returns the batched arrays, the scenes and the CSRs."""
    rng = np.random.default_rng(seed)
    P = len(n1s)
    d1 = _garbage(rng, (P, STRIDE, 32), np.uint8); a1 = _garbage(rng, (P, STRIDE), np.float32); v1 = _garbage(rng, (P, STRIDE), np.uint8)
    d2 = _garbage(rng, (P, STRIDE, 32), np.uint8); a2 = _garbage(rng, (P, STRIDE), np.float32); v2 = _garbage(rng, (P, STRIDE), np.uint8)
    scenes, f1, f2 = [], [], []
    for p, (n1, n2) in enumerate(zip(n1s, n2s)):
        s = S.bow_pair(n1, n2, seed * 100 + p); scenes.append(s)
        d1[p, :n1] = s["d1"]; a1[p, :n1] = s["a1"]; v1[p, :n1] = s["v1"]; d2[p, :n2] = s["d2"]; a2[p, :n2] = s["a2"]; v2[p, :n2] = s["v2"]
        f1.append(S.csr(s["node1"], STRIDE)); f2.append(S.csr(s["node2"], STRIDE))
    fv1, fv2 = list(pack_fv(f1, STRIDE)), list(pack_fv(f2, STRIDE))
    for fv in (fv1, fv2):   # garbage past each pair's CSR too
        for p in range(P):
            j = fv[3][p]
            fv[0][p, j:] = rng.integers(-5, 1 << 20, STRIDE - j); fv[2][p, fv[1][p, j]:] = rng.integers(-5, 1 << 20, STRIDE - fv[1][p, j])
            fv[1][p, j + 1:] = rng.integers(-5, 1 << 20, STRIDE - j)
    return dict(d1=d1, a1=a1, v1=v1, d2=d2, a2=a2, v2=v2), scenes, fv1, fv2


def _counts(ns, past):
    n = np.array(ns, np.int32)
    n[past] = STRIDE + 7 if n[past] == STRIDE else n[past]   # a count past the stride is clamped to it
    return n


@pytest.fixture(scope="module")
def matcher():
    m = ORBMatcher(0.7, True, max_pairs=len(COUNTS), max_features=64)   # the _fv entries do not depend on max_features
    yield m
    m.close()


@pytest.mark.parametrize("kfkf", [False, True])
@pytest.mark.parametrize("ratio,ori", [(0.7, True), (0.9, False)])
def test_search_by_bow_fv_ragged(oracle, matcher, kfkf, ratio, ori):
    n1s = COUNTS; n2s = COUNTS[::-1]
    b, scenes, fv1, fv2 = _bow_batch(n1s, n2s, 3 + kfkf)
    matcher.nnratio, matcher.check_ori = ratio, ori
    c1, c2 = _counts(n1s, COUNTS.index(STRIDE)), _counts(n2s, 0)
    if kfkf:
        nm, m = matcher.SearchByBoW_KF_fv(b["d1"], b["a1"], b["v1"], c1, fv1, b["d2"], b["a2"], b["v2"], c2, fv2)
    else:
        nm, m = matcher.SearchByBoW_fv(b["d1"], b["a1"], b["v1"], c1, fv1, b["d2"], b["a2"], c2, fv2)
    hi = 0
    for p, s in enumerate(scenes):
        o1, o2 = S.oracle_nodes(s["node1"], 0), S.oracle_nodes(s["node2"], 1)
        if kfkf:
            rn, rm = oracle.search_by_bow_kf(s["d1"], s["a1"], s["v1"], o1, s["d2"], s["a2"], s["v2"], o2, ratio, ori)
        else:
            rn, rm = oracle.search_by_bow(s["d1"], s["a1"], s["v1"], o1, s["d2"], s["a2"], o2, ratio, ori)
        want = np.full(STRIDE, -1, np.int32); want[:len(rm)] = rm
        assert nm[p] == rn and np.array_equal(m[p], want), p
        hi += int(((rm >= 4096) | ((np.arange(len(rm)) >= 4096) & (rm >= 0))).sum())
    assert hi > 500


def test_search_by_bow_fv_ties_and_taken(oracle, matcher):
    """Side-2 copies a, a + 4096, a + 8192 in one node tie at the best distance: with nnratio 1.5 a tie is accepted and the first position must win
    (not the last, not an index taken mod 4096), also between positions one lane scans. Side-1 copies b, b + 4096 in one node: the second must skip an F feature past 4095 that the first
    took. Both occur in the oracle's answer, and the GPU gives the same."""
    n = 12000
    s = S.bow_pair(n, n, 77)
    for k in ("node1", "node2"):   # one node: list position = feature index, so copies 4096 apart fall on the same lane of the scan
        s[k] = np.where(s[k] < 0, -1, 0).astype(np.int32)
    o1, o2 = S.oracle_nodes(s["node1"], 0), S.oracle_nodes(s["node2"], 1)
    rn, rm = oracle.search_by_bow(s["d1"], s["a1"], s["v1"], o1, s["d2"], s["a2"], o2, 1.5, False)
    ties = [a for a in range(0, n, 97) if a + 4096 < n and rm[a] >= 0 and rm[a + 4096] != rm[a]]
    f_of = {int(k): j for j, k in enumerate(rm) if k >= 0}
    taken = [b for b in range(0, n - 4096, 89) if f_of.get(b, -1) >= 4096 and b + 4096 in f_of]
    assert len(ties) > 20 and len(taken) > 5
    matcher.nnratio, matcher.check_ori = 1.5, False
    f1, f2 = pack_fv([S.csr(s["node1"], n)], n), pack_fv([S.csr(s["node2"], n)], n)
    nm, m = matcher.SearchByBoW_fv(s["d1"][None], s["a1"][None], s["v1"][None], [n], f1, s["d2"][None], s["a2"][None], [n], f2)
    assert nm[0] == rn and np.array_equal(m[0], rm)


def test_search_by_bow_fv_fed_by_transform_fv(oracle, matcher):
    """cslam_bow_transform_fv's outputs go into cslam_search_by_bow_fv unchanged."""
    from cubemapslam_b200 import synth
    voc = synth.vocabulary(k=10, L=4, seed=3, stop_frac=0.05)
    gv = Vocabulary(10, 4, voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"], max_frames=2, max_features=64)
    try:
        s = S.bow_pair(9024, 6024, 5)
        desc = np.zeros((2, 9024, 32), np.uint8); desc[0] = s["d1"]; desc[1, :6024] = s["d2"]
        out = gv.transform_fv(desc, n=[9024, 6024])
        fvs = [pack_fv([o[2:]], 9024) for o in out]
        matcher.nnratio, matcher.check_ori = 0.7, True
        nm, m = matcher.SearchByBoW_fv(desc[:1], s["a1"][None], s["v1"][None], [9024], fvs[0], desc[1:], np.resize(s["a2"], 9024)[None], [6024], fvs[1])
        node = [np.full(n, -1, np.int32) for n in (9024, 6024)]
        for f, o in enumerate(out):
            for j in range(len(o[2])):
                node[f][o[4][o[3][j]:o[3][j + 1]]] = o[2][j]
        rn, rm = oracle.search_by_bow(s["d1"], s["a1"], s["v1"], S.oracle_nodes(node[0], 0), s["d2"], s["a2"], S.oracle_nodes(node[1], 1), 0.7, True)
        assert nm[0] == rn > 100 and np.array_equal(m[0, :6024], rm) and (m[0, 6024:] == -1).all()
    finally:
        gv.close()


def _malformed():
    """(name, side, edit of a (node, start, feat, count) CSR of one pair)"""
    def dec(f): f[1][0, 2] = f[1][0, 1] - 1
    def past(f): f[1][0, f[3][0]] = 6025
    def neg(f): f[1][0, 0] = -1
    def idx(f): f[2][0, 3] = 6024
    def dup(f): f[2][0, 3] = f[2][0, 4]
    def asc(f): f[0][0, 5] = f[0][0, 4]
    def cnt(f): f[3][0] = STRIDE + 1
    return [("decreasing start", dec), ("start past the count", past), ("negative start", neg), ("index past the count", idx),
            ("feature twice", dup), ("nodes not ascending", asc), ("node count past the stride", cnt)]


@pytest.mark.parametrize("name,edit", _malformed())
@pytest.mark.parametrize("side", [1, 2])
def test_malformed_feature_vectors_are_rejected(matcher, name, edit, side):
    s = S.bow_pair(6024, 6024, 9)
    good = [pack_fv([S.csr(s["node%d" % k], 6024)], 6024) for k in (1, 2)]
    fv = [[x.copy() for x in g] for g in good]
    edit(fv[side - 1])
    one = lambda x: x[None]   # noqa: E731
    with pytest.raises(CslamError, match=BADARG + "cslam_search_by_bow_fv: malformed FeatureVector"):
        matcher.SearchByBoW_fv(one(s["d1"]), one(s["a1"]), one(s["v1"]), [6024], fv[0], one(s["d2"]), one(s["a2"]), [6024], fv[1])
    with pytest.raises(CslamError, match=BADARG + "cslam_search_by_bow_kf_fv: malformed FeatureVector"):
        matcher.SearchByBoW_KF_fv(one(s["d1"]), one(s["a1"]), one(s["v1"]), [6024], fv[0], one(s["d2"]), one(s["a2"]), one(s["v2"]), [6024], fv[1])
    sc = S.mapping_pair(6024, 4)
    z3, z1 = np.zeros((1, 6024, 3), np.float32), np.zeros((1, 6024), np.uint8)
    mp = Mapper()
    try:
        with pytest.raises(CslamError, match=BADARG + "cslam_search_for_triangulation_fv: malformed FeatureVector"):
            mp.SearchForTriangulation_fv(one(sc["kCur"][:6024]), one(sc["dCur"][:6024]), z3, z1, [6024], fv[0], one(sc["kLast"]), one(sc["dLast"]), z3, z1, [6024], fv[1],
                                         np.zeros((1, 3), np.float32), sc["TcwLast"].reshape(1, 16), sc["E12"].reshape(1, 9), sc["scale"], sc["level_sigma2"], 650, 650)
    finally:
        mp.close()
    n, _ = matcher.SearchByBoW_fv(one(s["d1"]), one(s["a1"]), one(s["v1"]), [6024], good[0], one(s["d2"]), one(s["a2"]), [6024], good[1])
    assert n[0] > 100   # the handle still works


def test_strides_past_the_bound_are_rejected(matcher):
    s = S.bow_pair(10, 10, 1)
    big = np.zeros((1, STRIDE + 1, 32), np.uint8); ang = np.zeros((1, STRIDE + 1), np.float32); v = np.zeros((1, STRIDE + 1), np.uint8)
    fvb = [np.zeros((1, STRIDE + 1), np.int32), np.zeros((1, STRIDE + 2), np.int32), np.zeros((1, STRIDE + 1), np.int32), np.zeros(1, np.int32)]
    fvs = pack_fv([S.csr(s["node2"], 10)], 10)
    with pytest.raises(CslamError, match=BADARG + r"cslam_search_by_bow_fv: bad argument \(pairs in \[1, 8\], strides in \[1, 16384\]\)"):
        matcher.SearchByBoW_fv(big, ang, v, [10], fvb, s["d2"][None], s["a2"][None], [10], fvs)
    with pytest.raises(CslamError, match=BADARG + "cslam_search_by_bow_kf_fv: bad argument"):
        matcher.SearchByBoW_KF_fv(s["d2"][None], s["a2"][None], s["v2"][None], [10], fvs, big, ang, v, [10], fvb)
    mp = Mapper()
    try:
        kb = np.zeros((1, STRIDE + 1), KP_DTYPE)
        with pytest.raises(CslamError, match=BADARG + r"cslam_search_for_triangulation_fv: bad argument \(strides in \[1, 16384\]\)"):
            mp.SearchForTriangulation_fv(kb, big, np.zeros((1, STRIDE + 1, 3), np.float32), v, [10], fvb, kb, big, np.zeros((1, STRIDE + 1, 3), np.float32), v, [10], fvb,
                                         np.zeros((1, 3), np.float32), np.eye(4, dtype=np.float32).reshape(1, 16), np.zeros((1, 9), np.float32), np.ones(8, np.float32),
                                         np.ones(8, np.float32), 650, 650)
        kk = np.zeros(STRIDE + 1, KP_DTYPE); kk["x"] = 700; kk["y"] = 700
        with pytest.raises(CslamError, match=BADARG + r"cslam_fuse_search_large: bad argument \(n_kf <= 16384"):
            mp.FuseSearch(kk, big[0], np.eye(4, dtype=np.float32), np.ones(1, np.uint8), np.zeros((1, 3), np.float32), np.zeros(1, np.int32), big[0, :1], 3.0,
                          np.ones(8, np.float32), np.ones(8, np.float32), 650, 650, large=True)
    finally:
        mp.close()


def _tri_inputs(oracle, n1s, n2s, seed):
    rng = np.random.default_rng(seed)
    P = len(n1s)
    k1 = np.zeros((P, STRIDE), KP_DTYPE); k2 = np.zeros((P, STRIDE), KP_DTYPE)
    for k in (k1, k2):
        k.view(np.uint8)[:] = rng.integers(0, 256, k.view(np.uint8).shape)
    d1 = _garbage(rng, (P, STRIDE, 32), np.uint8); d2 = _garbage(rng, (P, STRIDE, 32), np.uint8)
    r1 = _garbage(rng, (P, STRIDE, 3), np.float32); r2 = _garbage(rng, (P, STRIDE, 3), np.float32)
    h1 = _garbage(rng, (P, STRIDE), np.uint8); h2 = _garbage(rng, (P, STRIDE), np.uint8)
    Ow = np.zeros((P, 3), np.float32); T2 = np.zeros((P, 16), np.float32); E = np.zeros((P, 9), np.float32)
    f1, f2, want, ns = [], [], [], []
    for p, (n1, n2) in enumerate(zip(n1s, n2s)):
        s = S.mapping_pair(max(n1, n2, 2), seed * 10 + p)
        a = lambda x, n: np.ascontiguousarray(x[:n])   # noqa: E731
        n1, n2 = min(n1, len(s["kCur"])), min(n2, len(s["kLast"]))   # mapping_pair may keep a few key points fewer
        ns.append((n1, n2))
        kc, dc, hc, nc = a(s["kCur"], n1), a(s["dCur"], n1), a(s["hasMPCur"], n1), a(s["nodeCur"], n1)
        kl, dl, hl, nl = a(s["kLast"], n2), a(s["dLast"], n2), a(s["hasMPObs"], n2), a(s["nodeObs"], n2)
        ra, _ = oracle.key_point_rays(kc, 650, 650); rb, _ = oracle.key_point_rays(kl, 650, 650)
        k1[p, :n1] = kc; d1[p, :n1] = dc; r1[p, :n1] = ra; h1[p, :n1] = hc; k2[p, :n2] = kl; d2[p, :n2] = dl; r2[p, :n2] = rb; h2[p, :n2] = hl
        T1 = s["TcwCur"].astype(np.float64)
        Ow[p] = (-T1[:3, :3].T @ T1[:3, 3]).astype(np.float32); T2[p] = s["TcwLast"].reshape(16); E[p] = s["E12"].reshape(9)
        nc = nc.copy(); nc[rng.random(n1) < 0.05] = -1
        f1.append(S.csr(nc, STRIDE)); f2.append(S.csr(nl, STRIDE))
        want.append((kc, dc, ra, hc, S.oracle_nodes(nc, 0), kl, dl, rb, hl, nl, s))
    return (k1, d1, r1, h1, k2, d2, r2, h2, Ow, T2, E), pack_fv(f1, STRIDE), pack_fv(f2, STRIDE), want, [list(x) for x in zip(*ns)]


@pytest.mark.parametrize("ori", [False, True])
def test_search_for_triangulation_fv_ragged(oracle, ori):
    n1s = COUNTS; n2s = COUNTS[::-1]
    (k1, d1, r1, h1, k2, d2, r2, h2, Ow, T2, E), fv1, fv2, want, (n1s, n2s) = _tri_inputs(oracle, n1s, n2s, 11 + ori)
    s0 = want[0][-1]
    mp = Mapper()
    try:
        nm, m = mp.SearchForTriangulation_fv(k1, d1, r1, h1, _counts(n1s, COUNTS.index(STRIDE)), fv1, k2, d2, r2, h2, _counts(n2s, 0), fv2, Ow, T2, E, s0["scale"],
                                             s0["level_sigma2"], 650, 650, ori)
    finally:
        mp.close()
    hi = 0
    for p, w in enumerate(want):
        rn, rm = oracle.search_for_triangulation(*w[:10], Ow[p], T2[p], E[p], s0["scale"], s0["level_sigma2"], 650, 650, ori)
        full = np.full(STRIDE, -1, np.int32); full[:len(rm)] = rm
        assert nm[p] == rn and np.array_equal(m[p], full), p
        hi += int(((rm >= 4096) | ((np.arange(len(rm)) >= 4096) & (rm >= 0))).sum())
    assert hi > 500


@pytest.mark.parametrize("n,th", [(4097, 3.0), (6024, 3.0), (9024, 6.0), (16384, 3.0)])
def test_fuse_search_large(oracle, n, th):
    s = S.mapping_pair(n, 60 + n)
    k, d = np.ascontiguousarray(s["kCur"][:n]), np.ascontiguousarray(s["dCur"][:n])
    rng = np.random.default_rng(n)
    m = len(s["Xw"])
    valid = (rng.random(m) < 0.9).astype(np.uint8)
    level = np.clip(s["kLast"]["octave"] + rng.integers(-1, 2, m), 0, 7).astype(np.int32)
    g = oracle.FrameGrid(k, 650, 650)
    bi, bd = g.fuse_search(d, s["TcwCur"], s["scale"], s["inv_level_sigma2"], valid, s["Xw"], level, s["dLast"], th)
    mp = Mapper()
    try:
        gi, gd = mp.FuseSearch(k, d, s["TcwCur"], valid, s["Xw"], level, s["dLast"], th, s["scale"], s["inv_level_sigma2"], 650, 650, large=True)
    finally:
        mp.close()
    assert np.array_equal(gi, bi) and np.array_equal(gd, bd)
    assert ((bd <= 50) & (bi >= 4096)).sum() > (50 if n >= 6024 else -1)


# ------------------------------------------------------------------------------------------------ drop-ins on the reference's objects
LIB = os.path.join(ROOT, "oracle", "_ref", "libdropin_large.so")


@pytest.fixture
def dropin(oracle):
    if not os.path.exists(LIB):
        pytest.skip("oracle/_ref/libdropin_large.so is built in the build container (needs the reference tree)")
    L = C.CDLL(LIB)
    L.dropin_set_camera(C.byref(oracle.cam_params(config.front_1024())))
    return L


@pytest.mark.parametrize("n", [6024, 9024])
def test_search_by_bow_dropins_on_reference_objects(dropin, n):
    for kfkf in (0, 1):
        s = S.bow_pair(n, n - 17, 500 + n + kfkf)
        k1, k2 = S.key_points(s["a1"]), S.key_points(s["a2"])
        n2 = n - 17
        out = n if kfkf else n2
        mg = np.zeros(out, np.int32); mc = np.zeros(out, np.int32); ng = C.c_int32(); nc = C.c_int32()
        if kfkf:
            dropin.dropin_search_by_bow_kf(n, _p(k1), _p(s["d1"]), _p(s["v1"]), _p(s["node1"]), n2, _p(k2), _p(s["d2"]), _p(s["v2"]), _p(s["node2"]), C.c_float(0.75), 1,
                                           _p(mg), C.byref(ng), _p(mc), C.byref(nc))
        else:
            dropin.dropin_search_by_bow(n, _p(k1), _p(s["d1"]), _p(s["v1"]), _p(s["node1"]), n2, _p(k2), _p(s["d2"]), _p(s["node2"]), C.c_float(0.7), 1, _p(mg),
                                        C.byref(ng), _p(mc), C.byref(nc))
        assert ng.value == nc.value > 500
        assert np.array_equal(mg, mc)


@pytest.mark.parametrize("n", [6024, 9024])
def test_mapping_dropins_on_reference_objects(dropin, n):
    s = S.mapping_pair(n, 80 + n)
    a = lambda x: np.ascontiguousarray(x[:n])   # noqa: E731
    kc, dc = a(s["kCur"]), a(s["dCur"])
    m = len(s["Xw"])
    f = [kc, dc, np.ascontiguousarray(s["TcwCur"], np.float32), np.ascontiguousarray(s["Xw"], np.float32), np.ascontiguousarray(s["kLast"]),
         np.ascontiguousarray(s["dLast"]), np.ascontiguousarray(s["TcwLast"], np.float32)]
    ig = np.zeros(m, np.int32); ic = np.zeros(m, np.int32); bg = np.zeros(m, np.uint8); bc = np.zeros(m, np.uint8); ng = C.c_int32(); nc = C.c_int32()
    dropin.dropin_fuse(n, _p(f[0]), _p(f[1]), _p(f[2]), m, _p(f[3]), _p(f[4]), _p(f[5]), _p(f[6]), C.c_float(3.0), _p(ig), _p(bg), C.byref(ng), _p(ic), _p(bc),
                       C.byref(nc))
    assert ng.value == nc.value > 500
    assert np.array_equal(ig, ic) and np.array_equal(bg, bc) and (ig >= 4096).sum() > 50     # the final map state
    t = [kc, dc, np.ascontiguousarray(s["TcwCur"], np.float32), a(s["hasMPCur"]), a(s["nodeCur"]).astype(np.int32), np.ascontiguousarray(s["kLast"]),
         np.ascontiguousarray(s["dLast"]), np.ascontiguousarray(s["TcwLast"], np.float32), np.ascontiguousarray(s["hasMPObs"]),
         np.ascontiguousarray(s["nodeObs"], np.int32), np.ascontiguousarray(s["E12"], np.float32)]
    n2 = len(s["kLast"])
    for ori in (0, 1):
        mg = np.zeros(n, np.int32); mc = np.zeros(n, np.int32)
        dropin.dropin_search_for_triangulation(n, _p(t[0]), _p(t[1]), _p(t[2]), _p(t[3]), _p(t[4]), n2, _p(t[5]), _p(t[6]), _p(t[7]), _p(t[8]), _p(t[9]), _p(t[10]), ori,
                                               _p(mg), C.byref(ng), _p(mc), C.byref(nc))
        assert ng.value == nc.value > 300
        assert np.array_equal(mg, mc) and (mg[4096:] >= 0).sum() > 50
