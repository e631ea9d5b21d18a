"""oracle LocalMapping feature operations (oracle/mapping.h) == the reference's own MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cpp:243-303),
ORBMatcher::Fuse (src/ORBMatcher.cpp:1126-1240), ORBMatcher::SearchForTriangulation (:971-1124) and CamModelGeneral::GetVectorSigma
(src/CamModelGeneral.cpp:307-335) compiled in oracle/_ref/libref.so, run on reference KeyFrame / MapPoint objects; its answers are recorded for where the library cannot
be built (tests/refrecord.py)."""
import numpy as np
import pytest

from cubemapslam_b200 import config, synth

from oracle import ref
from tests import test_gpu_mapping_limits as L
from tests.refrecord import LIVE, RefRecord, same

REC = RefRecord("oracle_mapping")


@pytest.fixture(scope="module")
def cam(oracle):
    cp = oracle.cam_params(config.front_1024())
    return cp, ref.Ref(cp) if LIVE else None


def test_distinctive_descriptor(oracle, cam):
    cp, r = cam
    rng = np.random.default_rng(0)
    sets = []
    for N in (1, 2, 3, 4, 7, 12, 33):
        for rep in range(6):
            base = rng.integers(0, 256, 32, dtype=np.uint8)
            d = np.stack([base ^ np.packbits(rng.random(256) < rng.uniform(0.02, 0.3), bitorder="little") for _ in range(N)])
            if rep == 0 and N > 2:
                d[1] = d[0]                                # ties: the first index with the least median wins
            sets.append(d)
    rbest = REC("distinctive_descriptor", lambda: np.stack([r.distinctive_descriptor(d) for d in sets]))
    for d, rb in zip(sets, rbest):
        best = oracle.distinctive_descriptors(d, np.array([0, len(d)], np.int32))[0]
        assert np.array_equal(rb, d[best])
    assert oracle.distinctive_descriptors(np.zeros((0, 32), np.uint8), np.array([0, 0], np.int32))[0] == -1


def test_vector_sigma(oracle, cam):
    cp, r = cam
    rng = np.random.default_rng(1)
    tiles = [(1, 1), (0, 1), (2, 1), (1, 0), (1, 2)]
    q = []
    for i in range(400):
        c, rr = tiles[i % 5]
        kx = np.float32(c * 650 + rng.uniform(0, 649.9)); ky = np.float32(rr * 650 + rng.uniform(0, 649.9))
        q.append((kx, ky, rng.normal(0, 1, 3).astype(np.float32)))
    rs = REC("vector_sigma", lambda: np.array([r.vector_sigma(kx, ky, nrm) for kx, ky, nrm in q], np.float32))
    for i, ((kx, ky, nrm), b) in enumerate(zip(q, rs)):
        a = np.float32(oracle.vector_sigma(kx, ky, nrm, 650, 650))
        assert a == b or (np.isnan(a) and np.isnan(b)), (i, a, b)


@pytest.mark.parametrize("seed,th", [(0, 3.0), (1, 3.0), (2, 6.0)])
def test_fuse_search(oracle, cam, seed, th):
    cp, r = cam
    s = synth.mapping_pair(seed, n=1500, faceW=650)
    nf, valid, level, idx = REC("fuse_%d" % seed, lambda: r.fuse(s["kCur"], s["dCur"], s["TcwCur"], s["Xw"], s["kLast"], s["dLast"], s["TcwLast"], th))
    g = oracle.FrameGrid(s["kCur"], 650, 650)
    bi, bd = g.fuse_search(s["dCur"], s["TcwCur"], s["scale"], s["inv_level_sigma2"], valid, s["Xw"], level, s["dLast"], th)
    fused = bd <= 50
    assert nf == int(fused.sum()) and nf > 150
    # the reference's bookkeeping: a MapPoint that lost its key point to a later one was Replace()d by it, so it still resolves to the same index
    assert np.array_equal(np.where(fused, bi, -1), idx)
    assert valid.mean() > 0.5 and len(set(level.tolist())) >= 5


@pytest.mark.parametrize("seed,ori", [(0, False), (1, True), (2, False)])
def test_search_for_triangulation(oracle, cam, seed, ori):
    cp, r = cam
    s = synth.mapping_pair(10 + seed, n=1500, faceW=650)
    n2, m2, Ow1 = REC("triangulation_%d" % seed, lambda: r.search_for_triangulation(s["kCur"], s["dCur"], s["TcwCur"], s["hasMPCur"], s["nodeCur"], s["kLast"], s["dLast"],
                                                                                      s["TcwLast"], s["hasMPObs"], s["nodeObs"], s["E12"], ori), digest=(1,))
    rays1, _ = oracle.key_point_rays(s["kCur"], 650, 650); rays2, _ = oracle.key_point_rays(s["kLast"], 650, 650)
    n1, m1 = oracle.search_for_triangulation(s["kCur"], s["dCur"], rays1, s["hasMPCur"], s["nodeCur"], s["kLast"], s["dLast"], rays2, s["hasMPObs"], s["nodeObs"], Ow1,
                                             s["TcwLast"], s["E12"], s["scale"], s["level_sigma2"], 650, 650, ori)
    assert n1 == n2 and n1 > 100
    assert same(np.asarray(m1, np.int32), m2)
    good = m1 >= 0
    assert (s["src"][good] == m1[good]).mean() > 0.9


def test_fuse_on_face_boundaries(oracle, cam):
    """TransformRaysToCubemap leaves in-face coordinates (no tile offset) in (u, v) when its in-face bounds test fails, and Fuse does not look at the
    returned face - it only asks IsInImage(u, v) (src/ORBMatcher.cpp:1150-1154). MapPoints exactly on a face seam (|x/z| == 1 etc.) and behind the
    camera exercise that path: oracle == compiled reference."""
    cp, r = cam
    s, Xw, _ = L.face_boundary_points()
    I4 = np.eye(4, dtype=np.float32)
    nf, valid, level, idx = REC("fuse_face_boundaries", lambda: r.fuse(s["kCur"], s["dCur"], I4, Xw, s["kLast"], s["dLast"], I4, 4.0))
    g = oracle.FrameGrid(s["kCur"], 650, 650)
    bi, bd = g.fuse_search(s["dCur"], I4, s["scale"], s["inv_level_sigma2"], valid, Xw, level, s["dLast"], 4.0)
    fused = bd <= 50
    assert nf == int(fused.sum())
    assert np.array_equal(np.where(fused, bi, -1), idx)


# ---- the scenes of tests/test_gpu_mapping_limits.py that have a reference counterpart
@pytest.fixture(scope="module")
def cam450(oracle):
    cp = oracle.cam_params(config.lafida_450())
    return cp, ref.Ref(cp) if LIVE else None


def test_fuse_ties_and_complements(oracle, cam):
    """Ties at the least distance across cells, 32-cell chunks and seam rectangles (the first visited wins, not the lowest index), and
    complement-only windows: the reference fuses the first visited tied key point and nothing in a complement window."""
    cp, r = cam
    S = L.tie_scene(oracle); a = S.arrays()
    nf, valid, level, idx = REC("fuse_ties", lambda: r.fuse(a["kKF"], a["dKF"], a["Tcw"], a["Xw"], S.kobs(), a["dMP"], a["Tcw"], a["th"]))
    ms = [c["m"] for c in S.cases]
    assert (valid[ms] == 1).all() and np.array_equal(level[ms], a["level"][ms])   # the reference predicts the levels the GPU test uses
    bi, bd = oracle.FrameGrid(a["kKF"], 650, 650).fuse_search(a["dKF"], a["Tcw"], a["scale"], a["isg"], valid, a["Xw"], level, a["dMP"], a["th"])
    fused = bd <= 50
    assert nf == int(fused.sum())
    assert np.array_equal(np.where(fused, bi, -1), idx)
    for c in S.cases:
        assert idx[c["m"]] == (c["expect"] if c["dist"] <= 50 else -1), c


@pytest.mark.parametrize("seed,th", [(0, 3.0), (2, 12.0)])
def test_fuse_search_450(oracle, cam450, seed, th):
    cp, r = cam450
    s = synth.mapping_pair(seed, n=1500, faceW=450)
    nf, valid, level, idx = REC("fuse450_%d" % seed, lambda: r.fuse(s["kCur"], s["dCur"], s["TcwCur"], s["Xw"], s["kLast"], s["dLast"], s["TcwLast"], th))
    bi, bd = oracle.FrameGrid(s["kCur"], 450, 450).fuse_search(s["dCur"], s["TcwCur"], s["scale"], s["inv_level_sigma2"], valid, s["Xw"], level, s["dLast"], th)
    fused = bd <= 50
    assert nf == int(fused.sum()) and nf > 150
    assert np.array_equal(np.where(fused, bi, -1), idx)


def test_search_for_triangulation_450(oracle, cam450):
    """Three synthetic pairs, a pure rotation (camera centre exactly 0, E12 = 0) and an epipole on a face seam, at face width 450: KF1's
    pose [I | -Ow1] gives the reference exactly the camera centre the GPU test uses."""
    cp, r = cam450
    for i, p in enumerate(L.triangulation_pairs(oracle)):
        s = p["s"]; ori = i % 2 == 1
        T1 = s["TcwCur"] if i < 3 else np.eye(4, dtype=np.float32)
        if i == 4:
            T1 = T1.copy(); T1[:3, 3] = -p["Ow"]
        n2, m2, Ow1 = REC("triangulation450_%d" % i, lambda: r.search_for_triangulation(s["kCur"], s["dCur"], T1, s["hasMPCur"], s["nodeCur"], s["kLast"], s["dLast"],
                                                                                            p["T2"], s["hasMPObs"], s["nodeObs"], p["E"], ori), digest=(1,))
        assert i < 3 or np.array_equal(Ow1, p["Ow"]), i
        n1, m1 = L.oracle_triangulation(oracle, dict(p, Ow=Ow1), 450, ori)
        assert n1 == n2, i
        assert same(np.asarray(m1, np.int32), m2), i


def test_distinctive_descriptor_ties(oracle, cam):
    """Least-median ties first at rows 0, 31, 32, 127, 128, 129 (distinct descriptors, so the returned bytes name the row), all-identical
    sets and random sets of N = 1, 2, 3, 127, 128, 129 and small even N."""
    cp, r = cam
    sets = L.distinctive_sets(max_n=129)
    rbest = REC("distinctive_ties", lambda: np.stack([r.distinctive_descriptor(d) for d in sets]))
    for d, rb in zip(sets, rbest):
        best = oracle.distinctive_descriptors(d, np.array([0, len(d)], np.int32))[0]
        assert np.array_equal(rb, d[best])
