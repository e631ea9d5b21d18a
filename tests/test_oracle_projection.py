"""oracle projection matchers == the reference's own ORBMatcher::SearchByProjection (src/ORBMatcher.cpp:51-251) and
CamModelGeneral::TransformRaysToCubemap (src/CamModelGeneral.cpp:95-154) compiled in oracle/_ref/libref.so, on reference Frame / MapPoint objects; its answers are recorded for where the library cannot be
built (tests/refrecord.py)."""
import numpy as np
import pytest

from cubemapslam_b200 import config, synth

from oracle import ref
from tests import test_gpu_tracking_limits as L
from tests.refrecord import LIVE, RefRecord, same

REC = RefRecord("oracle_projection")


@pytest.fixture(scope="module")
def cam(oracle):
    cfg = config.front_1024()
    cp = oracle.cam_params(cfg)
    r = ref.Ref(cp) if LIVE else None
    return cp, r, float(REC("cos_fov_th", lambda: r.cos_fov_th()))


def test_ray_to_cubemap(oracle, cam):
    cp, r, _ = cam
    rng = np.random.default_rng(0)
    xyz = rng.normal(0, 1, (4000, 3)).astype(np.float32)
    xyz[::7, 2] = np.abs(xyz[::7, 0])                   # exactly on a face boundary (|x/z| == 1)
    xyz[::11] = 0
    uv, f = oracle.ray_to_cubemap(xyz, 650, 650)
    ruv, rf = REC("ray_to_cubemap", lambda: r.ray_to_cubemap(xyz), digest=(0, 1))
    assert same(f, rf) and same(uv, ruv)
    assert len(set(f.tolist())) == 6


@pytest.mark.parametrize("seed,th,ori", [(0, 15.0, True), (1, 7.0, True), (2, 15.0, False), (3, 30.0, True)])
def test_search_by_projection_last_frame(oracle, cam, seed, th, ori):
    cp, r, cth = cam
    s = synth.tracking_pair(seed, n=1500, faceW=650)
    g = oracle.FrameGrid(s["kCur"], 650, 650)
    n1, m1 = g.search_by_projection_last(s["dCur"], s["TcwCur"], s["scale"], s["kLast"], s["hasMP"], s["Xw"], s["dLast"], s["mpObs"], s["curTaken"], cth, th, ori)

    def run():
        n2, m2 = r.search_by_projection_last(s["kCur"], s["dCur"], s["TcwCur"], s["kLast"], s["TcwLast"], s["hasMP"], s["Xw"], s["dLast"], s["mpObs"], s["curTaken"], th, ori)
        return n2, np.where(m2 == -2, -1, m2)
    n2, m2 = REC("last_frame_%d" % seed, run, digest=(1,))
    assert n1 == n2 and n1 > 300
    assert same(np.asarray(m1, np.int32), m2)
    good = m1 >= 0
    assert (s["src"][good] == m1[good]).mean() > 0.9    # and the matches are the planted correspondences


@pytest.mark.parametrize("seed,th,nn", [(0, 1.0, 0.8), (1, 3.0, 0.8), (2, 5.0, 0.6)])
def test_search_by_projection_local_map(oracle, cam, seed, th, nn):
    cp, r, _ = cam
    s = synth.tracking_pair(10 + seed, n=1500, faceW=650)
    rng = np.random.default_rng(seed)
    # the local-map variant consumes what Frame::isInFrustum stored in each MapPoint: projection, predicted level, viewing cosine
    has = s["src"] >= 0
    nMP = 1200
    pick = rng.choice(np.nonzero(has)[0], nMP, replace=False)
    proj = np.stack([s["kCur"]["x"][pick], s["kCur"]["y"][pick]], 1).astype(np.float32) + rng.normal(0, 2.0, (nMP, 2)).astype(np.float32)
    lvl = np.clip(s["kCur"]["octave"][pick] + rng.integers(0, 2, nMP), 0, 7).astype(np.int32)
    vcos = rng.choice(np.array([0.9999, 0.99, 0.7], np.float32), nMP)
    dMP = s["dLast"][s["src"][pick]]
    inView = (rng.random(nMP) < 0.9).astype(np.uint8); obs = (rng.random(nMP) < 0.9).astype(np.int32)
    taken = (rng.random(len(s["kCur"])) < 0.05).astype(np.uint8)
    g = oracle.FrameGrid(s["kCur"], 650, 650)
    n1, m1 = g.search_by_projection_local(s["dCur"], s["scale"], inView, proj, lvl, vcos, dMP, obs, taken, th, nn)

    def run():
        n2, m2 = r.search_by_projection_local(s["kCur"], s["dCur"], inView, proj, lvl, vcos, dMP, obs, taken, th, nn)
        return n2, np.where(m2 == -2, -1, m2)
    n2, m2 = REC("local_map_%d" % seed, run, digest=(1,))
    assert n1 == n2 and n1 > 200
    assert same(np.asarray(m1, np.int32), m2)


# ---- the scenes of tests/test_gpu_tracking_limits.py: ties, thresholds, gates, projections, taken slots, histograms and sizes
CAMS = {650: dict(name="front_cam_params", Camera_Ih=1024, Camera_v0=512.0), 450: dict(name="lafida_cam0_params", CubeFace_w=450, CubeFace_h=450),
        610: dict(name="front_cam_params", Camera_Ih=1024, Camera_v0=512.0, CubeFace_w=610, CubeFace_h=610)}


@pytest.fixture(scope="module", params=sorted(CAMS))
def cam_w(request, oracle):
    W = request.param
    c = dict(CAMS[W]); name = c.pop("name")
    cp = oracle.cam_params(config.camera(name, **c))
    r = ref.Ref(cp) if LIVE else None
    cth = float(REC("cos_fov_th_%d" % W, lambda: r.cos_fov_th()))
    assert np.float32(cth) == L.cos_fov_th()                  # the GPU file's field-of-view threshold is the camera's
    return W, r, np.float32(cth)


def reference_can_take(a):
    """Every key point on a face with its cell corner on the same face: ComputeKeyPointRays exits and the debug build's PosInGrid asserts
    otherwise."""
    return all(L.ref_safe(x, y, a["W"]) for x, y in zip(a["k"]["x"], a["k"]["y"])) and all(L.ref_safe(x, y, a["W"]) for x, y in zip(a["kl"]["x"], a["kl"]["y"]))


@pytest.mark.parametrize("ori", [True, False])
def test_search_by_projection_last_limits(oracle, cam_w, ori):
    W, r, cth = cam_w
    for i, P in enumerate(L.last_batch(oracle, W)):
        a = P.arrays()
        assert reference_can_take(a), i

        def run():
            n2, m2 = r.search_by_projection_last(a["k"], a["d"], a["T"], a["kl"], a["T"], a["valid"], a["Xw"], a["dq"], a["obs"], a["taken"], L.TH_LAST, ori)
            return n2, np.where(m2 == -2, -1, m2)
        n2, m2 = REC("limits_last_%d_%d_%d" % (W, i, ori), run, digest=(1,))
        n1, m1 = L.oracle_search(oracle, a, 0, cth, ori)
        assert n1 == n2, (i, n1, n2)
        assert same(np.asarray(m1, np.int32), m2), i


@pytest.mark.parametrize("nn", L.NNRATIOS)
def test_search_by_projection_local_limits(oracle, cam_w, nn):
    W, r, _ = cam_w
    pairs = [(P, L.TH_LOCAL) for P in L.local_batch(oracle, W, nn)]
    if nn == 0.8:
        pairs += [(L.radius_pair(oracle, W, th), th) for th in (1.0, float(np.nextafter(np.float32(1), np.float32(2))))]
    for i, (P, th) in enumerate(pairs):
        a = P.arrays()
        assert reference_can_take(a), i

        def run():
            n2, m2 = r.search_by_projection_local(a["k"], a["d"], a["valid"], a["proj"], a["level"], a["vcos"], a["dq"], a["obs"], a["taken"], th, nn)
            return n2, np.where(m2 == -2, -1, m2)
        n2, m2 = REC("limits_local_%d_%s_%d" % (W, nn, i), run, digest=(1,))
        n1, m1 = L.oracle_search(oracle, a, 1, nn=nn, th=th)
        assert n1 == n2, (i, n1, n2)
        assert same(np.asarray(m1, np.int32), m2), i
