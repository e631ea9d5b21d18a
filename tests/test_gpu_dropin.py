"""The drop-in boundary, linked and run on the GPU: dropin/*.cpp (definitions of the reference's ORBextractor / ORBMatcher / Optimizer
methods on libcubemap_b200.so) compiled against the reference's own unmodified headers and linked with the reference's own Frame / KeyFrame /
MapPoint / Map classes (oracle/_ref/libdropin.so, recipe oracle/Makefile, harness oracle/dropin_api.cpp). The reference call sites
Frame::Frame -> (*mpORBextractor)(...), ORBMatcher::SearchByBoW(pKF, F, ...), Optimizer::PoseOptimization(&F),
Optimizer::LocalBundleAdjustment(pKF, &stop, pMap) run unchanged; results are compared with the oracle / the reference's CPU bodies."""
import ctypes as C
import os

import numpy as np
import pytest

from cubemapslam_b200 import config, synth
from oracle.oracle import KP_DTYPE, _p

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "oracle", "_ref", "libdropin.so")


@pytest.fixture
def dropin(oracle):
    """dropin(cfg): libdropin.so with the reference's CamModelGeneral, a process-wide singleton, set to cfg's camera. Every test sets its own
    camera first, so none depends on what an earlier test left there."""
    if not os.path.exists(LIB):
        pytest.skip("oracle/_ref/libdropin.so is built in the build container (needs the reference tree)")
    L = C.CDLL(LIB)

    def with_camera(cfg):
        L.dropin_set_camera(C.byref(oracle.cam_params(cfg)))
        return L
    return with_camera


def _in_fov(oracle, cfg, kpxy):
    """Which key points have their ray inside the field of view: Optimizer skips the others (src/Optimizer.cpp:84-86, :323-325, :520), so the
    tests drop them up front on both sides."""
    kp = np.zeros(len(kpxy), KP_DTYPE); kp["x"] = kpxy[:, 0]; kp["y"] = kpxy[:, 1]
    rays, _ = oracle.key_point_rays(kp, int(cfg["CubeFace.w"]), int(cfg["CubeFace.h"]))
    a = np.float32(cfg["Camera.fov"]) / np.float32(2) * (np.float32(3.1415926535897932384626) / np.float32(180))
    return rays[:, 2] >= np.float32(np.cos(np.float64(a)))


def _inv_sigma2(octave):
    """Frame::mvInvLevelSigma2[octave] of 8 levels with scale factor 1.2, in float32."""
    sc = np.float32(1.0); tab = []
    for _ in range(8):
        tab.append(np.float32(1.0) / (sc * sc)); sc = sc * np.float32(1.2)
    return np.array([tab[o] for o in octave], np.float32)


def test_frame_constructor_runs_gpu_extractor(oracle, dropin):
    """Frame::Frame(im, mask, ts, extractor, voc) of the reference with the drop-in ORBextractor: keypoints / descriptors equal the oracle,
    and the reference's own ComputeKeyPointRays / AssignFeaturesToGrid ran on them."""
    cfg = config.lafida_450()
    L = dropin(cfg)
    cp = oracle.cam_params(cfg)
    mask = config.load_mask("gray_lafida_cubemap_mask_450")
    m1, m2 = oracle.build_maps(cp)
    for fi in (0, 3):
        canvas = oracle.warp(cp, synth.fisheye_frame(cfg, fi), m1, m2)
        cap = 2100
        kps = np.zeros(cap, KP_DTYPE); desc = np.zeros((cap, 32), np.uint8); rays = np.zeros((cap, 3), np.float32); grid = np.zeros((5, 50, 50), np.int32)
        n = L.dropin_frame_from_image(_p(canvas), _p(mask), 1350, 1350, 2000, C.c_float(1.2), 8, 20, 7, cap, _p(kps), _p(desc), _p(rays), _p(grid))
        rk, rd = oracle.ORBextractor(2000, 1.2, 8, 20, 7, 450, 450)(canvas, mask)
        assert n == len(rk) > 1000
        assert np.array_equal(kps[:n].view(np.uint8), rk.view(np.uint8)) and np.array_equal(desc[:n], rd)
        assert grid.sum() == n and np.allclose(np.linalg.norm(rays[:n], axis=1), 1.0, atol=1e-6)


def test_search_by_bow_on_reference_objects(dropin):
    """ORBMatcher(0.7, true).SearchByBoW(pKF, F, matches) through the reference's KeyFrame / Frame / MapPoint objects: the GPU drop-in and the
    reference's own CPU body (src/ORBMatcher.cpp:409-539, same objects) must agree exactly."""
    L = dropin(config.lafida_450())
    for seed, n in ((0, 1500), (1, 700)):
        A, aA, B, aB, perm = synth.descriptor_pair(seed, n=n)
        rng = np.random.default_rng(40 + seed)
        nodeA = rng.integers(0, 60, n).astype(np.int32); nodeB = nodeA[perm].copy()
        nodeB[rng.random(n) < 0.1] = 61
        valid = (rng.random(n) < 0.8).astype(np.uint8)
        kA = np.zeros(n, KP_DTYPE); kB = np.zeros(n, KP_DTYPE)
        kA["x"] = 600; kA["y"] = 600; kB["x"] = 600; kB["y"] = 600; kA["angle"] = aA; kB["angle"] = aB
        mg = np.zeros(n, np.int32); mc = np.zeros(n, np.int32); ng = C.c_int32(); nc = C.c_int32()
        L.dropin_search_by_bow(n, _p(kA), _p(A), _p(valid), _p(nodeA), n, _p(kB), _p(B), _p(nodeB), C.c_float(0.7), 1, _p(mg), C.byref(ng), _p(mc), C.byref(nc))
        assert ng.value == nc.value > 50
        assert np.array_equal(mg, mc)


def test_pose_optimization_on_reference_frame(oracle, dropin):
    cfg = config.lafida_450()
    L = dropin(cfg)
    for seed in (5, 6):
        q = synth.pose_problem(n=300, faceW=450, seed=seed, outlier_frac=0.15)
        # feed both sides only correspondences inside the field of view, so that the oracle (which takes its edges as given) sees the same edge set
        keep = _in_fov(oracle, cfg, q["kpxy"])
        q = dict(q, Xw=q["Xw"][keep], kpxy=q["kpxy"][keep], inv_sigma2=q["inv_sigma2"][keep])
        n = len(q["Xw"])
        octave = np.zeros(n, np.int32)
        T = np.ascontiguousarray(q["Tcw"], np.float32).copy(); out = np.zeros(n, np.uint8)
        w = np.ones(n, np.float32)
        inl = L.dropin_pose_optimization(n, _p(np.ascontiguousarray(q["kpxy"], np.float32)), _p(octave), _p(np.ascontiguousarray(q["Xw"], np.float32)), _p(T), _p(out))
        r = oracle.pose_opt(q["Tcw"], q["Xw"], q["kpxy"], w, 450, 450)
        assert inl == r["inliers"] and np.array_equal(out, r["outlier"])
        assert np.allclose(T.reshape(4, 4), r["Tcw"], atol=2e-6)


def test_local_bundle_adjustment_on_reference_map(oracle, dropin):
    """Optimizer::LocalBundleAdjustment(pKF, &stop, pMap) on a Map built with the reference's KeyFrame / MapPoint / Map API; every key frame is
    covisible with the current one (every point is seen by all 6), so the local window is the whole problem and equals the oracle's input."""
    cfg = config.lafida_450()
    L = dropin(cfg)
    p = synth.ba_problem(nKF=6, nMP=400, kmin=6, kmax=6, faceW=450, seed=21, radius=1.5)
    keep = _in_fov(oracle, cfg, p["kpxy"])
    for key in ("eMP", "eKF", "kpxy", "inv_sigma2"):
        p[key] = np.ascontiguousarray(p[key][keep])
    nKF, nMP, nE = 6, 400, len(p["eMP"])
    rng = np.random.default_rng(2)
    octave = rng.integers(0, 8, nE).astype(np.int32)
    inv_sigma2 = _inv_sigma2(octave)
    T = np.ascontiguousarray(p["Tcw"], np.float32).reshape(nKF, 16).copy(); pts = np.ascontiguousarray(p["pts"], np.float32).copy()
    erased = np.zeros(nE, np.uint8)
    window = L.dropin_local_ba(nKF, nMP, nE, _p(T), _p(pts), _p(p["eMP"]), _p(p["eKF"]), _p(np.ascontiguousarray(p["kpxy"], np.float32)), _p(octave), 3, _p(erased))
    assert window == nKF
    r = oracle.local_ba(p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], inv_sigma2, 450, 450)
    assert r["iters"] >= 5
    # MapPoint::EraseObservation (src/MapPoint.cpp:96-124) drops the whole point once two or fewer observations remain: the harness reports
    # IsInKeyFrame, so the expected mask is the oracle's outlier edges plus every edge of a point that fell to <= 2 observations
    out = r["outlier"].astype(bool)
    nobs = np.bincount(p["eMP"], minlength=nMP); nout = np.bincount(p["eMP"], weights=out, minlength=nMP).astype(np.int64)
    bad = (nout > 0) & (nobs - nout <= 2)
    assert out.sum() > 0
    assert np.array_equal(erased.astype(bool), out | bad[p["eMP"]])
    assert np.allclose(T.reshape(nKF, 4, 4), r["Tcw"], atol=2e-6) and np.allclose(pts, r["pts"], atol=2e-6)


@pytest.mark.parametrize("seed,th", [(0, 15.0), (1, 30.0)])
def test_search_by_projection_on_reference_frames(dropin, seed, th):
    """ORBMatcher(0.9, true).SearchByProjection(CurrentFrame, LastFrame, th, true) (src/Tracking.cpp:634) on reference Frame / MapPoint objects:
    the GPU drop-in and the reference's own CPU body, from identical starting states, leave identical mvpMapPoints and return the same count."""
    L = dropin(config.front_1024())
    s = synth.tracking_pair(seed, n=1500, faceW=650)
    nC, nL = len(s["kCur"]), len(s["kLast"])
    mg = np.zeros(nC, np.int32); mc = np.zeros(nC, np.int32); ng = C.c_int32(); nc = C.c_int32()
    arrs = [np.ascontiguousarray(s["kCur"]), np.ascontiguousarray(s["dCur"]), np.ascontiguousarray(s["TcwCur"], np.float32), np.ascontiguousarray(s["kLast"]),
            np.ascontiguousarray(s["TcwLast"], np.float32), np.ascontiguousarray(s["hasMP"]), np.ascontiguousarray(s["Xw"]), np.ascontiguousarray(s["dLast"]),
            np.ascontiguousarray(s["mpObs"], np.int32), np.ascontiguousarray(s["curTaken"])]
    L.dropin_search_by_projection_last(nC, _p(arrs[0]), _p(arrs[1]), _p(arrs[2]), nL, _p(arrs[3]), _p(arrs[4]), _p(arrs[5]), _p(arrs[6]), _p(arrs[7]), _p(arrs[8]), _p(arrs[9]),
                                       C.c_float(th), 1, _p(mg), C.byref(ng), _p(mc), C.byref(nc))
    assert ng.value == nc.value > 300
    assert np.array_equal(mg, mc)


@pytest.mark.parametrize("seed,th", [(0, 3.0), (1, 6.0)])
def test_fuse_on_reference_key_frames(dropin, seed, th):
    """ORBMatcher(0.6).Fuse(pKF, vpMapPoints, th) (src/LocalMapping.cpp:402,423) on reference KeyFrame / MapPoint objects: the GPU drop-in (search on
    the device, Replace / AddObservation bookkeeping through the reference's own methods) and the reference's CPU body leave identical maps."""
    L = dropin(config.front_1024())
    s = synth.mapping_pair(seed, n=1500, faceW=650)
    n = len(s["Xw"])
    a = [np.ascontiguousarray(s["kCur"]), np.ascontiguousarray(s["dCur"]), np.ascontiguousarray(s["TcwCur"], np.float32), np.ascontiguousarray(s["Xw"], np.float32),
         np.ascontiguousarray(s["kLast"]), np.ascontiguousarray(s["dLast"]), np.ascontiguousarray(s["TcwLast"], np.float32)]
    ig = np.zeros(n, np.int32); ic = np.zeros(n, np.int32); bg = np.zeros(n, np.uint8); bc = np.zeros(n, np.uint8); ng = C.c_int32(); nc = C.c_int32()
    L.dropin_fuse(len(a[0]), _p(a[0]), _p(a[1]), _p(a[2]), n, _p(a[3]), _p(a[4]), _p(a[5]), _p(a[6]), C.c_float(th), _p(ig), _p(bg), C.byref(ng), _p(ic), _p(bc), C.byref(nc))
    assert ng.value == nc.value > 150
    assert np.array_equal(ig, ic) and np.array_equal(bg, bc)


@pytest.mark.parametrize("seed,ori", [(0, False), (1, True)])
def test_search_for_triangulation_on_reference_key_frames(dropin, seed, ori):
    """ORBMatcher(0.6, false).SearchForTriangulation(pKF1, pKF2, E12, pairs) (src/LocalMapping.cpp:262): drop-in == the reference's CPU body."""
    L = dropin(config.front_1024())
    s = synth.mapping_pair(30 + seed, n=1500, faceW=650)
    n1, n2 = len(s["kCur"]), len(s["kLast"])
    a = [np.ascontiguousarray(s["kCur"]), np.ascontiguousarray(s["dCur"]), np.ascontiguousarray(s["TcwCur"], np.float32), np.ascontiguousarray(s["hasMPCur"]),
         np.ascontiguousarray(s["nodeCur"], np.int32), np.ascontiguousarray(s["kLast"]), np.ascontiguousarray(s["dLast"]), np.ascontiguousarray(s["TcwLast"], np.float32),
         np.ascontiguousarray(s["hasMPObs"]), np.ascontiguousarray(s["nodeObs"], np.int32), np.ascontiguousarray(s["E12"], np.float32)]
    mg = np.zeros(n1, np.int32); mc = np.zeros(n1, np.int32); ng = C.c_int32(); nc = C.c_int32()
    L.dropin_search_for_triangulation(n1, _p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), _p(a[4]), n2, _p(a[5]), _p(a[6]), _p(a[7]), _p(a[8]), _p(a[9]), _p(a[10]), int(ori), _p(mg),
                                      C.byref(ng), _p(mc), C.byref(nc))
    assert ng.value == nc.value > 100
    assert np.array_equal(mg, mc)


def test_batched_distinctive_descriptors_on_reference_map_points(dropin):
    """cubemap_b200::DistinctiveDescriptors (one launch for all MapPoints of a key frame) == MapPoint::ComputeDistinctiveDescriptors per point."""
    L = dropin(config.front_1024())
    rng = np.random.default_rng(3)
    P = 400; off = [0]; rows = []
    for p in range(P):
        N = int(rng.choice([0, 1, 2, 3, 5, 8, 12]))
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        for _ in range(N):
            rows.append(base ^ np.packbits(rng.random(256) < rng.uniform(0.0, 0.25), bitorder="little"))
        off.append(off[-1] + N)
    desc = np.ascontiguousarray(np.stack(rows)); off = np.array(off, np.int32); eq = np.zeros(P, np.uint8)
    L.dropin_distinctive_batch(P, _p(off), _p(desc), _p(eq))
    assert eq.all()


def test_global_bundle_adjustment_on_reference_map(oracle, dropin):
    """Optimizer::GlobalBundleAdjustemnt(pMap, 20) (src/Tracking.cpp:514, src/LoopClosing.cpp:649; body src/Optimizer.cpp:461-621) through the drop-in on a
    Map built with the reference's API == the oracle's LM with one optimize(20), robust kernel on, no outlier stage."""
    cfg = config.lafida_450()
    L = dropin(cfg)
    p = synth.ba_problem(nKF=7, nMP=350, kmin=3, kmax=7, faceW=450, seed=31, radius=1.5)
    keep = _in_fov(oracle, cfg, p["kpxy"])
    for key in ("eMP", "eKF", "kpxy", "inv_sigma2"):
        p[key] = np.ascontiguousarray(p[key][keep])
    nKF, nMP, nE = 7, 350, len(p["eMP"])
    rng = np.random.default_rng(4)
    octave = rng.integers(0, 8, nE).astype(np.int32)
    inv_sigma2 = _inv_sigma2(octave)
    T = np.ascontiguousarray(p["Tcw"], np.float32).reshape(nKF, 16).copy(); pts = np.ascontiguousarray(p["pts"], np.float32).copy()
    L.dropin_global_ba(nKF, nMP, nE, _p(T), _p(pts), _p(p["eMP"]), _p(p["eKF"]), _p(np.ascontiguousarray(p["kpxy"], np.float32)), _p(octave), 20)
    fixed = np.zeros(nKF, np.uint8); fixed[0] = 1                 # only mnId == 0 is fixed
    r = oracle.local_ba(p["Tcw"], fixed, p["pts"], p["eMP"], p["eKF"], p["kpxy"], inv_sigma2, 450, 450, its1=20, its2=0)
    assert r["iters"] >= 5
    seen = np.bincount(p["eMP"], minlength=nMP) > 0
    assert np.allclose(T.reshape(nKF, 4, 4), r["Tcw"], atol=2e-6) and np.allclose(pts[seen], r["pts"][seen], atol=2e-6)
    assert not np.allclose(T.reshape(nKF, 4, 4)[1:], p["Tcw"][1:], atol=1e-4)      # it did move the free key frames
