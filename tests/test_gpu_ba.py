"""GPU parity: LocalBundleAdjustment / PoseOptimization vs the fp64 CPU oracle. Tolerance (north_star): 1e-5 relative on the
fp64 pose / point state (before the float32 cast); outlier sets and the LM trajectory (iterations, accepted steps) equal."""
import os
import numpy as np
import pytest

from cubemapslam_b200 import synth

pytestmark = pytest.mark.gpu
RTOL = 1e-5


@pytest.fixture(scope="module")
def opt():
    from cubemapslam_b200.optimizer import Optimizer
    o = Optimizer()
    yield o
    o.close()


def rel(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30)


def _compare_ba(oracle, opt, p, **kw):
    r = oracle.local_ba(p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], p["faceW"], p["faceH"], **kw)
    g = opt.LocalBundleAdjustment(p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], p["faceW"], p["faceH"], **kw)
    assert g["iters"] == r["iters"], (g["iters"], r["iters"])
    assert np.array_equal(g["log"][:, 2:], r["log"][:, 2:])                       # trials / accepted per iteration
    assert np.allclose(g["log"][:, 0], r["log"][:, 0], rtol=1e-8)                 # chi2 trajectory
    assert rel(g["pose64"], r["pose64"]) < RTOL and rel(g["pts64"], r["pts64"]) < RTOL
    assert np.array_equal(g["outlier"], r["outlier"])
    assert np.allclose(g["Tcw"], r["Tcw"], atol=2e-6) and np.allclose(g["pts"], r["pts"], atol=2e-6)
    return r, g


def test_local_ba_small_all_faces(oracle, opt):
    p = synth.ba_problem(nKF=8, nMP=300, kmin=2, kmax=6, faceW=450, seed=11, radius=1.5)
    r, g = _compare_ba(oracle, opt, p)
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "ba_small.npz"))
    assert rel(g["pose64"], gold["pose64"]) < RTOL and np.array_equal(g["outlier"], gold["outlier"])


def test_local_ba_first_trial(oracle, opt):
    p = synth.ba_problem(nKF=5, nMP=60, kmin=2, kmax=5, faceW=450, seed=8, radius=1.5)
    _compare_ba(oracle, opt, p, its1=1, its2=0)


def test_local_ba_medium_with_fixed_cameras(oracle, opt):
    p = synth.ba_problem(nKF=20, nMP=3000, kmin=2, kmax=10, faceW=650, seed=5, radius=2.0)
    p["kf_fixed"][[0, 7, 13]] = 1                                   # lFixedCameras
    r, g = _compare_ba(oracle, opt, p)
    assert np.allclose(g["pose64"][[7, 13]], r["pose64"][[7, 13]], rtol=0, atol=1e-15)
    assert r["outlier"].mean() > 0.02


def test_local_ba_edge_cases(oracle, opt):
    p = synth.ba_problem(nKF=6, nMP=80, kmin=2, kmax=4, faceW=450, seed=2, radius=1.5)
    # a landmark without observations, a keyframe without observations, and a raised stop flag
    keep = (p["eMP"] != 3) & (p["eKF"] != 4)
    for k in ("eMP", "eKF", "kpxy", "inv_sigma2"):
        p[k] = p[k][keep]
    _compare_ba(oracle, opt, p)
    stop = np.ones(1, np.uint8)
    g = opt.LocalBundleAdjustment(p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], 450, 450, stop_flag=stop)
    assert g["iters"] == 0 and np.array_equal(g["pts"], p["pts"]) and not g["outlier"].any()


def _all_fixed_problem():
    p = synth.ba_problem(nKF=6, nMP=200, kmin=2, kmax=5, faceW=450, seed=21, radius=1.5)
    p["kf_fixed"][:] = 1
    return p


def test_local_ba_all_keyframes_fixed(oracle, opt):
    """Every key frame fixed: only the points are free, so an LM trial has no Schur complement and no reduced solve."""
    p = _all_fixed_problem()
    r, g = _compare_ba(oracle, opt, p)
    assert r["iters"] > 0 and not np.array_equal(g["pts"], p["pts"])


def test_local_ba_all_keyframes_fixed_off_face(oracle, opt):
    """An off-face key point in a problem without free poses is reported with the caller's edge index, like one with free poses."""
    p = _all_fixed_problem()
    perm = np.random.default_rng(3).permutation(len(p["eMP"]))
    q = {k: (np.ascontiguousarray(p[k][perm]) if k in ("eMP", "eKF", "kpxy", "inv_sigma2") else p[k]) for k in p}
    bad = q["kpxy"].copy(); bad[23] = (10.0, 10.0)    # top-left corner of the canvas: no face
    with pytest.raises(Exception, match="edge 23"):
        opt.LocalBundleAdjustment(q["Tcw"], q["kf_fixed"], q["pts"], q["eMP"], q["eKF"], bad, q["inv_sigma2"], 450, 450)


def test_local_ba_no_edges(oracle, opt):
    p = synth.ba_problem(nKF=4, nMP=50, kmin=2, kmax=4, faceW=450, seed=6, radius=1.5)
    p["eMP"] = p["eMP"][:0]; p["eKF"] = p["eKF"][:0]; p["kpxy"] = p["kpxy"][:0]; p["inv_sigma2"] = p["inv_sigma2"][:0]
    r, g = _compare_ba(oracle, opt, p)
    assert g["iters"] == 0 and g["outlier"].size == 0 and np.array_equal(g["pts"], p["pts"])


def test_pose_optimization_batch(oracle, opt):
    probs = [synth.pose_problem(n=n, faceW=450, seed=s, outlier_frac=0.15) for n, s in ((300, 5), (200, 6), (40, 7), (2, 8), (9, 9))]
    off = np.cumsum([0] + [len(q["Xw"]) for q in probs]).astype(np.int32)
    T = np.stack([q["Tcw"] for q in probs]); Xw = np.concatenate([q["Xw"] for q in probs]); kp = np.concatenate([q["kpxy"] for q in probs])
    w = np.concatenate([q["inv_sigma2"] for q in probs])
    g = opt.PoseOptimization(T, Xw, kp, w, 450, 450, offset=off)
    for i, q in enumerate(probs):
        r = oracle.pose_opt(q["Tcw"], q["Xw"], q["kpxy"], q["inv_sigma2"], 450, 450)
        assert g["inliers"][i] == r["inliers"], i
        assert np.array_equal(g["outlier"][off[i]:off[i + 1]], r["outlier"]), i
        if len(q["Xw"]) >= 3:
            assert rel(g["pose64"][i], r["pose64"]) < RTOL, i
            assert np.allclose(g["Tcw"][i], r["Tcw"], atol=2e-6)
        else:
            assert np.array_equal(g["Tcw"][i], q["Tcw"])                       # untouched (src/Optimizer.cpp:133-134)
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "ba_small.npz"))
    q = synth.pose_problem(n=200, faceW=450, seed=5)
    o = opt.PoseOptimization(q["Tcw"], q["Xw"], q["kpxy"], q["inv_sigma2"], 450, 450)
    assert o["inliers"] == int(gold["po_inliers"]) and rel(o["pose64"], gold["po_pose64"]) < RTOL


def test_config4_scale_properties(opt):
    """BASELINE config-4 size (50 KF x 20k points, ~170k edges): oracle-free properties - chi2 decreases monotonically over
    accepted LM steps, fixed KF 0 unchanged, planted outlier fraction recovered, result close to the planted truth."""
    p = synth.ba_problem()
    g = opt.LocalBundleAdjustment(p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], 650, 650)
    assert g["iters"] >= 5
    acc = g["log"][g["log"][:, 3] == 1][:, 0]
    e0 = np.linalg.norm(p["Tcw"][:, :3, 3] - p["Tcw_true"][:, :3, 3], axis=1).mean()
    e1 = np.linalg.norm(g["Tcw"][:, :3, 3] - p["Tcw_true"][:, :3, 3], axis=1).mean()
    assert e1 < 0.3 * e0 and 0.03 < g["outlier"].mean() < 0.09
    assert np.allclose(g["Tcw"][0], p["Tcw"][0], atol=1e-6)


def test_config4_vs_oracle(oracle, opt):
    """BASELINE config 4 at full size (50 KF x 20k MapPoints, ~180k cubemap edges, optimize(5)+optimize(10)) against the fp64 oracle:
    1e-5 relative gate on poses and points, identical LM log (trials / accepted per iteration) and identical outlier set."""
    p = synth.ba_problem()
    r, g = _compare_ba(oracle, opt, p)
    assert len(p["eMP"]) > 150000 and r["iters"] >= 5


def test_local_ba_edge_order_is_free(oracle, opt):
    """Edges may come in any order (the drop-in emits them per MapPoint, other callers may not): a shuffled edge list takes the host counting
    sort + device gather path and must give the same answer as the grouped list, flags returned in the caller's order. A key point on no cube
    face is reported as an error naming the caller's edge index (the reference calls exit() there, src/CamModelGeneral.cpp FaceInCubemap)."""
    p = synth.ba_problem(nKF=8, nMP=300, kmin=2, kmax=6, faceW=450, seed=13, radius=1.5)
    g0 = opt.LocalBundleAdjustment(p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], 450, 450)
    perm = np.random.default_rng(5).permutation(len(p["eMP"]))
    q = {k: (np.ascontiguousarray(p[k][perm]) if k in ("eMP", "eKF", "kpxy", "inv_sigma2") else p[k]) for k in p}
    g1 = opt.LocalBundleAdjustment(q["Tcw"], q["kf_fixed"], q["pts"], q["eMP"], q["eKF"], q["kpxy"], q["inv_sigma2"], 450, 450)
    r = oracle.local_ba(q["Tcw"], q["kf_fixed"], q["pts"], q["eMP"], q["eKF"], q["kpxy"], q["inv_sigma2"], 450, 450)
    assert g1["iters"] == g0["iters"] == r["iters"]
    assert np.array_equal(g1["outlier"], g0["outlier"][perm]) and np.array_equal(g1["outlier"], r["outlier"])
    # a stable sort by landmark restores the grouped order edge for edge only if the shuffle kept the per-landmark order; sums are reordered otherwise
    assert rel(g1["pose64"], g0["pose64"]) < 1e-9 and rel(g1["pts64"], g0["pts64"]) < 1e-9
    assert rel(g1["pose64"], r["pose64"]) < RTOL
    bad = q["kpxy"].copy(); bad[17] = (10.0, 10.0)    # top-left corner of the canvas: no face
    with pytest.raises(Exception, match="edge 17"):
        opt.LocalBundleAdjustment(q["Tcw"], q["kf_fixed"], q["pts"], q["eMP"], q["eKF"], bad, q["inv_sigma2"], 450, 450)
