"""GPU: PoseOptimization (host, logged and device-resident entries) and LocalBA's classification against the oracle on the scenes of
tests/pose_limits_scenes.py, at every face width. Exact: inliers, outlier flags, the LM log's trials / accepted columns; chi2 and lambda to
1e-8 relative; pose64 to 1e-5 relative, bit-identical on the stationary frames."""
import numpy as np
import pytest

from cubemapslam_b200._capi import CslamError, lib, ptr
from tests import pose_limits_scenes as S

pytestmark = pytest.mark.gpu
GARBAGE = 0xA5


@pytest.fixture(scope="module")
def opt():
    from cubemapslam_b200.optimizer import Optimizer
    o = Optimizer()
    yield o
    o.close()


def rel(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


@pytest.mark.parametrize("W", S.WIDTHS)
def test_pose_limits_batch(oracle, opt, W):
    named = S.all_frames(W)
    b = S.batch([q for _, q in named])
    g = opt.PoseOptimization(b["Tcw"], b["Xw"], b["kpxy"], b["inv_sigma2"], W, W, offset=b["offset"], log=True)
    off = b["offset"]
    for i, (name, q) in enumerate(named):
        r = oracle.pose_opt(q["Tcw"], q["Xw"], q["kpxy"], q["inv_sigma2"], W, W)
        m = len(r["log"])
        assert g["inliers"][i] == r["inliers"], name
        assert np.array_equal(g["outlier"][off[i]:off[i + 1]], r["outlier"]), name
        assert g["nlog"][i] == m and not g["log"][i, m:].any(), name
        assert np.array_equal(g["log"][i, :m, 2:], r["log"][:, 2:]), name
        assert np.allclose(g["log"][i, :m, :2], r["log"][:, :2], rtol=1e-8, atol=0, equal_nan=True), name
        assert rel(g["pose64"][i], r["pose64"]) < 1e-5, name
        if name.startswith("stationary"):
            assert np.array_equal(bits(g["pose64"][i]), bits(r["pose64"])) and np.array_equal(g["Tcw"][i], q["Tcw"]), name
    plain = opt.PoseOptimization(b["Tcw"], b["Xw"], b["kpxy"], b["inv_sigma2"], W, W, offset=b["offset"])     # the log is only a hook
    for k in ("inliers", "outlier", "pose64", "Tcw"):
        assert np.array_equal(bits(plain[k]), bits(g[k])), k


@pytest.mark.parametrize("W", S.WIDTHS)
def test_pose_limits_dev_equals_host(opt, W):
    """The device-resident entry, strided with garbage past every count, is bit-identical to the host entry."""
    import torch
    frames = [q for _, q in S.all_frames(W)]
    F = len(frames); stride = max(len(q["Xw"]) for q in frames) + 5
    count = np.array([len(q["Xw"]) for q in frames], np.int32)
    X = np.full((F, stride, 3), np.float32(GARBAGE)); kp = np.full((F, stride, 2), np.float32(-7.5)); w = np.full((F, stride), np.float32(3.0))
    for f, q in enumerate(frames):
        X[f, :count[f]], kp[f, :count[f]], w[f, :count[f]] = q["Xw"], q["kpxy"], q["inv_sigma2"]
    T0 = np.stack([q["Tcw"] for q in frames])
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8).copy()).cuda()
    d = dict(count=dev(count), T=dev(T0), X=dev(X), kp=dev(kp), w=dev(w), outl=dev(np.full((F, stride), GARBAGE, np.uint8)),
             inl=dev(np.full(F, -1, np.int32)))
    torch.cuda.synchronize()
    opt.pose_optimization_dev(F, stride, d["count"].data_ptr(), d["T"].data_ptr(), d["X"].data_ptr(), d["kp"].data_ptr(), d["w"].data_ptr(), W, W,
                              d["outl"].data_ptr(), d["inl"].data_ptr())
    opt.sync()
    Tg = d["T"].cpu().numpy().view(np.float32).reshape(F, 4, 4); outl = d["outl"].cpu().numpy().reshape(F, stride)
    inl = d["inl"].cpu().numpy().view(np.int32)
    b = S.batch(frames)
    h = opt.PoseOptimization(b["Tcw"], b["Xw"], b["kpxy"], b["inv_sigma2"], W, W, offset=b["offset"])
    assert np.array_equal(bits(h["Tcw"]), bits(Tg)) and np.array_equal(h["inliers"], inl)
    for f in range(F):
        assert np.array_equal(h["outlier"][b["offset"][f]:b["offset"][f + 1]], outl[f, :count[f]]), f
        assert (outl[f, count[f]:] == GARBAGE).all(), f


@pytest.mark.parametrize("W", S.WIDTHS)
def test_local_ba_classification(oracle, opt, W):
    p = S.local_ba_scene(W)
    args = (p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], W, W)
    r = oracle.local_ba(*args)
    g = opt.LocalBundleAdjustment(*args)
    assert np.array_equal(g["outlier"], p["expected"]) and np.array_equal(r["outlier"], p["expected"])
    assert g["iters"] == r["iters"] and np.array_equal(g["log"][:, 2:], r["log"][:, 2:])
    assert np.allclose(g["log"][:, :2], r["log"][:, :2], rtol=1e-8, atol=0)
    assert np.array_equal(bits(g["pts"]), bits(p["pts"])) and np.array_equal(bits(g["pts64"]), bits(r["pts64"]))


@pytest.mark.parametrize("entry", ["cslam_pose_optimization", "cslam_pose_optimization_log"])
def test_off_face_correspondence_is_rejected(opt, entry):
    """A key point on no face, in a frame the optimizer runs on, is CSLAM_E_BADARG naming the frame and the correspondence; nothing is written."""
    b = S.batch(S.off_face_batch(650))
    F, n = len(b["Tcw"]), int(b["offset"][-1])
    T = b["Tcw"].copy(); outl = np.full(n, GARBAGE, np.uint8); inl = np.full(F, -1, np.int32); p64 = np.full((F, 7), -2.0)
    lg = np.full((F, 40, 4), -3.0); nlog = np.full(F, -4, np.int32)
    extra = (ptr(lg), ptr(nlog)) if entry.endswith("_log") else ()
    rc = getattr(lib(), entry)(opt._h, F, ptr(b["offset"]), ptr(T), ptr(b["Xw"]), ptr(b["kpxy"]), ptr(b["inv_sigma2"]), 650, 650, ptr(outl), ptr(inl),
                               ptr(p64), *extra)
    assert rc != 0
    assert "frame 2, correspondence 17" in lib().cslam_last_error().decode()
    assert np.array_equal(T, b["Tcw"]) and (outl == GARBAGE).all() and (inl == -1).all() and (p64 == -2.0).all() and (lg == -3.0).all() and (nlog == -4).all()
    with pytest.raises(CslamError, match="frame 2.*correspondence 17"):
        opt.PoseOptimization(b["Tcw"], b["Xw"], b["kpxy"], b["inv_sigma2"], 650, 650, offset=b["offset"], log=entry.endswith("_log"))
    few = S.batch([S.frame(b["Xw"][[0, 1]], b["kpxy"][[0, 1]], [1, 1]), S.frame(b["Xw"][:2], np.float32([[10, 10], [20, 20]]), [1, 1])])
    g = opt.PoseOptimization(few["Tcw"], few["Xw"], few["kpxy"], few["inv_sigma2"], 650, 650, offset=few["offset"])
    assert (g["inliers"] == 0).all()             # frames of < 3 correspondences never evaluate an edge, as in the reference
