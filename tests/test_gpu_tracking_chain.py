"""GPU parity of the device-resident tracking step against the oracle: frame index -> SearchByProjection(last frame) -> gather of the pose-only BA's
correspondences -> strided PoseOptimization, the pose-only BA at the sizes where its block reductions and schedule change, and the capacity edges
of the projection search (a 13-px cell with 16 / 17 passing key points, a window with 256 / 257 candidates)."""
import ctypes as C

import numpy as np
import pytest

from cubemapslam_b200 import synth
from cubemapslam_b200._capi import KP_DTYPE, CslamError, check, lib, ptr

pytestmark = pytest.mark.gpu

W = 650
RTOL = 1e-5
GARBAGE = 0xAB                       # fill byte of every row past a frame's count: a kernel that reads or writes past a count shows up


def cos_fov_th(fov_deg):
    """CamModelGeneral::SetCosFovTh (reference include/CamModelGeneral.h:224-229): float argument, double cos, float result."""
    a = np.float32(fov_deg) / np.float32(2) * (np.float32(3.1415926535897932384626) / np.float32(180))
    return np.float32(np.cos(np.float64(a)))


def level_tables():
    """mvScaleFactors / mvInvLevelSigma2 of an 8-level, 1.2 pyramid (reference src/ORBExtractor.cpp:388-402), float like the reference."""
    sc = np.ones(8, np.float32)
    for l in range(1, 8):
        sc[l] = sc[l - 1] * np.float32(1.2)
    return sc, (np.float32(1.0) / (sc * sc)).astype(np.float32)


def rel(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30)


def garbage(shape, dtype):
    dtype = np.dtype(dtype)
    return np.full(tuple(shape) + (dtype.itemsize,), GARBAGE, np.uint8).view(dtype)[..., 0].copy()


def to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8).copy()).cuda()


def from_dev(t, like):
    return t.cpu().numpy().view(like.dtype).reshape(like.shape)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


@pytest.fixture(scope="module")
def trk():
    from cubemapslam_b200.tracker import Tracker
    t = Tracker(max_frames=8, max_features=4096)
    yield t
    t.close()


@pytest.fixture(scope="module")
def opt():
    from cubemapslam_b200.optimizer import Optimizer
    o = Optimizer()
    yield o
    o.close()


# ------------------------------------------------------------------------------------------------ 1. chain parity
def pose_inputs_reference(match, kps, rays, Xw_last, inv_level_sigma2, cos_fov):
    """The correspondence loop of Optimizer::PoseOptimization (reference src/Optimizer.cpp:82-127): features in slot order, a feature whose
    ray leaves the field of view skipped (:84-86), only slots holding a MapPoint taken (:88-89; the orientation filter's cleared slots are
    NULL), the world point of that MapPoint (:118-121) and mvInvLevelSigma2[kp.octave] as the weight (:107)."""
    Xw, kp, w = [], [], []
    for i in range(len(kps)):
        if rays[i, 2] < cos_fov:
            continue
        if match[i] >= 0:
            Xw.append(Xw_last[match[i]]); kp.append((kps["x"][i], kps["y"][i])); w.append(inv_level_sigma2[kps["octave"][i]])
    return np.array(Xw, np.float32).reshape(-1, 3), np.array(kp, np.float32).reshape(-1, 2), np.array(w, np.float32)


def chain_pairs():
    """(pair, LastFrame count) of ragged sizes: an empty LastFrame, fewer than 3 correspondences, 9, 10 (the `< 10` rule), and large frames
    whose current frame nears the 4096 stride. 2 % of the current key points are turned by 90 degrees so that their matches land in a
    non-dominant rotation bin and the orientation filter clears them."""
    out = []
    for seed, n in ((20, 1000), (4, 2), (7, 16), (12, 26), (3, 1000), (2, 2500), (1, 3300), (0, 3500)):
        s = synth.tracking_pair(seed, n=n, faceW=W)
        turn = np.random.default_rng(seed).random(len(s["kCur"])) < 0.02
        s["kCur"]["angle"][turn] = np.mod(s["kCur"]["angle"][turn] + np.float32(90), np.float32(360))
        rng = np.random.default_rng(100 + seed)                 # the motion model's prediction is a little off
        T = s["TcwCur"].astype(np.float64)
        T[:3, :3] = synth._rodrigues(rng.normal(0, 0.003, 3)) @ T[:3, :3]; T[:3, 3] += rng.normal(0, 0.01, 3)
        s["TcwCur"] = T.astype(np.float32)
        s["curTaken"][:] = 0                                    # Tracking::TrackWithMotionModel clears mvpMapPoints first (src/Tracking.cpp:630)
        out.append((s, 0 if seed == 20 else n))
    return out


def test_tracking_chain_parity(oracle, trk, opt):
    """frame_index_dev -> search_by_projection_last_dev -> gather_pose_inputs_dev -> pose_optimization_dev over 8 ragged pairs, strides larger
    than every count, rows past each count filled with garbage; every stage against the oracle and the dev pose-only BA against the host entry."""
    import torch
    pairs = chain_pairs()
    P, cs, ls = len(pairs), 4096, 3600
    # a 170-degree lens (cosFovTh > 0): SearchByProjection tests the MapPoint's camera z unnormalised, PoseOptimization the key point's unit ray,
    # so some matched key points lie outside the field of view and the correspondence loop skips them
    cth = cos_fov_th(170.0)
    sc, invs2 = level_tables()
    kC, dC, taken = garbage((P, cs), KP_DTYPE), garbage((P, cs, 32), np.uint8), garbage((P, cs), np.uint8)
    kL, has, Xw, dL, obs = garbage((P, ls), KP_DTYPE), garbage((P, ls), np.uint8), garbage((P, ls, 3), np.float32), garbage((P, ls, 32), np.uint8), garbage((P, ls), np.uint8)
    nC, nL, T0 = np.zeros(P, np.int32), np.zeros(P, np.int32), np.zeros((P, 4, 4), np.float32)
    for f, (s, nl) in enumerate(pairs):
        nC[f] = len(s["kCur"]); nL[f] = nl; T0[f] = s["TcwCur"]
        kC[f, :nC[f]] = s["kCur"]; dC[f, :nC[f]] = s["dCur"]; taken[f, :nC[f]] = s["curTaken"]
        kL[f, :nl] = s["kLast"][:nl]; has[f, :nl] = s["hasMP"][:nl]; Xw[f, :nl] = s["Xw"][:nl]; dL[f, :nl] = s["dLast"][:nl]; obs[f, :nl] = s["mpObs"][:nl] > 0
    assert nC.max() > 3600 and nC.max() < cs and nL.max() < ls
    rays, cst, cid = garbage((P, cs, 3), np.float32), garbage((P, 12501), np.uint16), garbage((P, cs), np.uint16)
    match, nm = garbage((P, cs), np.int32), garbage((P,), np.int32)
    gX, gkp, gw, cnt = garbage((P, cs, 3), np.float32), garbage((P, cs, 2), np.float32), garbage((P, cs), np.float32), garbage((P,), np.int32)
    outl, inl = garbage((P, cs), np.uint8), garbage((P,), np.int32)
    d = {k: to_dev(v) for k, v in dict(kC=kC, dC=dC, taken=taken, kL=kL, has=has, Xw=Xw, dL=dL, obs=obs, nC=nC, nL=nL, T=T0, invs2=invs2, rays=rays, cst=cst,
                                      cid=cid, match=match, nm=nm, gX=gX, gkp=gkp, gw=gw, cnt=cnt, outl=outl, inl=inl).items()}
    a = {k: v.data_ptr() for k, v in d.items()}
    torch.cuda.synchronize()                                    # the handles' streams do not wait for torch's stream
    ts = torch.cuda.ExternalStream(trk.stream); os_ = torch.cuda.ExternalStream(opt.stream)
    trk.frame_index_dev(a["kC"], a["nC"], P, cs, W, W, a["rays"], a["cst"], a["cid"])
    trk.search_by_projection_last_dev(P, a["kC"], a["dC"], a["nC"], cs, a["cst"], a["cid"], a["taken"], a["T"], a["kL"], a["nL"], ls, a["has"], a["Xw"], a["dL"], a["obs"],
                                      W, W, cth, 15.0, 1, a["match"], a["nm"])
    trk.gather_pose_inputs_dev(P, a["match"], a["kC"], a["nC"], cs, a["rays"], cth, a["Xw"], ls, a["invs2"], a["gX"], a["gkp"], a["gw"], a["cnt"])
    os_.wait_stream(ts)
    opt.pose_optimization_dev(P, cs, a["cnt"], a["T"], a["gX"], a["gkp"], a["gw"], W, W, a["outl"], a["inl"])
    opt.sync(); trk.sync()
    match, nm, cnt = from_dev(d["match"], match), from_dev(d["nm"], nm), from_dev(d["cnt"], cnt)
    gX, gkp, gw = from_dev(d["gX"], gX), from_dev(d["gkp"], gkp), from_dev(d["gw"], gw)
    Tg, outl, inl = from_dev(d["T"], T0), from_dev(d["outl"], outl), from_dev(d["inl"], inl)

    refs, sizes = [], []
    for f, (s, nl) in enumerate(pairs):
        n = nC[f]
        g = oracle.FrameGrid(s["kCur"], W, W)
        nm_o, m_o = g.search_by_projection_last(s["dCur"], s["TcwCur"], sc, s["kLast"][:nl], s["hasMP"][:nl], s["Xw"][:nl], s["dLast"][:nl], s["mpObs"][:nl],
                                                s["curTaken"], cth, 15.0, True)
        assert nm[f] == nm_o and np.array_equal(np.where(match[f, :n] == -2, -1, match[f, :n]), m_o), f
        assert (bits(match[f, n:]) == GARBAGE).all(), f                 # nothing written past the count
        r_o, _ = oracle.key_point_rays(s["kCur"], W, W)
        X_o, kp_o, w_o = pose_inputs_reference(m_o, s["kCur"], r_o, s["Xw"], invs2, cth)
        c = len(X_o); sizes.append(c)
        assert cnt[f] == c, (f, cnt[f], c)
        assert np.array_equal(bits(gX[f, :c]), bits(X_o)) and np.array_equal(bits(gkp[f, :c]), bits(kp_o)) and np.array_equal(bits(gw[f, :c]), bits(w_o)), f
        assert (bits(gX[f, c:]) == GARBAGE).all() and (bits(gw[f, c:]) == GARBAGE).all(), f
        if nl >= 1000:                                                 # both skips of the correspondence loop are exercised
            assert ((m_o >= 0) & (r_o[:, 2] < cth)).sum() >= 1 and (match[f, :n] == -2).sum() >= 1, f
        r = oracle.pose_opt(s["TcwCur"], X_o, kp_o, w_o, W, W)
        refs.append(r)
        assert inl[f] == r["inliers"] and np.array_equal(outl[f, :c], r["outlier"]), f
        if c < 3:
            assert np.array_equal(bits(Tg[f]), bits(T0[f])), f               # returned untouched (src/Optimizer.cpp:133-134)
        else:
            assert np.allclose(Tg[f], r["Tcw"], atol=2e-6), f
    assert sizes[0] == 0 and 0 < sizes[1] < 3 and 3 <= sizes[2] < 10 and sizes[3] == 10 and min(sizes[4:]) > 300, sizes

    # the same kernel through the host entry on the gathered correspondences: bit-identical, and its fp64 pose within the 1e-5 gate
    off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    h = opt.PoseOptimization(T0, np.concatenate([gX[f, :cnt[f]] for f in range(P)]), np.concatenate([gkp[f, :cnt[f]] for f in range(P)]),
                             np.concatenate([gw[f, :cnt[f]] for f in range(P)]), W, W, offset=off)
    assert np.array_equal(bits(h["Tcw"]), bits(Tg)) and np.array_equal(h["inliers"], inl)
    for f in range(P):
        assert np.array_equal(h["outlier"][off[f]:off[f + 1]], outl[f, :cnt[f]]), f
        if cnt[f] >= 3:
            assert rel(h["pose64"][f], refs[f]["pose64"]) < RTOL, f


def test_pose_optimization_dev_count_past_stride(opt):
    """A frame of the strided form owns at most `stride` correspondences: a count past the stride is clamped and the frame never reads the
    next frame's rows. The gather never hands over such a count, so the rule is pinned here, against the host entry on the same rows."""
    import torch
    S = 300
    probs = [synth.pose_problem(n=S, faceW=W, seed=60 + i, outlier_frac=0.15, radius=1.5) for i in range(3)]
    count = np.array([S + 40, S, 200], np.int32)
    T0 = np.stack([q["Tcw"] for q in probs])
    X, kp, w = (np.stack([q[k] for q in probs]) for k in ("Xw", "kpxy", "inv_sigma2"))
    outl, inl = garbage((3, S), np.uint8), garbage((3,), np.int32)
    d = {k: to_dev(v) for k, v in dict(count=count, T=T0, X=X, kp=kp, w=w, outl=outl, inl=inl).items()}
    torch.cuda.synchronize()
    opt.pose_optimization_dev(3, S, d["count"].data_ptr(), d["T"].data_ptr(), d["X"].data_ptr(), d["kp"].data_ptr(), d["w"].data_ptr(), W, W, d["outl"].data_ptr(),
                              d["inl"].data_ptr())
    opt.sync()
    Tg, outl, inl = from_dev(d["T"], T0), from_dev(d["outl"], outl), from_dev(d["inl"], inl)
    n = np.minimum(count, S)
    off = np.concatenate([[0], np.cumsum(n)]).astype(np.int32)
    h = opt.PoseOptimization(T0, np.concatenate([X[f, :n[f]] for f in range(3)]), np.concatenate([kp[f, :n[f]] for f in range(3)]),
                             np.concatenate([w[f, :n[f]] for f in range(3)]), W, W, offset=off)
    assert np.array_equal(bits(h["Tcw"]), bits(Tg)) and np.array_equal(h["inliers"], inl)
    for f in range(3):
        assert np.array_equal(h["outlier"][off[f]:off[f + 1]], outl[f, :n[f]]), f


# ------------------------------------------------------------------------------------------------ 2. pose-only BA sizes and edges
SIZES = (3, 9, 10, 11, 255, 256, 257, 511, 512, 513, 1000, 2500, 4096)


def test_pose_optimization_size_sweep(oracle, opt):
    """One batched host call: sizes around the 256-thread CTA's strides and the `< 10` edge rule at three outlier rates, a frame that loses
    every edge after round 1 (later rounds have no active edge and restart from the prior) and a frame whose correspondences are all one point."""
    probs = [synth.pose_problem(n=n, faceW=W, seed=100 * k + j, outlier_frac=fr, radius=1.5) for k, fr in enumerate((0.0, 0.15, 0.5)) for j, n in enumerate(SIZES)]
    assert len({(int(x // W), int(y // W)) for x, y in probs[len(SIZES) - 1]["kpxy"]}) == 5      # observations on all five faces
    lost = synth.pose_problem(n=300, faceW=W, seed=31, outlier_frac=0.0, radius=1.5)
    T = lost["Tcw"].astype(np.float64)
    T[:3, :3] = synth._rodrigues(np.array([0.0, 1.5, 0.0])) @ T[:3, :3]                  # prior 86 degrees off: no edge survives round 1
    lost["Tcw"] = T.astype(np.float32)
    one = synth.pose_problem(n=40, faceW=W, seed=32, outlier_frac=0.0, radius=1.5)
    for k in ("Xw", "kpxy", "inv_sigma2"):
        one[k] = np.repeat(one[k][:1], 40, axis=0)                                          # rank-2 H: only lambda keeps the LDL^T positive
    probs += [lost, one]
    off = np.cumsum([0] + [len(q["Xw"]) for q in probs]).astype(np.int32)
    g = opt.PoseOptimization(np.stack([q["Tcw"] for q in probs]), np.concatenate([q["Xw"] for q in probs]), np.concatenate([q["kpxy"] for q in probs]),
                             np.concatenate([q["inv_sigma2"] for q in probs]), W, W, offset=off)
    for i, q in enumerate(probs):
        r = oracle.pose_opt(q["Tcw"], q["Xw"], q["kpxy"], q["inv_sigma2"], W, W)
        assert g["inliers"][i] == r["inliers"], (i, len(q["Xw"]))
        assert np.array_equal(g["outlier"][off[i]:off[i + 1]], r["outlier"]), (i, len(q["Xw"]))
        assert rel(g["pose64"][i], r["pose64"]) < RTOL, (i, len(q["Xw"]))
        assert np.allclose(g["Tcw"][i], r["Tcw"], atol=2e-6), (i, len(q["Xw"]))
    r = oracle.pose_opt(lost["Tcw"], lost["Xw"], lost["kpxy"], lost["inv_sigma2"], W, W)
    assert r["inliers"] == 0 and r["outlier"].all()
    assert g["inliers"][-2] == 0 and np.allclose(g["Tcw"][-2], lost["Tcw"], atol=1e-6)    # setEstimate(prior) at the top of every round (src/Optimizer.cpp:145)
    assert g["inliers"][-1] == 40 and np.isfinite(g["pose64"][-1]).all()


# ------------------------------------------------------------------------------------------------ 3. projection-search capacity
def flip(d, k, rng):
    m = np.zeros(256, bool); m[rng.choice(256, k, replace=False)] = True
    return d ^ np.packbits(m, bitorder="little")


NNRATIO = 0.8

# Both scenes search one MapPoint whose octave (mode 0) / predicted level (mode 1) is `octave`; both modes get the same window radius.
#   cell:   centre on the front face's right border, radius 7.5 px; the capacity is that of one 13-px cell of the right face, reached through
#           the seam rectangle (mode 0: th 7.5 at octave 0; mode 1: th 3, viewCos > 0.998 -> 2.5 * 3)
#   window: centre near the front face's lower right corner, radius 20 * 1.2^7 = 71.7 px; the candidates are spread over the front, right and
#           lower faces, three rectangles of the area table (mode 0: th 20 at octave 7; mode 1: th 5, viewCos <= 0.998 -> 4 * 5)
SCENES = {"cell": dict(uv=(1299.0, 975.0), octave=0, cap=16, th_last=7.5, th_local=3.0, vcos=0.9999, seed=1),
          "window": dict(uv=(1290.0, 1290.0), octave=7, cap=256, th_last=20.0, th_local=5.0, vcos=0.99, seed=2)}


def capacity_scene(oracle, edge, over):
    """CurrentFrame key points around one search window holding exactly `cap + over` candidates (checked against the oracle's
    GetFeaturesInArea in both modes), plus key points of the same cells that fail the level or the radius test and so do not count. The
    candidate the reference visits last has the best descriptor: a search that stopped early would pick another one."""
    s = dict(SCENES[edge]); u, v = s["uv"]; o = s["octave"]; sc, _ = level_tables()
    rng = np.random.default_rng(10 * s["seed"] + over)
    radius = np.float32(s["th_last"]) * sc[o]
    if edge == "cell":
        cell = [(1300.6 + 1.3 * i, 975.6 + 1.5 * j) for j in range(5) for i in range(5)]     # right face, cell column 0, row 25
        pts = [(1295.5, 970.0), (1297.0, 978.5), (1298.5, 973.0)] + cell[:s["cap"] + over]  # and 3 on the front face
        rest = [(1302.3, 984.0, 3), (1304.1, 985.5, 3), (1309.5, 978.0, 0), (1311.0, 983.0, 0)]  # same cell: wrong level / outside the window
    else:
        lat = [(u - radius + 3.25 + 6.5 * i, v - radius + 3.25 + 6.5 * j) for i in range(22) for j in range(22)]   # <= 4 per cell
        lat = [p for p in lat if max(abs(p[0] - u), abs(p[1] - v)) < radius - 0.5 and synth._pixel_to_ray(p[0], p[1], W) is not None]
        lat = [lat[i] for i in rng.permutation(len(lat))]
        pts = lat[:s["cap"] + over]
        rest = [(x, y, 2) for x, y in lat[s["cap"] + over:]]
        assert len({(int(x // W), int(y // W)) for x, y in pts}) == 3 and len(rest) >= 50
    k = np.zeros(len(pts) + len(rest), KP_DTYPE)
    k["x"] = [p[0] for p in pts] + [p[0] for p in rest]; k["y"] = [p[1] for p in pts] + [p[1] for p in rest]
    k["octave"] = [o] * len(pts) + [p[2] for p in rest]; k["size"] = 31; k["class_id"] = -1
    k = k[rng.permutation(len(k))]                              # candidates and non-candidates interleaved in slot order
    s["dq"] = rng.integers(0, 256, 32, dtype=np.uint8)
    s["d"] = np.stack([flip(s["dq"], int(rng.integers(30, 60)), rng) for _ in range(len(k))])
    s["Xw"] = (synth._pixel_to_ray(u, v, W) * 3.0).astype(np.float32)     # the LastFrame MapPoint, seen through TcwCur = identity
    uv, _ = oracle.ray_to_cubemap(s["Xw"], W, W)
    grid = oracle.FrameGrid(k, W, W)
    r_local = np.float32(2.5 if s["vcos"] > 0.998 else 4.0) * np.float32(s["th_local"]) * sc[o]
    assert r_local == radius
    last = grid.features_in_area(uv[0, 0], uv[0, 1], radius, o - 1, o + 1)      # src/ORBMatcher.cpp:179
    local = grid.features_in_area(u, v, radius, o - 1, o)                       # src/ORBMatcher.cpp:75
    assert len(last) == len(pts) and np.array_equal(last, local) and (k["octave"][last] == o).all()
    s["d"][last[-1]] = flip(s["dq"], 5, rng)
    s.update(k=k, best=int(last[-1]))
    return s


def search_local_dev(trk, s, a, match, nm):
    """cslam_search_by_projection_local_dev on device arrays (one frame, one MapPoint)."""
    return lib().cslam_search_by_projection_local_dev(trk._h, 1, ptr(a["k"]), ptr(a["d"]), ptr(a["n"]), len(s["k"]), ptr(a["cs"]), ptr(a["ci"]), ptr(a["taken"]),
                                                      ptr(a["one"]), 1, ptr(a["one8"]), ptr(a["proj"]), ptr(a["level"]), ptr(a["vcos"]), ptr(a["dq"]), ptr(a["one8"]),
                                                      W, W, C.c_float(s["th_local"]), C.c_float(NNRATIO), C.c_float(1.2), 8, ptr(match), ptr(nm))


def run_search(oracle, trk, s, mode, path):
    """One MapPoint searched in the scene: (GPU nmatches, GPU match, oracle nmatches, oracle match). Mode 0 (SearchByProjection_last) sees
    the MapPoint through TcwCur = identity; mode 1 (SearchByProjection_local) gets its projection, predicted level and viewing cosine."""
    import torch
    k, n = s["k"], len(s["k"])
    sc, _ = level_tables(); cth = cos_fov_th(190.0)
    taken = np.zeros(n, np.uint8); T = np.eye(4, dtype=np.float32)
    kl = np.zeros(1, KP_DTYPE); kl["octave"] = s["octave"]; kl["size"] = 31; kl["class_id"] = -1
    one8, one = np.ones(1, np.uint8), np.ones(1, np.int32)
    proj, lvl, vcos = np.array([s["uv"]], np.float32), np.array([s["octave"]], np.int32), np.array([s["vcos"]], np.float32)
    g = oracle.FrameGrid(k, W, W)
    if mode == "last":
        ref = g.search_by_projection_last(s["d"], T, sc, kl, one8, s["Xw"][None], s["dq"][None], one, taken, cth, s["th_last"], True)
    else:
        ref = g.search_by_projection_local(s["d"], sc, one8, proj, lvl, vcos, s["dq"][None], one, taken, s["th_local"], NNRATIO)
    if path == "host":
        if mode == "last":
            out = trk.SearchByProjection_last(k, s["d"], T, kl, one8, s["Xw"][None], s["dq"][None], one, taken, W, W, cth, s["th_last"], True)
        else:
            out = trk.SearchByProjection_local(k, s["d"], one8, proj, lvl, vcos, s["dq"][None], one, taken, W, W, s["th_local"], NNRATIO)
        return out + ref
    d = {key: to_dev(v) for key, v in dict(k=k, d=s["d"], n=np.array([n], np.int32), taken=taken, T=T, kl=kl, one8=one8, one=one, Xw=s["Xw"], dq=s["dq"], proj=proj,
                                          level=lvl, vcos=vcos, cs=np.zeros(12501, np.uint16), ci=np.zeros(n, np.uint16)).items()}
    a = {key: v.data_ptr() for key, v in d.items()}
    match, nm = to_dev(np.zeros(n, np.int32)), to_dev(np.zeros(1, np.int32))
    torch.cuda.synchronize()
    trk.frame_index_dev(a["k"], a["n"], 1, n, W, W, None, a["cs"], a["ci"])
    if mode == "last":
        trk.search_by_projection_last_dev(1, a["k"], a["d"], a["n"], n, a["cs"], a["ci"], a["taken"], a["T"], a["kl"], a["one"], 1, a["one8"], a["Xw"], a["dq"], a["one8"],
                                          W, W, cth, s["th_last"], 1, match.data_ptr(), nm.data_ptr())
    else:
        check(search_local_dev(trk, s, a, match.data_ptr(), nm.data_ptr()))
    trk.sync()                                                  # a window over capacity is reported here
    return (int(from_dev(nm, one)[0]), from_dev(match, np.zeros(n, np.int32))) + ref


@pytest.mark.parametrize("path", ["host", "dev"])
@pytest.mark.parametrize("mode", ["last", "local"])
@pytest.mark.parametrize("edge", ["cell", "window"])
def test_projection_search_capacity(oracle, trk, edge, mode, path):
    """At capacity the search equals the oracle; one more candidate is reported as CSLAM_E_CAPACITY (by the host entry, or by sync() after
    the _dev call), never truncated; the next call on the same handle succeeds, so the device error flag was cleared."""
    fit, over = capacity_scene(oracle, edge, 0), capacity_scene(oracle, edge, 1)
    for attempt in range(2):
        nm, m, nm_o, m_o = run_search(oracle, trk, fit, mode, path)
        assert nm == nm_o == 1 and m_o[fit["best"]] == 0 and np.array_equal(m, m_o), (attempt, nm, nm_o)
        if attempt == 0:
            with pytest.raises(CslamError, match="capacity"):
                run_search(oracle, trk, over, mode, path)
