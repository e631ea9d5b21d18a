"""The host entry points stage their inputs, outputs and scratch in their handle's device arena (common.cuh DevArena), which keeps its chunks
across calls. Host calls of changing size on one handle (large, small, large), interleaved with the device-pointer forms on the same handle,
must give the bytes the device-pointer forms give on the same inputs, and the limits a handle is created with still bound its host calls."""
import numpy as np
import pytest

from cubemapslam_b200 import synth
from cubemapslam_b200._capi import KP_DTYPE, CslamError, check, lib, ptr

pytestmark = pytest.mark.gpu

BADARG = "error -2:"


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def empty(shape, dtype):
    import torch
    return torch.empty(shape, dtype=dtype, device="cuda")


def host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def keypoints(rng, n, W=650):
    k = np.zeros(n, KP_DTYPE)
    k["x"] = rng.uniform(0, 3 * W, n); k["y"] = rng.uniform(0, 3 * W, n); k["angle"] = rng.uniform(0, 360, n); k["octave"] = rng.integers(0, 8, n)
    return k


def test_matcher_host_calls_match_the_device_forms():
    import torch
    from cubemapslam_b200.matcher import ORBMatcher
    m = ORBMatcher(0.6, True, max_pairs=4, max_features=2048)
    rng = np.random.default_rng(0)
    try:
        for n in (1800, 300, 2000):
            A, aA, B, aB, perm = synth.descriptor_pair(n, n=n)
            # all-pairs matcher (row-split launch for n > 256)
            hn, hm, hd, hs = m.match_bruteforce(A, aA, B, aB)
            dA, daA, dB, daB = dev(A), dev(aA), dev(B), dev(aB)
            match, dist, sec, nm = empty(n, torch.int32), empty(n, torch.int32), empty(n, torch.int32), empty(1, torch.int32)
            torch.cuda.synchronize()
            m.match_bruteforce_dev(dA.data_ptr(), daA.data_ptr(), n, dB.data_ptr(), daB.data_ptr(), n, 1, match.data_ptr(), nm.data_ptr(), dist12=dist.data_ptr(),
                                   second12=sec.data_ptr())
            m.sync()
            assert hn == host(nm)[0] and hn > 0
            assert np.array_equal(hm, host(match)) and np.array_equal(hd, host(dist)) and np.array_equal(hs, host(sec))
            # consecutive frames of a ragged batch in the front end's layout
            F = 3
            kps = np.zeros((F, n), KP_DTYPE); desc = np.zeros((F, n, 32), np.uint8); cnt = np.array([n, n - 17, n // 2], np.int32)
            for f in range(F):
                src, ang = (B, aB) if f % 2 else (A, aA)
                kps[f, :cnt[f]] = keypoints(rng, cnt[f]); kps[f, :cnt[f]]["angle"] = ang[:cnt[f]]; desc[f, :cnt[f]] = src[:cnt[f]]
            hnm, hmatch = m.match_frames(kps, desc, cnt)
            dk, dd, dn = dev(kps.view(np.uint8)), dev(desc), dev(cnt)
            match, nm = empty((F - 1, n), torch.int32), empty(F - 1, torch.int32)
            torch.cuda.synchronize()
            m.match_frames_dev(dk.data_ptr(), dd.data_ptr(), dn.data_ptr(), n, F, match.data_ptr(), nm.data_ptr())
            m.sync()
            gm = host(match)
            assert np.array_equal(hnm, host(nm)) and hnm.min() > 0
            for f in range(F - 1):
                assert np.array_equal(hmatch[f, :cnt[f]], gm[f, :cnt[f]]), (n, f)
            # SearchByBoW(KeyFrame, Frame)
            nodeA = rng.integers(0, 60, n).astype(np.int32); nodeB = nodeA[perm]; valid = (rng.random(n) < 0.9).astype(np.uint8)
            hb, hmf = m.SearchByBoW(A, aA, valid, nodeA, B, aB, nodeB)
            dv, dnA, dnB = dev(valid), dev(nodeA), dev(nodeB)
            mf, nm = empty(n, torch.int32), empty(1, torch.int32)
            torch.cuda.synchronize()
            m.search_by_bow_dev(dA.data_ptr(), daA.data_ptr(), dv.data_ptr(), dnA.data_ptr(), n, dB.data_ptr(), daB.data_ptr(), dnB.data_ptr(), n, 1, mf.data_ptr(), nm.data_ptr())
            m.sync()
            assert hb == host(nm)[0] and hb > 0 and np.array_equal(hmf, host(mf))
    finally:
        m.close()


def test_tracker_host_calls_match_the_device_forms():
    import torch
    from cubemapslam_b200.tracker import NCELLS, Tracker
    trk = Tracker(max_frames=2, max_features=4096)
    cth = np.float32(np.cos(np.deg2rad(95.0)))
    try:
        for i, n in enumerate((1500, 300, 1800)):
            s = synth.tracking_pair(30 + i, n=n, faceW=650)
            kC, kL = s["kCur"], s["kLast"]; nc, nl = len(kC), len(kL)
            # frame index: rays and the cell CSR (cell_idx holds the key points that lie on a face)
            rays, cs, ci = trk.frame_index(kC, 650, 650)
            dk, dn = dev(kC.view(np.uint8)), dev(np.array([nc], np.int32))
            drays, dcs, dci = empty((nc, 3), torch.float32), empty(NCELLS + 1, torch.int16), empty(nc, torch.int16)
            torch.cuda.synchronize()
            trk.frame_index_dev(dk.data_ptr(), dn.data_ptr(), 1, nc, 650, 650, drays.data_ptr(), dcs.data_ptr(), dci.data_ptr())
            trk.sync()
            gcs = host(dcs).view(np.uint16)
            assert np.array_equal(rays, host(drays)) and np.array_equal(cs, gcs) and 0 < cs[-1] <= nc
            assert np.array_equal(ci[:cs[-1]], host(dci).view(np.uint16)[:cs[-1]])
            # SearchByProjection(Frame&, const Frame&): the host call builds the frame index itself
            obs = (s["mpObs"] > 0).astype(np.uint8)
            hn, hm = trk.SearchByProjection_last(kC, s["dCur"], s["TcwCur"], kL, s["hasMP"], s["Xw"], s["dLast"], obs, s["curTaken"], 650, 650, cth, 15.0, True)
            dd, dt, dT, dkl, dnl, dh, dX, dm, do = (dev(s["dCur"]), dev(s["curTaken"]), dev(s["TcwCur"].astype(np.float32)), dev(kL.view(np.uint8)), dev(np.array([nl], np.int32)),
                                                    dev(s["hasMP"]), dev(s["Xw"].astype(np.float32)), dev(s["dLast"]), dev(obs))
            match, nm = empty(nc, torch.int32), empty(1, torch.int32)
            torch.cuda.synchronize()
            trk.frame_index_dev(dk.data_ptr(), dn.data_ptr(), 1, nc, 650, 650, None, dcs.data_ptr(), dci.data_ptr())
            trk.search_by_projection_last_dev(1, dk.data_ptr(), dd.data_ptr(), dn.data_ptr(), nc, dcs.data_ptr(), dci.data_ptr(), dt.data_ptr(), dT.data_ptr(), dkl.data_ptr(),
                                              dnl.data_ptr(), nl, dh.data_ptr(), dX.data_ptr(), dm.data_ptr(), do.data_ptr(), 650, 650, cth, 15.0, 1, match.data_ptr(), nm.data_ptr())
            trk.sync()
            assert hn == host(nm)[0] and hn > 20 and np.array_equal(hm, host(match))
    finally:
        trk.close()


def test_vocabulary_host_transform_matches_the_device_form():
    import torch
    from cubemapslam_b200.vocabulary import Vocabulary
    voc = synth.vocabulary(k=10, L=4, seed=3)
    gv = Vocabulary(10, 4, voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"], max_frames=2, max_features=2048)
    rng = np.random.default_rng(3)
    leaves = np.nonzero(voc["is_leaf"])[0]
    try:
        for stride in (2000, 300, 2048):
            cnt = np.array([stride, stride // 3], np.int32)
            d = voc["desc"][rng.choice(leaves, (2, stride))] ^ np.packbits(rng.random((2, stride, 256)) < 0.05, axis=2, bitorder="little")
            res = gv.transform(d, n=cnt, levelsup=2)
            dd, dn = dev(d), dev(cnt)
            word, leaf, node, bw = (empty((2, stride), torch.int32) for _ in range(4))
            bv, bc = empty((2, stride), torch.float64), empty(2, torch.int32)
            torch.cuda.synchronize()
            check(lib().cslam_bow_transform_dev(gv._h, ptr(dd.data_ptr()), ptr(dn.data_ptr()), stride, 2, 2, ptr(word.data_ptr()), ptr(leaf.data_ptr()), ptr(node.data_ptr()),
                                                ptr(bw.data_ptr()), ptr(bv.data_ptr()), ptr(bc.data_ptr())))
            check(lib().cslam_vocabulary_sync(gv._h))
            gw, gn, gbw, gbv, gbc = host(word), host(node), host(bw), host(bv), host(bc)
            for f in range(2):
                hw, hn, hbw, hbv = res[f]
                c = gbc[f]
                assert c > 0 and np.array_equal(hw, gw[f, :cnt[f]]) and np.array_equal(hn, gn[f, :cnt[f]])
                assert np.array_equal(hbw, gbw[f, :c]) and np.array_equal(hbv.view(np.uint64), gbv[f, :c].view(np.uint64))
    finally:
        gv.close()


def _triangulation_inputs(oracle, P, seed):
    ss = [synth.mapping_pair(seed + p, n=900 + 150 * p, faceW=650) for p in range(P)]
    s1 = max(len(s["kCur"]) for s in ss); s2 = max(len(s["kLast"]) for s in ss)
    k1 = np.zeros((P, s1), KP_DTYPE); d1 = np.zeros((P, s1, 32), np.uint8); r1 = np.zeros((P, s1, 3), np.float32); h1 = np.zeros((P, s1), np.uint8); nd1 = np.zeros((P, s1), np.int32)
    k2 = np.zeros((P, s2), KP_DTYPE); d2 = np.zeros((P, s2, 32), np.uint8); r2 = np.zeros((P, s2, 3), np.float32); h2 = np.zeros((P, s2), np.uint8); nd2 = np.zeros((P, s2), np.int32)
    n1 = np.zeros(P, np.int32); n2 = np.zeros(P, np.int32); Ow = np.zeros((P, 3), np.float32); T2 = np.zeros((P, 16), np.float32); E = np.zeros((P, 9), np.float32)
    for p, s in enumerate(ss):
        a, b = len(s["kCur"]), len(s["kLast"]); n1[p] = a; n2[p] = b
        k1[p, :a] = s["kCur"]; d1[p, :a] = s["dCur"]; r1[p, :a] = oracle.key_point_rays(s["kCur"], 650, 650)[0]; h1[p, :a] = s["hasMPCur"]; nd1[p, :a] = s["nodeCur"]
        k2[p, :b] = s["kLast"]; d2[p, :b] = s["dLast"]; r2[p, :b] = oracle.key_point_rays(s["kLast"], 650, 650)[0]; h2[p, :b] = s["hasMPObs"]; nd2[p, :b] = s["nodeObs"]
        T1 = s["TcwCur"].astype(np.float64)
        Ow[p] = (-T1[:3, :3].T @ T1[:3, 3]).astype(np.float32); T2[p] = s["TcwLast"].reshape(16); E[p] = s["E12"].reshape(9)
    return (k1, d1, r1, h1, nd1, n1, k2, d2, r2, h2, nd2, n2, Ow, T2, E, ss[0]["scale"], ss[0]["level_sigma2"], 650, 650, True), n1


def test_mapper_host_calls_on_one_handle_match_fresh_handles(oracle):
    from cubemapslam_b200.mapper import Mapper
    rng = np.random.default_rng(4)
    calls = []
    for i, (P, n, pairs) in enumerate(((3000, 1800, 4), (200, 300, 1), (4000, 2000, 5))):
        nobs = rng.integers(0, 40, P); off = np.concatenate([[0], np.cumsum(nobs)]).astype(np.int32)
        desc = rng.integers(0, 256, (int(off[-1]), 32), dtype=np.uint8)
        s = synth.mapping_pair(50 + i, n=n, faceW=650)
        nm = len(s["Xw"])
        valid = (rng.random(nm) < 0.9).astype(np.uint8); level = np.clip(s["kLast"]["octave"] + rng.integers(-1, 2, nm), 0, 7).astype(np.int32)
        fuse = (s["kCur"], s["dCur"], s["TcwCur"], valid, s["Xw"], level, s["dLast"], 3.0, s["scale"], s["inv_level_sigma2"], 650, 650)
        tri, n1 = _triangulation_inputs(oracle, pairs, 60 + 10 * i)
        calls.append((desc, off, fuse, tri, n1))

    def run(m, c):
        desc, off, fuse, tri, n1 = c
        tn, tm = m.SearchForTriangulation(*tri)
        return [m.ComputeDistinctiveDescriptors(desc, off), *m.FuseSearch(*fuse), tn] + [tm[p, :n1[p]] for p in range(len(n1))]

    shared = Mapper()
    try:
        for c in calls:
            got = run(shared, c)
            fresh = Mapper()
            try:
                want = run(fresh, c)
            finally:
                fresh.close()
            assert len(got) == len(want) and all(np.array_equal(g, w) for g, w in zip(got, want))
            assert (got[0] >= 0).sum() > 100 and got[3].sum() > 0
    finally:
        shared.close()


def test_pose_optimization_host_calls_on_one_handle_match_fresh_handles():
    from cubemapslam_b200.optimizer import Optimizer
    probs = [synth.pose_problem(n=n, seed=s) for n, s in ((600, 1), (80, 2), (900, 3))]

    def run(o, p):
        r = o.PoseOptimization(p["Tcw"], p["Xw"], p["kpxy"], p["inv_sigma2"], p["faceW"], p["faceH"])
        return [np.asarray(r["inliers"]), r["Tcw"], r["outlier"], r["pose64"]]

    shared = Optimizer()
    try:
        for p in probs:
            got = run(shared, p)
            fresh = Optimizer()
            try:
                want = run(fresh, p)
            finally:
                fresh.close()
            assert got[0] > 0 and all(np.array_equal(g, w) for g, w in zip(got, want))
    finally:
        shared.close()


def test_host_calls_above_the_create_time_limits_are_bad_arguments():
    from cubemapslam_b200.mapper import Mapper
    from cubemapslam_b200.matcher import ORBMatcher
    from cubemapslam_b200.tracker import Tracker
    from cubemapslam_b200.vocabulary import Vocabulary
    rng = np.random.default_rng(5)
    n = 300
    A, aA, B, aB, _ = synth.descriptor_pair(0, n=n)
    node = np.zeros(n, np.int32); valid = np.ones(n, np.uint8); kps = keypoints(rng, n)
    m = ORBMatcher(max_pairs=2, max_features=256)
    try:
        for call in (lambda: m.match_bruteforce(A, aA, B, aB), lambda: m.SearchByBoW(A, aA, valid, node, B, aB, node),
                     lambda: m.SearchByBoW_KF(A, aA, valid, node, B, aB, valid, node), lambda: m.DescriptorDistance(np.tile(A, (2, 1)), np.tile(B, (2, 1))),
                     lambda: m.match_frames(np.stack([kps[:200]] * 3), np.stack([A[:200]] * 3), np.full(3, 200, np.int32))):
            with pytest.raises(CslamError, match=BADARG):
                call()
        assert m.match_bruteforce(A[:256], aA[:256], B[:256], aB[:256])[0] > 0   # at the limits
    finally:
        m.close()
    trk = Tracker(max_frames=1, max_features=64)
    try:
        T = np.eye(4, dtype=np.float32); xyz = np.zeros((n, 3), np.float32)
        for call in (lambda: trk.frame_index(kps, 650, 650),
                     lambda: trk.SearchByProjection_last(kps, A, T, kps[:10], valid[:10], xyz[:10], A[:10], valid[:10], valid, 650, 650, 0.0, 15.0),
                     lambda: trk.SearchByProjection_local(kps[:10], A[:10], valid, np.zeros((n, 2), np.float32), node, np.ones(n, np.float32), A, valid, valid[:10],
                                                          650, 650, 1.0, 0.8)):
            with pytest.raises(CslamError, match=BADARG):
                call()
    finally:
        trk.close()
    voc = synth.vocabulary(k=6, L=3, seed=1)
    gv = Vocabulary(6, 3, voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"], max_frames=1, max_features=64)
    try:
        with pytest.raises(CslamError, match=BADARG):
            gv.transform(A[:100])
        with pytest.raises(CslamError, match=BADARG):
            gv.transform(np.stack([A[:10]] * 2))
    finally:
        gv.close()
    mp = Mapper()   # no create-time limits: at most 4096 key points per key frame
    try:
        big = keypoints(rng, 4097); bigd = np.zeros((4097, 32), np.uint8)
        with pytest.raises(CslamError, match=BADARG):
            mp.FuseSearch(big, bigd, np.eye(4, dtype=np.float32), valid, xyz, node, A, 3.0, np.ones(8, np.float32), np.ones(8, np.float32), 650, 650)
    finally:
        mp.close()
