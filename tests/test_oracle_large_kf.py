"""The oracle's SearchByBoW (both forms) and SearchForTriangulation against the compiled reference at 4097, 6024 and 9024 features per key frame,
the sizes of the initialisation extractor's key frames that the _fv entries take. SearchByBoW runs the reference's CPU body on its own KeyFrame /
Frame / MapPoint objects (oracle/_ref/libdropin_large.so, no GPU needed); SearchForTriangulation runs through libref.so. The reference's answers
are recorded in tests/golden/refcalls_oracle_large_kf.npz, so the test also runs where oracle/_ref cannot be built."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import ref
from oracle.oracle import _p

from . import large_kf_scenes as S
from .refrecord import RefRecord

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LARGE = os.path.join(ROOT, "oracle", "_ref", "libdropin_large.so")
REC = RefRecord("oracle_large_kf")


def _ref_bow(kfkf, s, nnratio, ori):
    L = C.CDLL(LARGE)
    n1, n2 = len(s["d1"]), len(s["d2"])
    k1, k2 = S.key_points(s["a1"]), S.key_points(s["a2"])
    m = np.zeros(n2 if not kfkf else n1, np.int32)
    n = L.ref_search_by_bow_cpu(int(kfkf), n1, _p(k1), _p(s["d1"]), _p(s["v1"]), _p(s["node1"]), n2, _p(k2), _p(s["d2"]), _p(s["v2"]), _p(s["node2"]),
                                C.c_float(nnratio), int(ori), _p(m))
    return n, m


@pytest.mark.parametrize("n", S.SIZES)
@pytest.mark.parametrize("kfkf", [0, 1])
def test_search_by_bow_oracle_vs_reference(oracle, n, kfkf):
    for seed, n2, ratio, ori in ((n, n, 0.7, True), (n + 1, n - 1000, 0.75, False)):
        s = S.bow_pair(n, n2, seed)
        rn, rm = REC("bow%d_%d_%d" % (kfkf, n, seed), lambda: _ref_bow(kfkf, s, ratio, ori))
        o1, o2 = S.oracle_nodes(s["node1"], 0), S.oracle_nodes(s["node2"], 1)
        if kfkf:
            on, om = oracle.search_by_bow_kf(s["d1"], s["a1"], s["v1"], o1, s["d2"], s["a2"], s["v2"], o2, ratio, ori)
        else:
            on, om = oracle.search_by_bow(s["d1"], s["a1"], s["v1"], o1, s["d2"], s["a2"], o2, ratio, ori)
        assert on == rn > 200 and np.array_equal(om, rm)
        if n >= 6024:   # matches with a feature index past 4095
            assert ((om >= 4096) | ((np.arange(len(om)) >= 4096) & (om >= 0))).sum() > 50


@pytest.mark.parametrize("n", S.SIZES)
def test_search_for_triangulation_oracle_vs_reference(oracle, n):
    from cubemapslam_b200 import config
    s = S.mapping_pair(n, 50 + n)
    cut = lambda a: np.ascontiguousarray(a[:n])   # noqa: E731 - KF1 = the current frame's first n key points
    k1, d1, h1, nd1 = cut(s["kCur"]), cut(s["dCur"]), cut(s["hasMPCur"]), cut(s["nodeCur"])
    k2, d2, h2, nd2 = s["kLast"], s["dLast"], s["hasMPObs"], s["nodeObs"]
    T1 = s["TcwCur"].astype(np.float64); Ow = (-T1[:3, :3].T @ T1[:3, 3]).astype(np.float32)
    for ori in (False, True):
        def live():
            r = ref.Ref(oracle.cam_params(config.front_1024()))
            rn, rm, _ = r.search_for_triangulation(k1, d1, s["TcwCur"], h1, nd1, k2, d2, s["TcwLast"], h2, nd2, s["E12"], ori)
            return rn, rm
        rn, rm = REC("tri_%d_%d" % (n, ori), live)
        r1, _ = oracle.key_point_rays(k1, 650, 650); r2, _ = oracle.key_point_rays(k2, 650, 650)
        on, om = oracle.search_for_triangulation(k1, d1, r1, h1, nd1, k2, d2, r2, h2, nd2, Ow, s["TcwLast"], s["E12"], s["scale"], s["level_sigma2"], 650, 650, ori)
        assert on == rn > 100 and np.array_equal(om, rm)
        if n >= 6024:   # KF1 and KF2 indices past 4095
            assert (om[4096:] >= 0).sum() > 50 and (om >= 4096).sum() > 50
