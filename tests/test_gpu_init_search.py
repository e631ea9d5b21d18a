"""cslam_search_for_initialization (Tracker.SearchForInitialization) against the oracle, bit for bit, on every scene of
tests/init_search_scenes.py; the drop-in ORBMatcher::SearchForInitialization against the reference's own CPU body on the same reference
Frames (oracle/_ref/libdropin_init.so), including a chain of calls; bad arguments rejected before anything is enqueued."""
import ctypes as C
import os

import numpy as np
import pytest

from cubemapslam_b200._capi import CslamError, lib, ptr
from cubemapslam_b200.tracker import CSLAM_BOW_FV_MAX_FEATURES, Tracker
from oracle.oracle import KP_DTYPE, _p

from . import init_search_scenes as S

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BADARG = -2


@pytest.fixture(scope="module")
def trk():
    t = Tracker(max_frames=1, max_features=4096)   # the drop-in's handle: its max_features does not bound this entry
    yield t
    t.close()


def gpu_vs_oracle(oracle, trk, scene, W, nn=0.9, ori=True):
    k1, d1, k2, d2, xy = scene
    gn, gm, gxy = trk.SearchForInitialization(k1, d1, xy, k2, d2, W, W, 100, nn, ori)
    on, om, oxy = S.oracle_search(scene, W, 100, nn, ori)
    assert gn == on and np.array_equal(gm, om) and np.array_equal(gxy, oxy)
    return gn, gm, gxy


@pytest.mark.parametrize("W", sorted(S.EXTRACTED))
def test_extracted_frames(oracle, trk, W):
    n, _, _ = gpu_vs_oracle(oracle, trk, S.extracted(oracle, W), W)
    assert n >= 100


@pytest.mark.parametrize("W", sorted(S.EXTRACTED))
def test_chain(oracle, trk, W):
    views = S.chain(oracle, W)
    k1, d1 = views[0]
    xy = np.stack([k1["x"], k1["y"]], 1).astype(np.float32)
    for k2, d2 in views[1:]:
        _, _, xy = gpu_vs_oracle(oracle, trk, (k1, d1, k2, d2, xy), W)


@pytest.mark.parametrize("W", (333, 650))
@pytest.mark.parametrize("n1,n2", [(3000, 4000), (16384, 16384), (0, 500), (500, 0), (1, 1)])
@pytest.mark.parametrize("ori", (True, False))
def test_dense(oracle, trk, W, n1, n2, ori):
    gpu_vs_oracle(oracle, trk, S.dense(n1 + n2 + W, W, n1, n2), W, 0.9, ori)


@pytest.mark.parametrize("nn", (0.6, 0.9, 1.0))
def test_dense_ratios(oracle, trk, nn):
    gpu_vs_oracle(oracle, trk, S.dense(11, 450, 6024, 9024), 450, nn, True)


def test_steal_changes_three_maxima(oracle, trk):
    n, m, _ = gpu_vs_oracle(oracle, trk, S.steal(), 650)
    assert n == 4 and m[5] == -1


def test_bad_arguments(trk):
    k1, d1, k2, d2, xy = S.dense(3, 650, 200, 200)
    launches = trk.launches
    m = np.empty(len(k1), np.int32); nm = np.zeros(1, np.int32)

    def call(k1=k1, d1=d1, n1=len(k1), xy=xy, k2=k2, d2=d2, n2=len(k2), W=650, H=650, ws=100, match=m, nmp=nm):
        return lib().cslam_search_for_initialization(trk._h, ptr(k1), ptr(d1), n1, ptr(xy), ptr(k2), ptr(d2), n2, W, H, ws, C.c_float(0.9), 1, ptr(match), ptr(nmp))
    assert call() == 0
    launches = trk.launches
    big = np.zeros(CSLAM_BOW_FV_MAX_FEATURES + 1, KP_DTYPE)
    neg = k1.copy(); neg["octave"][7] = -1
    for kw in (dict(n1=-1), dict(n2=-1), dict(k1=big, n1=len(big)), dict(k2=big, n2=len(big)), dict(k1=None), dict(d1=None), dict(xy=None), dict(k2=None), dict(d2=None),
               dict(match=None), dict(nmp=None), dict(W=650, H=640), dict(W=0, H=0), dict(k1=neg), dict(ws=0), dict(ws=-5), dict(ws=326), dict(W=199, H=199)):
        assert call(**kw) == BADARG, kw
    assert trk.launches == launches
    with pytest.raises(CslamError):
        trk.SearchForInitialization(k1, d1, xy, k2, d2, 650, 650, 326)


def test_dropin_equals_reference_cpu_body(oracle):
    """The drop-in definition and the reference's body on the same reference Frames (extracted frames, a chain of calls, dense scenes)."""
    path = os.path.join(ROOT, "oracle", "_ref", "libdropin_init.so")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/libdropin_init.so is built only where the reference tree exists")
    L = C.CDLL(path)
    for W in (450, 650):
        L.dropin_set_camera(C.byref(oracle.cam_params(S.cam_cfg(W))))
        views = S.chain(oracle, W)
        k1, d1 = views[0]
        scenes = [S.dense(W, W, 6024, 9024), S.dense(W + 1, W, 16384, 16384), S.dense(W + 2, W, 0, 10), S.dense(W + 3, W, 10, 0)]
        xyg = np.stack([k1["x"], k1["y"]], 1).astype(np.float32); xyc = xyg.copy()
        runs = [(k1, d1, k2, d2, None) for k2, d2 in views[1:]] + scenes
        for i, (a1, b1, a2, b2, xy) in enumerate(runs):
            chained = xy is None
            if not chained:
                xyg = xy.copy(); xyc = xy.copy()
            n1 = len(a1)
            mg = np.zeros(n1, np.int32); mc = np.zeros(n1, np.int32); ng = C.c_int32(); nc = C.c_int32()
            L.dropin_search_for_initialization(n1, _p(np.ascontiguousarray(a1)), _p(np.ascontiguousarray(b1)), len(a2), _p(np.ascontiguousarray(a2)), _p(np.ascontiguousarray(b2)), 100,
                                               C.c_float(0.9), 1, _p(xyg), _p(mg), C.byref(ng), _p(xyc), _p(mc), C.byref(nc))
            assert ng.value == nc.value and np.array_equal(mg, mc) and np.array_equal(xyg, xyc), (W, i)
            if chained:
                assert ng.value >= 100
