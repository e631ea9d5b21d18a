"""cslam_search_by_projection_local_large (Tracker.SearchByProjection_local_large) against the oracle, exactly, on local maps past 4096
MapPoints (tests/local_map_scenes.py): ragged batches up to CSLAM_LOCAL_MAP_MAX_POINTS, cslam_search_by_projection_local against the oracle up to
4096, every bad argument of both host entries, window capacity, and the drop-in ORBMatcher::SearchByProjection(F, vpMapPoints, th) on the
reference's own Frame / MapPoint objects up to 65 537 MapPoints."""
import ctypes as C
import os

import numpy as np
import pytest

from cubemapslam_b200 import config
from cubemapslam_b200._capi import CslamError, lib
from cubemapslam_b200.tracker import CSLAM_LOCAL_MAP_MAX_POINTS, Tracker
from oracle.oracle import KP_DTYPE, _p

from . import local_map_scenes as S

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NN = 0.8
BADARG, CAPACITY = -2, -4


@pytest.fixture(scope="module")
def trk():
    t = Tracker(max_frames=8, max_features=4096)
    yield t
    t.close()


def batch(counts, mp_stride, W, nlevels, seed, nkp=(4096,)):
    """One frame per count (key point counts cycling through nkp, garbage past them) and its map at mp_stride (garbage past each count)."""
    frames, maps = [], []
    for i, n in enumerate(counts):
        fr = S.frame(seed + i, W, nkp[i % len(nkp)], nlevels)
        frames.append(fr); maps.append(S.local_map(fr, min(max(n, 0), mp_stride), seed + 31 * i, mp_stride))
    fs = max(len(f["k"]) for f in frames)
    rng = np.random.default_rng(seed)
    k = np.zeros((len(frames), fs), KP_DTYPE); d = rng.integers(0, 256, (len(frames), fs, 32), dtype=np.uint8); taken = np.zeros((len(frames), fs), np.uint8)
    for i, f in enumerate(frames):
        m = len(f["k"]); k[i, :m] = f["k"]; d[i, :m] = f["d"]; taken[i, :m] = f["taken"]
        k[i, m:]["x"] = rng.uniform(0, 3 * W, fs - m); k[i, m:]["y"] = rng.uniform(0, 3 * W, fs - m); k[i, m:]["octave"] = rng.integers(0, nlevels, fs - m)
    st = {key: np.stack([mp[key] for mp in maps]) for key in maps[0]}
    nf = np.array([len(f["k"]) for f in frames], np.int32)
    return frames, maps, dict(k=k, d=d, taken=taken, nf=nf, nmp=np.array(counts, np.int32), **st)


def run_large(trk, B, W, th, nlevels, nn=NN):
    return trk.SearchByProjection_local_large(B["k"], B["d"], B["in_view"], B["proj"], B["level"], B["vcos"], B["dq"], B["obs"], B["taken"], W, W, th, nn, S.NLEVELS[nlevels],
                                              nlevels, nF=B["nf"], nMP=B["nmp"])


def check_against_oracle(oracle, frames, maps, B, nm, m, th, mp_stride):
    for i, (fr, mp) in enumerate(zip(frames, maps)):
        n = min(max(int(B["nmp"][i]), 0), mp_stride)
        on, om = S.oracle_search(oracle, fr, mp, n, th, NN)
        nf = len(fr["k"])
        assert nm[i] == on, (i, n, nm[i], on)
        assert np.array_equal(m[i, :nf], om), (i, n)
        assert (m[i, nf:] == -1).all()
        if n > 4096:
            assert (om >= 4096).any()


@pytest.mark.parametrize("W,nlevels,th", [(450, 8, 5.0), (650, 12, 1.0), (650, 8, 5.0), (450, 12, 1.0)])
def test_ragged_batch_equals_oracle(oracle, trk, W, nlevels, th):
    counts = [0, 1, 4095, 4096, 4097, 65536, 65537, 65541]   # the last: one past the stride (clamped)
    frames, maps, B = batch(counts, 65540, W, nlevels, 100 * W + nlevels, nkp=(4096, 3001))
    nm, m = run_large(trk, B, W, th, nlevels)
    check_against_oracle(oracle, frames, maps, B, nm, m, th, 65540)
    assert (m[6] >= 65536).any() or (m[5] >= 4096).any()


@pytest.mark.parametrize("W,th", [(450, 5.0), (650, 1.0)])
def test_largest_local_map(oracle, trk, W, th):
    counts = [CSLAM_LOCAL_MAP_MAX_POINTS, CSLAM_LOCAL_MAP_MAX_POINTS + 1, 70001]
    frames, maps, B = batch(counts, CSLAM_LOCAL_MAP_MAX_POINTS, W, 8, 7 * W)
    nm, m = run_large(trk, B, W, th, 8)
    check_against_oracle(oracle, frames, maps, B, nm, m, th, CSLAM_LOCAL_MAP_MAX_POINTS)
    assert (m[0] >= 65536).any()


@pytest.mark.parametrize("W,nlevels,th", [(450, 8, 5.0), (650, 12, 1.0), (650, 8, 5.0)])
def test_equals_existing_entry_up_to_4096(oracle, trk, W, nlevels, th):
    for counts in ([4096, 4000, 1, 0, 2048], [4096] * 3):
        frames, maps, B = batch(counts, 4096, W, nlevels, 300 + W + len(counts))
        B["nf"][:] = 4096
        nm, m = trk.SearchByProjection_local(B["k"], B["d"], B["in_view"], B["proj"], B["level"], B["vcos"], B["dq"], B["obs"], B["taken"], W, W, th, NN,
                                             S.NLEVELS[nlevels], nlevels, nF=B["nf"], nMP=B["nmp"])
        check_against_oracle(oracle, frames, maps, B, nm, m, th, 4096)
        assert nm.max() > 1000


def _call(trk, entry, B, nframes=None, f_stride=None, mp_stride=None, W=450, H=None, nlevels=8, null=None):
    P, fs = B["k"].shape
    ms = B["in_view"].shape[1]
    arrs = dict(k=B["k"], d=B["d"], nf=B["nf"], taken=B["taken"], nmp=B["nmp"], in_view=B["in_view"], proj=B["proj"], level=B["level"], vcos=B["vcos"], dq=B["dq"],
                obs=B["obs"])
    ptrs = {key: (None if key == null else _p(v)) for key, v in arrs.items()}
    match = np.full((P, fs), 12345, np.int32); nm = np.full(P, 777, np.int32)
    rc = getattr(lib(), entry)(trk._h, P if nframes is None else nframes, ptrs["k"], ptrs["d"], ptrs["nf"], fs if f_stride is None else f_stride, ptrs["taken"], ptrs["nmp"],
                               ms if mp_stride is None else mp_stride, ptrs["in_view"], ptrs["proj"], ptrs["level"], ptrs["vcos"], ptrs["dq"], ptrs["obs"], W,
                               W if H is None else H, C.c_float(5.0), C.c_float(NN), C.c_float(1.2), nlevels, None if null == "match" else _p(match),
                               None if null == "nm" else _p(nm))
    return rc, match, nm


def _bad_arguments_write_nothing(trk, entry, mp_max, stride):
    """Every bad argument of a host entry whose mp_stride bound is mp_max, on a batch of two frames with maps of 100 and `stride` MapPoints."""
    _, _, B = batch([100, stride], stride, 450, 8, 11)
    rc, m, nm = _call(trk, entry, B)
    assert rc == 0 and nm.max() > 0
    cases = [dict(nframes=0), dict(nframes=9), dict(f_stride=0), dict(f_stride=4097), dict(mp_stride=0), dict(mp_stride=mp_max + 1), dict(W=450, H=451),
             dict(W=0, H=0), dict(nlevels=0), dict(nlevels=17)] + [dict(null=key) for key in ("k", "d", "nf", "taken", "nmp", "in_view", "proj", "level", "vcos", "dq", "obs")]
    for c in cases:
        rc, m, nm = _call(trk, entry, B, **c)
        assert rc == BADARG, c
        assert (m == 12345).all() and (nm == 777).all(), c
    for lv in (-1, 8):   # an in-view row's level outside [0, nlevels)
        B2 = dict(B); B2["level"] = B["level"].copy(); B2["in_view"] = B["in_view"].copy()
        B2["level"][1, stride - 1] = lv; B2["in_view"][1, stride - 1] = 1
        rc, m, nm = _call(trk, entry, B2)
        assert rc == BADARG and (m == 12345).all() and (nm == 777).all(), lv
        B2["nmp"] = np.array([100, stride - 1], np.int32)   # the same row past the count is not read
        assert _call(trk, entry, B2)[0] == 0


def test_bad_arguments_write_nothing(trk):
    _bad_arguments_write_nothing(trk, "cslam_search_by_projection_local_large", CSLAM_LOCAL_MAP_MAX_POINTS, 5000)


def test_local_entry_bad_arguments_write_nothing(trk):
    """cslam_search_by_projection_local takes the checks of _large, with mp_stride bounded by the handle's max_features (4096)."""
    _bad_arguments_write_nothing(trk, "cslam_search_by_projection_local", 4096, 4000)


def test_window_capacity(trk):
    """A window of more than 256 candidates is CSLAM_E_CAPACITY, from both entries."""
    W = 450
    rng = np.random.default_rng(3)
    k = np.zeros(600, KP_DTYPE)
    k["x"] = rng.uniform(W + 100, W + 220, 600); k["y"] = rng.uniform(W + 100, W + 220, 600); k["octave"] = 7
    d = rng.integers(0, 256, (600, 32), dtype=np.uint8)
    one = lambda x: np.asarray(x)[None]   # noqa: E731
    args = (one(k), one(d), one([1]), one([[W + 160, W + 160]]).astype(np.float32), one([7]).astype(np.int32), one([0.5]).astype(np.float32), one(d[:1]), one([1]),
            one(np.zeros(600, np.uint8)), W, W, 5.0, NN)
    for fn in (trk.SearchByProjection_local_large, trk.SearchByProjection_local):
        with pytest.raises(CslamError, match="error %d" % CAPACITY):
            fn(*args)
    nm, _ = trk.SearchByProjection_local_large(*args[:-2], 1.0, NN)   # the handle is usable afterwards
    assert nm >= 0


# ------------------------------------------------------------------------------------------------ the drop-in on the reference's objects
LIB = os.path.join(ROOT, "oracle", "_ref", "libdropin_local_map.so")


@pytest.fixture
def dropin(oracle):
    if not os.path.exists(LIB):
        pytest.skip("oracle/_ref/libdropin_local_map.so is built where the reference tree exists")
    L = C.CDLL(LIB)
    L.dropin_set_camera(C.byref(oracle.cam_params(config.front_1024())))
    return L


@pytest.mark.parametrize("n", [3000, 4096, 4097, 20000, 65537])
def test_dropin_on_reference_objects(dropin, n):
    W = 650
    fr = S.frame(n, W)
    mp = S.local_map(fr, n, 2 * n)
    nk = len(fr["k"])
    for th in (1.0, 5.0):
        mg = np.zeros(nk, np.int32); mc = np.zeros(nk, np.int32); ng = C.c_int32(); nc = C.c_int32()
        obs = mp["obs"].astype(np.int32)
        dropin.dropin_search_by_projection_local(nk, _p(fr["k"]), _p(fr["d"]), n, _p(mp["in_view"]), _p(mp["proj"]), _p(mp["level"]), _p(mp["vcos"]), _p(mp["dq"]), _p(obs),
                                                 _p(fr["taken"]), C.c_float(th), C.c_float(NN), _p(mg), C.byref(ng), _p(mc), C.byref(nc))
        assert ng.value == nc.value > 0
        assert np.array_equal(mg, mc)
        if n > 4096:
            assert (mg >= 4096).any()
