"""The oracle's SearchForInitialization (oracle/frame_index.h) against the reference's own body (ref_search_for_initialization in
oracle/ref_api.cpp, on reference Frames) on the scenes of tests/init_search_scenes.py, and GetFeaturesInArea against the reference at the
search's window (r = 100) and at r = W/2 for every face and overflow case at faces 333, 450 and 650. The reference's answers are recorded in
tests/golden/refcalls_oracle_init_search.npz, so the test also runs where oracle/_ref cannot be built."""
import numpy as np
import pytest

from oracle import init_search

from . import init_search_scenes as S
from .refrecord import LIVE, RefRecord, same

REC = RefRecord("oracle_init_search")


def _ref(oracle, W):
    return init_search.RefInit(oracle.cam_params(S.cam_cfg(W))) if LIVE else None


def check(oracle, r, key, scene, W, nn=0.9, ori=True):
    on, om, oxy = S.oracle_search(scene, W, 100, nn, ori)
    rn, rm, rxy = REC(key, lambda: r.search_for_initialization(*scene, 100, nn, ori), digest=(1, 2))
    assert on == rn and same(om, rm) and same(oxy, rxy), key
    return on, om, oxy


@pytest.mark.parametrize("W", sorted(S.EXTRACTED))
def test_extracted_frames(oracle, W):
    sc = S.extracted(oracle, W)
    assert len(sc[0]) > 0.75 * S.EXTRACTED[W]   # lafida's mask leaves about 80 % of 6000
    n, m, _ = check(oracle, _ref(oracle, W), "extracted_%d" % W, sc, W)
    assert n >= 100 and (m >= 0).sum() == n


@pytest.mark.parametrize("W", sorted(S.EXTRACTED))
def test_chain(oracle, W):
    """Tracking calls SearchForInitialization(mInitialFrame, mCurrentFrame, mvbPrevMatched, ...) frame after frame, carrying the centres."""
    r = _ref(oracle, W)
    views = S.chain(oracle, W)
    k1, d1 = views[0]
    xy = np.stack([k1["x"], k1["y"]], 1).astype(np.float32)
    for i, (k2, d2) in enumerate(views[1:]):
        n, m, xy = check(oracle, r, "chain_%d_%d" % (W, i), (k1, d1, k2, d2, xy), W)
        assert n >= 100


@pytest.mark.parametrize("W", (333, 650))
@pytest.mark.parametrize("n1,n2", [(3000, 4000), (16384, 16384), (0, 500), (500, 0)])
@pytest.mark.parametrize("ori", (True, False))
def test_dense(oracle, W, n1, n2, ori):
    sc = S.dense(n1 + n2 + W, W, n1, n2)
    n, m, _ = check(oracle, _ref(oracle, W), "dense_%d_%d_%d_%d" % (W, n1, n2, ori), sc, W, 0.9, ori)
    if n1 and n2:
        assert n > 10
        counts, _ = init_search.features_in_area(sc[2], W, [(x, y, 100.0, 0, 0) for x, y in sc[4][::25]])
        big = counts.max()
        assert big > 256   # windows past window_candidates' 256
        start, idx = oracle.FrameGrid(sc[2], W, W).csr()
        lv0 = np.zeros(len(start) - 1, np.int64)
        np.add.at(lv0, np.searchsorted(start, np.arange(len(idx)), side="right") - 1, sc[2]["octave"][idx] == 0)
        assert lv0.max() > 16   # 13-px cells past window_candidates' 16


def test_steal_changes_three_maxima(oracle):
    sc = S.steal()
    n, m, _ = check(oracle, _ref(oracle, 650), "steal", sc, 650)
    assert n == 4 and list(m) == [0, 1, 2, 3, -1, -1]
    n2, m2, _ = S.oracle_search(sc, 650, check_ori=False)
    assert n2 == 5 and m2[5] == 4 and m2[4] == -1   # without the filter q1 keeps X


@pytest.mark.parametrize("W", (333, 450, 650))
def test_features_in_area_at_the_search_window(oracle, W):
    rng = np.random.default_rng(W)
    sc = S.dense(W, W, 10, 6000)
    k2 = sc[2]
    queries = []
    for fx, fy in S.FACES:
        for k in range(240):
            u, v = rng.uniform(1, W - 1, 2)
            mode = k % 4   # inside, against an x edge, a y edge, a corner: every overflow case at r = 100 and W / 2
            if mode in (1, 3):
                u = rng.choice([rng.uniform(1, 60), rng.uniform(W - 60, W - 1)])
            if mode in (2, 3):
                v = rng.choice([rng.uniform(1, 60), rng.uniform(W - 60, W - 1)])
            r = 100.0 if k % 2 == 0 else W / 2.0
            lo, hi = (-1, -1) if k % 3 == 0 else (0, 0)
            queries.append((np.float32(fx * W + u), np.float32(fy * W + v), np.float32(r), lo, hi))
    queries.append((np.float32(W * 0.5), np.float32(W * 0.5), np.float32(100.0), 0, 0))   # a corner tile: nothing
    rc, ri = REC("area_%d" % W, lambda: _ref(oracle, W).features_in_area_given(k2, queries), digest=(0, 1))
    lens, idx = init_search.features_in_area(k2, W, queries)
    assert same(lens, rc) and same(idx, ri)
    assert lens[-1] == 0 and (lens > 256).any()
