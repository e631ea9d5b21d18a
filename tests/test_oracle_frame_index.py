"""oracle/frame_index.h (rays, 5x50x50 grid, GetFeaturesInArea with its cube-face wrap-around cases) == the reference's own Frame code
compiled in oracle/_ref/libref.so (src/Frame.cpp:158-176,251-716,728-760, include/CamModelGeneral.h:494-513); its answers are recorded for
where the library cannot be built (tests/refrecord.py)."""
import numpy as np
import pytest

from cubemapslam_b200 import config, synth

from oracle import ref
from tests import test_gpu_tracking_limits as L
from tests.refrecord import LIVE, RefRecord, same

REC = RefRecord("oracle_frame_index")


@pytest.fixture(scope="module", params=[("lafida", 450), ("front", 650)])
def frame(request, oracle):
    name, W = request.param
    if name == "lafida":
        cfg = config.lafida_450(); mask = config.load_mask("gray_lafida_cubemap_mask_450"); nf = 2000
    else:
        cfg = config.front_1024(); mask = np.full((1950, 1950), 255, np.uint8); nf = 3000      # full mask: features near every face seam
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    canvas = oracle.warp(cp, synth.fisheye_frame(cfg, 2), m1, m2)
    kps, _ = oracle.ORBextractor(nf, 1.2, 8, 20, 7, W, W)(canvas, mask)       # == the reference's extractor (test_oracle_ref.py)
    F = None
    if LIVE:
        r = ref.Ref(cp)
        F = ref.RefFrame(r.extractor(nf, 1.2, 8, 20, 7), canvas, mask)
    assert same(kps, REC(name + "/kps", lambda: F.kps, digest=(0,)))
    return name, W, kps, F


def test_rays_and_grid(oracle, frame):
    name, W, kps, F = frame
    rng = np.random.default_rng(0)
    cells = [(int(rng.integers(0, 5)), int(rng.integers(0, 50)), int(rng.integers(0, 50))) for _ in range(300)]

    def run():
        got = [F.grid_cell(f, c, r_) for f, c, r_ in cells]
        return F.rays, F.grid_count, np.concatenate(got), np.array([len(a) for a in got])
    rrays, rcount, rcells, rlens = REC(name + "/rays_and_grid", run, digest=(0, 1, 2, 3))
    rays, faces = oracle.key_point_rays(kps, W, W)
    assert same(rays, rrays)                                  # bit-exact unit bearing vectors
    g = oracle.FrameGrid(kps, W, W)
    start, idx = g.csr()
    counts = np.diff(start).reshape(5, 50, 50).astype(np.int32)
    assert len(idx) == len(kps) == counts.sum()
    assert same(counts, rcount)
    got = [idx[start[(f * 50 + c) * 50 + r_]:start[(f * 50 + c) * 50 + r_ + 1]].astype(np.int32) for f, c, r_ in cells]
    assert same(np.array([len(a) for a in got]), rlens) and same(np.concatenate(got), rcells)


def test_features_in_area_all_wraparound_cases(oracle, frame):
    name, W, kps, F = frame
    g = oracle.FrameGrid(kps, W, W)
    rng = np.random.default_rng(1)
    tiles = {0: (1, 1), 1: (0, 1), 2: (2, 1), 3: (1, 0), 4: (1, 2)}
    queries = []
    for face, (tc, tr) in tiles.items():
        for k in range(1500):
            # uniform in the face, with half of the samples pushed against an edge / a corner so that every overflow case is exercised
            u, v = rng.uniform(0, W, 2)
            mode = k % 4
            if mode >= 1:
                u = rng.choice([rng.uniform(0, 40), rng.uniform(W - 40, W - 0.01)])
            if mode >= 2:
                v = rng.choice([rng.uniform(0, 40), rng.uniform(W - 40, W - 0.01)])
            if mode == 3:
                u, v = v, u
            x = np.float32(tc * W + u); y = np.float32(tr * W + v)
            r = np.float32(rng.choice([7.0, 15.0, 15.0 * 1.728, 40.0, 75.0]))
            lv = int(rng.integers(0, 8)); lo, hi = [(-1, -1), (lv - 1, lv), (lv - 1, lv + 1), (0, 3)][k % 4]
            queries.append((x, y, r, lo, hi))
    queries.append((np.float32(10.0), np.float32(10.0), np.float32(30.0), -1, -1))     # a centre outside the five faces: nothing

    def run():
        got = [F.features_in_area(*q) for q in queries]
        return np.concatenate(got).astype(np.int32), np.array([len(b) for b in got])
    rall, rlens = REC(name + "/features_in_area", run, digest=(0, 1))
    got = [g.features_in_area(*q) for q in queries]
    lens = np.array([len(a) for a in got])
    assert same(lens, rlens) and same(np.concatenate(got).astype(np.int32), rall)
    assert lens[-1] == 0
    assert (lens[:-1] > 0).sum() > 0.2 * (len(queries) - 1)


@pytest.mark.parametrize("W,name,over", [(650, "front_cam_params", {}), (450, "lafida_cam0_params", {"CubeFace_w": 450, "CubeFace_h": 450}), (610, "front_cam_params", {"CubeFace_w": 610, "CubeFace_h": 610})])
def test_rays_and_grid_of_given_key_points(oracle, W, name, over):
    """The frames of tests/test_gpu_tracking_limits.py (seams, the float below each seam, cell edges, a 300-key-point cell, n = 0 / 257 /
    4096) through the reference's Frame: rays bit for bit, mGrid sizes and contents. Key points off the faces are left out here
    (ComputeKeyPointRays exits on them), and so are key points whose cell corner lies on another face (the debug build's PosInGrid asserts;
    x = 1949.9999 at W = 650 is one): the GPU file compares those with the oracle only."""
    cp = oracle.cam_params(config.camera(name, **over))
    r = ref.Ref(cp) if LIVE else None
    for i, (k, n) in enumerate(L.index_frames(W, with_off=False)):
        k = k[:min(n, 4096)]
        assert all(L.ref_safe(x, y, W) for x, y in zip(k["x"], k["y"])), i
        rrays, rcount, ridx = REC("given_%d_%d" % (W, i), lambda: r.frame_index(k), digest=(0, 1, 2))
        rays, _ = oracle.key_point_rays(k, W, W)
        start, idx = oracle.FrameGrid(k, W, W).csr()
        assert same(rays, rrays), i
        assert same(np.diff(start).reshape(5, 50, 50).astype(np.int32), rcount), i
        assert same(idx.astype(np.int32), ridx), i
