"""GPU parity of k_pyramid and k_describe against the CPU oracle, bit for bit (tests marked gpu).

k_pyramid reads each CTA's source rows as one window described at create time; windows wider than the small instantiation's bound
(scale factors above about 1.4) run the wide one. k_describe runs one warp per output slot and finds its level and kept-list slot from
the frame's kept counts. Level sizes here include widths that are not multiples of 4 and heights that are not multiples of 8."""
import numpy as np
import pytest

from cubemapslam_b200 import config, synth

pytestmark = pytest.mark.gpu

BATCHES = (1, 3, 13)


def _cfg(geom, face, scale, nlevels, nfeatures=None):
    kw = {"CubeFace_w": face, "CubeFace_h": face, "ORBextractor_scaleFactor": scale, "ORBextractor_nLevels": nlevels}
    if nfeatures is not None:
        kw["ORBextractor_nFeatures"] = nfeatures
    if geom == "front":   # the benchmark's 1280 x 1024 sensor
        return config.camera("front_cam_params", Camera_Ih=1024, Camera_v0=512.0, **kw)
    return config.camera("lafida_cam0_params", **kw)


def _fe(cfg, max_batch):
    from cubemapslam_b200.frontend import FrontEnd
    face = int(cfg["CubeFace.w"])
    return FrontEnd(cfg, np.full((3 * face, 3 * face), 255, np.uint8), max_batch=max_batch)


def _chain(oracle, level0, fe, f):
    """Every level of frame f against the oracle's resize_linear chain from level0."""
    lvl = level0
    assert np.array_equal(fe.level_image(f, 0), lvl)
    for l in range(1, fe.nlevels):
        h, w = fe.level_image(f, l).shape
        lvl = oracle.resize_linear(lvl, w, h)
        assert np.array_equal(fe.level_image(f, l), lvl), "frame %d level %d (%dx%d)" % (f, l, w, h)


PYR_CASES = [("front", 650, 1.2, 8), ("front", 650, 1.5, 7), ("front", 650, 2.0, 5),
             ("lafida", 450, 1.5, 6), ("lafida", 333, 1.2, 8), ("lafida", 333, 2.0, 4)]


def test_pyramid_cases_cover_ragged_levels():
    """Some level of the cases has a width that is not a multiple of 4 and a height that is not a multiple of 8."""
    ragged = False
    for _, face, s, nl in PYR_CASES:
        for l in range(1, nl):
            n = int(np.rint(np.float32(3 * face) * np.float32(1.0 / np.float32(s) ** l)))
            ragged |= n % 4 != 0 and n % 8 != 0
    assert ragged


@pytest.mark.parametrize("geom,face,scale,nlevels", PYR_CASES)
def test_pyramid_warp_path(oracle, geom, face, scale, nlevels):
    cfg = _cfg(geom, face, scale, nlevels)
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in range(max(BATCHES))])
    fe = _fe(cfg, max(BATCHES))
    try:
        for b in BATCHES:
            fe.run(frames[-b:])
            for f in range(b):
                _chain(oracle, oracle.warp(cp, frames[len(frames) - b + f], m1, m2), fe, f)
    finally:
        fe.close()


@pytest.mark.parametrize("scale,nlevels", [(1.2, 8), (2.0, 4)])
def test_pyramid_caller_canvas_then_warp(oracle, scale, nlevels):
    """Caller canvases (textured corners) build every level from the whole canvas; a warp-path run afterwards sees zeroed corners."""
    cfg = _cfg("lafida", 333, scale, nlevels)
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    rng = np.random.default_rng(1)
    canv = np.stack([oracle.warp(cp, synth.fisheye_frame(cfg, i), m1, m2) for i in range(3)])
    canv[:, :333, :333] = rng.integers(0, 256, (3, 333, 333), dtype=np.uint8)
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in (4, 5, 6)])
    fe = _fe(cfg, 3)
    try:
        fe.extract(canv)
        for f in range(3):
            _chain(oracle, canv[f], fe, f)
        fe.run(frames)
        for f in range(3):
            _chain(oracle, oracle.warp(cp, frames[f], m1, m2), fe, f)
    finally:
        fe.close()


@pytest.mark.parametrize("geom,face,scale,nlevels,nfeatures", [
    ("lafida", 450, 1.2, 8, 300),     # short per-level lists
    ("front", 650, 1.2, 8, 5000),     # long per-level lists
    ("front", 650, 1.5, 7, 3000),
    ("lafida", 333, 2.0, 4, 1000),
])
def test_keypoints_and_descriptors(oracle, geom, face, scale, nlevels, nfeatures):
    cfg = _cfg(geom, face, scale, nlevels, nfeatures)
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    mask = np.full((3 * face, 3 * face), 255, np.uint8)
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in range(3)])
    fe = _fe(cfg, 3)
    ex = oracle.ORBextractor(nfeatures, scale, nlevels, 20, 7, face, face)
    try:
        res = fe.run(frames)
        for f in range(3):
            kps, desc = ex(oracle.warp(cp, frames[f], m1, m2), mask)
            gk, gd = res[f]
            assert len(gk) == len(kps) > 0, "frame %d: %d vs %d key points" % (f, len(gk), len(kps))
            assert np.array_equal(gk.view(np.uint8), kps.view(np.uint8)), "key points, frame %d" % f
            assert np.array_equal(gd, desc), "descriptors, frame %d" % f
    finally:
        fe.close()


def test_blank_frame_then_textured(oracle):
    """A blank frame keeps no key point on any level (every k_describe warp exits); the next frame is complete again."""
    cfg = _cfg("lafida", 450, 1.2, 8)
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    fe = _fe(cfg, 2)
    try:
        frames = np.stack([np.zeros((cp.Ih, cp.Iw), np.uint8), synth.fisheye_frame(cfg, 2)])
        (k0, d0), (k1, d1) = fe.run(frames)
        assert len(k0) == 0 and d0.shape == (0, 32)
        rk, rd = oracle.ORBextractor(2000, 1.2, 8, 20, 7, 450, 450)(oracle.warp(cp, frames[1], m1, m2), np.full((1350, 1350), 255, np.uint8))
        assert np.array_equal(k1.view(np.uint8), rk.view(np.uint8)) and np.array_equal(d1, rd)
    finally:
        fe.close()
