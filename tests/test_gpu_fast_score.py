"""k_fast's arc score and NMS against the CPU oracle, bit for bit, at several FAST threshold pairs (tests marked gpu).

k_fast scores two pixels per u16 lane pair with the intensities in the high bytes of the lanes and the neighbouring pixels in the low bytes,
and stores (max(s, minThFAST) - minThFAST) << 8. These inputs make a wrong lane decode visible: ring pixels that tie in value while the
bytes next to them differ (stripes, checkerboards), saturated 0/255 regions (scores of 255, the largest the encoding holds), isolated
single-pixel spikes, and thresholds at both ends of the range. Candidates (x, y, response), key points and descriptors are compared on
caller canvases (every detection pixel scored) and on the warp path (only the live work items scored)."""
import os

import numpy as np
import pytest

from cubemapslam_b200 import _capi, config, synth

pytestmark = pytest.mark.gpu
NTHREADS = max(1, min(32, os.cpu_count() or 1))
THRESHOLDS = [(20, 7), (7, 7), (12, 1), (40, 0), (255, 254)]
FACE = 450
P = 40   # pattern patch edge


def _patch(kind, rng):
    yy, xx = np.mgrid[0:P, 0:P]
    if kind == 0:    # 1-px vertical stripes, 0/255
        return np.where(xx % 2 == 0, 0, 255)
    if kind == 1:    # period-3 stripes: two equal columns beside a different one
        return np.choose(xx % 3, [90, 90, 200])
    if kind == 2:    # 1-px checkerboard
        return np.where((xx + yy) % 2 == 0, 30, 230)
    if kind == 3:    # 2-px checkerboard with a saturated half
        return np.where(((xx // 2) + (yy // 2)) % 2 == 0, 0, np.where(xx < P // 2, 255, 128))
    if kind == 4:    # saturated blocks: 0 / 255 quadrants with a diagonal edge
        return np.where(xx + yy < P, 0, 255) ^ np.where((xx // 10 + yy // 10) % 2 == 0, 0, 255)
    if kind == 5:    # single-pixel spikes (0, 255, +-1) on a flat field
        p = np.full((P, P), 128)
        for v in (0, 255, 127, 129):
            p[rng.integers(3, P - 3, 6), rng.integers(3, P - 3, 6)] = v
        return p
    if kind == 6:    # sparse spikes on saturated fields: scores of exactly 255
        p = np.where(yy < P // 2, 255, 0)
        p[rng.integers(3, P // 2 - 3, 5), rng.integers(3, P - 3, 5)] = 0
        p[rng.integers(P // 2 + 3, P - 3, 5), rng.integers(3, P - 3, 5)] = 255
        return p
    return rng.choice(np.array([0, 1, 127, 128, 254, 255]), (P, P))   # few levels: many ties between ring pixels


def _stamp(img, origin, size, step, seed):
    """Pattern patches on a sparse grid of img (so the textured area stays within the candidate buffers)."""
    rng = np.random.default_rng(seed)
    y0, x0 = origin
    k = 0
    for y in range(y0, y0 + size - P, step):
        for x in range(x0, x0 + size - P, step):
            img[y:y + P, x:x + P] = _patch(k % 8, rng)
            k += 1
    return img


def _canvas(oracle, cp, maps, cfg, i):
    c = oracle.warp(cp, synth.fisheye_frame(cfg, i), *maps)
    c[:FACE, :FACE] = 60   # flat corner tile: scored on caller canvases, no corners
    return _stamp(c, (3 * i, FACE - 30 + 5 * i), 2 * FACE, 3 * P + 7, i)


def _orb(cfg, ini, mn):
    o = _capi.orb_params(cfg)
    o.ini_th_fast, o.min_th_fast = ini, mn
    return o


def _odd_width_level(cfg):
    """Some k_fast tile of the level pyramid has a detection width that is not a multiple of 4 (checked, not assumed)."""
    for l in range(int(cfg["ORBextractor.nLevels"])):
        side = int(np.rint(np.float32(3 * FACE) * (np.float32(1.0) / np.float32(np.float32(1.2) ** l))))
        minB, maxBX = 16, side - 16
        width = np.float32(maxBX - minB)
        nCols = int(width / np.float32(30))
        wCell = int(np.ceil(width / np.float32(nCols)))
        nColsEff = max(j + 1 for j in range(nCols) if not minB + j * wCell >= maxBX - 6)
        for cx in range(-(-nColsEff // 4)):
            tx0 = minB + cx * 4 * wCell
            nx = min(tx0 + min(4, nColsEff - 4 * cx) * wCell + 6, maxBX) - tx0 - 6
            if nx % 4:
                return True
    return False


@pytest.fixture(scope="module")
def geom(oracle):
    cfg = config.camera("lafida_cam0_params", CubeFace_w=FACE, CubeFace_h=FACE)
    cp = oracle.cam_params(cfg)
    return cfg, cp, oracle.build_maps(cp), np.full((3 * FACE, 3 * FACE), 255, np.uint8)


def _key(a):
    return a[np.lexsort((a[:, 0], a[:, 1]))]


@pytest.mark.parametrize("ini,mn", THRESHOLDS)
def test_caller_canvas(oracle, geom, ini, mn):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, cp, maps, mask = geom
    assert _odd_width_level(cfg)
    canv = np.stack([_canvas(oracle, cp, maps, cfg, i) for i in range(2)])
    fe = FrontEnd(cfg, mask, max_batch=2, orb=_orb(cfg, ini, mn))
    try:
        got = fe.extract(canv)
        for f in range(2):
            ex = oracle.ORBextractor(2000, 1.2, 8, ini, mn, FACE, FACE)
            kps, desc = ex(canv[f], mask)
            for l in range(8):
                c = ex.stage(l, 0)
                ref = np.stack([c["x"], c["y"], c["response"]], 1).astype(np.int32)
                g = fe.candidates(f, l)
                assert len(g) == len(ref), "(%d,%d) canvas %d level %d: %d candidates vs %d" % (ini, mn, f, l, len(g), len(ref))
                assert np.array_equal(_key(g), _key(ref)), "(%d,%d) canvas %d level %d candidates" % (ini, mn, f, l)
            gk, gd = got[f]
            assert len(gk) == len(kps), "(%d,%d) canvas %d: %d key points vs %d" % (ini, mn, f, len(gk), len(kps))
            assert np.array_equal(gk.view(np.uint8), kps.view(np.uint8)) and np.array_equal(gd, desc), "(%d,%d) canvas %d" % (ini, mn, f)
    finally:
        fe.close()


@pytest.mark.parametrize("ini,mn", THRESHOLDS)
def test_warp_path(oracle, geom, ini, mn):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, cp, maps, mask = geom
    Iw, Ih = int(cfg["Camera.Iw"]), int(cfg["Camera.Ih"])
    frames = np.stack([_stamp(synth.fisheye_frame(cfg, i).copy(), (Ih // 4 + 9 * i, Iw // 4 + 5 * i), min(Iw, Ih) // 2, 2 * P + 5, 10 + i)
                       for i in range(2)]).astype(np.uint8)
    fe = FrontEnd(cfg, mask, max_batch=2, orb=_orb(cfg, ini, mn))
    try:
        got = fe.run(frames)
        rk, rd, rn = oracle.warp_extract_batch_out(cp, frames, maps[0], maps[1], mask, 2000, 1.2, 8, ini, mn, NTHREADS, fe.kp_cap)
        for f in range(2):
            ex = oracle.ORBextractor(2000, 1.2, 8, ini, mn, FACE, FACE)
            ex(oracle.warp(cp, frames[f], *maps), mask)
            for l in range(8):
                c = ex.stage(l, 0)
                ref = np.stack([c["x"], c["y"], c["response"]], 1).astype(np.int32)
                assert np.array_equal(_key(fe.candidates(f, l)), _key(ref)), "(%d,%d) frame %d level %d candidates" % (ini, mn, f, l)
            gk, gd = got[f]
            assert len(gk) == rn[f], "(%d,%d) frame %d: %d key points vs %d" % (ini, mn, f, len(gk), rn[f])
            assert np.array_equal(gk.view(np.uint8), rk[f, :rn[f]].view(np.uint8)) and np.array_equal(gd, rd[f, :rn[f]]), "(%d,%d) frame %d" % (ini, mn, f)
    finally:
        fe.close()
