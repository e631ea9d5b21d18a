"""GPU parity of k_fast's live work-item lists against the CPU oracle, bit for bit (tests marked gpu).

On the warp path k_fast scores only the 4-pixel work items that hold a pixel whose 7x7 window is not all one static class: the black canvas
corners (0) or the face pixels outside the image circle, whose warp map is (0, 0) and which therefore all hold the frame's S(0, 0), on every
pyramid level. These tests make S(0, 0) differ from 0 so that the two classes differ and the borders between them carry texture, and compare
key points, descriptors and the bench pipeline's matches with the oracle's warp + extract at several geometries and batch sizes."""
import math
import os

import numpy as np
import pytest

from cubemapslam_b200 import config, synth

pytestmark = pytest.mark.gpu
NTHREADS = max(1, min(32, os.cpu_count() or 1))


def _cfg(geom, face):
    if geom == "front":   # the benchmark's 1280 x 1024 sensor (config.front_1024) at another face size
        return config.camera("front_cam_params", Camera_Ih=1024, Camera_v0=512.0, CubeFace_w=face, CubeFace_h=face)
    return config.camera("lafida_cam0_params", CubeFace_w=face, CubeFace_h=face)


def _mask(cfg):
    face = int(cfg["CubeFace.w"])
    return np.full((3 * face, 3 * face), 255, np.uint8)


def _unmasked(cfg, i, s00):
    """A recipe frame whose region outside the image circle is textured too (another recipe frame, shifted by half the sensor), S(0,0) = s00."""
    Iw, Ih = int(cfg["Camera.Iw"]), int(cfg["Camera.Ih"])
    invp = [cfg.get("Camera.pol%d" % k, 0.0) for k in range(int(cfg["Camera.nrinvpol"]))]
    fov = cfg["Camera.fov"] / 2.0 * math.pi / 180.0
    rho = synth._horner(invp, math.atan(-math.cos(fov) / math.sin(fov)))
    yy, xx = np.mgrid[0:Ih, 0:Iw]
    inside = (xx - cfg["Camera.u0"]) ** 2 + (yy - cfg["Camera.v0"]) ** 2 <= rho ** 2
    img = np.where(inside, synth.fisheye_frame(cfg, i), np.roll(synth.fisheye_frame(cfg, i + 50), (Ih // 2, Iw // 2), (0, 1))).astype(np.uint8)
    img[0, 0] = s00
    return img


def _reference(oracle, cfg, fe, frames, mask):
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    o = fe.orb
    return oracle.warp_extract_batch_out(cp, frames, m1, m2, mask, o.nfeatures, o.scale_factor, o.nlevels, o.ini_th_fast, o.min_th_fast,
                                         NTHREADS, fe.kp_cap)


def _check(got, ref, frames, what):
    rk, rd, rn = ref
    for i in range(len(frames)):
        gk, gd = got[i]
        assert len(gk) == rn[i], "%s frame %d: %d key points vs %d" % (what, i, len(gk), rn[i])
        assert np.array_equal(gk.view(np.uint8), rk[i, :rn[i]].view(np.uint8)), "%s frame %d key points" % (what, i)
        assert np.array_equal(gd, rd[i, :rn[i]]), "%s frame %d descriptors" % (what, i)


def test_bench_frames_and_matches(oracle):
    """The benchmark's frames (zero outside the image circle, so S(0,0) = 0), its mask, and the checkOri matches of consecutive frames."""
    from cubemapslam_b200.frontend import FrontEnd
    from cubemapslam_b200.matcher import ORBMatcher
    cfg = config.front_1024()
    mask = config.load_mask("gray_cubemap_front_mask_650")
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in range(6)])
    assert (frames[:, 0, 0] == 0).all()
    fe = FrontEnd(cfg, mask, max_batch=6)
    mt = ORBMatcher(0.6, True, max_pairs=8, max_features=fe.kp_cap)
    try:
        rk, rd, rn = ref = _reference(oracle, cfg, fe, frames, mask)
        kps = np.empty_like(rk); desc = np.empty_like(rd); n = np.empty_like(rn)
        fe.run_raw(frames, kps, desc, n)
        _check([(kps[i, :n[i]], desc[i, :n[i]]) for i in range(6)], ref, frames, "bench")
        nm, m = mt.match_frames(kps, desc, n)
        rnm, rm = oracle.match_frames_batch(rk, rd, rn, checkOri=True, nthreads=NTHREADS)
        assert np.array_equal(np.asarray(nm), rnm)
        for p in range(5):
            assert np.array_equal(np.asarray(m)[p, :rn[p]], rm[p, :rn[p]]), "matches of pair %d" % p
    finally:
        fe.close(); mt.close()


@pytest.mark.parametrize("s00", [1, 128, 255])
def test_unmasked_frames_origin_constant(oracle, s00):
    """Texture up to the image's edges and a non-zero S(0,0): the out-of-view class differs from the black corners on every level."""
    from cubemapslam_b200.frontend import FrontEnd
    cfg = config.front_1024()
    mask = config.load_mask("gray_cubemap_front_mask_650")
    frames = np.stack([_unmasked(cfg, i, s00) for i in range(3)])
    fe = FrontEnd(cfg, mask, max_batch=3)
    try:
        _check(fe.run(frames), _reference(oracle, cfg, fe, frames, mask), frames, "S(0,0)=%d" % s00)
    finally:
        fe.close()


@pytest.mark.parametrize("geom,face", [("lafida", 450), ("front", 333), ("front", 560), ("front", 570), ("front", 610), ("front", 650)])
def test_geometries_and_batches(oracle, geom, face):
    cfg = _cfg(geom, face)
    from cubemapslam_b200.frontend import FrontEnd
    mask = _mask(cfg)
    frames = np.stack([_unmasked(cfg, i, (37 * i + 1) % 256) if i % 2 else synth.fisheye_frame(cfg, i) for i in range(13)])
    frames[4, 0, 0] = 200   # a masked frame whose out-of-view class is not black
    fe = FrontEnd(cfg, mask, max_batch=13)
    try:
        ref = _reference(oracle, cfg, fe, frames, mask)
        for b in (1, 3, 13):
            got = fe.run(frames[:b])
            _check(got, tuple(r[:b] for r in ref), frames[:b], "%s %d batch %d" % (geom, face, b))
    finally:
        fe.close()


def test_caller_canvas_then_warp_path(oracle):
    """A caller-canvas extract scores every pixel of arbitrary canvases; the next warp-path run goes back to the live lists and must
    equal a fresh front end and the oracle."""
    from cubemapslam_b200.frontend import FrontEnd
    cfg = config.front_1024()
    mask = config.load_mask("gray_cubemap_front_mask_650")
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    canv = np.stack([oracle.warp(cp, _unmasked(cfg, i, 90), m1, m2) for i in range(3)])
    for c in canv:   # flat grey corners: non-zero on every level, but no texture to flood the candidate buffers
        for v, (ty, tx) in zip((37, 90, 150, 220), ((0, 0), (0, 1300), (1300, 0), (1300, 1300))):
            c[ty:ty + 650, tx:tx + 650] = v
    frames = np.stack([_unmasked(cfg, i, s) for i, s in zip((4, 5, 6), (0, 128, 255))])
    fe = FrontEnd(cfg, mask, max_batch=3); fresh = FrontEnd(cfg, mask, max_batch=3)
    try:
        fe.extract(canv)
        got = fe.run(frames)
        want = fresh.run(frames)
        for f in range(3):
            assert np.array_equal(got[f][0].view(np.uint8), want[f][0].view(np.uint8)) and np.array_equal(got[f][1], want[f][1]), "frame %d" % f
        _check(got, _reference(oracle, cfg, fe, frames, mask), frames, "after a caller canvas")
    finally:
        fe.close(); fresh.close()
