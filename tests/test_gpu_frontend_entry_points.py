"""One front end serves its host entry points (cslam_frontend_run with pageable and with page-locked buffers, cslam_orb_extract, cslam_warp)
and its device form (cslam_frontend_run_dev) interleaved, at batches from 1 to max_batch. The host calls stage through the handle's device arena
and its lanes; every call must give the bytes a fresh front end gives for the same frames."""
import numpy as np
import pytest

from cubemapslam_b200 import config, synth
from cubemapslam_b200._capi import KP_DTYPE

pytestmark = pytest.mark.gpu

MAX_BATCH = 64


def _fe():
    from cubemapslam_b200.frontend import FrontEnd
    return FrontEnd(config.lafida_450(), config.load_mask("gray_lafida_cubemap_mask_450"), max_batch=MAX_BATCH)


def fisheye(first, batch):
    cfg = config.lafida_450()
    return np.stack([synth.fisheye_frame(cfg, first + i) for i in range(batch)])


def rows(kps, desc, n):
    """Per frame, the key point bytes and descriptors in [0, n[f]); bytes past a frame's count are unspecified."""
    return [(kps[f, :n[f]].view(np.uint8).copy(), desc[f, :n[f]].copy()) for f in range(len(n))]


def split(res):   # FrontEnd.run / extract output of a batch
    return [(k.view(np.uint8), d) for k, d in res]


def assert_same(got, want, what):
    assert len(got) == len(want), what
    for f, ((gk, gd), (wk, wd)) in enumerate(zip(got, want)):
        assert len(wk) > 0, "%s frame %d: no key points" % (what, f)
        assert len(gk) == len(wk) and np.array_equal(gk, wk) and np.array_equal(gd, wd), "%s frame %d" % (what, f)


def fresh(call):
    fe = _fe()
    try:
        return call(fe)
    finally:
        fe.close()


def run_dev(fe, frames):
    """cslam_frontend_run_dev on device copies of `frames`; returns the device outputs without synchronising."""
    import torch
    B = len(frames)
    fish = torch.from_numpy(frames).cuda()
    kps = torch.zeros((B, fe.kp_cap * KP_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
    desc = torch.zeros((B, fe.kp_cap, 32), dtype=torch.uint8, device="cuda"); n = torch.zeros(B, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    fe.run_dev(fish.data_ptr(), B, kps.data_ptr(), desc.data_ptr(), n.data_ptr())
    return fish, kps, desc, n


def dev_rows(out):
    import torch
    torch.cuda.synchronize()
    _, kps, desc, n = out
    return rows(kps.cpu().numpy().view(KP_DTYPE), desc.cpu().numpy(), n.cpu().numpy())


def pinned(shape, dtype):
    """A page-locked numpy array (it keeps its torch storage alive)."""
    import torch
    dtype = np.dtype(dtype)
    return torch.empty(int(np.prod(shape)) * dtype.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(dtype).reshape(shape)


def test_interleaved_entry_points_match_a_fresh_front_end():
    fe = _fe()
    try:
        nl, kc = fe.nlevels, fe.kp_cap
        # cslam_frontend_run, pageable buffers: 13 frames, 4 chunks on 4 lanes
        f13 = fisheye(0, 13)
        got13 = split(fe.run(f13))
        want13 = fresh(lambda g: split(g.run(f13)))
        assert_same(got13, want13, "run 13")
        # cslam_orb_extract on caller canvases with textured corner tiles
        canvases = fresh(lambda g: g.warp(fisheye(20, 3)))
        canvases[:, :450, :450] = np.random.default_rng(0).integers(0, 256, (3, 450, 450), dtype=np.uint8)
        assert_same(split(fe.extract(canvases)), fresh(lambda g: split(g.extract(canvases))), "extract 3")
        # cslam_frontend_run_dev, then at once a page-locked host batch of max_batch frames (8 chunks on 4 lanes) on the same stream
        f5 = fisheye(30, 5)
        dev5 = run_dev(fe, f5)
        f64 = fisheye(40, MAX_BATCH)
        fish_p = pinned(f64.shape, np.uint8)
        fish_p[:] = f64
        kps_p, desc_p, n_p = pinned((MAX_BATCH, kc), KP_DTYPE), pinned((MAX_BATCH, kc, 32), np.uint8), pinned((MAX_BATCH,), np.int32)
        fe.run_raw(fish_p, kps_p, desc_p, n_p)
        got64 = rows(kps_p, desc_p, n_p)
        assert_same(dev_rows(dev5), fresh(lambda g: dev_rows(run_dev(g, f5))), "run_dev 5")
        assert_same(got64, fresh(lambda g: split(g.run(f64))), "pinned run 64")
        # cslam_warp into caller canvases whose corner tiles must stay as the caller left them
        f2 = fisheye(110, 2)
        canvas = np.full((2, 1350, 1350), 7, np.uint8)
        warped = fe.warp(f2, canvas.copy())
        want = fresh(lambda g: g.warp(f2, canvas.copy()))
        assert np.array_equal(warped, want) and np.all(warped[:, :450, :450] == 7) and np.all(warped[:, 900:, 900:] == 7)
        # cslam_frontend_run, one frame
        f1 = fisheye(120, 1)
        assert_same(split(fe.run(f1)), fresh(lambda g: split(g.run(f1))), "run 1")
        # a timed host batch runs as one lane and one chunk: every launch counted once, the same bytes
        fe.set_timing(True)
        l0 = fe.launches
        timed = split(fe.run(f13))
        launched = fe.launches - l0
        tm = fe.timing()
        fe.set_timing(False)
        want_counts = {"k_warp": 1, "k_pyramid": nl - 1, "k_fast": nl, "k_distribute": 1, "k_describe": 1}
        assert {k: c for k, (_, c) in tm.items()} == want_counts and launched == sum(want_counts.values())
        assert all(ms > 0 for ms, _ in tm.values()), tm
        assert_same(timed, want13, "timed run 13")
    finally:
        fe.close()
