"""cslam_frontend_submit / cslam_frontend_wait: batches pipelined through the asynchronous host entry, interleaved with every other call of
the front end, must give the bytes a fresh front end's cslam_frontend_run gives for the same frames; each ticket reports its own errors."""
import gc
import math
import weakref

import numpy as np
import pytest

from cubemapslam_b200 import config
from cubemapslam_b200._capi import KP_DTYPE
from tests.test_gpu_frontend_entry_points import MAX_BATCH, _fe, assert_same, dev_rows, fisheye, fresh, pinned, rows, run_dev, split

pytestmark = pytest.mark.gpu


def inputs(frames, page_locked):
    if not page_locked:
        return frames.copy()
    p = pinned(frames.shape, np.uint8)
    p[:] = frames
    return p


def outputs(fe, batch, page_locked):
    make = pinned if page_locked else np.empty
    return make((batch, fe.kp_cap), KP_DTYPE), make((batch, fe.kp_cap, 32), np.uint8), make((batch,), np.int32)


def submit(fe, frames, page_locked_in=False, page_locked_out=False):
    """Submits `frames`; returns the ticket and the output buffers."""
    out = outputs(fe, len(frames), page_locked_out)
    return fe.submit_raw(inputs(frames, page_locked_in), *out), out


def want_run(frames):
    return fresh(lambda g: split(g.run(frames)))


def badarg(call):
    from cubemapslam_b200._capi import CslamError
    with pytest.raises(CslamError, match="error -2"):
        call()


def test_pipelined_batches_match_run():
    sizes = [1, 7, 64, 64, 33, 64, 2]
    batches = []
    first = 0
    for b in sizes:
        batches.append(fisheye(first, b))
        first += b
    fe = _fe()
    try:
        got = {}
        prev = None
        for i, frames in enumerate(batches):   # submit batch i, then wait for batch i - 1
            t, out = submit(fe, frames, page_locked_in=i % 2 == 1, page_locked_out=i % 3 != 1)
            if prev is not None:
                fe.wait(prev[0])
                got[i - 1] = rows(*prev[1])
            prev = (t, out)
        fe.wait(prev[0])
        got[len(batches) - 1] = rows(*prev[1])
        for i, frames in enumerate(batches):
            assert_same(got[i], want_run(frames), "ticket %d (%d frames)" % (i, len(frames)))
    finally:
        fe.close()


def test_pageable_input_may_be_reused_after_submit():
    frames = fisheye(300, 9)
    fe = _fe()
    try:
        buf = frames.copy()
        out = outputs(fe, len(frames), False)
        t = fe.submit_raw(buf, *out)
        buf[:] = fisheye(400, 9)
        fe.wait(t)
        assert_same(rows(*out), want_run(frames), "reused input")
    finally:
        fe.close()


def test_other_calls_with_two_tickets_pending_match_a_fresh_front_end():
    fa, fb, fc = fisheye(0, MAX_BATCH), fisheye(64, 5), fisheye(70, 11)
    fe = _fe()
    try:
        ta, oa = submit(fe, fa)
        tb, ob = submit(fe, fb, page_locked_in=True, page_locked_out=True)
        # the debug reads show the most recently enqueued batch
        level = fe.level_image(0, 0)
        assert np.array_equal(level, fresh(lambda g: (g.run(fb[:1]), g.level_image(0, 0))[1])), "get_level with tickets pending"
        f13 = fisheye(200, 13)
        assert_same(split(fe.run(f13)), want_run(f13), "run 13")
        f2 = fisheye(110, 2)
        canvas = np.full((2, 1350, 1350), 7, np.uint8)
        warped = fe.warp(f2, canvas.copy())
        assert np.array_equal(warped, fresh(lambda g: g.warp(f2, canvas.copy())))
        assert np.all(warped[:, :450, :450] == 7) and np.all(warped[:, 900:, 900:] == 7)
        f5 = fisheye(30, 5)
        assert_same(dev_rows(run_dev(fe, f5)), fresh(lambda g: dev_rows(run_dev(g, f5))), "run_dev 5")
        # caller canvases with textured corner tiles last: the next submit must clear the corners again
        canvases = fresh(lambda g: g.warp(fisheye(20, 3)))
        canvases[:, :450, :450] = np.random.default_rng(0).integers(0, 256, (3, 450, 450), dtype=np.uint8)
        assert_same(split(fe.extract(canvases)), fresh(lambda g: split(g.extract(canvases))), "extract 3")
        fe.wait(ta)
        fe.wait(tb)
        assert_same(rows(*oa), want_run(fa), "ticket a")
        assert_same(rows(*ob), want_run(fb), "ticket b")
        tc, oc = submit(fe, fc)
        fe.wait(tc)
        assert_same(rows(*oc), want_run(fc), "ticket after a caller canvas")
        fe.sync()
    finally:
        fe.close()


def test_ticket_rules():
    import ctypes as C
    from cubemapslam_b200._capi import lib, ptr
    fa, fb, fc = fisheye(500, 3), fisheye(503, 4), fisheye(507, 2)
    fe = _fe()
    try:
        ta, oa = submit(fe, fa)
        tb, ob = submit(fe, fb, page_locked_out=True)
        assert 0 < ta < tb
        badarg(lambda: submit(fe, fc))   # a third pending ticket
        fe.wait(tb)   # out of order
        fe.wait(ta)
        assert_same(rows(*oa), want_run(fa), "ticket a")
        assert_same(rows(*ob), want_run(fb), "ticket b")
        for t in (ta, tb, tb + 1, tb + 1000, 0, -1):   # waited, never issued, not a ticket
            badarg(lambda: fe.wait(t))
        # failed submits issue no ticket
        out = outputs(fe, MAX_BATCH + 1, False)
        t = C.c_int64(-7)
        assert lib().cslam_frontend_submit(fe._h, None, 1, ptr(out[0]), ptr(out[1]), ptr(out[2]), C.byref(t)) == -2 and t.value == -7
        badarg(lambda: fe.submit_raw(fc[:0], *out))
        badarg(lambda: fe.submit_raw(np.zeros((MAX_BATCH + 1,) + fc.shape[1:], np.uint8), *out))
        assert not fe._pending
        tc, oc = submit(fe, fc)
        assert tc == tb + 1
        fe.wait(tc)
        assert_same(rows(*oc), want_run(fc), "ticket after failed submits")
    finally:
        fe.close()


def level0_list_capacity(face):
    """k_fast's candidate list of level 0 (cslam_frontend_create): 32 per FAST cell of the whole level, at least 4096."""
    w = 3 * face
    width = w - 32   # EDGE_THRESHOLD - 3 inset on both sides
    n = int(width / 30)
    cell = math.ceil(width / n)
    cols = max(j + 1 for j in range(n) if not 16 + j * cell >= w - 16 - 6)
    rws = max(i + 1 for i in range(n) if not 16 + i * cell >= w - 16 - 3)
    return max(4096, cols * rws * 32)


def test_an_overflow_is_reported_by_its_own_ticket(oracle):
    from cubemapslam_b200._capi import CslamError
    cfg = config.lafida_450()
    mask = config.load_mask("gray_lafida_cubemap_mask_450")
    noise = np.random.default_rng(5).integers(0, 256, (1, int(cfg["Camera.Ih"]), int(cfg["Camera.Iw"])), dtype=np.uint8)
    # the reference's level-0 candidates of the noise frame exceed the list: the front end must report the overflow
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    ex = oracle.ORBextractor(int(cfg["ORBextractor.nFeatures"]), cfg["ORBextractor.scaleFactor"], int(cfg["ORBextractor.nLevels"]),
                             int(cfg["ORBextractor.iniThFAST"]), int(cfg["ORBextractor.minThFAST"]), 450, 450)
    ex(oracle.warp(cp, noise[0], m1, m2), mask)
    assert len(ex.stage(0, 0)) > level0_list_capacity(450)
    fa, fc = fisheye(600, 6), fisheye(606, 40)
    fe = _fe()
    try:
        ta, oa = submit(fe, fa)
        tb, _ = submit(fe, noise)
        fe.wait(ta)
        tc, oc = submit(fe, fc, page_locked_out=True)
        with pytest.raises(CslamError, match="error -4"):
            fe.wait(tb)
        fe.wait(tc)
        fe.sync()   # the ticket's error is not the handle's
        assert_same(rows(*oa), want_run(fa), "ticket before the overflow")
        assert_same(rows(*oc), want_run(fc), "ticket after the overflow")
    finally:
        fe.close()


def test_buffers_outlive_the_callers_references_and_close_waits():
    fa, fb = fisheye(700, 16), fisheye(716, 8)
    fe = _fe()
    try:
        def go(frames):   # every reference to the ticket's buffers goes out of scope here
            t, out = submit(fe, frames, page_locked_in=True, page_locked_out=True)
            return t, [weakref.ref(a) for a in out]
        ta, wa = go(fa)
        tb, wb = go(fb)
        gc.collect()
        junk = [outputs(fe, 16, True) for _ in range(2)]   # page-locked memory a freed buffer would come back as
        for o in junk:
            for a in o:
                a.fill(0xAB)
        oa, ob = [w() for w in wa], [w() for w in wb]
        assert all(a is not None for a in oa + ob), "the wrapper keeps a pending ticket's buffers"
        fe.wait(ta)
        fe.wait(tb)
        assert_same(rows(*oa), want_run(fa), "ticket a")
        assert_same(rows(*ob), want_run(fb), "ticket b")
        # close with two tickets pending, then a new front end on the same device
        submit(fe, fa)
        submit(fe, fb, page_locked_in=True)
    finally:
        fe.close()
    assert not fe._pending
    fe2 = _fe()
    try:
        assert_same(split(fe2.run(fb)), want_run(fb), "front end after a close with tickets pending")
    finally:
        fe2.close()


def test_launches_and_timing_of_a_submitted_batch():
    fe = _fe()
    try:
        nl = fe.nlevels
        for frames in (fisheye(800, 7), fisheye(807, MAX_BATCH)):
            l0 = fe.launches
            fe.run(frames)
            by_run = fe.launches - l0
            l0 = fe.launches
            t, _ = submit(fe, frames)
            fe.wait(t)
            assert fe.launches - l0 == by_run, len(frames)
        f13 = fisheye(0, 13)
        fe.set_timing(True)
        l0 = fe.launches
        t, out = submit(fe, f13)
        fe.wait(t)
        launched = fe.launches - l0
        tm = fe.timing()
        fe.set_timing(False)
        want_counts = {"k_warp": 1, "k_pyramid": nl - 1, "k_fast": nl, "k_distribute": 1, "k_describe": 1}
        assert {k: c for k, (_, c) in tm.items()} == want_counts and launched == sum(want_counts.values())
        assert all(ms > 0 for ms, _ in tm.values()), tm
        assert_same(rows(*out), want_run(f13), "timed ticket")
    finally:
        fe.close()
