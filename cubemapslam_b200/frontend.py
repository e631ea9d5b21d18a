"""Host-side mirror of the reference's warp + ORBextractor interface on top of the C ABI.

  System::CvtFisheyeToCubeMap_reverseQuery_withInterpolation  (reference src/System.cpp:327-355)  -> FrontEnd.warp
  ORBextractor::operator()                                     (reference src/ORBExtractor.cpp:838-926) -> FrontEnd.extract
FrontEnd.run / run_dev fuse both for batches (BASELINE config 2); submit_raw / wait are run_raw in two halves, so that one batch computes while the
next uploads and the previous downloads. PyTorch is only used by callers for device memory."""
import ctypes as C

import numpy as np

from . import _capi
from ._capi import KP_DTYPE, check, lib, ptr


class FrontEnd(_capi.Handle):
    KIND = "frontend"

    def __init__(self, cfg, mask, max_batch=8, device=0, orb=None):
        self.cfg = cfg
        self.cam = _capi.cam_params(cfg)
        self.orb = orb if orb is not None else _capi.orb_params(cfg)
        mask = np.ascontiguousarray(mask, np.uint8)
        self.CW, self.CH = 3 * self.cam.face_w, 3 * self.cam.face_h
        if mask.shape != (self.CH, self.CW):
            raise ValueError("mask must be %dx%d (same size as the cubemap canvas, reference src/ORBExtractor.cpp:848)" % (self.CH, self.CW))
        self._pending = {}   # ticket -> the arrays of a submitted batch, kept alive until it is waited or the handle is closed
        super().__init__(int(device), C.byref(self.cam), C.byref(self.orb), ptr(mask), mask.shape[1], int(max_batch))
        self.max_batch = max_batch
        self.kp_cap = lib().cslam_frontend_kp_capacity(self._h)
        self.nlevels = self.orb.nlevels

    # ---- reference-facing calls (host buffers)
    def warp(self, fisheye, canvas=None):
        fisheye = np.ascontiguousarray(fisheye, np.uint8)
        single = fisheye.ndim == 2
        f = fisheye[None] if single else fisheye
        assert f.shape[1:] == (self.cam.Ih, self.cam.Iw)
        if canvas is None:
            canvas = np.zeros((f.shape[0], self.CH, self.CW), np.uint8)   # the caller's zeroed canvas (Examples/cubemap_lafida.cpp:111)
        c = canvas[None] if canvas.ndim == 2 else canvas
        check(lib().cslam_warp(self._h, ptr(f), f.shape[0], ptr(c), c.shape[2]))
        return canvas[0] if single and canvas.ndim == 3 else canvas

    def _split(self, kps, desc, n, single):
        out = [(kps[i, :n[i]].copy(), desc[i, :n[i]].copy()) for i in range(len(n))]
        return out[0] if single else out

    def extract(self, canvas):
        canvas = np.ascontiguousarray(canvas, np.uint8)
        single = canvas.ndim == 2
        c = canvas[None] if single else canvas
        assert c.shape[1:] == (self.CH, self.CW)
        B = c.shape[0]
        kps = np.empty((B, self.kp_cap), KP_DTYPE); desc = np.empty((B, self.kp_cap, 32), np.uint8); n = np.empty(B, np.int32)
        check(lib().cslam_orb_extract(self._h, ptr(c), c.shape[2], B, ptr(kps), ptr(desc), ptr(n)))
        return self._split(kps, desc, n, single)

    def run(self, fisheye):
        fisheye = np.ascontiguousarray(fisheye, np.uint8)
        single = fisheye.ndim == 2
        f = fisheye[None] if single else fisheye
        B = f.shape[0]
        kps = np.empty((B, self.kp_cap), KP_DTYPE); desc = np.empty((B, self.kp_cap, 32), np.uint8); n = np.empty(B, np.int32)
        check(lib().cslam_frontend_run(self._h, ptr(f), B, ptr(kps), ptr(desc), ptr(n)))
        return self._split(kps, desc, n, single)

    def run_raw(self, fisheye, kps, desc, n):
        """Batched host call into caller-provided (pinned) buffers; no per-frame splitting."""
        check(lib().cslam_frontend_run(self._h, ptr(fisheye), int(fisheye.shape[0]), ptr(kps), ptr(desc), ptr(n)))

    def submit_raw(self, fisheye, kps, desc, n):
        """run_raw's batch, enqueued without waiting: returns the ticket to wait() on. The four arrays are referenced here until then, as the
        GPU reads a page-locked input and writes the outputs until the ticket is waited."""
        t = C.c_int64()
        check(lib().cslam_frontend_submit(self._h, ptr(fisheye), int(fisheye.shape[0]), ptr(kps), ptr(desc), ptr(n), C.byref(t)))
        self._pending[t.value] = (fisheye, kps, desc, n)
        return t.value

    def wait(self, ticket):
        """Waits for a submitted batch; its buffers then hold what run_raw writes. Raises for the ticket's own errors; the ticket is waited
        either way."""
        try:
            check(lib().cslam_frontend_wait(self._h, C.c_int64(int(ticket))))
        finally:
            self._pending.pop(int(ticket), None)

    def close(self):
        super().close()   # waits for the pending tickets' device work
        self._pending = {}

    # ---- device-resident path (addresses as ints, e.g. torch.Tensor.data_ptr())
    def run_dev(self, fisheye_dev, batch, kps_dev, desc_dev, n_dev):
        check(lib().cslam_frontend_run_dev(self._h, ptr(fisheye_dev), int(batch), ptr(kps_dev), ptr(desc_dev), ptr(n_dev)))

    def set_timing(self, enable):
        check(lib().cslam_frontend_set_timing(self._h, int(enable)))

    def timing(self):
        out = {}
        for kind in range(5):
            name = C.c_char_p(); ms = C.c_double(); cnt = C.c_int64()
            check(lib().cslam_frontend_get_timing(self._h, kind, C.byref(name), C.byref(ms), C.byref(cnt)))
            out[name.value.decode()] = (ms.value, cnt.value)
        return out

    # ---- stage access for parity tests
    def level_image(self, frame, level):
        w = C.c_int(); h = C.c_int()
        check(lib().cslam_frontend_level_size(self._h, level, C.byref(w), C.byref(h)))
        out = np.empty((h.value, w.value), np.uint8)
        check(lib().cslam_frontend_get_level(self._h, frame, level, ptr(out)))
        return out

    def candidates(self, frame, level):
        cap = 1 << 18
        out = np.empty((cap, 3), np.int32); n = C.c_int()
        check(lib().cslam_frontend_get_candidates(self._h, frame, level, ptr(out), cap, C.byref(n)))
        return out[:n.value].copy()

    def maps(self):
        m1 = np.empty((self.CH, self.CW), np.float32); m2 = np.empty_like(m1)
        check(lib().cslam_frontend_get_maps(self._h, ptr(m1), ptr(m2)))
        return m1, m2

    def tables(self):
        nl = self.nlevels
        sc = [np.empty(nl, np.float32) for _ in range(4)]; per = np.empty(nl, np.int32); um = np.empty(16, np.int32)
        check(lib().cslam_frontend_tables(self._h, ptr(sc[0]), ptr(sc[1]), ptr(sc[2]), ptr(sc[3]), ptr(per), ptr(um)))
        return dict(scale=sc[0], inv_scale=sc[1], sigma2=sc[2], inv_sigma2=sc[3], features_per_level=per, umax=um)
