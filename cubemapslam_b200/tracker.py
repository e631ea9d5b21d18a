"""Host-side mirror of the reference's per-frame indexing and projection matchers on top of the C ABI.

  Frame::ComputeKeyPointRays / AssignFeaturesToGrid   (reference src/Frame.cpp:746-760,158-176)   -> Tracker.frame_index
  Frame::GetFeaturesInArea cell rectangles            (src/Frame.cpp:251-716)                     -> area_rects (host utility)
  ORBMatcher::SearchByProjection(Frame&, const Frame&, th, mono)        (src/ORBMatcher.cpp:130-251) -> Tracker.SearchByProjection_last
  ORBMatcher::SearchByProjection(Frame&, vector<MapPoint*>&, th)        (src/ORBMatcher.cpp:51-128)  -> Tracker.SearchByProjection_local
                                                                        local maps past 4096 MapPoints -> Tracker.SearchByProjection_local_large
  ORBMatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) (src/ORBMatcher.cpp:676-794) -> Tracker.SearchForInitialization
All calls but SearchForInitialization (one pair per call) are batched over independent frames (leading axis)."""
import ctypes as C

import numpy as np

from ._capi import KP_DTYPE, Handle, check, lib, ptr

NCELLS = 5 * 50 * 50
CSLAM_LOCAL_MAP_MAX_POINTS = 1 << 20   # MapPoints per frame of SearchByProjection_local_large
CSLAM_BOW_FV_MAX_FEATURES = 16384      # key points per frame of SearchForInitialization


def area_rects(x, y, r, face_w, face_h):
    out = np.zeros((3, 5), np.int32)
    n = lib().cslam_area_rects(C.c_float(x), C.c_float(y), C.c_float(r), int(face_w), int(face_h), ptr(out))
    return out[:n].copy()


def _b(a, dtype, single):
    a = np.ascontiguousarray(a, dtype)
    return a[None] if single else a


class Tracker(Handle):
    KIND = "tracker"

    def __init__(self, max_frames=8, max_features=4096, device=0):
        super().__init__(int(device), int(max_frames), int(max_features))
        self.max_frames, self.max_features = max_frames, max_features

    def frame_index(self, kps, face_w, face_h, n=None):
        """kps: (stride,) or (F, stride) cv::KeyPoint records. Returns rays (F, stride, 3), cell_start (F, 12501) u16, cell_idx (F, stride) u16."""
        kps = np.ascontiguousarray(kps, KP_DTYPE); single = kps.ndim == 1
        k = kps[None] if single else kps
        F, stride = k.shape
        n = np.full(F, stride, np.int32) if n is None else np.ascontiguousarray(n, np.int32).reshape(F)
        rays = np.zeros((F, stride, 3), np.float32); cs = np.zeros((F, NCELLS + 1), np.uint16); ci = np.zeros((F, stride), np.uint16)
        check(lib().cslam_frame_index(self._h, ptr(k), ptr(n), F, stride, int(face_w), int(face_h), ptr(rays), ptr(cs), ptr(ci)))
        return (rays[0], cs[0], ci[0]) if single else (rays, cs, ci)

    def frame_index_dev(self, kps, n, nframes, stride, face_w, face_h, rays, cell_start, cell_idx):
        check(lib().cslam_frame_index_dev(self._h, ptr(kps), ptr(n), int(nframes), int(stride), int(face_w), int(face_h), ptr(rays), ptr(cell_start), ptr(cell_idx)))

    def SearchByProjection_last(self, kCur, dCur, TcwCur, kLast, hasMP, Xw, dMP, mpObs, curTaken, face_w, face_h, cos_fov_th, th, check_ori=True, scale_factor=1.2, nlevels=8,
                                nCur=None, nLast=None):
        kCur = np.ascontiguousarray(kCur, KP_DTYPE); single = kCur.ndim == 1
        kC = kCur[None] if single else kCur
        P, cs = kC.shape
        kL = _b(kLast, KP_DTYPE, single); ls = kL.shape[1]
        a = [_b(dCur, np.uint8, single), _b(TcwCur, np.float32, single).reshape(P, 16), _b(hasMP, np.uint8, single), _b(Xw, np.float32, single), _b(dMP, np.uint8, single),
             _b(np.asarray(mpObs) > 0, np.uint8, single), _b(curTaken, np.uint8, single)]
        nC = np.full(P, cs, np.int32) if nCur is None else np.ascontiguousarray(nCur, np.int32).reshape(P)
        nL = np.full(P, ls, np.int32) if nLast is None else np.ascontiguousarray(nLast, np.int32).reshape(P)
        match = np.empty((P, cs), np.int32); nm = np.empty(P, np.int32)
        check(lib().cslam_search_by_projection_last(self._h, P, ptr(kC), ptr(a[0]), ptr(nC), cs, ptr(a[6]), ptr(a[1]), ptr(kL), ptr(nL), ls, ptr(a[2]), ptr(a[3]), ptr(a[4]), ptr(a[5]),
                                                    int(face_w), int(face_h), C.c_float(cos_fov_th), C.c_float(th), int(check_ori), C.c_float(scale_factor), int(nlevels),
                                                    ptr(match), ptr(nm)))
        return (int(nm[0]), match[0]) if single else (nm, match)

    def SearchByProjection_local(self, kF, dF, inView, projXY, level, viewCos, dMP, mpObs, fTaken, face_w, face_h, th, nnratio, scale_factor=1.2, nlevels=8, nF=None, nMP=None):
        return self._local("cslam_search_by_projection_local", kF, dF, inView, projXY, level, viewCos, dMP, mpObs, fTaken, face_w, face_h, th, nnratio, scale_factor, nlevels,
                           nF, nMP)

    def SearchByProjection_local_large(self, kF, dF, inView, projXY, level, viewCos, dMP, mpObs, fTaken, face_w, face_h, th, nnratio, scale_factor=1.2, nlevels=8, nF=None,
                                       nMP=None):
        """SearchByProjection_local for local maps of up to CSLAM_LOCAL_MAP_MAX_POINTS MapPoints per frame, whatever max_features (frames stay
        within it). Same arguments and results; match rows past a frame's count are -1."""
        return self._local("cslam_search_by_projection_local_large", kF, dF, inView, projXY, level, viewCos, dMP, mpObs, fTaken, face_w, face_h, th, nnratio, scale_factor,
                           nlevels, nF, nMP)

    def _local(self, entry, kF, dF, inView, projXY, level, viewCos, dMP, mpObs, fTaken, face_w, face_h, th, nnratio, scale_factor, nlevels, nF, nMP):
        kF = np.ascontiguousarray(kF, KP_DTYPE); single = kF.ndim == 1
        k = kF[None] if single else kF
        P, fs = k.shape
        a = [_b(dF, np.uint8, single), _b(inView, np.uint8, single), _b(projXY, np.float32, single), _b(level, np.int32, single), _b(viewCos, np.float32, single),
             _b(dMP, np.uint8, single), _b(np.asarray(mpObs) > 0, np.uint8, single), _b(fTaken, np.uint8, single)]
        ms = a[1].shape[1]
        nf = np.full(P, fs, np.int32) if nF is None else np.ascontiguousarray(nF, np.int32).reshape(P)
        nm_ = np.full(P, ms, np.int32) if nMP is None else np.ascontiguousarray(nMP, np.int32).reshape(P)
        match = np.empty((P, fs), np.int32); nm = np.empty(P, np.int32)
        check(getattr(lib(), entry)(self._h, P, ptr(k), ptr(a[0]), ptr(nf), fs, ptr(a[7]), ptr(nm_), ms, ptr(a[1]), ptr(a[2]), ptr(a[3]), ptr(a[4]), ptr(a[5]), ptr(a[6]),
                                      int(face_w), int(face_h), C.c_float(th), C.c_float(nnratio), C.c_float(scale_factor), int(nlevels), ptr(match), ptr(nm)))
        return (int(nm[0]), match[0]) if single else (nm, match)

    def SearchForInitialization(self, k1, d1, prev_xy, k2, d2, face_w, face_h, window_size=100, nnratio=0.9, check_ori=True):
        """One pair of frames of up to CSLAM_BOW_FV_MAX_FEATURES key points each, whatever max_features. prev_xy: (n1, 2) window centres
        (vbPrevMatched). Returns (nmatches, match12, prev_xy updated with F2's key point of every surviving match)."""
        k1 = np.ascontiguousarray(k1, KP_DTYPE); k2 = np.ascontiguousarray(k2, KP_DTYPE)
        d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8); xy = np.ascontiguousarray(prev_xy, np.float32).reshape(-1, 2)
        match = np.empty(len(k1), np.int32); nm = np.zeros(1, np.int32)
        check(lib().cslam_search_for_initialization(self._h, ptr(k1), ptr(d1), len(k1), ptr(xy), ptr(k2), ptr(d2), len(k2), int(face_w), int(face_h), int(window_size),
                                                    C.c_float(nnratio), int(check_ori), ptr(match), ptr(nm)))
        out = xy.copy()
        live = match >= 0
        out[live, 0] = k2["x"][match[live]]; out[live, 1] = k2["y"][match[live]]
        return int(nm[0]), match, out

    def search_by_projection_last_dev(self, npairs, kCur, dCur, nCur, cur_stride, cell_start, cell_idx, curTaken, TcwCur, kLast, nLast, last_stride, hasMP, Xw, dMP, mpObs,
                                      face_w, face_h, cos_fov_th, th, check_ori, match, nmatches, scale_factor=1.2, nlevels=8):
        check(lib().cslam_search_by_projection_last_dev(self._h, int(npairs), ptr(kCur), ptr(dCur), ptr(nCur), int(cur_stride), ptr(cell_start), ptr(cell_idx), ptr(curTaken), ptr(TcwCur),
                                                        ptr(kLast), ptr(nLast), int(last_stride), ptr(hasMP), ptr(Xw), ptr(dMP), ptr(mpObs), int(face_w), int(face_h),
                                                        C.c_float(cos_fov_th), C.c_float(th), int(check_ori), C.c_float(scale_factor), int(nlevels), ptr(match), ptr(nmatches)))

    def gather_pose_inputs_dev(self, npairs, match, kCur, nCur, cur_stride, rays, cos_fov_th, XwLast, last_stride, inv_sigma2_levels, XwOut, kpOut, wOut, count):
        check(lib().cslam_tracker_gather_pose_inputs_dev(self._h, int(npairs), ptr(match), ptr(kCur), ptr(nCur), int(cur_stride), ptr(rays), C.c_float(cos_fov_th), ptr(XwLast),
                                                         int(last_stride), ptr(inv_sigma2_levels), ptr(XwOut), ptr(kpOut), ptr(wOut), ptr(count)))
