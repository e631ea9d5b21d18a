"""Host-side mirror of the LocalMapping feature operations on top of the C ABI (SURVEY §8(f) rank 4).

  MapPoint::ComputeDistinctiveDescriptors             (reference src/MapPoint.cpp:243-303)     -> Mapper.ComputeDistinctiveDescriptors (batched over MapPoints)
  ORBMatcher::Fuse(KeyFrame*, vector<MapPoint*>&, th) (src/ORBMatcher.cpp:1126-1240)           -> Mapper.FuseSearch (the search; the map bookkeeping stays with the caller)
  ORBMatcher::SearchForTriangulation                  (src/ORBMatcher.cpp:971-1124)            -> Mapper.SearchForTriangulation (batched over key-frame pairs)"""
import ctypes as C

import numpy as np

from ._capi import KP_DTYPE, Handle, check, lib, ptr


class Mapper(Handle):
    KIND = "mapper"

    def __init__(self, device=0):
        super().__init__(int(device))

    def ComputeDistinctiveDescriptors(self, desc, offset):
        desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32); offset = np.ascontiguousarray(offset, np.int32)
        n = len(offset) - 1
        best = np.empty(max(n, 0), np.int32)
        check(lib().cslam_distinctive_descriptors(self._h, ptr(desc), ptr(offset), n, ptr(best)))
        return best

    def FuseSearch(self, kKF, dKF, Tcw, valid, Xw, level, dMP, th, scale_factors, inv_level_sigma2, face_w, face_h):
        kKF = np.ascontiguousarray(kKF, KP_DTYPE); dKF = np.ascontiguousarray(dKF, np.uint8); Tcw = np.ascontiguousarray(Tcw, np.float32).reshape(16)
        valid = np.ascontiguousarray(valid, np.uint8); Xw = np.ascontiguousarray(Xw, np.float32); level = np.ascontiguousarray(level, np.int32)
        dMP = np.ascontiguousarray(dMP, np.uint8); sf = np.ascontiguousarray(scale_factors, np.float32); isg = np.ascontiguousarray(inv_level_sigma2, np.float32)
        n = len(valid)
        bi = np.empty(n, np.int32); bd = np.empty(n, np.int32)
        check(lib().cslam_fuse_search(self._h, ptr(kKF), ptr(dKF), len(kKF), ptr(Tcw), n, ptr(valid), ptr(Xw), ptr(level), ptr(dMP), C.c_float(th), ptr(sf), ptr(isg), len(sf),
                                      int(face_w), int(face_h), ptr(bi), ptr(bd)))
        return bi, bd

    def SearchForTriangulation(self, k1, d1, rays1, hasMP1, node1, n1, k2, d2, rays2, hasMP2, node2, n2, Ow1, Tcw2, E12, scale_factors, level_sigma2, face_w, face_h, checkOri=False):
        """All per-feature arrays carry a leading pair axis: (P, stride, ...). Returns (nmatches[P], match12[P, stride1])."""
        k1 = np.ascontiguousarray(k1, KP_DTYPE); k2 = np.ascontiguousarray(k2, KP_DTYPE)
        P, s1 = k1.shape; s2 = k2.shape[1]
        a = [np.ascontiguousarray(d1, np.uint8), np.ascontiguousarray(rays1, np.float32), np.ascontiguousarray(hasMP1, np.uint8), np.ascontiguousarray(node1, np.int32),
             np.ascontiguousarray(n1, np.int32), np.ascontiguousarray(d2, np.uint8), np.ascontiguousarray(rays2, np.float32), np.ascontiguousarray(hasMP2, np.uint8),
             np.ascontiguousarray(node2, np.int32), np.ascontiguousarray(n2, np.int32), np.ascontiguousarray(Ow1, np.float32), np.ascontiguousarray(Tcw2, np.float32),
             np.ascontiguousarray(E12, np.float32), np.ascontiguousarray(scale_factors, np.float32), np.ascontiguousarray(level_sigma2, np.float32)]
        m = np.empty((P, s1), np.int32); nm = np.empty(P, np.int32)
        check(lib().cslam_search_for_triangulation(self._h, P, ptr(k1), ptr(a[0]), ptr(a[1]), ptr(a[2]), ptr(a[3]), ptr(a[4]), s1, ptr(k2), ptr(a[5]), ptr(a[6]), ptr(a[7]), ptr(a[8]),
                                                   ptr(a[9]), s2, ptr(a[10]), ptr(a[11]), ptr(a[12]), ptr(a[13]), ptr(a[14]), len(a[13]), int(face_w), int(face_h), int(checkOri),
                                                   ptr(m), ptr(nm)))
        return nm, m
