"""Host-side mirror of the reference ORBMatcher interface (reference include/ORBMatcher.h:42-104) on top of the C ABI.

  ORBMatcher(nnratio, checkOri)          constructor arguments kept
  DescriptorDistance(a, b)               src/ORBMatcher.cpp:951-967
  SearchByBoW(KF, F)                     src/ORBMatcher.cpp:409-539   (arrays instead of KeyFrame*/Frame&)
  SearchByBoW_fv / SearchByBoW_KF_fv     the same searches for key frames of up to Vocabulary.MAX_FV_FEATURES features, FeatureVectors as CSRs
  match_bruteforce                       BASELINE config 3 (definition: DESIGN.md §matcher)
All calls are batched over `npairs` independent pairs (leading axis)."""
import ctypes as C

import numpy as np

from ._capi import Handle, check, lib, ptr
from .vocabulary import Vocabulary

TH_HIGH = 100
TH_LOW = 50
HISTO_LENGTH = 12


class ORBMatcher(Handle):
    KIND = "matcher"

    def __init__(self, nnratio=0.6, checkOri=True, max_pairs=64, max_features=2048, device=0):
        self.nnratio = float(nnratio); self.check_ori = bool(checkOri)
        super().__init__(int(device), int(max_pairs), int(max_features))
        self.max_pairs, self.max_features = max_pairs, max_features

    def DescriptorDistance(self, a, b):
        a = np.ascontiguousarray(a, np.uint8).reshape(-1, 32); b = np.ascontiguousarray(b, np.uint8).reshape(-1, 32)
        out = np.empty(a.shape[0], np.int32)
        check(lib().cslam_hamming(self._h, ptr(a), ptr(b), a.shape[0], ptr(out)))
        return out if out.size != 1 else int(out[0])

    @staticmethod
    def _batched(*arrs):
        single = arrs[0].ndim == 2
        return single, [a[None] if single else a for a in arrs]

    def match_bruteforce(self, descA, angA, descB, angB, th_low=TH_LOW):
        descA = np.ascontiguousarray(descA, np.uint8); descB = np.ascontiguousarray(descB, np.uint8)
        angA = np.ascontiguousarray(angA, np.float32); angB = np.ascontiguousarray(angB, np.float32)
        single = descA.ndim == 2
        if single:
            descA, descB, angA, angB = descA[None], descB[None], angA[None], angB[None]
        P, nA, nB = descA.shape[0], descA.shape[1], descB.shape[1]
        m = np.empty((P, nA), np.int32); d = np.empty((P, nA), np.int32); s = np.empty((P, nA), np.int32); n = np.empty(P, np.int32)
        check(lib().cslam_match_bruteforce(self._h, ptr(descA), ptr(angA), nA, ptr(descB), ptr(angB), nB, P, C.c_float(self.nnratio), int(th_low),
                                           int(self.check_ori), ptr(m), ptr(d), ptr(s), ptr(n)))
        return (int(n[0]), m[0], d[0], s[0]) if single else (n, m, d, s)

    def match_bruteforce_dev(self, descA, angA, nA, descB, angB, nB, npairs, match12, nmatches, dist12=None, second12=None, th_low=TH_LOW):
        check(lib().cslam_match_bruteforce_dev(self._h, ptr(descA), ptr(angA), int(nA), ptr(descB), ptr(angB), int(nB), int(npairs), C.c_float(self.nnratio),
                                               int(th_low), int(self.check_ori), ptr(match12), ptr(dist12), ptr(second12), ptr(nmatches)))

    def match_frames_dev(self, kps, desc, n, kp_stride, nframes, match12, nmatches, th_low=TH_LOW):
        check(lib().cslam_match_frames_dev(self._h, ptr(kps), ptr(desc), ptr(n), int(kp_stride), int(nframes), C.c_float(self.nnratio), int(th_low), int(self.check_ori),
                                           ptr(match12), ptr(nmatches)))

    def match_frames(self, kps, desc, n, th_low=TH_LOW):
        """Host arrays as FrontEnd.run_raw fills them: kps (F, stride) records, desc (F, stride, 32), n (F,). Returns nmatches (F-1,), match12 (F-1, stride)."""
        F, stride = kps.shape[0], kps.shape[1]
        match = np.empty((F - 1, stride), np.int32); nm = np.empty(F - 1, np.int32)
        check(lib().cslam_match_frames(self._h, ptr(kps), ptr(desc), ptr(n), int(stride), int(F), C.c_float(self.nnratio), int(th_low), int(self.check_ori), ptr(match), ptr(nm)))
        return nm, match

    def ubench_popc(self):
        v = C.c_double()
        check(lib().cslam_ubench_popc(self._h, C.byref(v)))
        return v.value

    def ubench_bmma(self):
        """(BMMA, IMMA) rates in 256-bit products (= Hamming distances) per second, register-only chains."""
        b = C.c_double(); i = C.c_double()
        check(lib().cslam_ubench_bmma(self._h, C.byref(b), C.byref(i)))
        return b.value, i.value

    def ubench_minmax3(self):
        v = C.c_double()
        check(lib().cslam_ubench_minmax3(self._h, C.byref(v)))
        return v.value

    def SearchByBoW(self, descKF, angKF, kf_valid, node_kf, descF, angF, node_f):
        a = [np.ascontiguousarray(descKF, np.uint8), np.ascontiguousarray(angKF, np.float32), np.ascontiguousarray(kf_valid, np.uint8),
             np.ascontiguousarray(node_kf, np.int32), np.ascontiguousarray(descF, np.uint8), np.ascontiguousarray(angF, np.float32),
             np.ascontiguousarray(node_f, np.int32)]
        single = a[0].ndim == 2
        if single:
            a = [x[None] for x in a]
        P, nKF, nF = a[0].shape[0], a[0].shape[1], a[4].shape[1]
        mf = np.empty((P, nF), np.int32); n = np.empty(P, np.int32)
        check(lib().cslam_search_by_bow(self._h, ptr(a[0]), ptr(a[1]), ptr(a[2]), ptr(a[3]), nKF, ptr(a[4]), ptr(a[5]), ptr(a[6]), nF, P,
                                        C.c_float(self.nnratio), int(self.check_ori), ptr(mf), ptr(n)))
        return (int(n[0]), mf[0]) if single else (n, mf)

    def SearchByBoW_KF(self, desc1, ang1, valid1, node1, desc2, ang2, valid2, node2):
        """SearchByBoW(KeyFrame*, KeyFrame*, ...) (reference src/ORBMatcher.cpp:541-674); match12 per feature of key frame 1."""
        a = [np.ascontiguousarray(desc1, np.uint8), np.ascontiguousarray(ang1, np.float32), np.ascontiguousarray(valid1, np.uint8), np.ascontiguousarray(node1, np.int32),
             np.ascontiguousarray(desc2, np.uint8), np.ascontiguousarray(ang2, np.float32), np.ascontiguousarray(valid2, np.uint8), np.ascontiguousarray(node2, np.int32)]
        single = a[0].ndim == 2
        if single:
            a = [x[None] for x in a]
        P, n1, n2 = a[0].shape[0], a[0].shape[1], a[4].shape[1]
        m12 = np.empty((P, n1), np.int32); n = np.empty(P, np.int32)
        check(lib().cslam_search_by_bow_kf(self._h, ptr(a[0]), ptr(a[1]), ptr(a[2]), ptr(a[3]), n1, ptr(a[4]), ptr(a[5]), ptr(a[6]), ptr(a[7]), n2, P,
                                           C.c_float(self.nnratio), int(self.check_ori), ptr(m12), ptr(n)))
        return (int(n[0]), m12[0]) if single else (n, m12)

    def search_by_bow_dev(self, descKF, angKF, kf_valid, node_kf, nKF, descF, angF, node_f, nF, npairs, match_f, nmatches):
        check(lib().cslam_search_by_bow_dev(self._h, ptr(descKF), ptr(angKF), ptr(kf_valid), ptr(node_kf), int(nKF), ptr(descF), ptr(angF), ptr(node_f),
                                            int(nF), int(npairs), C.c_float(self.nnratio), int(self.check_ori), ptr(match_f), ptr(nmatches)))

    def SearchByBoW_fv(self, descKF, angKF, kf_valid, n_kf, fv_kf, descF, angF, n_f, fv_f):
        """cslam_search_by_bow_fv: SearchByBoW(KeyFrame*, Frame&) for strides up to Vocabulary.MAX_FV_FEATURES, whatever max_features.
        Per-feature arrays are (P, stride, ...), n_* (P,); fv_* = (node, start, feat, count), batched as pack_fv returns them (the layout
        cslam_bow_transform_fv writes). Returns (nmatches (P,), match_f (P, f_stride)), -1 past n_f."""
        return self._bow_fv(lib().cslam_search_by_bow_fv, descKF, angKF, kf_valid, n_kf, fv_kf, descF, angF, None, n_f, fv_f)

    def SearchByBoW_KF_fv(self, desc1, ang1, valid1, n1, fv1, desc2, ang2, valid2, n2, fv2):
        """cslam_search_by_bow_kf_fv: SearchByBoW(KeyFrame*, KeyFrame*) likewise. Returns (nmatches (P,), match12 (P, stride1))."""
        return self._bow_fv(lib().cslam_search_by_bow_kf_fv, desc1, ang1, valid1, n1, fv1, desc2, ang2, valid2, n2, fv2)

    def _bow_fv(self, fn, d1, a1, v1, n1, fv1, d2, a2, v2, n2, fv2):
        d1 = np.ascontiguousarray(d1, np.uint8); d2 = np.ascontiguousarray(d2, np.uint8)
        P, s1, s2 = d1.shape[0], d1.shape[1], d2.shape[1]
        a1 = np.ascontiguousarray(a1, np.float32); a2 = np.ascontiguousarray(a2, np.float32); v1 = np.ascontiguousarray(v1, np.uint8)
        n1 = np.ascontiguousarray(n1, np.int32); n2 = np.ascontiguousarray(n2, np.int32)
        f1 = [np.ascontiguousarray(x, np.int32) for x in fv1]; f2 = [np.ascontiguousarray(x, np.int32) for x in fv2]
        out = np.empty((P, s1 if v2 is not None else s2), np.int32); nm = np.empty(P, np.int32)
        v2 = None if v2 is None else np.ascontiguousarray(v2, np.uint8)
        side2 = [ptr(d2), ptr(a2)] + ([ptr(v2)] if v2 is not None else [])
        check(fn(self._h, P, ptr(d1), ptr(a1), ptr(v1), ptr(n1), s1, *[ptr(x) for x in f1], *side2, ptr(n2), s2, *[ptr(x) for x in f2],
                 C.c_float(self.nnratio), int(self.check_ori), ptr(out), ptr(nm)))
        return nm, out


def pack_fv(fvs, stride):
    """Per-frame FeatureVectors [(node (j,), start (j + 1,), feat (start[-1],)), ...] (Vocabulary.transform_fv's last three outputs) ->
    the batched CSR (node (P, stride), start (P, stride + 1), feat (P, stride), count (P,)) of the _fv entries."""
    assert stride <= Vocabulary.MAX_FV_FEATURES
    P = len(fvs)
    node = np.zeros((P, stride), np.int32); start = np.zeros((P, stride + 1), np.int32); feat = np.zeros((P, stride), np.int32); count = np.zeros(P, np.int32)
    for p, (nd, st, ft) in enumerate(fvs):
        j = len(nd); count[p] = j; node[p, :j] = nd; start[p, :j + 1] = st; feat[p, :len(ft)] = ft
    return node, start, feat, count
