"""Host-side mirror of ORBVocabulary::transform (reference include/ORBVocabulary.h:35-36, ThirdParty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1262) on the C ABI."""

import numpy as np

from ._capi import Handle, check, lib, ptr


class Vocabulary(Handle):
    KIND = "vocabulary"

    def __init__(self, k, L, parent, is_leaf, desc, weight, max_frames=8, max_features=4096, device=0):
        parent = np.ascontiguousarray(parent, np.int32); is_leaf = np.ascontiguousarray(is_leaf, np.uint8); desc = np.ascontiguousarray(desc, np.uint8)
        weight = np.ascontiguousarray(weight, np.float64)
        super().__init__(int(device), int(k), int(L), len(parent), ptr(parent), ptr(is_leaf), ptr(desc), ptr(weight), int(max_frames), int(max_features))

    def transform(self, desc, n=None, levelsup=4):
        """desc: (stride, 32) or (F, stride, 32). Returns per frame: word (stride,), node (stride,), bow_word (m,), bow_val (m,)."""
        desc = np.ascontiguousarray(desc, np.uint8); single = desc.ndim == 2
        d = desc[None] if single else desc
        F, stride = d.shape[0], d.shape[1]
        n = np.full(F, stride, np.int32) if n is None else np.ascontiguousarray(n, np.int32).reshape(F)
        word = np.zeros((F, stride), np.int32); node = np.zeros((F, stride), np.int32); bw = np.zeros((F, stride), np.int32); bv = np.zeros((F, stride), np.float64); bc = np.zeros(F, np.int32)
        check(lib().cslam_bow_transform(self._h, ptr(d), ptr(n), stride, F, int(levelsup), ptr(word), ptr(node), ptr(bw), ptr(bv), ptr(bc)))
        out = [(word[f, :n[f]], node[f, :n[f]], bw[f, :bc[f]].copy(), bv[f, :bc[f]].copy()) for f in range(F)]
        return out[0] if single else out

    MAX_FV_FEATURES = 16384        # CSLAM_BOW_FV_MAX_FEATURES

    def transform_fv(self, desc, n=None, levelsup=4):
        """BowVector and FeatureVector (cslam_bow_transform_fv), stride <= 16384 whatever max_features. desc: (stride, 32) or (F, stride, 32).
        Returns per frame: bow_word (m,), bow_val (m,), fv_node (j,), fv_start (j + 1,), fv_feat (fv_start[-1],) - node fv_node[i] holds the
        features fv_feat[fv_start[i]:fv_start[i + 1]], ascending."""
        desc = np.ascontiguousarray(desc, np.uint8); single = desc.ndim == 2
        d = desc[None] if single else desc
        F, stride = d.shape[0], d.shape[1]
        n = np.full(F, stride, np.int32) if n is None else np.ascontiguousarray(n, np.int32).reshape(F)
        bw = np.zeros((F, stride), np.int32); bv = np.zeros((F, stride), np.float64); bc = np.zeros(F, np.int32)
        fn = np.zeros((F, stride), np.int32); fs = np.zeros((F, stride + 1), np.int32); ff = np.zeros((F, stride), np.int32); fc = np.zeros(F, np.int32)
        check(lib().cslam_bow_transform_fv(self._h, ptr(d), ptr(n), stride, F, int(levelsup), ptr(bw), ptr(bv), ptr(bc), ptr(fn), ptr(fs), ptr(ff), ptr(fc)))
        out = []
        for f in range(F):
            j = fc[f]
            out.append((bw[f, :bc[f]].copy(), bv[f, :bc[f]].copy(), fn[f, :j].copy(), fs[f, :j + 1].copy(), ff[f, :fs[f, j]].copy()))
        return out[0] if single else out
