"""ctypes wrappers for SearchForInitialization (ORACLE: test infrastructure, not product code; recipe oracle/init_search_dropin.mk):
  search / features_in_area      the oracle's restatement, oracle/liboracle_init.so (init_search.h);
  RefInit                        the reference's own body and GetFeaturesInArea, oracle/_ref/libref_init.so (built where the reference tree exists)."""
import ctypes as C
import os
import subprocess

import numpy as np

from .oracle import _f32, _p, _u8

_HERE = os.path.dirname(os.path.abspath(__file__))
_MK = ["make", "-s", "-C", _HERE, "-f", "init_search_dropin.mk"]
_LIBS = {}


def build():
    subprocess.check_call(_MK + ["liboracle_init.so"])


def _lib(name):
    if name not in _LIBS:
        path = os.path.join(_HERE, name)
        if name == "liboracle_init.so" and not os.path.exists(path):
            build()
        elif name.startswith("_ref/") and os.path.isdir(os.environ.get("REF", "/root/reference")):
            subprocess.check_call(_MK + ["-j8", name])
        _LIBS[name] = C.CDLL(path)
    return _LIBS[name]


def _windows(queries):
    q = np.asarray(queries, np.float64)
    return _f32(q[:, :3]), np.ascontiguousarray(q[:, 3:5], np.int32)


def search(k1, d1, k2, d2, prev_xy, face_w, window_size=100, nnratio=0.9, checkOri=True):
    """ORBMatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) (reference src/ORBMatcher.cpp:676-794).
    Returns (nmatches, match12, prev_xy updated)."""
    k1 = np.ascontiguousarray(k1); k2 = np.ascontiguousarray(k2); d1 = _u8(d1); d2 = _u8(d2); xy = _f32(prev_xy).reshape(-1, 2).copy()
    m = np.empty(len(k1), np.int32)
    n = _lib("liboracle_init.so").orc_init_search(_p(k2), _p(d2), len(k2), int(face_w), _p(k1), _p(d1), len(k1), _p(xy), int(window_size), C.c_float(nnratio), int(checkOri), _p(m))
    return n, m, xy


def _area(fn, head, queries):
    xyr, lv = _windows(queries)
    counts = np.zeros(len(xyr), np.int32); cap = 1 << 24; idx = np.zeros(cap, np.int32)
    m = fn(*head, len(xyr), _p(xyr), _p(lv), _p(counts), _p(idx), cap)
    assert m <= cap
    return counts, idx[:m].copy()


def features_in_area(kps, face_w, queries):
    """The oracle's Frame::GetFeaturesInArea, uncapped, per query (x, y, r, min_level, max_level): (counts, indices concatenated)."""
    kps = np.ascontiguousarray(kps)
    return _area(_lib("liboracle_init.so").orc_init_features_in_area, (_p(kps), len(kps), int(face_w)), queries)


def ref_available():
    return os.path.exists(os.path.join(_HERE, "_ref", "libref_init.so"))


class RefInit:
    """The reference's own SearchForInitialization / GetFeaturesInArea on Frames of given key points, one camera configuration."""

    def __init__(self, cam_params):
        self.L = _lib("_ref/libref_init.so"); self.cp = cam_params

    def _cam(self):
        self.L.ref_init_set_camera(C.byref(self.cp))
        return self.L

    def search_for_initialization(self, k1, d1, k2, d2, prev_xy, window_size=100, nnratio=0.9, checkOri=True):
        k1 = np.ascontiguousarray(k1); k2 = np.ascontiguousarray(k2); d1 = _u8(d1); d2 = _u8(d2); xy = _f32(prev_xy).reshape(-1, 2).copy()
        m = np.empty(len(k1), np.int32)
        n = self._cam().ref_init_search_for_initialization(len(k1), _p(k1), _p(d1), len(k2), _p(k2), _p(d2), _p(xy), int(window_size), C.c_float(nnratio), int(checkOri), _p(m))
        return n, m, xy

    def features_in_area_given(self, kps, queries):
        kps = np.ascontiguousarray(kps)
        return _area(self._cam().ref_init_features_in_area, (len(kps), _p(kps)), queries)
