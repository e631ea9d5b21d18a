"""ctypes binding of libcubemap_b200.so (the C ABI declared in include/cubemap_b200.h).

The CUDA library is mandatory: importing this module without the built .so, or creating a handle without a CUDA
device, raises — there is no CPU fallback anywhere in the package."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcubemap_b200.so")

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])


class CslamError(RuntimeError):
    pass


class CamParams(C.Structure):
    _fields_ = [("c", C.c_double), ("d", C.c_double), ("e", C.c_double), ("u0", C.c_double), ("v0", C.c_double),
                ("poly", C.c_double * 5), ("invpoly", C.c_double * 12), ("Iw", C.c_int32), ("Ih", C.c_int32),
                ("face_w", C.c_int32), ("face_h", C.c_int32), ("fov_deg", C.c_double)]


class OrbParams(C.Structure):
    _fields_ = [("nfeatures", C.c_int32), ("scale_factor", C.c_float), ("nlevels", C.c_int32), ("ini_th_fast", C.c_int32),
                ("min_th_fast", C.c_int32)]


class BAProblem(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("n_mp", C.c_int32), ("n_edges", C.c_int32), ("Tcw", C.c_void_p), ("kf_fixed", C.c_void_p),
                ("points", C.c_void_p), ("edge_mp", C.c_void_p), ("edge_kf", C.c_void_p), ("kp_xy", C.c_void_p),
                ("inv_sigma2", C.c_void_p), ("face_w", C.c_int32), ("face_h", C.c_int32)]


class BAResult(C.Structure):
    _fields_ = [("outlier", C.c_void_p), ("pose_fp64", C.c_void_p), ("points_fp64", C.c_void_p), ("lm_log", C.c_void_p),
                ("log_cap", C.c_int32), ("iterations", C.c_int32), ("trials", C.c_int32), ("stop_after_trials", C.c_int32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CslamError("libcubemap_b200.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                             "the package has no CPU fallback")
        _lib = C.CDLL(LIB_PATH)
        _lib.cslam_last_error.restype = C.c_char_p
        for kind in ("frontend", "matcher", "vocabulary", "tracker", "optimizer"):
            getattr(_lib, "cslam_%s_stream" % kind).restype = C.c_void_p
        for kind in ("frontend", "matcher", "tracker", "optimizer", "mapper"):
            getattr(_lib, "cslam_%s_launches" % kind).restype = C.c_int64
    return _lib


def check(rc):
    if rc != 0:
        raise CslamError("libcubemap_b200: error %d: %s" % (rc, lib().cslam_last_error().decode()))


class Handle:
    """One handle of the C ABI: cslam_<KIND>_create(&h, *args) on construction, cslam_<KIND>_destroy on close() (safe to call twice) or
    garbage collection. stream, launches and sync forward to cslam_<KIND>_stream / _launches / _sync; a handle whose C ABI lacks one of
    them raises AttributeError there."""
    KIND = None

    def __init__(self, *args):
        self._h = C.c_void_p()
        check(getattr(lib(), "cslam_%s_create" % self.KIND)(C.byref(self._h), *args))

    def close(self):
        if getattr(self, "_h", None):
            getattr(lib(), "cslam_%s_destroy" % self.KIND)(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def stream(self):
        return getattr(lib(), "cslam_%s_stream" % self.KIND)(self._h)

    @property
    def launches(self):
        return getattr(lib(), "cslam_%s_launches" % self.KIND)(self._h)

    def sync(self):
        check(getattr(lib(), "cslam_%s_sync" % self.KIND)(self._h))


def ptr(a):
    """Host numpy array or raw device address (int) -> c_void_p."""
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    return a.ctypes.data_as(C.c_void_p)


def cam_params(cfg):
    cp = CamParams()
    cp.c, cp.d, cp.e = cfg["Camera.c"], cfg["Camera.d"], cfg["Camera.e"]
    cp.u0, cp.v0 = cfg["Camera.u0"], cfg["Camera.v0"]
    for i in range(5):
        cp.poly[i] = cfg.get("Camera.a%d" % i, 0.0) if i < int(cfg["Camera.nrpol"]) else 0.0
    for i in range(12):
        cp.invpoly[i] = cfg.get("Camera.pol%d" % i, 0.0) if i < int(cfg["Camera.nrinvpol"]) else 0.0
    cp.Iw, cp.Ih = int(cfg["Camera.Iw"]), int(cfg["Camera.Ih"])
    cp.face_w, cp.face_h = int(cfg["CubeFace.w"]), int(cfg["CubeFace.h"])
    cp.fov_deg = cfg["Camera.fov"]
    return cp


def orb_params(cfg=None, **kw):
    op = OrbParams()
    if cfg is not None:
        op.nfeatures = int(cfg["ORBextractor.nFeatures"]); op.scale_factor = cfg["ORBextractor.scaleFactor"]
        op.nlevels = int(cfg["ORBextractor.nLevels"]); op.ini_th_fast = int(cfg["ORBextractor.iniThFAST"])
        op.min_th_fast = int(cfg["ORBextractor.minThFAST"])
    for k, v in kw.items():
        setattr(op, k, v)
    return op
