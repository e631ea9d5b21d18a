"""ctypes wrapper around oracle/_ref/libref.so = the reference's own sources compiled unmodified against the cv:: shim
(ORACLE: test infrastructure, not product code; recipe in oracle/Makefile, entry points in oracle/ref_api.cpp, scenes in oracle/ref_scene.cpp).

The library is built in the build container (where /root/reference exists) and travels to the GPU box as a prebuilt file;
nothing here reads /root/reference at run time."""
import ctypes as C
import os
import subprocess

import numpy as np

from .oracle import KP_DTYPE, _f32, _p, _u8

_HERE = os.path.dirname(os.path.abspath(__file__))
PIN_ALLOC, PIN_SINCOS = 1, 2
_LIBS = {}


def available(variant="libref.so"):
    return os.path.exists(os.path.join(_HERE, "_ref", variant))


def build(target="ref"):
    """Only possible where the reference tree is present (the build container)."""
    if os.path.isdir(os.environ.get("REF", "/root/reference")):
        subprocess.check_call(["make", "-s", "-j8", "-C", _HERE, target])


def lib(variant="libref.so"):
    if variant not in _LIBS:
        path = os.path.join(_HERE, "_ref", variant)
        build("_ref/" + variant)       # where the reference tree exists, make brings the library up to date with its sources' contents
        L = C.CDLL(path)
        for name, t in (("ref_orb_create", C.c_void_p), ("ref_frame_from_image", C.c_void_p), ("ref_voc_load", C.c_void_p), ("ref_cos_fov_th", C.c_float),
                        ("ref_vector_sigma", C.c_float), ("ref_arena_used", C.c_size_t), ("ref_warp_extract_batch_out", C.c_long)):
            getattr(L, name).restype = t
        _LIBS[variant] = L
    return _LIBS[variant]


class Ref:
    """One camera configuration of the compiled reference (CamModelGeneral is a process-wide singleton, src/System.cpp:89)."""

    def __init__(self, cam_params, pins=PIN_ALLOC | PIN_SINCOS, variant="libref.so"):
        self.L = lib(variant)
        self.cp = cam_params
        self.L.ref_set_pins(0)
        self._cam()
        self.pins = pins

    def _cam(self):
        """The library, with the singleton camera set to this configuration."""
        self.L.ref_set_camera(C.byref(self.cp))
        return self.L

    def _pinned(self):
        self._cam().ref_set_pins(int(self.pins))

    def cos_fov_th(self):
        return float(self.L.ref_cos_fov_th())

    def build_maps(self):
        W3, H3 = 3 * self.cp.faceW, 3 * self.cp.faceH
        m1 = np.empty((H3, W3), np.float32); m2 = np.empty((H3, W3), np.float32)
        self._cam().ref_build_maps(_p(m1), _p(m2))
        return m1, m2

    def warp(self, fisheye, m1, m2, canvas=None):
        fisheye = _u8(fisheye)
        if canvas is None:
            canvas = np.zeros((3 * self.cp.faceH, 3 * self.cp.faceW), np.uint8)
        self._cam().ref_warp(_p(fisheye), _p(m1), _p(m2), _p(canvas))
        return canvas

    def extractor(self, nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST):
        return RefORBextractor(self, nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST)

    def search_by_projection_last(self, kCur, dCur, TcwCur, kLast, TcwLast, hasMP, Xw, dMP, mpObs, curTaken, th, checkOri=True):
        kCur = np.ascontiguousarray(kCur); kLast = np.ascontiguousarray(kLast)
        a = [_u8(dCur), _f32(TcwCur).reshape(16), _f32(TcwLast).reshape(16), _u8(hasMP), _f32(Xw), _u8(dMP), np.ascontiguousarray(mpObs, np.int32), _u8(curTaken)]
        match = np.empty(len(kCur), np.int32)
        n = self._cam().ref_search_by_projection_last(len(kCur), _p(kCur), _p(a[0]), _p(a[1]), len(kLast), _p(kLast), _p(a[2]), _p(a[3]), _p(a[4]), _p(a[5]), _p(a[6]), _p(a[7]),
                                                 C.c_float(th), int(checkOri), _p(match))
        return n, match

    def search_by_projection_local(self, kF, dF, inView, projXY, level, viewCos, dMP, mpObs, fTaken, th, nnratio):
        kF = np.ascontiguousarray(kF)
        a = [_u8(dF), _u8(inView), _f32(projXY), np.ascontiguousarray(level, np.int32), _f32(viewCos), _u8(dMP), np.ascontiguousarray(mpObs, np.int32), _u8(fTaken)]
        match = np.empty(len(kF), np.int32)
        n = self._cam().ref_search_by_projection_local(len(kF), _p(kF), _p(a[0]), len(a[1]), _p(a[1]), _p(a[2]), _p(a[3]), _p(a[4]), _p(a[5]), _p(a[6]), _p(a[7]), C.c_float(th),
                                                  C.c_float(nnratio), _p(match))
        return n, match

    def frame_index(self, kps):
        """Rays, mGrid sizes (5 x 50 x 50) and the cell contents in (face, col, row) order of a Frame holding the given key points."""
        kps = np.ascontiguousarray(kps); n = len(kps)
        rays = np.zeros((n, 3), np.float32); count = np.zeros((5, 50, 50), np.int32); idx = np.zeros(max(n, 1), np.int32)
        self._cam().ref_frame_index(n, _p(kps), _p(rays), _p(count), _p(idx))
        return rays, count, idx[:int(count.sum())].copy()

    def ray_to_cubemap(self, xyz):
        xyz = _f32(xyz).reshape(-1, 3); uv = np.zeros((len(xyz), 2), np.float32); faces = np.zeros(len(xyz), np.int32)
        self._cam()
        for i in range(len(xyz)):
            u = C.c_float(); v = C.c_float()
            faces[i] = self.L.ref_ray_to_cubemap(C.c_float(xyz[i, 0]), C.c_float(xyz[i, 1]), C.c_float(xyz[i, 2]), C.byref(u), C.byref(v))
            uv[i] = (u.value, v.value)
        return uv, faces

    def warp_extract_batch_out(self, fisheyes, m1, m2, mask, nfeatures, scaleFactor, nlevels, iniTh, minTh, nthreads, cap):
        fisheyes = _u8(fisheyes); mask = _u8(mask); F = fisheyes.shape[0]
        kps = np.zeros((F, cap), KP_DTYPE); desc = np.zeros((F, cap, 32), np.uint8); n = np.zeros(F, np.int32)
        self._cam().ref_set_pins(0)                    # the timed baseline runs the stock code paths (glibc malloc / sincosf)
        self.L.ref_warp_extract_batch_out(_p(fisheyes), F, _p(m1), _p(m2), _p(mask), int(nfeatures), C.c_float(scaleFactor), int(nlevels), int(iniTh), int(minTh), int(nthreads), int(cap),
                                          _p(kps), _p(desc), _p(n))
        return kps, desc, n

    # ---- LocalMapping feature operations (src/MapPoint.cpp:243-303, src/ORBMatcher.cpp:971-1240) on reference KeyFrame / MapPoint objects
    def distinctive_descriptor(self, desc):
        desc = _u8(desc).reshape(-1, 32); out = np.zeros(32, np.uint8)
        self._cam().ref_distinctive_descriptor(len(desc), _p(desc), _p(out))
        return out

    def fuse(self, kKF, dKF, Tcw, Xw, kObs, dMP, TcwObs, th=3.0):
        """Returns nFused, valid, level (the pre-tests / PredictScale of Fuse, from the reference's own getters), idxInKF per MapPoint."""
        kKF = np.ascontiguousarray(kKF); kObs = np.ascontiguousarray(kObs); Xw = _f32(Xw); n = len(Xw)
        a = [_u8(dKF), _f32(Tcw).reshape(16), _u8(dMP), _f32(TcwObs).reshape(16)]
        valid = np.zeros(n, np.uint8); level = np.zeros(n, np.int32); idx = np.zeros(n, np.int32)
        nf = self._cam().ref_fuse(len(kKF), _p(kKF), _p(a[0]), _p(a[1]), n, _p(Xw), _p(kObs), _p(a[2]), _p(a[3]), C.c_float(th), _p(valid), _p(level), _p(idx))
        return nf, valid, level, idx

    def search_for_triangulation(self, k1, d1, Tcw1, hasMP1, node1, k2, d2, Tcw2, hasMP2, node2, E12, checkOri=False):
        k1 = np.ascontiguousarray(k1); k2 = np.ascontiguousarray(k2)
        a = [_u8(d1), _f32(Tcw1).reshape(16), _u8(hasMP1), np.ascontiguousarray(node1, np.int32), _u8(d2), _f32(Tcw2).reshape(16), _u8(hasMP2), np.ascontiguousarray(node2, np.int32),
             _f32(E12).reshape(9)]
        Ow1 = np.zeros(3, np.float32); m = np.empty(len(k1), np.int32)
        n = self._cam().ref_search_for_triangulation(len(k1), _p(k1), _p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), len(k2), _p(k2), _p(a[4]), _p(a[5]), _p(a[6]), _p(a[7]), _p(a[8]),
                                                int(checkOri), _p(Ow1), _p(m))
        return n, m, Ow1

    def vector_sigma(self, kx, ky, normal_rig):
        nr = _f32(normal_rig)
        return float(self._cam().ref_vector_sigma(C.c_float(kx), C.c_float(ky), _p(nr)))

    def descriptor_distance(self, a, b):
        a = _u8(a); b = _u8(b)
        return self.L.ref_descriptor_distance(_p(a), _p(b))


class RefORBextractor:
    def __init__(self, ref, nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST):
        self.ref = ref; self.nlevels = nlevels
        self._h = C.c_void_p(ref.L.ref_orb_create(int(nfeatures), C.c_float(scaleFactor), int(nlevels), int(iniThFAST), int(minThFAST)))

    def __del__(self):
        try:
            self.ref.L.ref_set_pins(0)
            self.ref.L.ref_orb_destroy(self._h)
        except Exception:
            pass

    def __call__(self, image, mask):
        image = _u8(image); mask = _u8(mask)
        assert image.shape == mask.shape
        self.ref._pinned()
        n = self.ref.L.ref_orb_extract(self._h, _p(image), image.shape[1], image.shape[0], _p(mask))
        self.ref.L.ref_set_pins(0)
        kps = np.empty(n, KP_DTYPE); desc = np.empty((n, 32), np.uint8)
        self.ref.L.ref_orb_result(self._h, _p(kps), _p(desc))
        return kps, desc

    def level_image(self, level):
        w = C.c_int(); h = C.c_int()
        self.ref.L.ref_orb_level_size(self._h, level, C.byref(w), C.byref(h))
        out = np.zeros((h.value, w.value), np.uint8)
        self.ref.L.ref_orb_level_image(self._h, level, _p(out))
        return out


class RefFrame:
    """The reference's Frame built from an image like Tracking does (extraction, ComputeKeyPointRays, AssignFeaturesToGrid)."""
    GRID = (5, 50, 50)

    def __init__(self, rex, image, mask):
        image = _u8(image); mask = _u8(mask)
        self.ref = rex.ref; self.rex = rex
        self.ref._pinned()
        self._h = C.c_void_p(self.ref.L.ref_frame_from_image(rex._h, _p(image), _p(mask), image.shape[0], image.shape[1]))
        self.ref.L.ref_set_pins(0)
        self.N = self.ref.L.ref_frame_n(self._h)
        n = self.N
        self.kps = np.empty(n, KP_DTYPE); self.desc = np.empty((n, 32), np.uint8); self.rays = np.empty((n, 3), np.float32)
        self.grid_count = np.empty(self.GRID, np.int32)
        self.ref.L.ref_frame_get(self._h, _p(self.kps), _p(self.desc), _p(self.rays), _p(self.grid_count))

    def __del__(self):
        try:
            self.ref.L.ref_frame_destroy(self._h)
        except Exception:
            pass

    def grid_cell(self, face, col, row):
        buf = np.empty(4096, np.int32)
        n = self.ref.L.ref_frame_grid_cell(self._h, int(face), int(col), int(row), _p(buf), 4096)
        return buf[:n].copy()

    def features_in_area(self, x, y, r, min_level=-1, max_level=-1):
        buf = np.empty(8192, np.int32)
        n = self.ref.L.ref_frame_features_in_area(self._h, C.c_float(x), C.c_float(y), C.c_float(r), int(min_level), int(max_level), _p(buf), 8192)
        return buf[:n].copy()


class RefVocabulary:
    """The reference's ORBVocabulary (DBoW2 TemplatedVocabulary<FORB>) loaded from a text file in ORBvoc.txt's format."""

    def __init__(self, path, variant="libref.so"):
        self.L = lib(variant)
        self._h = C.c_void_p(self.L.ref_voc_load(str(path).encode()))
        if not self._h:
            raise RuntimeError("vocabulary load failed: " + str(path))

    def __del__(self):
        try:
            self.L.ref_voc_destroy(self._h)
        except Exception:
            pass

    def size(self):
        return self.L.ref_voc_size(self._h)

    def transform(self, feats, levelsup=4):
        feats = _u8(feats); n = len(feats)
        bw = np.zeros(max(n, 1), np.int32); bv = np.zeros(max(n, 1), np.float64); node = np.zeros(max(n, 1), np.int32)
        m = self.L.ref_voc_transform(self._h, _p(feats), n, int(levelsup), _p(bw), _p(bv), _p(node))
        return bw[:m].copy(), bv[:m].copy(), node[:n].copy()
