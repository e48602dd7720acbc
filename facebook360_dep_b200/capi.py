"""ctypes binding of include/derp_b200.h.

``load_cuda()`` -> facebook360_dep_b200/libderp_b200.so, the product (sm_90a CUDA).  It raises if the library is
missing or reports a different backend: there is no CPU fallback.  The checker libraries that export the same ABI
(the oracle, the compiled reference) are loaded by tests/oracle_libs.py — test infrastructure lives outside
this package; ``Library`` below is just the generic ctypes binding of the header.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
# DERP_B200_LIB: kernel-tuning experiments load an alternative build of the SAME CUDA library
CUDA_LIB = os.environ.get("DERP_B200_LIB") or os.path.join(_HERE, "libderp_b200.so")

CAM_FTHETA, CAM_RECTILINEAR, CAM_EQUISOLID, CAM_ORTHOGRAPHIC = 0, 1, 2, 3
CAM_TYPES = {"FTHETA": 0, "RECTILINEAR": 1, "EQUISOLID": 2, "ORTHOGRAPHIC": 3}

OK, EINVAL, ECUDA, ENOMEM, ESTATE, ECOVERAGE = 0, -1, -2, -3, -4, -5


class CameraDesc(C.Structure):
    _fields_ = [
        ("type", C.c_int32),
        ("has_principal", C.c_int32),
        ("has_fov", C.c_int32),
        ("reserved", C.c_int32),
        ("origin", C.c_double * 3),
        ("forward", C.c_double * 3),
        ("up", C.c_double * 3),
        ("right", C.c_double * 3),
        ("resolution", C.c_double * 2),
        ("principal", C.c_double * 2),
        ("focal", C.c_double * 2),
        ("distortion", C.c_double * 3),
        ("fov", C.c_double),
    ]


class LevelParams(C.Structure):
    _fields_ = [
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("level", C.c_int32),
        ("num_levels", C.c_int32),
        ("full_width", C.c_int32),
        ("full_height", C.c_int32),
        ("var_noise_floor", C.c_float),
        ("var_high_thresh", C.c_float),
        ("use_foreground_masks", C.c_int32),
        ("reserved", C.c_int32),
    ]


class ProcessOpts(C.Structure):
    _fields_ = [
        ("num_depths", C.c_int32),
        ("min_depth_m", C.c_float),
        ("max_depth_m", C.c_float),
        ("partial_coverage", C.c_int32),
        ("random_proposals", C.c_int32),
        ("ping_pong_iterations", C.c_int32),
        ("mismatches_start_level", C.c_int32),
        ("do_bilateral_filter", C.c_int32),
        ("do_median_filter", C.c_int32),
        ("reserved", C.c_int32),
    ]


def camera_desc_from_json(cam):
    """One entry of the rig JSON's "cameras" array -> CameraDesc (Camera.cpp:30-75)."""
    d = CameraDesc()
    d.type = CAM_TYPES[cam["type"]]
    for k in ("origin", "forward", "up", "right"):
        for i in range(3):
            getattr(d, k)[i] = float(cam[k][i])
    for i in range(2):
        d.resolution[i] = float(cam["resolution"][i])
        d.focal[i] = float(cam["focal"][i])
    if "principal" in cam:
        d.has_principal = 1
        for i in range(2):
            d.principal[i] = float(cam["principal"][i])
    dist = list(cam.get("distortion", []))
    if len(dist) > 3:
        raise ValueError("bad distortion")
    for i in range(3):
        d.distortion[i] = float(dist[i]) if i < len(dist) else 0.0
    if "fov" in cam:
        d.has_fov = 1
        d.fov = float(cam["fov"])
    return d


def rig_descs(rig_json):
    cams = rig_json["cameras"]
    arr = (CameraDesc * len(cams))()
    for i, c in enumerate(cams):
        arr[i] = camera_desc_from_json(c)
    return arr


_p = C.POINTER
_SIGS = {
    "derp_backend": (C.c_char_p, []),
    "derp_last_error": (C.c_char_p, []),
    "derp_set_threads": (C.c_int, [C.c_int]),
    "derp_create": (C.c_int, [_p(CameraDesc), C.c_int, _p(C.c_int32), C.c_int, C.c_int, _p(C.c_void_p)]),
    "derp_destroy": (None, [C.c_void_p]),
    "derp_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "derp_sync": (C.c_int, [C.c_void_p]),
    "derp_get_launch_count": (C.c_int, [C.c_void_p, _p(C.c_uint64)]),
    "derp_profile": (C.c_int, [C.c_void_p, C.c_int]),
    "derp_get_profile": (C.c_int, [C.c_void_p, _p(C.c_double), _p(C.c_uint64)]),
    "derp_get_profile_ping_pong": (C.c_int, [C.c_void_p, _p(C.c_double), _p(C.c_uint64), _p(C.c_uint64), _p(C.c_uint64)]),
    "derp_set_sweep_mode": (C.c_int, [C.c_void_p, C.c_int]),
    "derp_get_sweep_stats": (C.c_int, [C.c_void_p, _p(C.c_uint64), _p(C.c_uint64)]),
    "derp_level_begin": (C.c_int, [C.c_void_p, _p(LevelParams)]),
    "derp_set_colors": (C.c_int, [C.c_void_p, _p(C.c_void_p)]),
    "derp_set_foreground_masks": (C.c_int, [C.c_void_p, _p(C.c_void_p)]),
    "derp_set_background_disparity": (C.c_int, [C.c_void_p, _p(C.c_void_p)]),
    "derp_reproject": (C.c_int, [C.c_void_p, C.c_int]),
    "derp_brute_force": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_void_p]),
    "derp_random_proposals": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float]),
    "derp_ping_pong": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "derp_mismatches": (C.c_int, [C.c_void_p]),
    "derp_bilateral": (C.c_int, [C.c_void_p, C.c_int]),
    "derp_median": (C.c_int, [C.c_void_p, C.c_int]),
    "derp_mask_fov": (C.c_int, [C.c_void_p, C.c_int]),
    "derp_upsample_from": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "derp_level_keep": (C.c_int, [C.c_void_p]),
    "derp_upsample_from_kept": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "derp_process_level": (C.c_int, [C.c_void_p, _p(ProcessOpts)]),
    "derp_level_estimate": (C.c_int, [C.c_void_p, _p(ProcessOpts)]),
    "derp_level_filter": (C.c_int, [C.c_void_p, _p(ProcessOpts)]),
    "derp_disparity_device_ptr": (C.c_void_p, [C.c_void_p, C.c_int]),
    "derp_gather_disparities": (C.c_int, [C.c_void_p, C.c_void_p]),
    "derp_mismatches_gathered": (C.c_int, [C.c_void_p]),
    "derp_eval_cost": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "derp_set_disparity": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "derp_get_disparity": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "derp_get_fov_mask": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "derp_get_mismatch_mask": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "derp_get_variance": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "derp_get_var_noise_floor": (C.c_int, [C.c_void_p, _p(C.c_float)]),
    "derp_get_proj_warp": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "derp_get_proj_color": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "derp_get_proj_bias": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "derp_get_counters": (C.c_int, [C.c_void_p, _p(C.c_uint64), _p(C.c_uint64)]),
    "derp_temporal_filter": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, _p(C.c_void_p), _p(C.c_void_p),
                                       _p(C.c_void_p), C.c_int, C.c_float, C.c_int, C.c_float, C.c_float,
                                       C.c_float, C.c_void_p]),
    "derp_joint_bilateral_f32": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p]),
    "derp_upsample_disparity": (C.c_int, [C.c_int, _p(CameraDesc), C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "derp_device_alloc": (C.c_int, [C.c_int, C.c_size_t, _p(C.c_void_p)]),
    "derp_device_free": (C.c_int, [C.c_int, C.c_void_p]),
    "derp_device_copy": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]),
    "derp_downscale_area": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]),
    "derp_foreground_mask": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int,
                                       C.c_void_p]),
    "derp_camera_mesh_size": (C.c_int, [C.c_int, C.c_int, C.c_double, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "derp_camera_mesh": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double,
                                   C.c_float, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                   C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "derp_camera_mesh_simplified": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double,
                                              C.c_double, C.c_float, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                              C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "derp_bc7_compress": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "derp_bc7_compress_image": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
}

ABI_SYMBOLS = sorted(_SIGS)


class DerpError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("derp error %d: %s" % (code, msg))
        self.code = code


def _bind(library, sigs, optional=()):
    """Opens `library` (a path, or a binding of one) and sets restype and argtypes of every entry point in `sigs`.
    Returns (path, CDLL).  A missing entry point raises AttributeError unless its name is in `optional`."""
    path = getattr(library, "path", library)
    if not os.path.exists(path):
        raise FileNotFoundError(
            "%s not found — build it first (python -c 'import __graft_entry__ as g; g.build()')" % path)
    lib = C.CDLL(path, mode=C.RTLD_LOCAL)
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name, None) if name in optional else getattr(lib, name)
        if fn is not None:
            fn.restype = res
            fn.argtypes = args
    return path, lib


class _Binding:
    """A library whose entry points return a DERP_* code and leave the message in derp_last_error."""

    def _check(self, rc):
        if rc != 0:
            raise DerpError(rc, self.lib.derp_last_error().decode())


class Library(_Binding):
    """One loaded shared library exporting the derp_b200.h ABI."""

    def __init__(self, path):
        self.path, self.lib = _bind(path, _SIGS)
        self.backend = self.lib.derp_backend().decode()

    check = _Binding._check

    def set_threads(self, n):
        self.check(self.lib.derp_set_threads(int(n)))

    # ---- stand-alone entry points ----------------------------------------------------------
    def temporal_filter(self, guides, disps, masks, frame_offset, sigma, spatial_radius, w0, w1, w2, device=0):
        T = len(guides)
        H, W = disps[0].shape
        g = [np.ascontiguousarray(x, np.uint16) for x in guides]
        d = [np.ascontiguousarray(x, np.float32) for x in disps]
        m = [np.ascontiguousarray(x, np.uint8) for x in masks]
        out = np.empty((H, W), np.float32)
        self.check(self.lib.derp_temporal_filter(
            device, W, H, T, _ptr_array(g), _ptr_array(d), _ptr_array(m), frame_offset, sigma,
            spatial_radius, w0, w1, w2, out.ctypes.data))
        return out

    def joint_bilateral_f32(self, image, guide, mask, radius, sigma, w0, w1, w2, device=0):
        H, W = image.shape
        image = np.ascontiguousarray(image, np.float32)
        guide = np.ascontiguousarray(guide, np.float32)
        mask = np.ascontiguousarray(mask, np.uint8)
        out = np.empty((H, W), np.float32)
        self.check(self.lib.derp_joint_bilateral_f32(device, W, H, image.ctypes.data, guide.ctypes.data,
                                                     mask.ctypes.data, radius, sigma, w0, w1, w2,
                                                     out.ctypes.data))
        return out

    def downscale_area(self, image, out_w, out_h, device=0):
        """cv::resize INTER_AREA of a u16 HxWx3 image (shrinking)."""
        image = np.ascontiguousarray(image, np.uint16)
        h, w = image.shape[:2]
        out = np.empty((out_h, out_w, 3), np.uint16)
        self.check(self.lib.derp_downscale_area(device, image.ctypes.data, w, h, out.ctypes.data, out_w, out_h))
        return out

    def foreground_mask(self, templ, frame, blur_radius=1, threshold=0.04, morph_closing_size=4, device=0):
        """generateForegroundMask (BackgroundSubtractionUtil.h:20-59) for one camera; returns a uint8 0/1 mask."""
        templ = np.ascontiguousarray(templ, np.uint16)
        frame = np.ascontiguousarray(frame, np.uint16)
        h, w = templ.shape[:2]
        out = np.empty((h, w), np.uint8)
        self.check(self.lib.derp_foreground_mask(device, templ.ctypes.data, frame.ctypes.data, w, h, blur_radius, threshold,
                                                 morph_closing_size, out.ctypes.data))
        return out

    def camera_mesh(self, disparity, resolution, scalar_focal, depth_scale=1.0, tear_ratio=0.95, foreground_mask=None,
                    device=0, triangles=0):
        """The camera mesh ConvertToBinary builds from one disparity map before simplification
        (ConvertToBinary.cpp:150-183, MeshUtil.h): returns (vertexes float32 [nv, 3], faces uint32 [nf, 3])."""
        disparity = np.ascontiguousarray(disparity, np.float32)
        h, w = disparity.shape
        mw, mh = C.c_int(), C.c_int()
        self.check(self.lib.derp_camera_mesh_size(w, h, depth_scale, C.byref(mw), C.byref(mh)))
        cells = mw.value * mh.value
        vtx = np.empty((max(cells, 1), 3), np.float32)
        idx = np.empty((max(2 * cells, 1), 3), np.uint32)
        fm = None if foreground_mask is None else np.ascontiguousarray(foreground_mask, np.uint8)
        nv, nf = C.c_uint64(), C.c_uint64()
        head = (device, disparity.ctypes.data, w, h, depth_scale, float(resolution[0]), float(resolution[1]),
                float(scalar_focal), tear_ratio, _dp(fm), 0 if fm is None else fm.shape[1], 0 if fm is None else fm.shape[0])
        tail = (vtx.ctypes.data, idx.ctypes.data, C.byref(nv), C.byref(nf))
        if triangles > 0:  # + MeshSimplifier with convertDepth's constants (ConvertToBinary.cpp:186-203)
            self.check(self.lib.derp_camera_mesh_simplified(*head, int(triangles), *tail))
        else:
            self.check(self.lib.derp_camera_mesh(*head, *tail))
        return vtx[:nv.value].copy(), idx[:nf.value].copy()

    def bc7_compress(self, rgba, device=0):
        """CompressBlocksBC7 with the veryfast profile (BC7Util.h:69-76) of an opaque RGBA8 surface [h, w, 4]:
        returns the w * h output bytes as [w * h / 16, 16] (16-byte blocks; rows of partial blocks stay zero)."""
        rgba = np.ascontiguousarray(rgba, np.uint8)
        h, w, c = rgba.shape
        assert c == 4
        out = np.empty(w * h, np.uint8)
        self.check(self.lib.derp_bc7_compress(device, rgba.ctypes.data, w, h, out.ctypes.data))
        return out

    def bc7_compress_image(self, pixels, gamma=2.2 / 1.8, device=0):
        """bc7_util::compressBC7 up to the file write (BC7Util.h:45-76) of an image as cv2.imread(IMREAD_UNCHANGED)
        returns it: uint8 / uint16 [h, w, 3 or 4] in B, G, R[, A] order.  Returns the w * h bytes of the .bc7 file."""
        pixels = np.ascontiguousarray(pixels)
        assert pixels.dtype in (np.uint8, np.uint16) and pixels.ndim == 3 and pixels.shape[2] in (3, 4)
        h, w, c = pixels.shape
        out = np.empty(w * h, np.uint8)
        self.check(self.lib.derp_bc7_compress_image(device, pixels.ctypes.data, pixels.dtype.itemsize * 8, c, w, h, gamma,
                                                    out.ctypes.data))
        return out

    def upsample_disparity(self, cam_desc, coarse, out_w, out_h, background_up=None, coarse_mask=None,
                           fine_mask=None, use_foreground_masks=False, device=0):
        coarse = np.ascontiguousarray(coarse, np.float32)
        ch, cw = coarse.shape
        bg = None if background_up is None else np.ascontiguousarray(background_up, np.float32)
        cm = None if coarse_mask is None else np.ascontiguousarray(coarse_mask, np.uint8)
        fm = None if fine_mask is None else np.ascontiguousarray(fine_mask, np.uint8)
        out = np.empty((out_h, out_w), np.float32)
        self.check(self.lib.derp_upsample_disparity(
            device, C.byref(cam_desc), coarse.ctypes.data, cw, ch, _dp(bg), _dp(cm), _dp(fm), out_w, out_h,
            int(use_foreground_masks), out.ctypes.data))
        return out


def _dp(a):
    return None if a is None else a.ctypes.data


def _ptr_array(arrs):
    pa = (C.c_void_p * len(arrs))()
    for i, a in enumerate(arrs):
        pa[i] = a.ctypes.data
    return pa


# ---- include/derp_blur.h ------------------------------------------------------------------------------------------
_BLUR_SIGS = {
    "derp_last_error": (C.c_char_p, []),
    "derp_gaussian_blur": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
}
BLUR_SYMBOLS = ["derp_gaussian_blur"]


class Blur(_Binding):
    """ctypes binding of include/derp_blur.h on a loaded library: ``Blur(load_cuda())``."""

    def __init__(self, library):
        self.path, self.lib = _bind(library, _BLUR_SIGS)

    check = _Binding._check

    def gaussian_blur(self, image, radius, device=0):
        """cv::GaussianBlur((2 radius + 1)^2, sigma 0) of a u16 HxWx3 image (cv_util::gaussianBlur), radius 0 to 64."""
        image = np.ascontiguousarray(image, np.uint16)
        h, w = image.shape[:2]
        out = np.empty((h, w, 3), np.uint16)
        self.check(self.lib.derp_gaussian_blur(device, image.ctypes.data, w, h, radius, out.ctypes.data))
        return out


# ---- include/derp_resize.h ----------------------------------------------------------------------------------------
_RESIZE_SIGS = {
    "derp_last_error": (C.c_char_p, []),
    "derp_resize_area": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                   C.c_int]),
}
RESIZE_SYMBOLS = ["derp_resize_area"]
RESIZE_DTYPES = {np.dtype(np.uint8): 8, np.dtype(np.uint16): 16, np.dtype(np.float32): 32}


class Resize(_Binding):
    """ctypes binding of include/derp_resize.h on a loaded library: ``Resize(load_cuda())``."""

    def __init__(self, library):
        self.path, self.lib = _bind(library, _RESIZE_SIGS)

    check = _Binding._check

    def resize_area(self, image, out_w, out_h, threshold=None, device=0):
        """cv2.resize(image, (out_w, out_h), interpolation=INTER_AREA) [then cv2.threshold(., threshold, 255,
        THRESH_BINARY)] of a uint8, uint16 or float32 HxW or HxWxC image, C = 1, 3 or 4; the result has image's layout."""
        image = np.ascontiguousarray(image)
        bits = RESIZE_DTYPES.get(image.dtype)
        if bits is None:
            raise ValueError("resize_area: uint8, uint16 or float32 samples, not %s" % image.dtype)
        h, w = image.shape[:2]
        c = image.shape[2] if image.ndim == 3 else 1
        out = np.empty((out_h, out_w) + image.shape[2:], image.dtype)
        self.check(self.lib.derp_resize_area(device, image.ctypes.data, bits, c, w, h, out.ctypes.data, out_w, out_h,
                                             -1 if threshold is None else int(threshold)))
        return out


# ---- include/derp_rephoto.h ---------------------------------------------------------------------------------------
_REPHOTO_SIGS = {
    "derp_last_error": (C.c_char_p, []),
    "derp_rephoto_cubemap": (C.c_int, [C.c_int, _p(CameraDesc), C.c_int, _p(C.c_void_p), _p(C.c_void_p), C.c_int, C.c_int,
                                       C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "derp_rephoto_score": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p]),
}
REPHOTO_SYMBOLS = sorted(k for k in _REPHOTO_SIGS if k.startswith("derp_rephoto_"))
REPHOTO_METHODS = {"MSSIM": 0, "NCC": 1}


class Rephoto(_Binding):
    """ctypes binding of include/derp_rephoto.h on a loaded library: ``Rephoto(load_cuda())`` for the product, or a
    path to another library exporting the same entry points (the CPU checker the tests build)."""

    def __init__(self, library):
        self.path, self.lib = _bind(library, _REPHOTO_SIGS)

    def rephoto_cubemap(self, descs, disparities, colors_bgra, center, edge, want_color=True, want_disparity=False,
                        want_winners=False, device=0):
        """CanopyScene(rig, disparities, colors).cubemap(edge, center) (ComputeRephotographyErrors.cpp:77-95): float
        B, G, R, A cubemaps [6 * edge, edge, 4] (faces +X, -X, +Y, -Y, +Z, -Z stacked), NaN set to 0.  disparities:
        float [h, w] per camera; colors_bgra: float [h, w, 4] per camera at the disparity's size.  Returns
        (color, disparity, winners), each None unless asked for; winners int32 [num_cams, 6 * edge, edge]."""
        S = len(disparities)
        d = [np.ascontiguousarray(x, np.float32) for x in disparities]
        h, w = d[0].shape if S else (2, 2)
        assert all(x.shape == (h, w) for x in d)
        cols = None
        if want_color and S:
            cols = [np.ascontiguousarray(x, np.float32) for x in colors_bgra]
            assert all(x.shape == (h, w, 4) for x in cols)
        ctr = np.ascontiguousarray(center, np.float32)
        oc = np.empty((6 * edge, edge, 4), np.float32) if want_color else None
        od = np.empty((6 * edge, edge, 4), np.float32) if want_disparity else None
        wn = np.empty((max(S, 1), 6 * edge, edge), np.int32) if want_winners else None
        dp = _ptr_array(d) if S else None
        cp = _ptr_array(cols) if cols else None
        self._check(self.lib.derp_rephoto_cubemap(device, descs, S, dp, cp, w, h, ctr.ctypes.data, edge, _dp(oc), _dp(od),
                                                 _dp(wn)))
        return oc, od, (wn[:S] if wn is not None else None)

    def rephoto_score(self, ref_bgr, ren_bgr, mask, method="MSSIM", stat_radius=1, device=0):
        """computeScoreMap + averageScore (RephotographyUtil.h:39-120): returns (score map float [h, w, 3] B, G, R,
        per-channel averages over the mask without NaN as a float64 [3] in B, G, R order)."""
        x = np.ascontiguousarray(ref_bgr, np.float32)
        y = np.ascontiguousarray(ren_bgr, np.float32)
        m = np.ascontiguousarray(mask, np.uint8)
        h, w = x.shape[:2]
        assert x.shape == (h, w, 3) and y.shape == (h, w, 3) and m.shape == (h, w)
        score = np.empty((h, w, 3), np.float32)
        avg = np.empty(3, np.float64)
        self._check(self.lib.derp_rephoto_score(device, x.ctypes.data, y.ctypes.data, m.ctypes.data, w, h,
                                               REPHOTO_METHODS[method], stat_radius, score.ctypes.data, avg.ctypes.data))
        return score, avg


# ---- include/derp_canopy.h ----------------------------------------------------------------------------------------
_CANOPY_SIGS = {
    "derp_last_error": (C.c_char_p, []),
    "derp_canopy_render": (C.c_int, [C.c_int, _p(CameraDesc), C.c_int, _p(C.c_void_p), C.c_int, C.c_int, _p(C.c_void_p),
                                     C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float,
                                     C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "derp_canopy_snapshot_matrix": (C.c_int, [C.c_void_p] * 3 + [C.c_double, C.c_int, C.c_int, C.c_void_p]),
}
CANOPY_SYMBOLS = sorted(k for k in _CANOPY_SIGS if k.startswith("derp_canopy_"))
CANOPY_PROJECTIONS = {"cubemap": 0, "equirect": 1, "perspective": 2}
CANOPY_SHADERS = {"on_screen": 0, "svd": 1}


class Canopy(_Binding):
    """ctypes binding of include/derp_canopy.h on a loaded library: ``Canopy(load_cuda())`` for the product, or a path
    to another library exporting derp_canopy_render (the CPU checker the tests build)."""

    def __init__(self, library):
        self.path, self.lib = _bind(library, _CANOPY_SIGS, optional=("derp_canopy_snapshot_matrix",))

    def snapshot_matrix(self, position, forward, up, horizontal_fov=90.0, width=3072, height=1536):
        """SimpleMeshRenderer's snapshot clip matrix (computed on the host): float32 [4, 4]."""
        vec = [np.ascontiguousarray(v, np.float32) for v in (position, forward, up)]
        out = np.empty(16, np.float32)
        self._check(self.lib.derp_canopy_snapshot_matrix(vec[0].ctypes.data, vec[1].ctypes.data, vec[2].ctypes.data,
                                                         horizontal_fov, width, height, out.ctypes.data))
        return out.reshape(4, 4)

    def render(self, descs, disparities, colors_bgra, position, projection="cubemap", size=(64, 64), matrix=None,
               ipd=0.0, alpha_blend=True, shader="svd", want_color=True, want_disparity=False, want_winners=False,
               device=0):
        """CanopyScene(rig, disparities, colors).cubemap / equirect / render from `position` (derp_canopy.h).
        disparities: float [h, w] per camera (the mesh); colors_bgra: float [ch, cw, 4] per camera at any one size.
        size = (out_width, out_height): (edge, edge) for the cubemap, (2 h, h) for the equirect.  Returns (color,
        disparity, winners), each None unless asked for: float B, G, R, A images with NaN where nothing covers, winners
        int32 [num_cams, raster rows, raster width]."""
        S = len(disparities)
        d = [np.ascontiguousarray(x, np.float32) for x in disparities]
        h, w = d[0].shape if S else (2, 2)
        assert all(x.shape == (h, w) for x in d)
        cols, ch, cw = None, 0, 0
        if want_color:
            cols = [np.ascontiguousarray(x, np.float32) for x in colors_bgra]
            ch, cw = cols[0].shape[:2] if S else (1, 1)
            assert all(x.shape == (ch, cw, 4) for x in cols)
        proj = CANOPY_PROJECTIONS[projection]
        W, H = size
        shape = {0: (6 * H, W), 1: (H, 2 * H), 2: (H, W)}[proj]
        raster = (6 * H, H) if proj != 2 else (H, W)
        pos = np.ascontiguousarray(position, np.float32)
        m = None if matrix is None else np.ascontiguousarray(matrix, np.float32).reshape(16)
        oc = np.empty(shape + (4,), np.float32) if want_color else None
        od = np.empty(shape + (4,), np.float32) if want_disparity else None
        wn = np.empty((max(S, 1),) + raster, np.int32) if want_winners else None
        self._check(self.lib.derp_canopy_render(device, descs, S, _ptr_array(d) if S else None, w, h,
                                                _ptr_array(cols) if cols else None, cw, ch, proj, pos.ctypes.data,
                                                _dp(m), W, H, float(ipd), int(bool(alpha_blend)), CANOPY_SHADERS[shader],
                                                _dp(oc), _dp(od), _dp(wn)))
        return oc, od, (wn[:S] if wn is not None else None)


def snapshot_matrix(position, forward, up, horizontal_fov=90.0, width=3072, height=1536, library=None):
    """SimpleMeshRenderer's snapshot clip matrix (derp_canopy_snapshot_matrix, computed on the host): float32 [4, 4].
    `library`: a Library or Canopy binding, the product by default."""
    canopy = library if isinstance(library, Canopy) else Canopy(library or load_cuda())
    return canopy.snapshot_matrix(position, forward, up, horizontal_fov, width, height)


class Context:
    """One DerpCtx: a (frame, level) of a rig on one device."""

    def __init__(self, library, descs, dst_to_src=None, device=0):
        self.L = library
        self.S = len(descs)
        if dst_to_src is None:
            dst_to_src = list(range(self.S))
        self.dst_to_src = list(dst_to_src)
        self.Sd = len(self.dst_to_src)
        d2s = (C.c_int32 * self.Sd)(*self.dst_to_src)
        h = C.c_void_p()
        library.check(library.lib.derp_create(descs, self.S, d2s, self.Sd, device, C.byref(h)))
        self.h = h
        self.W = self.H = 0
        self._keep = []

    def close(self):
        if self.h:
            self.L.lib.derp_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream):
        self.L.check(self.L.lib.derp_set_stream(self.h, C.c_void_p(cuda_stream)))

    def sync(self):
        self.L.check(self.L.lib.derp_sync(self.h))

    def profile(self, enable=True):
        self.L.check(self.L.lib.derp_profile(self.h, int(enable)))

    def get_profile(self):
        ms, n = C.c_double(), C.c_uint64()
        self.L.check(self.L.lib.derp_get_profile(self.h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def get_profile_ping_pong(self):
        ms, n, e, h = C.c_double(), C.c_uint64(), C.c_uint64(), C.c_uint64()
        self.L.check(self.L.lib.derp_get_profile_ping_pong(self.h, C.byref(ms), C.byref(n), C.byref(e), C.byref(h)))
        return ms.value, n.value, e.value, h.value

    def set_sweep_mode(self, mode):
        """0 automatic, 1 plain sweep, 2 filtered sweep (derp_b200.h)."""
        self.L.check(self.L.lib.derp_set_sweep_mode(self.h, int(mode)))

    def sweep_stats(self):
        a, b = C.c_uint64(), C.c_uint64()
        self.L.check(self.L.lib.derp_get_sweep_stats(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def launch_count(self):
        n = C.c_uint64()
        self.L.check(self.L.lib.derp_get_launch_count(self.h, C.byref(n)))
        return n.value

    def level_begin(self, width, height, level=0, num_levels=1, full_width=None, full_height=None,
                    var_noise_floor=4e-5, var_high_thresh=1e-3, use_foreground_masks=False):
        p = LevelParams()
        p.width, p.height, p.level, p.num_levels = width, height, level, num_levels
        p.full_width = full_width if full_width else width
        p.full_height = full_height if full_height else height
        p.var_noise_floor, p.var_high_thresh = var_noise_floor, var_high_thresh
        p.use_foreground_masks = int(use_foreground_masks)
        self.L.check(self.L.lib.derp_level_begin(self.h, C.byref(p)))
        self.W, self.H = width, height

    def set_colors(self, colors):
        a = [np.ascontiguousarray(c, np.uint16) for c in colors]
        assert len(a) == self.S and all(x.shape == (self.H, self.W, 3) for x in a)
        self.L.check(self.L.lib.derp_set_colors(self.h, _ptr_array(a)))

    def set_colors_ptr(self, ptrs):
        """colors as raw addresses (host or device memory), one u16 HxWx3 image per camera."""
        assert len(ptrs) == self.S
        pa = (C.c_void_p * self.S)(*[int(p) for p in ptrs])
        self.L.check(self.L.lib.derp_set_colors(self.h, pa))

    def set_foreground_masks(self, masks):
        a = [np.ascontiguousarray(m, np.uint8) for m in masks]
        assert len(a) == self.S
        self.L.check(self.L.lib.derp_set_foreground_masks(self.h, _ptr_array(a)))

    def set_background_disparity(self, bgs):
        a = [np.ascontiguousarray(m, np.float32) for m in bgs]
        assert len(a) == self.Sd
        self.L.check(self.L.lib.derp_set_background_disparity(self.h, _ptr_array(a)))

    def reproject(self, dst):
        self.L.check(self.L.lib.derp_reproject(self.h, dst))

    def brute_force(self, dst, num_depths=150, min_depth_m=0.5, max_depth_m=1e4, partial_coverage=True,
                    want_index=True):
        idx = np.empty((self.H, self.W), np.int32) if want_index else None
        self.L.check(self.L.lib.derp_brute_force(self.h, dst, num_depths, min_depth_m, max_depth_m,
                                                 int(partial_coverage), _dp(idx)))
        return idx

    def random_proposals(self, dst, n=2, min_depth_m=0.5, max_depth_m=1e4):
        self.L.check(self.L.lib.derp_random_proposals(self.h, dst, n, min_depth_m, max_depth_m))

    def ping_pong(self, dst, iterations=1):
        self.L.check(self.L.lib.derp_ping_pong(self.h, dst, iterations))

    def mismatches(self):
        self.L.check(self.L.lib.derp_mismatches(self.h))

    def bilateral(self, dst):
        self.L.check(self.L.lib.derp_bilateral(self.h, dst))

    def median(self, dst):
        self.L.check(self.L.lib.derp_median(self.h, dst))

    def mask_fov(self, dst):
        self.L.check(self.L.lib.derp_mask_fov(self.h, dst))

    def upsample_from(self, dst, coarse, coarse_mask=None, fine_mask=None):
        coarse = np.ascontiguousarray(coarse, np.float32)
        ch, cw = coarse.shape
        cm = None if coarse_mask is None else np.ascontiguousarray(coarse_mask, np.uint8)
        fm = None if fine_mask is None else np.ascontiguousarray(fine_mask, np.uint8)
        self.L.check(self.L.lib.derp_upsample_from(self.h, dst, coarse.ctypes.data, cw, ch, _dp(cm), _dp(fm)))

    def level_keep(self):
        """Snapshot the finished level's disparities inside the context for upsample_from_kept."""
        self.L.check(self.L.lib.derp_level_keep(self.h))

    def upsample_from_kept(self, dst, coarse_mask=None, fine_mask=None):
        cm = None if coarse_mask is None else np.ascontiguousarray(coarse_mask, np.uint8)
        fm = None if fine_mask is None else np.ascontiguousarray(fine_mask, np.uint8)
        self.L.check(self.L.lib.derp_upsample_from_kept(self.h, dst, _dp(cm), _dp(fm)))

    @staticmethod
    def _opts(num_depths=150, min_depth_m=0.5, max_depth_m=1e4, partial_coverage=True,
              random_proposals=2, ping_pong_iterations=1, mismatches_start_level=-1,
              do_bilateral_filter=True, do_median_filter=True):
        o = ProcessOpts()
        o.num_depths, o.min_depth_m, o.max_depth_m = num_depths, min_depth_m, max_depth_m
        o.partial_coverage = int(partial_coverage)
        o.random_proposals, o.ping_pong_iterations = random_proposals, ping_pong_iterations
        o.mismatches_start_level = mismatches_start_level
        o.do_bilateral_filter, o.do_median_filter = int(do_bilateral_filter), int(do_median_filter)
        return o

    def process_level(self, **kw):
        o = self._opts(**kw)
        self.L.check(self.L.lib.derp_process_level(self.h, C.byref(o)))

    def level_estimate(self, **kw):
        """First half of process_level (everything before mismatch handling)."""
        o = self._opts(**kw)
        self.L.check(self.L.lib.derp_level_estimate(self.h, C.byref(o)))

    def level_filter(self, **kw):
        """Second half of process_level (bilateral, median, maskFov)."""
        o = self._opts(**kw)
        self.L.check(self.L.lib.derp_level_filter(self.h, C.byref(o)))

    def disparity_ptr(self, dst):
        """Address of the context's own disparity plane (device memory on the CUDA library)."""
        p = self.L.lib.derp_disparity_device_ptr(self.h, dst)
        if not p:
            raise DerpError(-1, self.L.lib.derp_last_error().decode())
        return p

    def gather_disparities(self, planes):
        """planes: one entry per rig camera — int address (host / this device / peer device), a float32
        numpy array (H, W), or None for a camera this context owns as a destination."""
        keep, arr = [], (C.c_void_p * self.S)()
        assert len(planes) == self.S
        for s, pl in enumerate(planes):
            if pl is None:
                arr[s] = None
            elif isinstance(pl, int):
                arr[s] = pl
            else:
                a = np.ascontiguousarray(pl, np.float32)
                assert a.shape == (self.H, self.W)
                keep.append(a)
                arr[s] = a.ctypes.data
        self.L.check(self.L.lib.derp_gather_disparities(self.h, arr))

    def mismatches_gathered(self):
        self.L.check(self.L.lib.derp_mismatches_gathered(self.h))

    def eval_cost(self, dst, disparity):
        d = np.ascontiguousarray(disparity, np.float32)
        cost = np.empty((self.H, self.W), np.float32)
        conf = np.empty((self.H, self.W), np.float32)
        self.L.check(self.L.lib.derp_eval_cost(self.h, dst, d.ctypes.data, cost.ctypes.data, conf.ctypes.data))
        return cost, conf

    def set_disparity(self, dst, disparity=None, cost=None, confidence=None):
        a = [None if x is None else np.ascontiguousarray(x, np.float32) for x in (disparity, cost, confidence)]
        self.L.check(self.L.lib.derp_set_disparity(self.h, dst, _dp(a[0]), _dp(a[1]), _dp(a[2])))

    def get_disparity(self, dst, want_cost=True):
        d = np.empty((self.H, self.W), np.float32)
        c = np.empty((self.H, self.W), np.float32) if want_cost else None
        f = np.empty((self.H, self.W), np.float32) if want_cost else None
        self.L.check(self.L.lib.derp_get_disparity(self.h, dst, d.ctypes.data, _dp(c), _dp(f)))
        return (d, c, f) if want_cost else d

    def get_fov_mask(self, dst):
        m = np.empty((self.H, self.W), np.uint8)
        self.L.check(self.L.lib.derp_get_fov_mask(self.h, dst, m.ctypes.data))
        return m

    def get_mismatch_mask(self, dst):
        m = np.empty((self.H, self.W), np.uint8)
        self.L.check(self.L.lib.derp_get_mismatch_mask(self.h, dst, m.ctypes.data))
        return m

    def get_variance(self, src):
        v = np.empty((self.H, self.W), np.float32)
        self.L.check(self.L.lib.derp_get_variance(self.h, src, v.ctypes.data))
        return v

    def get_var_noise_floor(self):
        f = C.c_float()
        self.L.check(self.L.lib.derp_get_var_noise_floor(self.h, C.byref(f)))
        return f.value

    def get_proj_warp(self, src):
        w = np.empty((self.H, self.W, 2), np.float32)
        self.L.check(self.L.lib.derp_get_proj_warp(self.h, src, w.ctypes.data))
        return w

    def get_proj_color(self, src):
        w = np.empty((self.H, self.W, 3), np.uint16)
        self.L.check(self.L.lib.derp_get_proj_color(self.h, src, w.ctypes.data))
        return w

    def get_proj_bias(self, src):
        w = np.empty((self.H, self.W, 3), np.uint16)
        self.L.check(self.L.lib.derp_get_proj_bias(self.h, src, w.ctypes.data))
        return w

    def get_counters(self):
        a, b = C.c_uint64(), C.c_uint64()
        self.L.check(self.L.lib.derp_get_counters(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value


_cache = {}


def load_cuda():
    """The product library. Fails loudly when it is missing — there is no CPU fallback."""
    if "cuda" not in _cache:
        lib = Library(CUDA_LIB)
        if not lib.backend.startswith("cuda"):
            raise RuntimeError("%s reports backend %r, expected the CUDA library" % (CUDA_LIB, lib.backend))
        _cache["cuda"] = lib
    return _cache["cuda"]


# ---- include/derp_sweepview.h -------------------------------------------------------------------------------------
_SWEEP_SIGS = {
    "derp_last_error": (C.c_char_p, []),
    "derp_sweep_overlaps": (C.c_int, [C.c_int, _p(CameraDesc), C.c_int, _p(C.c_void_p), C.c_void_p, C.c_int, C.c_void_p,
                                      C.c_int, C.c_void_p]),
    "derp_sweep_crop_bounds": (C.c_int, [C.c_int, _p(CameraDesc), C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_int,
                                         C.c_void_p]),
    "derp_sweep_equirect": (C.c_int, [C.c_int, _p(CameraDesc), C.c_int, C.c_int, _p(C.c_void_p), C.c_void_p, C.c_uint64,
                                      C.c_void_p, C.c_int, C.c_void_p, C.c_int, _p(C.c_void_p)]),
    "derp_sweep_center_rig": (C.c_int, [_p(CameraDesc), C.c_int, C.c_int, _p(CameraDesc), C.c_void_p]),
    "derp_sweep_last_hits": (C.c_uint64, []),
    "derp_sweep_crop_width": (C.c_int, [C.c_uint64, C.c_void_p, _p(C.c_uint64)]),
    "derp_project_equirect_masks": (C.c_int, [C.c_int, _p(CameraDesc), C.c_int, C.c_double, _p(C.c_void_p), C.c_void_p,
                                              _p(C.c_void_p)]),
    "derp_project_last_host_pixels": (C.c_uint64, []),
    "derp_test_eqr_index_proven": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "derp_test_eqr_index_host": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
}
# derp_test_sweep_*_host: the same arguments as the entry point without the device
_SWEEP_HOST_SIGS = {"derp_test_sweep_%s_host" % k: (C.c_int, _SWEEP_SIGS["derp_sweep_" + k][1][1:])
                    for k in ("overlaps", "equirect")}
SWEEP_SYMBOLS = sorted(k for k in _SWEEP_SIGS if k.startswith("derp_sweep_"))
SWEEP_TEST_HOOKS = sorted(_SWEEP_HOST_SIGS)
_SWEEP_HOST_SIGS["derp_test_project_equirect_masks_host"] = (C.c_int,
                                                            _SWEEP_SIGS["derp_project_equirect_masks"][1][1:])
PROJECT_SYMBOLS = ["derp_project_equirect_masks", "derp_project_last_host_pixels",
                   "derp_test_project_equirect_masks_host"]


def rescaled_descs(descs, scale):
    """The rig as GenerateCameraOverlaps / GenerateEquirect hold it after Camera::rescale(resolution * scale)
    (Camera.cpp:217-223): resolution * scale, principal and focal times newResolution / resolution, in fp64."""
    out = (CameraDesc * len(descs))()
    for i, d in enumerate(descs):
        r = CameraDesc()
        C.pointer(r)[0] = d
        for k in range(2):
            res = d.resolution[k]
            nr = res * scale
            p = d.principal[k] if d.has_principal else res / 2
            r.principal[k] = p * (nr / res)
            r.focal[k] = d.focal[k] * (nr / res)
            r.resolution[k] = nr
        r.has_principal = 1
        out[i] = r
    return out


class SweepView(_Binding):
    """ctypes binding of include/derp_sweepview.h on a loaded library: ``SweepView(load_cuda())`` for the product, or a
    path to a library exporting some of the same entry points (the CPU checkers the tests build).  ``host=True`` runs
    the product's DERP_HD per-pixel code on the host (derp_test_sweep_*_host)."""

    def __init__(self, library, host=False):
        sigs = dict(_SWEEP_SIGS, **_SWEEP_HOST_SIGS) if host else _SWEEP_SIGS
        self.path, self.lib = _bind(library, sigs, optional=_SWEEP_SIGS)
        self.host = host

    @staticmethod
    def _images(images):
        ims = [np.ascontiguousarray(x, np.float32) for x in images]
        assert all(x.ndim == 3 and x.shape[2] == 4 for x in ims)
        sizes = np.array([[x.shape[1], x.shape[0]] for x in ims], np.int32).reshape(-1)
        return ims, sizes

    def overlaps(self, descs, images, dst, disparities, device=0):
        """projectSrcsToDst of camera `dst` at each disparity: float [n, int(res.y), int(res.x), 4] (B, G, R, A)."""
        ims, sizes = self._images(images)
        disp = np.ascontiguousarray(disparities, np.float32)
        W, H = int(descs[dst].resolution[0]), int(descs[dst].resolution[1])
        out = np.empty((len(disp), H, W, 4), np.float32)
        if self.host:
            rc = self.lib.derp_test_sweep_overlaps_host(descs, len(descs), _ptr_array(ims), sizes.ctypes.data, dst,
                                                        disp.ctypes.data, len(disp), out.ctypes.data)
        else:
            rc = self.lib.derp_sweep_overlaps(device, descs, len(descs), _ptr_array(ims), sizes.ctypes.data, dst,
                                              disp.ctypes.data, len(disp), out.ctypes.data)
        self._check(rc)
        return out

    def crop_bounds(self, descs, height, depths, center=-1, device=0):
        """createCroppedEquirect's box per depth: float64 [n, 4] = minX, maxX, minY, maxY."""
        dep = np.ascontiguousarray(depths, np.float32)
        out = np.empty((len(dep), 4), np.float64)
        self._check(self.lib.derp_sweep_crop_bounds(device, descs, len(descs), center, height, dep.ctypes.data, len(dep),
                                                    out.ctypes.data))
        return out

    def crop_width(self, height, box):
        b = np.ascontiguousarray(box, np.float64)
        w = C.c_uint64()
        self._check(self.lib.derp_sweep_crop_width(height, b.ctypes.data, C.byref(w)))
        return w.value

    def equirect(self, descs, images, height, depths, bounds=None, black_bg=False, center=-1, widths=None, device=0):
        """createEquirect (bounds None) or createCroppedEquirect per depth: a list of float [height, width_k, 4]."""
        ims, sizes = self._images(images)
        dep = np.ascontiguousarray(depths, np.float32)
        b = None if bounds is None else np.ascontiguousarray(bounds, np.float64)
        if widths is None:
            widths = [2 * height] * len(dep) if b is None else [self.crop_width(height, b[k]) for k in range(len(dep))]
        outs = [np.empty((height, w, 4), np.float32) for w in widths]
        args = (descs, len(descs), center, _ptr_array(ims), sizes.ctypes.data, height, dep.ctypes.data, len(dep), _dp(b),
                int(bool(black_bg)), _ptr_array(outs))
        if self.host:
            self._check(self.lib.derp_test_sweep_equirect_host(*args))
        else:
            self._check(self.lib.derp_sweep_equirect(device, *args))
        return outs

    def project_masks(self, descs, masks, depth, device=0):
        """ProjectEquirectsToCameras at `depth` m: masks[i] is camera i's equirect mask (uint8 [h, w], 0 / non-zero, or
        a device pointer given as (ptr, w, h)); returns uint8 [int(res.y), int(res.x)] per camera, 0 or 255."""
        ptrs, sizes, keep = [], [], []
        for m in masks:
            if isinstance(m, tuple):
                ptrs.append(m[0])
                sizes += [m[1], m[2]]
            else:
                m = np.ascontiguousarray(m, np.uint8)
                keep.append(m)
                ptrs.append(m.ctypes.data)
                sizes += [m.shape[1], m.shape[0]]
        sz = np.array(sizes, np.int32)
        outs = [np.empty((int(d.resolution[1]), int(d.resolution[0])), np.uint8) for d in descs]
        args = (descs, len(descs), float(depth), (C.c_void_p * len(ptrs))(*ptrs), sz.ctypes.data, _ptr_array(outs))
        if self.host:
            self._check(self.lib.derp_test_project_equirect_masks_host(*args))
        else:
            self._check(self.lib.derp_project_equirect_masks(device, *args))
        return outs

    def eqr_index(self, pts_or_boxes, width, height, proven=False, device=0):
        """int64 [n]: eqrIndex of points [n, 3] on the host (the index or -1), or with ``proven`` the device's
        eqrIndexProven of boxes [n, 6] (x lo, x hi, y lo, y hi, z lo, z hi; -2 where it does not decide)."""
        a = np.ascontiguousarray(pts_or_boxes, np.float64).reshape(-1, 6 if proven else 3)
        out = np.empty(len(a), np.int64)
        if proven:
            self._check(self.lib.derp_test_eqr_index_proven(device, a.ctypes.data, len(a), width, height,
                                                            out.ctypes.data))
        else:
            self._check(self.lib.derp_test_eqr_index_host(a.ctypes.data, len(a), width, height, out.ctypes.data))
        return out

    def last_host_pixels(self):
        """Pixels this thread's last project_masks call resolved on the host (the device could not prove them)."""
        return int(self.lib.derp_project_last_host_pixels())

    def last_hits(self):
        """(sample, camera) pairs whose camera saw the point in this thread's last overlaps / equirect call."""
        return int(self.lib.derp_sweep_last_hits())

    def center_rig(self, descs, center):
        """centerRig: (centred descriptors, float64 [n, 3, 3] rotations, float64 [n, 3] origins)."""
        out = (CameraDesc * len(descs))()
        rot = np.empty((len(descs), 3, 3), np.float64)
        self._check(self.lib.derp_sweep_center_rig(descs, len(descs), center, out, rot.ctypes.data))
        org = np.array([[out[i].origin[k] for k in range(3)] for i in range(len(descs))], np.float64)
        return out, rot, org


# ---- include/derp_eqrmesh.h ---------------------------------------------------------------------------------------
_EQR_SIGS = {
    "derp_last_error": (C.c_char_p, []),
    "derp_equirect_mesh_size": (C.c_int, [C.c_int, C.c_int, C.c_double, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "derp_equirect_mesh": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_float, C.c_void_p,
                                     C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "derp_equirect_mesh_simplified": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_float,
                                                C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64),
                                                C.POINTER(C.c_uint64)]),
}
EQR_SYMBOLS = sorted(k for k in _EQR_SIGS if k.startswith("derp_equirect_"))


class EqrMesh(_Binding):
    """ctypes binding of include/derp_eqrmesh.h on a loaded library: ``EqrMesh(load_cuda())`` for the product, or a path
    to a library exporting the same entry points (the CPU checkers the tests build)."""

    def __init__(self, library):
        self.path, self.lib = _bind(library, _EQR_SIGS)

    def mesh(self, disparity, scale=1.0, max_depth=700.0, tear_ratio=0.95, num_faces=200000, strictness=0.0,
             device=0):
        """CreateObjFromDisparityEquirect's mesh of a disparity equirect (float32 [h, w], or a device pointer given as
        (ptr, w, h)): returns (vertexes float64 [nv, 3], faces uint32 [nf, 3]); simplified when strictness > 0."""
        if isinstance(disparity, tuple):
            ptr, w, h = disparity
        else:
            disparity = np.ascontiguousarray(disparity, np.float32)
            h, w = disparity.shape
            ptr = disparity.ctypes.data
        mw, mh = C.c_int(), C.c_int()
        self._check(self.lib.derp_equirect_mesh_size(w, h, scale, C.byref(mw), C.byref(mh)))
        cells = mw.value * mh.value
        vtx = np.empty((cells, 3), np.float64)
        idx = np.empty((2 * cells, 3), np.uint32)
        nv, nf = C.c_uint64(), C.c_uint64()
        head = (device, ptr, w, h, float(scale), float(max_depth), tear_ratio)
        tail = (vtx.ctypes.data, idx.ctypes.data, C.byref(nv), C.byref(nf))
        if strictness > 0:
            self._check(self.lib.derp_equirect_mesh_simplified(*head, int(num_faces), float(strictness), *tail))
        else:
            self._check(self.lib.derp_equirect_mesh(*head, *tail))
        return vtx[:nv.value].copy(), idx[:nf.value].copy()


# ---- include/derp_rigsim.h ----------------------------------------------------------------------------------------
RIGSIM_SCENES = {"icosahedron": 0, "cube": 1, "ground_plane": 2}


class RigsimSceneParams(C.Structure):
    _fields_ = [("scene", C.c_int32), ("num_random_icosahedrons", C.c_int32), ("red_triangle", C.c_int32),
                ("reserved", C.c_int32), ("min_icosahedron_dist", C.c_double), ("max_icosahedron_dist", C.c_double),
                ("min_icosahedron_radius", C.c_double), ("max_icosahedron_radius", C.c_double),
                ("ground_plane_dist_m", C.c_double)]


class RigsimRender(C.Structure):
    _fields_ = [("anti_alias_supersample", C.c_int32), ("marble", C.c_int32), ("marble_scale", C.c_double),
                ("interpupillary_radius", C.c_double), ("skybox_bgr", C.c_void_p), ("skybox_width", C.c_int32),
                ("skybox_height", C.c_int32), ("ceiling_bgr", C.c_void_p), ("ceiling_cols", C.c_int32),
                ("ceiling_rows", C.c_int32), ("ceiling_position", C.c_double), ("ceiling_width", C.c_double),
                ("ceiling_depth", C.c_double)]


RIGSIM_TRIANGLE = np.dtype([(k, np.float32, (3,)) for k in ("v0", "v1", "v2", "e1", "e2", "normal", "color")])
RIGSIM_NODE = np.dtype([("center", np.float32, (3,)), ("radius", np.float32), ("first", np.int32),
                        ("count", np.int32), ("escape", np.int32), ("reserved", np.int32)])

_RIGSIM_SIGS = {
    "derp_last_error": (C.c_char_p, []),
    "derp_rigsim_scene_create": (C.c_int, [_p(RigsimSceneParams), _p(C.c_void_p)]),
    "derp_rigsim_scene_destroy": (None, [C.c_void_p]),
    "derp_rigsim_scene_info": (C.c_int, [C.c_void_p, _p(C.c_int32), _p(C.c_int32), _p(C.c_int32)]),
    "derp_rigsim_scene_get": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "derp_rigsim_render_cameras": (C.c_int, [C.c_int, C.c_void_p, _p(RigsimRender), _p(CameraDesc), C.c_int,
                                             _p(C.c_void_p), _p(C.c_void_p)]),
    "derp_rigsim_render_equirect": (C.c_int, [C.c_int, C.c_void_p, _p(RigsimRender), C.c_int, C.c_int, C.c_int,
                                              C.c_void_p, C.c_void_p]),
    "derp_rigsim_last_host_rays": (C.c_uint64, []),
    "derp_rigsim_last_rays": (C.c_uint64, []),
    "derp_rigsim_trace_host": (C.c_int, [C.c_void_p, _p(RigsimRender), C.c_void_p, C.c_int, C.c_void_p]),
    "derp_test_rigsim_area": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "derp_test_sky_texel": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "derp_test_sky_texel_host": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
}
RIGSIM_SYMBOLS = sorted(k for k in _RIGSIM_SIGS if k.startswith("derp_rigsim_"))


class RigSim(_Binding):
    """ctypes binding of include/derp_rigsim.h on a loaded library: ``RigSim(load_cuda())``.

    ``scene(...)`` builds the scene and its BVH on the host from the process's rand() stream (seed it with
    ``srand``); the render calls take the scene handle, an 8-bit BGR skybox and RigSimulator's rendering flags."""

    def __init__(self, library):
        self.path, self.lib = _bind(library, _RIGSIM_SIGS)
        self.libc = C.CDLL(None)
        self.libc.rand.restype = C.c_int

    def srand(self, seed):
        """Seeds the C library's rand(), which the scene and the BVH consume (the same stream the process shares)."""
        self.libc.srand(C.c_uint(seed))

    def rand(self):
        """The next rand() value (tests compare the stream position a scene build leaves)."""
        return int(self.libc.rand())

    def scene(self, scene="icosahedron", num_random_icosahedrons=250, min_icosahedron_dist=100.0,
              max_icosahedron_dist=250.0, min_icosahedron_radius=20.0, max_icosahedron_radius=50.0,
              red_triangle=False, ground_plane_dist_m=1.70):
        p = RigsimSceneParams(RIGSIM_SCENES[scene], num_random_icosahedrons, int(bool(red_triangle)), 0,
                              min_icosahedron_dist, max_icosahedron_dist, min_icosahedron_radius,
                              max_icosahedron_radius, ground_plane_dist_m)
        h = C.c_void_p()
        self._check(self.lib.derp_rigsim_scene_create(C.byref(p), C.byref(h)))
        return h

    def destroy(self, scene):
        self.lib.derp_rigsim_scene_destroy(scene)

    def scene_arrays(self, scene):
        """(triangles RIGSIM_TRIANGLE [nt], nodes RIGSIM_NODE [nn], leaf triangle indices int32 [nl]), BVH in preorder."""
        nt, nn, nl = C.c_int32(), C.c_int32(), C.c_int32()
        self._check(self.lib.derp_rigsim_scene_info(scene, C.byref(nt), C.byref(nn), C.byref(nl)))
        tris = np.zeros(max(nt.value, 1), RIGSIM_TRIANGLE)
        nodes = np.zeros(nn.value, RIGSIM_NODE)
        leaf = np.zeros(max(nl.value, 1), np.int32)
        self._check(self.lib.derp_rigsim_scene_get(scene, tris.ctypes.data, nodes.ctypes.data, leaf.ctypes.data))
        return tris[:nt.value], nodes, leaf[:nl.value]

    @staticmethod
    def render_opts(skybox, aas=1, marble=False, marble_scale=0.1, interpupillary_radius=3.2, ceiling=None,
                    ceiling_position=0.0, ceiling_width=0.0, ceiling_depth=0.0):
        """The rendering flags as a RigsimRender; skybox / ceiling are uint8 [h, w, 3] BGR arrays (kept alive by the
        returned tuple's second element)."""
        sky = np.ascontiguousarray(skybox, np.uint8)
        ceil = None if ceiling is None else np.ascontiguousarray(ceiling, np.uint8)
        o = RigsimRender(int(aas), int(bool(marble)), marble_scale, interpupillary_radius, sky.ctypes.data,
                         sky.shape[1], sky.shape[0], None if ceil is None else ceil.ctypes.data,
                         0 if ceil is None else ceil.shape[1], 0 if ceil is None else ceil.shape[0],
                         ceiling_position, ceiling_width, ceiling_depth)
        return o, (sky, ceil)

    def render_cameras(self, scene, descs, skybox, outs=None, device=0, **opts):
        """renderCamera for every camera (no noise): a list of (bgr float32 [h, w, 3] = 255 * B, G, R, depth float32
        [h, w]).  ``outs``: optional (bgr pointers, depth pointers) of device memory written in place."""
        o, keep = self.render_opts(skybox, **opts)
        if isinstance(descs, (list, tuple)):
            descs = (CameraDesc * len(descs))(*descs)
        if outs is None:
            res = [(np.empty((int(d.resolution[1]), int(d.resolution[0]), 3), np.float32),
                    np.empty((int(d.resolution[1]), int(d.resolution[0])), np.float32)) for d in descs]
            b, dp = _ptr_array([r[0] for r in res]), _ptr_array([r[1] for r in res])
        else:
            res = None
            b, dp = (C.c_void_p * len(descs))(*outs[0]), (C.c_void_p * len(descs))(*outs[1])
        self._check(self.lib.derp_rigsim_render_cameras(device, scene, C.byref(o), descs, len(descs), b, dp))
        return res

    def render_equirect(self, scene, width, height, skybox, stereo=False, device=0, **opts):
        """renderMonoEquirect: (bgr [h, w, 3], clamp(1 / depth) [h, w]); stereo: (left bgr, right bgr)."""
        o, keep = self.render_opts(skybox, **opts)
        out0 = np.empty((height, width, 3), np.float32)
        out1 = np.empty((height, width, 3) if stereo else (height, width), np.float32)
        self._check(self.lib.derp_rigsim_render_equirect(device, scene, C.byref(o), int(bool(stereo)), width, height,
                                                         out0.ctypes.data, out1.ctypes.data))
        return out0, out1

    def area(self, src, k, device=0):
        """The render's INTER_AREA by the integer factor k on the GPU (derp_test_rigsim_area): float [h / k, w / k(, cn)]."""
        s = np.ascontiguousarray(src, np.float32)
        cn = 1 if s.ndim == 2 else s.shape[2]
        out = np.empty((s.shape[0] // k, s.shape[1] // k) + s.shape[2:], np.float32)
        self._check(self.lib.derp_test_rigsim_area(device, s.ctypes.data, out.shape[1], out.shape[0], cn, k,
                                                   out.ctypes.data))
        return out

    def last_host_rays(self):
        """(rays whose sky texel the host resolved, supersample rays traced) in this thread's last render."""
        return int(self.lib.derp_rigsim_last_host_rays()), int(self.lib.derp_rigsim_last_rays())

    def sky_texel(self, dirs, rows, cols, host=False, device=0):
        """int32 [n, 2] (row, column) of float32 directions [n, 3] in a rows x cols skybox: the device's proven texel
        ((-1, -1) where it leaves the ray to the host), or with ``host`` the C library's."""
        d = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3)
        out = np.empty((len(d), 2), np.int32)
        if host:
            self._check(self.lib.derp_test_sky_texel_host(d.ctypes.data, len(d), rows, cols, out.ctypes.data))
        else:
            self._check(self.lib.derp_test_sky_texel(device, d.ctypes.data, len(d), rows, cols, out.ctypes.data))
        return out

    def trace_host(self, scene, rays, skybox, **opts):
        """traceRayToGetColor on the host for float32 rays [n, 6] (origin, direction): float32 [n, 4] = B, G, R, depth."""
        o, keep = self.render_opts(skybox, **opts)
        r = np.ascontiguousarray(rays, np.float32).reshape(-1, 6)
        out = np.empty((len(r), 4), np.float32)
        self._check(self.lib.derp_rigsim_trace_host(scene, C.byref(o), r.ctypes.data, len(r), out.ctypes.data))
        return out


# ---- include/derp_riganalysis.h -----------------------------------------------------------------------------------
_RIGANALYSIS_SIGS = {
    "derp_last_error": (C.c_char_p, []),
    "derp_rig_coverage": (C.c_int, [C.c_int, _p(CameraDesc), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                    C.c_int, C.c_void_p]),
    "derp_rig_equirect_coverage": (C.c_int, [C.c_int, _p(CameraDesc), C.c_void_p, C.c_int, C.c_int, C.c_int,
                                             C.c_double, C.c_void_p, C.c_void_p]),
    "derp_rig_camera_coverage": (C.c_int, [C.c_int, _p(CameraDesc), C.c_void_p, C.c_int, C.c_int, C.c_double,
                                           C.c_void_p]),
    "derp_rig_cross_section": (C.c_int, [C.c_int, _p(CameraDesc), C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "derp_rig_analysis_last_host_points": (C.c_uint64, []),
    "derp_test_rig_coverage_host": (C.c_int, [_p(CameraDesc), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                              C.c_int, C.c_void_p]),
    "derp_test_rig_equirect_coverage_host": (C.c_int, [_p(CameraDesc), C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                       C.c_double, C.c_void_p, C.c_void_p]),
    "derp_test_rig_camera_coverage_host": (C.c_int, [_p(CameraDesc), C.c_void_p, C.c_int, C.c_int, C.c_double,
                                                     C.c_void_p]),
    "derp_test_rig_cross_section_host": (C.c_int, [_p(CameraDesc), C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "derp_test_math": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "derp_test_acosf_exhaustive": (C.c_int, [C.c_int, C.c_void_p]),
    "derp_test_rig_point_iv": (C.c_int, [C.c_int, _p(CameraDesc), C.c_void_p, C.c_int, C.c_double, C.c_void_p]),
    "derp_test_sees_iv": (C.c_int, [C.c_int, _p(CameraDesc), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "derp_test_sees_device": (C.c_int, [C.c_int, _p(CameraDesc), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "derp_test_proven_count": (C.c_int, [C.c_int, _p(CameraDesc), C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_void_p]),
    "derp_test_count_timing_host": (C.c_int, [_p(CameraDesc), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                              C.c_void_p]),
}
MATH_FNS = {"sin": 0, "cos": 1, "atan": 2, "asin": 3, "atan2": 4, "acosf": 5, "atan2f": 6, "atan2Pos": 7}
RIGANALYSIS_SYMBOLS = sorted(k for k in _RIGANALYSIS_SIGS if k.startswith("derp_rig_"))


class RigAnalysis(_Binding):
    """ctypes binding of include/derp_riganalysis.h on a loaded library: ``RigAnalysis(load_cuda())``.

    Every call takes the rig as CameraDesc entries (a list or a ctypes array) and, optionally, ``rot``: float64
    [n, 3, 3] rotation matrices (rows right, up, backward) used as given.  ``host=True`` runs the host per-point code
    (derp_test_rig_*_host) instead of the GPU.  ``out`` (where taken) is a device pointer written in place."""

    def __init__(self, library):
        self.path, self.lib = _bind(library, _RIGANALYSIS_SIGS)

    @staticmethod
    def _rig(descs, rot):
        if isinstance(descs, (list, tuple)):
            descs = (CameraDesc * len(descs))(*descs)
        r = None if rot is None else np.ascontiguousarray(rot, np.float64).reshape(len(descs), 9)
        return descs, r, (None if r is None else r.ctypes.data)

    def coverage(self, descs, samples, distances, rot=None, host=False, device=0):
        """uint64 [len(distances), n + 1]: per distance, the number of samples seen by exactly k cameras."""
        descs, keep, r = self._rig(descs, rot)
        s = np.ascontiguousarray(samples, np.float64).reshape(-1, 3)
        d = np.ascontiguousarray(distances, np.float64)
        hist = np.zeros((len(d), len(descs) + 1), np.uint64)
        if host:
            self._check(self.lib.derp_test_rig_coverage_host(descs, r, len(descs), s.ctypes.data, len(s),
                                                             d.ctypes.data, len(d), hist.ctypes.data))
        else:
            self._check(self.lib.derp_rig_coverage(device, descs, r, len(descs), s.ctypes.data, len(s), d.ctypes.data,
                                                   len(d), hist.ctypes.data))
        return hist

    def equirect(self, descs, width, height, distance, rot=None, host=False, device=0, out=None):
        """(counts int32 [height, width], minTimingDiff float32 [height, width]); with ``out`` = (counts, timing)
        device pointers they are written in place and (None, None) is returned."""
        descs, keep, r = self._rig(descs, rot)
        if out is None:
            counts, timing = np.empty((height, width), np.int32), np.empty((height, width), np.float32)
            pc, pt = counts.ctypes.data, timing.ctypes.data
        else:
            counts = timing = None
            pc, pt = out
        if host:
            self._check(self.lib.derp_test_rig_equirect_coverage_host(descs, r, len(descs), width, height, distance,
                                                                      pc, pt))
        else:
            self._check(self.lib.derp_rig_equirect_coverage(device, descs, r, len(descs), width, height, distance,
                                                            pc, pt))
        return counts, timing

    def camera(self, descs, cam, distance, rot=None, host=False, device=0, out=None):
        """int32 [int(res.y), int(res.x)] of camera ``cam``."""
        descs, keep, r = self._rig(descs, rot)
        d = descs[cam]
        counts = None if out is not None else np.empty((int(d.resolution[1]), int(d.resolution[0])), np.int32)
        p = out if out is not None else counts.ctypes.data
        if host:
            self._check(self.lib.derp_test_rig_camera_coverage_host(descs, r, len(descs), cam, distance, p))
        else:
            self._check(self.lib.derp_rig_camera_coverage(device, descs, r, len(descs), cam, distance, p))
        return counts

    def cross_section(self, descs, dim=400, rot=None, host=False, device=0, out=None):
        """int32 [dim, dim]."""
        descs, keep, r = self._rig(descs, rot)
        counts = None if out is not None else np.empty((dim, dim), np.int32)
        p = out if out is not None else counts.ctypes.data
        if host:
            self._check(self.lib.derp_test_rig_cross_section_host(descs, r, len(descs), dim, p))
        else:
            self._check(self.lib.derp_rig_cross_section(device, descs, r, len(descs), dim, p))
        return counts

    def last_host_points(self):
        """The points this thread's last GPU call resolved on the host."""
        return int(self.lib.derp_rig_analysis_last_host_points())

    # ---- probes of the device's interval proofs (derp_test_*) ----
    def math(self, fn, a, b=None, device=0):
        """The device's ``fn`` (a MATH_FNS name) of a (and b): float64 [n, 3] = value, widened interval lo, hi."""
        a = np.ascontiguousarray(a, np.float64).ravel()
        b = None if b is None else np.ascontiguousarray(b, np.float64).ravel()
        out = np.empty((len(a), 3))
        self._check(self.lib.derp_test_math(device, MATH_FNS[fn], a.ctypes.data, None if b is None else b.ctypes.data,
                                            len(a), out.ctypes.data))
        return out

    def acosf_exhaustive(self, device=0):
        """Every float in [-1, 1]: dict of the device's and host's greatest errors (ulps), their greatest distance in
        float steps, and the host values outside the device value's widenF."""
        st = np.zeros(4, np.uint32)
        self._check(self.lib.derp_test_acosf_exhaustive(device, st.ctypes.data))
        return {"device_ulps": st[0] / 2.0 ** 20, "host_ulps": st[1] / 2.0 ** 20, "steps": int(st[2]),
                "outside": int(st[3])}

    def rig_point_iv(self, desc, pix, depth, device=0):
        """rigPointIv of int pixels [n, 2]: float64 [n, 7] = x lo, x hi, y lo, y hi, z lo, z hi, undistort's r."""
        p = np.ascontiguousarray(pix, np.int32).reshape(-1, 2)
        out = np.empty((len(p), 7))
        self._check(self.lib.derp_test_rig_point_iv(device, C.byref(desc), p.ctypes.data, len(p), depth,
                                                    out.ctypes.data))
        return out

    def sees_iv(self, desc, boxes, device=0):
        """seesIv of boxes [n, 6] (x lo, x hi, y lo, y hi, z lo, z hi): (int32 decision 1 / 0 / -1, float64 py [n, 2])."""
        b = np.ascontiguousarray(boxes, np.float64).reshape(-1, 6)
        dec, py = np.empty(len(b), np.int32), np.empty((len(b), 2))
        self._check(self.lib.derp_test_sees_iv(device, C.byref(desc), b.ctypes.data, len(b), dec.ctypes.data,
                                               py.ctypes.data))
        return dec, py

    def sees_device(self, desc, pts, device=0):
        """The device's Camera::sees of points [n, 3]: (float64 pixel [n, 2], bool seen [n])."""
        p = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
        pix, seen = np.empty((len(p), 2)), np.empty(len(p), np.uint8)
        self._check(self.lib.derp_test_sees_device(device, C.byref(desc), p.ctypes.data, len(p), pix.ctypes.data,
                                                   seen.ctypes.data))
        return pix, seen.astype(bool)

    def proven_count(self, descs, pts, rot=None, host=False, device=0):
        """provenCount<true> of points [n, 3] (count -1: left to the host), or with ``host`` its host twin
        countTiming: (int32 counts [n], float32 minTimingDiff [n])."""
        descs, keep, r = self._rig(descs, rot)
        p = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
        counts, timing = np.empty(len(p), np.int32), np.empty(len(p), np.float32)
        if host:
            self._check(self.lib.derp_test_count_timing_host(descs, r, len(descs), p.ctypes.data, len(p),
                                                             counts.ctypes.data, timing.ctypes.data))
        else:
            self._check(self.lib.derp_test_proven_count(device, descs, r, len(descs), p.ctypes.data, len(p),
                                                        counts.ctypes.data, timing.ctypes.data))
        return counts, timing
