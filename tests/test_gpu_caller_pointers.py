"""The CUDA library's pointer convention (include/derp_b200.h): every image, plane, mask and output argument may be host,
pinned, device or managed memory.  Each entry point of derp_b200.h that takes caller memory runs once with numpy arrays
and once with the same bytes as CUDA tensors on device 0, as pinned host tensors, at a device address one byte off every
alignment the kernels read with (so the library must stage it), and on a second GPU when there is one.  All inputs and
outputs of a run are of one kind; every output must equal the numpy run's bit for bit."""
import ctypes as C

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests.parity_util import scene_inputs

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


@pytest.fixture(params=["device", "pinned", "misaligned", "device1"])
def kind(request):
    if request.param == "device1" and torch.cuda.device_count() < 2:
        pytest.skip("needs a second CUDA device")
    return request.param


def _sync():
    for d in range(torch.cuda.device_count()):
        torch.cuda.synchronize(d)


class Mem:
    """nbytes of caller memory of one kind ("host" = a numpy array), holding a copy of `data` when given."""

    def __init__(self, kind, data=None, nbytes=None):
        raw = None if data is None else np.ascontiguousarray(data).view(np.uint8).reshape(-1).copy()
        self.kind = kind
        self.nbytes = raw.size if raw is not None else nbytes
        self.off = 1 if kind == "misaligned" else 0
        if kind == "host":
            self.a = raw if raw is not None else np.zeros(self.nbytes, np.uint8)
            self.ptr = self.a.ctypes.data
            return
        src = torch.from_numpy(raw) if raw is not None else torch.zeros(self.nbytes, dtype=torch.uint8)
        if kind == "pinned":
            self.t = src.pin_memory()
        else:
            self.t = torch.zeros(self.nbytes + self.off, dtype=torch.uint8, device="cuda:1" if kind == "device1" else "cuda:0")
            self.t[self.off:].copy_(src)
        self.ptr = self.t.data_ptr() + self.off
        _sync()

    def bytes(self):
        _sync()
        if self.kind == "host":
            return self.a.copy()
        return self.t[self.off:].cpu().numpy().copy()


class Run:
    """One run of entry points with every caller buffer of one kind; `out` collects what the library wrote."""

    def __init__(self, kind):
        self.kind, self.keep, self.outs = kind, [], []

    def inp(self, data):
        m = Mem(self.kind, data)
        self.keep.append(m)
        return m.ptr

    def ptrs(self, arrays):
        pa = (C.c_void_p * len(arrays))()
        for i, a in enumerate(arrays):
            pa[i] = self.inp(a)
        return pa

    def out(self, nbytes):
        m = Mem(self.kind, nbytes=nbytes)
        self.keep.append(m)
        self.outs.append(m)
        return m.ptr

    def results(self):
        return [m.bytes() for m in self.outs]


def same_as_host(body, kind):
    want, got = Run("host"), Run(kind)
    extra_want, extra_got = body(want), body(got)
    a, b = want.results(), got.results()
    assert len(a) == len(b) and len(a) > 0
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), (kind, "output", i)
    assert extra_want == extra_got, kind


def test_context_entry_points(cuda, kind):
    """Colours, masks, background, the level hand-off, both upsampling paths, brute force, eval cost, the getters and
    setters, and the gathered mismatch stage."""
    S, W, H = 4, 48, 40
    rig, colors, _ = scene_inputs(num_cams=S, width=W, height=H, kind="FTHETA")
    coarse_colors = [cuda.downscale_area(c, W // 2, H // 2) for c in colors]
    rng = np.random.RandomState(3)
    yy, xx = np.mgrid[0:H, 0:W]
    masks = [(((xx - W / 2 - 3 * s) ** 2 + (yy - H / 2) ** 2) < (0.4 * W) ** 2).astype(np.uint8) for s in range(S)]
    cmasks = [m[::2, ::2].copy() for m in masks]
    bgs = [(0.05 + rng.uniform(0, 0.01, (H, W))).astype(np.float32) for _ in range(S)]
    coarse = [rng.uniform(0.05, 1.0, (H // 2, W // 2)).astype(np.float32) for _ in range(S)]
    for c in coarse:
        c[rng.uniform(size=c.shape) < 0.05] = np.nan
    hyp = rng.uniform(0.05, 1.0, (H, W)).astype(np.float32)
    n = W * H

    def body(r):
        L = cuda.lib
        ctx = capi.Context(cuda, capi.rig_descs(rig))
        h = ctx.h
        try:
            ctx.level_begin(W // 2, H // 2, level=1, num_levels=2, full_width=W, full_height=H, use_foreground_masks=True)
            cuda.check(L.derp_set_colors(h, r.ptrs(coarse_colors)))
            for d in range(S):
                cuda.check(L.derp_set_disparity(h, d, r.inp(coarse[d]), r.inp(coarse[d] * 2), r.inp(coarse[d] * 3)))
            ctx.level_keep()
            ctx.level_begin(W, H, level=0, num_levels=2, full_width=W, full_height=H, use_foreground_masks=True)
            cuda.check(L.derp_set_colors(h, r.ptrs(colors)))
            cuda.check(L.derp_set_foreground_masks(h, r.ptrs(masks)))
            cuda.check(L.derp_set_background_disparity(h, r.ptrs(bgs)))
            for d in range(S):
                cuda.check(L.derp_upsample_from_kept(h, d, r.inp(cmasks[d]), r.inp(masks[d])))
                cuda.check(L.derp_get_disparity(h, d, r.out(4 * n), None, None))
            cuda.check(L.derp_upsample_from(h, 1, r.inp(coarse[1]), W // 2, H // 2, r.inp(cmasks[1]), r.inp(masks[1])))
            cuda.check(L.derp_reproject(h, 0))
            cuda.check(L.derp_brute_force(h, 0, 16, 0.5, 1e4, 1, r.out(4 * n)))
            cuda.check(L.derp_get_disparity(h, 0, r.out(4 * n), r.out(4 * n), r.out(4 * n)))
            cuda.check(L.derp_eval_cost(h, 0, r.inp(hyp), r.out(4 * n), r.out(4 * n)))
            cuda.check(L.derp_get_fov_mask(h, 0, r.out(n)))
            cuda.check(L.derp_get_variance(h, 1, r.out(4 * n)))
            cuda.check(L.derp_get_proj_warp(h, 1, r.out(8 * n)))
            cuda.check(L.derp_get_proj_color(h, 1, r.out(6 * n)))
            cuda.check(L.derp_get_proj_bias(h, 1, r.out(6 * n)))
            cuda.check(L.derp_mismatches(h))
            cuda.check(L.derp_get_mismatch_mask(h, 2, r.out(n)))
            planes = [ctx.get_disparity(d, want_cost=False) * np.float32(1.5) for d in range(S)]
            cuda.check(L.derp_gather_disparities(h, r.ptrs(planes)))
            cuda.check(L.derp_mismatches_gathered(h))
            for d in range(S):
                cuda.check(L.derp_get_disparity(h, d, r.out(4 * n), None, None))
            cuda.check(L.derp_get_mismatch_mask(h, 3, r.out(n)))
            return ctx.launch_count()
        finally:
            ctx.close()

    same_as_host(body, kind)


def test_downscale_area(cuda, kind):
    img = np.random.RandomState(4).randint(0, 65536, (60, 84, 3)).astype(np.uint16)

    def body(r):
        for w, h in ((42, 30), (35, 25)):  # integer ratio (resizeAreaFast_), general ratio
            cuda.check(cuda.lib.derp_downscale_area(0, r.inp(img), 84, 60, r.out(w * h * 6), w, h))

    same_as_host(body, kind)


def test_foreground_mask(cuda, kind):
    rng = np.random.RandomState(6)
    H, W = 50, 71
    bg = np.clip(rng.normal(30000, 9000, (H, W, 3)), 0, 65535).astype(np.uint16)
    fr = np.clip(bg.astype(np.int64) + rng.randint(-1500, 1500, bg.shape), 0, 65535).astype(np.uint16)
    fr[10:30, 20:50] = rng.randint(0, 65536, (20, 30, 3)).astype(np.uint16)

    def body(r):
        for blur, close in ((1, 4), (0, 0)):
            cuda.check(cuda.lib.derp_foreground_mask(0, r.inp(bg), r.inp(fr), W, H, blur, 0.04, close, r.out(W * H)))

    same_as_host(body, kind)


def test_upsample_disparity(cuda, kind):
    rig, _, _ = scene_inputs(num_cams=4, width=96, height=64, kind="FTHETA")
    desc = capi.camera_desc_from_json(rig["cameras"][1])
    rng = np.random.RandomState(2)
    coarse = rng.uniform(1e-4, 2, (32, 48)).astype(np.float32)
    coarse[3:6, 7:9] = np.nan
    cm = (rng.uniform(size=(32, 48)) > 0.3).astype(np.uint8)
    fm = (rng.uniform(size=(64, 96)) > 0.2).astype(np.uint8)
    bg = rng.uniform(0.01, 0.02, (64, 96)).astype(np.float32)

    def body(r):
        L = cuda.lib
        cuda.check(L.derp_upsample_disparity(0, C.byref(desc), r.inp(coarse), 48, 32, None, None, None, 100, 70, 0,
                                             r.out(100 * 70 * 4)))
        cuda.check(L.derp_upsample_disparity(0, C.byref(desc), r.inp(coarse), 48, 32, r.inp(bg), r.inp(cm), r.inp(fm), 96,
                                             64, 1, r.out(96 * 64 * 4)))

    same_as_host(body, kind)


def test_temporal_and_joint_bilateral(cuda, kind):
    rng = np.random.RandomState(11)
    H, W, T = 30, 38, 3
    base = rng.randint(0, 65536, (H, W, 3))
    guides = [np.clip(base + rng.randint(-300, 300, (H, W, 3)), 0, 65535).astype(np.uint16) for _ in range(T)]
    disps = [rng.uniform(1e-3, 2, (H, W)).astype(np.float32) for _ in range(T)]
    masks = [(rng.uniform(size=(H, W)) > 0.15).astype(np.uint8) for _ in range(T)]
    guide = guides[0].astype(np.float32) * (np.float32(1.0) / np.float32(65535.0))

    def body(r):
        L = cuda.lib
        cuda.check(L.derp_temporal_filter(0, W, H, T, r.ptrs(guides), r.ptrs(disps), r.ptrs(masks), 1, 0.01, 1, 0.5, 1.0,
                                          0.5, r.out(W * H * 4)))
        for radius in (3, 20):  # the shared-memory tile and the global-memory kernel
            cuda.check(L.derp_joint_bilateral_f32(0, W, H, r.inp(disps[0]), r.inp(guide), r.inp(masks[0]), radius, 0.05,
                                                  0.5, 0.5, 1.0, r.out(W * H * 4)))

    same_as_host(body, kind)


def test_device_copy(cuda, kind):
    data = np.random.RandomState(1).randint(0, 256, 1000).astype(np.uint8)

    def body(r):
        cuda.check(cuda.lib.derp_device_copy(0, r.out(1000), r.inp(data), 1000))

    same_as_host(body, kind)


def test_camera_mesh(cuda, kind):
    rng = np.random.RandomState(9)
    H, W = 40, 52
    disp = rng.uniform(0.05, 1.0, (H, W)).astype(np.float32)
    disp[5:9, 10:14] = np.nan
    fg = (rng.uniform(size=(H // 2, W // 2)) > 0.2).astype(np.uint8)

    def body(r):
        L, counts = cuda.lib, []
        for triangles in (0, 500):
            nv, nf = C.c_uint64(), C.c_uint64()
            head = (0, r.inp(disp), W, H, 1.0, float(W), float(H), 30.0, 0.95, r.inp(fg), W // 2, H // 2)
            tail = (r.out(W * H * 12), r.out(W * H * 24), C.byref(nv), C.byref(nf))
            if triangles:
                cuda.check(L.derp_camera_mesh_simplified(*head, triangles, *tail))
            else:
                cuda.check(L.derp_camera_mesh(*head, *tail))
            counts.append((nv.value, nf.value))
        return counts

    same_as_host(body, kind)


def test_bc7(cuda, kind):
    rng = np.random.RandomState(7)
    h, w = 22, 36  # partial block rows stay zero
    rgba = rng.randint(0, 256, (h, w, 4)).astype(np.uint8)
    bgr16 = rng.randint(0, 65536, (h, w, 3)).astype(np.uint16)
    bgr8 = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)

    def body(r):
        L = cuda.lib
        cuda.check(L.derp_bc7_compress(0, r.inp(rgba), w, h, r.out(w * h)))
        cuda.check(L.derp_bc7_compress_image(0, r.inp(bgr16), 16, 3, w, h, 2.2 / 1.8, r.out(w * h)))
        cuda.check(L.derp_bc7_compress_image(0, r.inp(bgr8), 8, 3, w, h, 2.2 / 1.8, r.out(w * h)))

    same_as_host(body, kind)
