"""derp_resize_area and ResizeFrames on the GPU: the library against tests/golden/resize_vectors.npz and live cv2 (0
differing values; NaN compared as NaN, -0 as -0), every kind of caller pointer, all ten levels of the golden rig's 3360 x
2160 images for every sample type and channel count, the app end to end against resize_camera restated with cv2, and
DerpCLI on the app's levels against DerpCLI on cv2's, disparity files byte for byte."""
import json
import os
import subprocess

import numpy as np
import pytest

from facebook360_dep_b200 import capi
from tests.golden import gen_resize_vectors as gv
from tests.test_resize_frames import APP, BIN, GOLDEN_RIG, VECTORS, level_sizes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rs(cuda):
    return capi.Resize(cuda)


def test_golden_vectors(rs):
    vec = np.load(VECTORS)
    n = 0
    for key, bits, ch, src, dst, content, seed, thr in gv.cases():
        img = gv.source(bits, ch, src[0], src[1], content, seed)
        got = rs.resize_area(img, dst[0], dst[1], thr)
        assert gv.same_values(got, vec[key]), key
        assert gv.same_values(got, gv.cv_resize(img, dst, thr)), key
        n += 1
    assert n == len(vec.files)


@pytest.mark.parametrize("bits", [8, 16, 32])
def test_random_shapes_against_cv2(rs, bits):
    """Random sizes in both directions, from 1 x 1 up, against live cv2."""
    rng = np.random.RandomState(bits)
    for i in range(120):
        ch = [1, 3, 4][i % 3]
        sw, sh, dw, dh = (int(v) for v in rng.randint(1, 90, 4))
        img = gv.source(bits, ch, sw, sh, "special" if bits == 32 and i % 2 else "random", 1000 * bits + i)
        thr = 127 if bits == 8 and i % 4 == 0 else None
        assert gv.same_values(rs.resize_area(img, dw, dh, thr), gv.cv_resize(img, (dw, dh), thr)), (ch, sw, sh, dw, dh)


@pytest.mark.parametrize("kind", ["device", "pinned", "misaligned", "device1"])
def test_caller_pointers(rs, kind):
    import torch
    from tests.test_gpu_caller_pointers import same_as_host
    if kind == "device1" and torch.cuda.device_count() < 2:
        pytest.skip("needs a second CUDA device")
    cases = [(8, 3, (83, 45), (40, 22), -1), (16, 4, (83, 45), (166, 91), -1), (32, 1, (83, 45), (20, 15), -1),
             (8, 1, (83, 45), (83, 45), 127), (16, 3, (84, 46), (42, 23), -1), (32, 4, (83, 45), (83, 45), -1)]

    def body(r):
        for bits, ch, (sw, sh), (dw, dh), thr in cases:
            img = gv.source(bits, ch, sw, sh, "random", bits + ch)
            out = r.out(dw * dh * ch * img.itemsize)
            rs.check(rs.lib.derp_resize_area(0, r.inp(img), bits, ch, sw, sh, out, dw, dh, thr))

    same_as_host(body, kind)


@pytest.mark.parametrize("bits", [8, 16, 32])
@pytest.mark.parametrize("channels", [1, 3, 4])
def test_golden_rig_levels(rs, bits, channels):
    """The ten levels of a 3360 x 2160 image, from a device copy of it as the app passes it, each against cv2."""
    import torch
    img = gv.source(bits, channels, 3360, 2160, "random", 7 * bits + channels)
    dsrc = torch.from_numpy(img.copy()).cuda()
    for W, H in level_sizes((3360, 2160)):
        out = np.empty((H, W) + img.shape[2:], img.dtype)
        rs.check(rs.lib.derp_resize_area(0, dsrc.data_ptr(), bits, channels, 3360, 2160, out.ctypes.data, W, H, -1))
        assert gv.same_values(out, gv.cv_resize(img, (W, H))), (W, H)


# ---- the app -----------------------------------------------------------------------------------------------------------
RESOLUTIONS = [(640, 427), (300, 200)]  # an odd height; a camera narrower than every level above 256


def read_level(path):
    import cv2
    return cv2.imread(str(path), cv2.IMREAD_UNCHANGED)


def resize_camera(src, dst, cid, resolution, frame, ext, threshold):
    """resize_camera (resize.py:51-85) with cv2: imread(UNCHANGED), resize, threshold, imwrite.  For .pfm, cv2.imread and
    cv2.imwrite order the rows as imageio (FreeImage) does in resize.py: the file's last row is the image's first."""
    import cv2
    img = cv2.imread(os.path.join(src, cid, frame + ext), cv2.IMREAD_UNCHANGED)
    for level, (W, H) in enumerate(level_sizes(resolution)):
        d = os.path.join(dst, "level_%d" % level, cid)
        os.makedirs(d, exist_ok=True)
        assert cv2.imwrite(os.path.join(d, frame + ext), gv.cv_resize(img, (W, H), threshold))


def listing(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


def write_pfm(path, img):
    """A PFM as the project writes it (io::writePfm, DerpCLI's disparities): the top row first."""
    with open(path, "wb") as f:
        f.write(b"Pf\n%d %d\n-1.0\n" % (img.shape[1], img.shape[0]) + np.ascontiguousarray(img, np.float32).tobytes())


def make_frame(kind, w, h, rng, seed):
    if kind == "color8":
        return rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
    if kind == "color16":
        return rng.randint(0, 65536, (h, w, 3)).astype(np.uint16)
    if kind == "color16_rgba":
        return rng.randint(0, 65536, (h, w, 4)).astype(np.uint16)
    if kind == "masks":
        return (rng.uniform(size=(h, w)) < 0.5).astype(np.uint8) * 255
    return gv.source(32, 1, w, h, "special", seed)


@pytest.mark.parametrize("kind", ["color8", "color16", "color16_rgba", "masks", "pfm", "mixed"])
def test_app_matches_resize_camera(tmp_path, cuda, kind):
    """Decoded level files and their names against resize_camera with cv2.  "mixed": one camera of PNG, one of PFM (each
    camera's extension is its own)."""
    import cv2
    from tests.test_resize_frames import write_rig
    ids = write_rig(tmp_path / "rig.json", RESOLUTIONS)
    threshold = 127 if kind == "masks" else None
    frames = ["000011", "000012"]
    rng = np.random.RandomState(len(kind))
    kinds = {"mixed": ["color16", "pfm"]}.get(kind, [kind, kind])
    for cid, (w, h), k in zip(ids, RESOLUTIONS, kinds):
        os.makedirs(tmp_path / "src" / cid)
        for f in frames:
            img = make_frame(k, w, h, rng, len(f) + w)
            if k == "pfm":
                write_pfm(tmp_path / "src" / cid / (f + ".pfm"), img)
            else:
                assert cv2.imwrite(str(tmp_path / "src" / cid / (f + ".png")), img)
    args = [APP, "--rig=" + str(tmp_path / "rig.json"), "--src_dir=" + str(tmp_path / "src"),
            "--dst_dir=" + str(tmp_path / "app")]
    if threshold is not None:
        args.append("--threshold=%d" % threshold)
    r = subprocess.run(args, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    for f in frames:
        for cid, res, k in zip(ids, RESOLUTIONS, kinds):
            resize_camera(str(tmp_path / "src"), str(tmp_path / "cv"), cid, res, f, ".pfm" if k == "pfm" else ".png",
                          threshold)
    names = listing(tmp_path / "app")
    assert names == listing(tmp_path / "cv") and len(names) == 10 * len(ids) * len(frames)
    for name in names:
        got, want = read_level(tmp_path / "app" / name), read_level(tmp_path / "cv" / name)
        assert gv.same_values(got, want), name
    if "pfm" in kinds:  # the row order matters: resizing the rows top-down would differ
        cid, res = [(c, r) for c, r, k in zip(ids, RESOLUTIONS, kinds) if k == "pfm"][0]
        img = make_frame("pfm", res[0], res[1], np.random.RandomState(0), 1)
        W, H = level_sizes(res)[0]
        assert not gv.same_values(gv.cv_resize(img, (W, H)), gv.cv_resize(img[::-1].copy(), (W, H))[::-1])


def test_derpcli_on_app_levels_matches_cv2_levels(tmp_path, cuda):
    """DerpCLI over the coarsest four levels (--level_end=6) of a 4-camera rig: the pyramid ResizeFrames made and the one
    resize_camera makes with cv2 give byte-identical disparity files."""
    import cv2
    from facebook360_dep_b200 import synth
    W, H = 320, 213
    rig = synth.ring_rig(4, W, H, kind="FTHETA")
    colors, _ = synth.render_rig(rig, W, H)
    ids = [c["id"] for c in rig["cameras"]]
    full = tmp_path / "full"
    for cid, img in zip(ids, colors):
        os.makedirs(full / cid)
        assert cv2.imwrite(str(full / cid / "000000.png"), img)
    outs = []
    for maker in ("app", "cv"):
        root = tmp_path / maker
        os.makedirs(root / "rigs")
        json.dump(rig, open(root / "rigs" / "rig_calibrated.json", "w"))
        levels = root / "video" / "color_levels"
        if maker == "app":
            subprocess.run([APP, "--rig=" + str(root / "rigs" / "rig_calibrated.json"), "--src_dir=" + str(full),
                            "--dst_dir=" + str(levels)], check=True, capture_output=True)
        else:
            for cid in ids:
                resize_camera(str(full), str(levels), cid, (W, H), "000000", ".png", None)
        out = tmp_path / (maker + "_out")
        subprocess.run([os.path.join(BIN, "DerpCLI"), "--input_root=" + str(root), "--output_root=" + str(out),
                        "--first=000000", "--last=000000", "--level_end=6", "--partial_coverage=true", "--num_depths=64",
                        "--gpus=1"], check=True, capture_output=True)
        outs.append(out)
    names = [n for n in listing(outs[0]) if n.endswith(".pfm")]
    assert names == [n for n in listing(outs[1]) if n.endswith(".pfm")]
    assert {n.split(os.sep)[1] for n in names if n.startswith("disparity_levels")} == {"level_6", "level_7", "level_8",
                                                                                       "level_9"}
    for n in names:
        assert open(outs[0] / n, "rb").read() == open(outs[1] / n, "rb").read(), n
