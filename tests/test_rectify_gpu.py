"""GPU parity of util::stereo_rectifier: b200_rectifier_maps, b200_stereo_rectify and b200_stereo_rectify_device against the CPU
restatement (tests/rectify_oracle.c, itself pinned to OpenCV in test_rectify_cpu.py), bit for bit; and the stereo front end from a
RAW pair: rectify on the device -> one ORB extract over both eyes -> match::stereo, against oracle remap -> oracle extract -> oracle
stereo."""
import ctypes as C

import numpy as np
import pytest

import rectify_oracle as R
from golden.natural import load_images
from oracle import pyoracle as O
from stella_vslam_b200 import feature, match
from stella_vslam_b200._lib import ERR_INVALID, KP_DTYPE, RectifierParams, check, lib
from workloads import synth

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def _rot(w):
    w = np.asarray(w, np.float64)
    t = np.linalg.norm(w)
    if t == 0:
        return np.eye(3)
    k = w / t
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(t) * Kx + (1 - np.cos(t)) * Kx @ Kx


def _random_calib(seed, cols, rows, model, n_dist):
    rng = np.random.default_rng(seed)
    f = rng.uniform(300, 900)
    K = (f, 0, cols / 2 + rng.uniform(-30, 30), 0, f * rng.uniform(0.98, 1.02), rows / 2 + rng.uniform(-30, 30), 0, 0, 1)
    fr = f * (0.9 if model == "perspective" else 0.4)
    sig = [0.2, 0.05, 1e-3, 1e-3, 0.01, 0.1, 0.02, 0.01] if model == "perspective" else [0.05, 0.01, 0.005, 0.001]
    return dict(model=model, cols=cols, rows=rows, K_rect=(fr, 0, cols / 2, 0, fr, rows / 2, 0, 0, 1), K=(K, K),
                D=(tuple(rng.normal(0, sig[:n_dist])), tuple(rng.normal(0, sig[:n_dist]))),
                R=(tuple(_rot(rng.normal(0, 0.05, 3)).ravel()), tuple(_rot(rng.normal(0, 0.05, 3)).ravel())))


def _shifted(cols, rows):
    """Identity rotation, no distortion, principal points moved so that the maps leave the source on every side (left eye: up and
    left, right eye: down and right) and land on integer coordinates in the middle."""
    Kr = (100.0, 0, cols / 2, 0, 100.0, rows / 2, 0, 0, 1)
    return dict(model="perspective", cols=cols, rows=rows, K_rect=Kr, K=((100.0, 0, cols / 2 - 7, 0, 100.0, rows / 2 - 5, 0, 0, 1),
                                                                            (100.0, 0, cols / 2 + 6.5, 0, 100.0, rows / 2 + 3.25, 0, 0, 1)),
                D=((0, 0, 0, 0), (0, 0, 0, 0, 0)), R=(tuple(np.eye(3).ravel()), tuple(np.eye(3).ravel())))


def _behind():
    cal = dict(synth.TUM_VI_STEREO)
    cal["R"] = (tuple(_rot([0.0, 1.9, 0.0]).ravel()), tuple(_rot([0.0, -1.9, 0.3]).ravel()))
    return cal


CASES = {
    "euroc": synth.EUROC_STEREO, "tum_vi": synth.TUM_VI_STEREO, "fisheye_behind": _behind(),
    "persp4_1241": _random_calib(1, 1241, 376, "perspective", 4), "persp5_1920": _random_calib(2, 1920, 1080, "perspective", 5),
    "persp8_1241": _random_calib(3, 1241, 376, "perspective", 8), "fisheye_1920": _random_calib(4, 1920, 1080, "fisheye", 4),
    "shifted_752": _shifted(752, 480), "tiny_1x1": _shifted(1, 1), "tiny_3x5": _shifted(3, 5),
}


def _rectifier(cal):
    return feature.stereo_rectifier(cal["model"], cal["cols"], cal["rows"], cal["K_rect"], cal["K"][0], cal["D"][0], cal["R"][0], cal["K"][1],
                                    cal["D"][1], cal["R"][1])


def _frames(cal, channels, n, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (n, cal["rows"], cal["cols"]) + (() if channels == 1 else (channels,)), dtype=np.uint8)


@pytest.mark.parametrize("name", list(CASES))
def test_maps_bit_identical_to_oracle(name):
    cal = CASES[name]
    rect = _rectifier(cal)
    for eye in range(2):
        want = R.rect_map(cal["model"], cal["cols"], cal["rows"], cal["K"][eye], cal["D"][eye], cal["R"][eye], cal["K_rect"])
        got = rect.maps(eye)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("channels", [1, 3, 4])
def test_host_rectify_bit_identical_to_oracle(name, channels):
    cal = CASES[name]
    rect = _rectifier(cal)
    left, right = _frames(cal, channels, 2, seed=channels)
    got = rect.rectify(left, right)
    want = R.rectify_pair(cal, left, right)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_host_rectify_natural_euroc_frame(golden_dir):
    img = load_images(golden_dir)["euroc_752x480"]
    rect = _rectifier(synth.EUROC_STEREO)
    got = rect.rectify(img, img[::-1].copy())
    want = R.rectify_pair(synth.EUROC_STEREO, img, img[::-1].copy())
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def _device_run(rect, cal, channels, batch, src_pad, out_pad, interleave, seed=0):
    """Frames in padded device buffers (row pitch = cols * channels + pad); returns (got_left, got_right) and the oracle's."""
    rows, row = cal["rows"], cal["cols"] * channels
    left, right = _frames(cal, channels, batch, seed), _frames(cal, channels, batch, seed + 1)
    sp, op = row + src_pad, row + out_pad

    def upload(frames):
        buf = torch.zeros((batch, rows, sp), dtype=torch.uint8, device="cuda")
        buf[:, :, :row] = torch.from_numpy(frames.reshape(batch, rows, row)).cuda()
        return buf

    dl, dr = upload(left), upload(right)
    out = torch.full((2 * batch, rows, op), 7, dtype=torch.uint8, device="cuda")
    rect.set_stream(torch.cuda.current_stream())    # ordered after the uploads and the fill
    if interleave:   # eye e of pair f at frame 2 f + e
        ol, orr, ofs = out[0::2], out[1::2], 2 * rows * op
    else:
        ol, orr, ofs = out[:batch], out[batch:], rows * op
    check(lib().b200_stereo_rectify_device(rect._h, channels, dl.data_ptr(), dr.data_ptr(), sp, rows * sp, ol.data_ptr(), orr.data_ptr(), op,
                                           ofs, batch))
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert (o[:, :, row:] == 7).all()    # the row padding is never written
    got_l, got_r = (o[0::2], o[1::2]) if interleave else (o[:batch], o[batch:])
    got_l, got_r = got_l[:, :, :row].reshape(left.shape), got_r[:, :, :row].reshape(right.shape)
    maps = [R.rect_map(cal["model"], cal["cols"], rows, cal["K"][e], cal["D"][e], cal["R"][e], cal["K_rect"]) for e in range(2)]
    want_l = np.stack([R.remap(f, *maps[0]) for f in left])
    want_r = np.stack([R.remap(f, *maps[1]) for f in right])
    return (got_l, got_r), (want_l, want_r)


@pytest.mark.parametrize("name", ["euroc", "tum_vi", "fisheye_behind", "persp4_1241", "shifted_752", "tiny_3x5", "tiny_1x1"])
@pytest.mark.parametrize("channels", [1, 3, 4])
@pytest.mark.parametrize("batch", [1, 64])
@pytest.mark.parametrize("pads", [(0, 0), (16, 16), (3, 5)], ids=["dense", "pad16", "unaligned"])
@pytest.mark.parametrize("interleave", [False, True], ids=["planar", "interleaved"])
def test_device_rectify_bit_identical_to_oracle(name, channels, batch, pads, interleave):
    cal = CASES[name]
    if batch == 64 and cal["cols"] * cal["rows"] > 400000:
        batch = 8    # keeps the oracle's share of the run short; 64 is covered on the EuRoC and TUM-VI sizes
    rect = _rectifier(cal)
    got, want = _device_run(rect, cal, channels, batch, pads[0], pads[1], interleave, seed=batch + channels)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_device_rectify_on_torch_stream():
    cal = synth.EUROC_STEREO
    rect = _rectifier(cal)
    s = torch.cuda.Stream()
    rect.set_stream(s)
    left, right = _frames(cal, 1, 4, 1), _frames(cal, 1, 4, 2)
    with torch.cuda.stream(s):
        dl, dr = torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda()
        out = torch.empty((8, cal["rows"], cal["cols"]), dtype=torch.uint8, device="cuda")
        rect.rectify_device(dl, dr, out[0::2], out[1::2])
    s.synchronize()
    rect.set_stream(None)
    o = out.cpu().numpy()
    for f in range(4):
        want = R.rectify_pair(cal, left[f], right[f])
        assert np.array_equal(o[2 * f], want[0]) and np.array_equal(o[2 * f + 1], want[1])


@pytest.mark.parametrize("name", ["euroc", "tum_vi"])
def test_raw_pair_chain_bit_identical_to_oracle(name):
    """raw pair -> b200_stereo_rectify_device (eyes interleaved) -> b200_orb_extract_device over 2B frames -> b200_stereo_compute(h, 2p,
    h, 2p + 1), on one torch stream, against oracle remap -> oracle extract -> oracle stereo."""
    cal = {"euroc": synth.EUROC_STEREO, "tum_vi": synth.TUM_VI_STEREO}[name]
    B, rows, cols = 2, cal["rows"], cal["cols"]
    raw = [synth.make_raw_stereo_pair(cal, seed=31 + p) for p in range(B)]
    rect = _rectifier(cal)
    ex = feature.orb_extractor(feature.orb_params(), 800, max_batch=2 * B)
    s = torch.cuda.Stream()
    rect.set_stream(s)
    check(lib().b200_orb_set_stream(ex._h, C.c_void_p(s.cuda_stream), 0))
    with torch.cuda.stream(s):
        dl = torch.from_numpy(np.stack([r[0] for r in raw])).cuda()
        dr = torch.from_numpy(np.stack([r[1] for r in raw])).cuda()
        frames = torch.empty((2 * B, rows, cols), dtype=torch.uint8, device="cuda")
        rect.rectify_device(dl, dr, frames[0::2], frames[1::2])
        check(lib().b200_orb_extract_device(ex._h, C.c_void_p(frames.data_ptr()), cols, rows, cols, rows * cols, 2 * B, None, 0))
    cap = lib().b200_orb_max_keypoints(ex._h, cols, rows)
    kps, desc, counts = np.zeros((2 * B, cap), KP_DTYPE), np.zeros((2 * B, cap, 32), np.uint8), np.zeros(2 * B, np.int32)
    check(lib().b200_orb_fetch(ex._h, kps.ctypes.data, desc.ctypes.data, cap, counts.ctypes.data))
    s.synchronize()
    assert np.array_equal(frames.cpu().numpy()[0], R.rectify_pair(cal, *raw[0])[0])
    for p in range(B):
        want_l, want_r = R.rectify_pair(cal, *raw[p])
        a = O.orb_extract(want_l, min_area=800, want_pyramid=True)
        b = O.orb_extract(want_r, min_area=800, want_pyramid=True)
        kl, kr = kps[2 * p, :counts[2 * p]], kps[2 * p + 1, :counts[2 * p + 1]]
        dl_, dr_ = desc[2 * p, :counts[2 * p]], desc[2 * p + 1, :counts[2 * p + 1]]
        assert np.array_equal(kl, a["kps"]) and np.array_equal(dl_, a["desc"])
        assert np.array_equal(kr, b["kps"]) and np.array_equal(dr_, b["desc"])
        fxb = cal["fxb"]
        xr_want, dep_want, n_want = O.stereo_compute(a["pyramid"], b["pyramid"], a["kps"], a["desc"], b["kps"], b["desc"], fxb, fxb / cal["K_rect"][0])
        st = match.stereo(ex, ex, kl, kr, dl_, dr_, fxb, fxb / cal["K_rect"][0], frame_left=2 * p, frame_right=2 * p + 1)
        xr, dep = st.compute()
        assert np.array_equal(xr, xr_want) and np.array_equal(dep, dep_want) and st.num_matched_ == n_want
        assert n_want > 0.1 * len(kl), (n_want, len(kl))
    rect.set_stream(None)
    check(lib().b200_orb_set_stream(ex._h, None, 1))


def test_invalid_input_writes_nothing():
    cal = synth.EUROC_STEREO
    rect = _rectifier(cal)
    rows, cols = cal["rows"], cal["cols"]
    L = lib()
    src = torch.zeros((2, rows, cols), dtype=torch.uint8, device="cuda")
    out = torch.full((2, rows, cols), 9, dtype=torch.uint8, device="cuda")
    a, b, o0, o1 = src[0].data_ptr(), src[1].data_ptr(), out[0].data_ptr(), out[1].data_ptr()
    bad = [(rect._h, 2, a, b, cols, 0, o0, o1, cols, 0, 1), (rect._h, 1, a, b, cols - 1, 0, o0, o1, cols, 0, 1),
           (rect._h, 1, a, b, cols, 0, o0, o1, cols - 1, 0, 1), (rect._h, 3, a, b, cols, 0, o0, o1, cols, 0, 1),
           (rect._h, 1, None, b, cols, 0, o0, o1, cols, 0, 1), (rect._h, 1, a, b, cols, 0, o0, None, cols, 0, 1),
           (rect._h, 1, a, b, cols, rows * cols - 1, o0, o1, cols, rows * cols, 2), (rect._h, 1, a, b, cols, 0, o0, o1, cols, 0, -1),
           (None, 1, a, b, cols, 0, o0, o1, cols, 0, 1)]
    for args in bad:
        assert L.b200_stereo_rectify_device(*args) == ERR_INVALID, args
    assert L.b200_stereo_rectify_device(rect._h, 1, a, b, cols, 0, o0, o1, cols, 0, 0) == 0     # batch 0: nothing to do
    torch.cuda.synchronize()
    assert (out == 9).all()
    h_out = np.full((2, rows, cols), 9, np.uint8)
    h_src = np.zeros((rows, cols), np.uint8)
    assert L.b200_stereo_rectify(rect._h, 1, h_src.ctypes.data, cols - 1, h_src.ctypes.data, cols, h_out[0].ctypes.data, cols,
                                 h_out[1].ctypes.data, cols) == ERR_INVALID
    assert L.b200_stereo_rectify(rect._h, 5, h_src.ctypes.data, cols, h_src.ctypes.data, cols, h_out[0].ctypes.data, cols,
                                 h_out[1].ctypes.data, cols) == ERR_INVALID
    assert (h_out == 9).all()
    mx = np.zeros((rows, cols), np.float32)
    assert L.b200_rectifier_maps(rect._h, 2, mx.ctypes.data, mx.ctypes.data) == ERR_INVALID


def test_create_rejects_bad_parameters():
    cal = synth.EUROC_STEREO
    L = lib()

    def params(**kw):
        p = RectifierParams()
        p.model, p.cols, p.rows, p.device = kw.get("model", 0), kw.get("cols", 752), kw.get("rows", 480), 0
        p.K_rect[:] = list(cal["K_rect"])
        for e in range(2):
            p.K[e][:] = list(cal["K"][e])
            p.R[e][:] = list(kw.get("R", cal["R"][e]))
            p.D[e][:5] = list(cal["D"][e])
            p.n_dist[e] = kw.get("n_dist", 5)
        return p

    for kw in (dict(n_dist=12), dict(n_dist=14), dict(n_dist=3), dict(model=1, n_dist=5), dict(model=2), dict(cols=0), dict(rows=40000),
               dict(R=(0,) * 9)):
        h = C.c_void_p()
        assert L.b200_rectifier_create(C.byref(params(**kw)), C.byref(h)) == ERR_INVALID, kw
        assert not h.value
    h = C.c_void_p()
    assert L.b200_rectifier_create(C.byref(params(n_dist=8)), C.byref(h)) == 0 and h.value
    L.b200_rectifier_destroy(h)
