"""GPU tests of the per-frame undistortion (ldso_b200_set_undistort / ldso_b200_undistort_frame): the device's rectified image against
the fixtures the undistortion pin wrote (the reference's own Undistort::undistort<T>, bit for bit), the pyramid and a tracker run built
from it against make_images of the host-rectified image, the edge rule against the restatement, and the error returns."""
import ctypes as C

import numpy as np
import pytest

from ldso_b200 import capi, synth
from tests import undistort_oracle as U

pytestmark = pytest.mark.gpu

LEVELS = 3


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _set(ctx, c, rx, ry, G, vinv):
    ctx.set_undistort(int(c["wOrg"]), int(c["hOrg"]), rx, ry, G, vinv, int(c["mode"]), bool(c["use_exposure"]))


@pytest.mark.parametrize("cam", U.CAMERAS)
def test_level0_matches_the_reference_bit_for_bit(cam):
    """Every fixture case: 8- and 16-bit frames, modes 0 / 1 / 2, the factor path (no valid G, exposure <= 0), no exposure, and
    passthrough (pinhole_none): the device's level-0 intensity equals the reference's image at every pixel, and the exposure time
    equals processFrame's."""
    t = U.tables()
    (rx, ry), cases = U.camera(cam)
    c0 = cases[0][0]
    ctx = capi.Context(int(c0["w"]), int(c0["h"]), LEVELS)
    for c, expected, past in cases:
        raw, G, vinv = U.case_inputs(t, c)
        _set(ctx, c, rx, ry, G, vinv)
        e = ctx.undistort_frame(0, raw, float(c["exposure"]), float(c["factor"]))
        assert np.float32(e) == c["exposure_out"], (cam, c["name"])
        got = ctx.download_frame_level(0, 0)[..., 0]
        assert np.array_equal(_bits(got), _bits(expected)), (cam, c["name"], int((_bits(got) != _bits(expected)).sum()))
    ctx.close()


@pytest.mark.parametrize("cam", ["radtan_crop", "kb_crop", "pinhole_none"])
def test_pyramid_equals_make_images_of_the_rectified_image(cam):
    t = U.tables()
    (rx, ry), cases = U.camera(cam)
    for c, expected, _ in cases:
        if c["name"] not in ("u8_m2", "u16_m1", "u8_nogamma"):
            continue
        ctx = capi.Context(int(c["w"]), int(c["h"]), LEVELS)
        raw, G, vinv = U.case_inputs(t, c)
        _set(ctx, c, rx, ry, G, vinv)
        ctx.undistort_frame(0, raw, float(c["exposure"]), float(c["factor"]))
        ctx.make_images(1, expected)
        for l in range(LEVELS):
            assert np.array_equal(_bits(ctx.download_frame_level(0, l)), _bits(ctx.download_frame_level(1, l))), (cam, c["name"], l)
        ctx.close()


def _edge_remap(w, h, wOrg, hOrg, rng):
    """A remap table that reaches every branch: outside (-1), the two past-the-end offsets, xxi = wOrg-1 (row wrap), offsets beyond the
    range check, integer coordinates, and random interior points."""
    rx = rng.uniform(0, wOrg - 1, (h, w)).astype(np.float32)
    ry = rng.uniform(0, hOrg - 1, (h, w)).astype(np.float32)
    special = [(0.25, hOrg - 1 + 0.5), (wOrg - 1 + 0.75, hOrg - 2 + 0.125), (wOrg - 1 + 0.5, 3.5), (wOrg - 1 + 0.99, 0.0),
               (1.5, hOrg - 1 + 0.25), (3.0, wOrg - 1.5), (-1.0, -1.0), (-0.0, 5.5), (7.0, 9.0), (0.0, 0.0)]
    flat_x, flat_y = rx.reshape(-1), ry.reshape(-1)
    for k, (x, y) in enumerate(special * 8):
        i = rng.integers(0, w * h)
        flat_x[i], flat_y[i] = x, y
    return rx, ry


@pytest.mark.parametrize("bpp,mode", [(1, 2), (2, 2), (1, 0), (2, 1)])
def test_edge_rule_matches_the_restatement(bpp, mode):
    """Taps past the end of the raw frame read 0, a tap at xxi = wOrg-1 wraps to the next row, offsets past the range check give 0."""
    rng = np.random.default_rng(5 + bpp + 3 * mode)
    w, h, wOrg, hOrg = 64, 48, 40, 30
    rx, ry = _edge_remap(w, h, wOrg, hOrg, rng)
    raw = rng.integers(0, 256 if bpp == 1 else 65536, (hOrg, wOrg)).astype(np.uint8 if bpp == 1 else np.uint16)
    G = np.sort(rng.uniform(0, 255, 256 if bpp == 1 else 65536)).astype(np.float32)
    vinv = rng.uniform(1.0, 2.5, (hOrg, wOrg)).astype(np.float32)
    exp_img, e, past = U.undistort(raw, w, h, rx, ry, G, vinv, mode, 1, 1.25, 0.5)
    assert past.sum() > 0
    ctx = capi.Context(w, h, LEVELS)
    ctx.set_undistort(wOrg, hOrg, rx, ry, G, vinv, mode, True)
    assert ctx.undistort_frame(2, raw, 1.25, 0.5) == e
    got = ctx.download_frame_level(2, 0)[..., 0]
    assert np.array_equal(_bits(got), _bits(exp_img)), int((_bits(got) != _bits(exp_img)).sum())
    ctx.close()


def test_tracker_from_undistort_frame_equals_make_images():
    """trackNewestCoarse on a new frame built by undistort_frame gives the same bits as on the one make_images built from the
    host-rectified image."""
    pair = synth.make_track_pair(w=320, h=240, n_pts=400, seed=7)
    from tests import oracle_py
    ot = oracle_py.OracleTracker(pair)
    ctx = capi.Context(pair.w, pair.h, pair.levels)
    ctx.upload_frame(0, pair.ref_pyr)
    ctx.tracker_make_k(*[float(x) for x in pair.K])
    for l in range(pair.levels):
        ctx.tracker_set_ref_level(l, *ot.pc(l))
    # a raw 8-bit frame one pixel larger on each side than the new image, remapped back with a sub-pixel shift
    wOrg, hOrg = pair.w + 2, pair.h + 2
    img = np.pad(np.asarray(pair.new_pyr[0])[..., 0].reshape(pair.h, pair.w), 1, mode="edge")
    raw = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    ys, xs = np.mgrid[0:pair.h, 0:pair.w].astype(np.float32)
    rx, ry = xs + np.float32(1.3), ys + np.float32(0.8)
    G = (255.0 * np.linspace(0.0, 1.0, 256) ** 0.8).astype(np.float32)
    vinv = np.full((hOrg, wOrg), 1.0625, np.float32)
    host, _, _ = U.undistort(raw, pair.w, pair.h, rx, ry, G, vinv, 2, 1, 1.0, 1.0)
    results = []
    for use_device in (False, True):
        if use_device:
            ctx.set_undistort(wOrg, hOrg, rx, ry, G, vinv, 2, True)
            ctx.undistort_frame(1, raw, 1.0, 1.0)
        else:
            ctx.make_images(1, host)
        ctx.tracker_set_frames(pair.ref_aff[0], pair.ref_aff[1], 1.0, 1, 1.0)
        results.append(ctx.tracker_track(np.eye(3), np.zeros(3), 0.0, 0.0, pair.levels - 1))
    a, b = results
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y), equal_nan=True), (x, y)
    ctx.close()


def test_error_returns():
    L = capi.load()
    ctx = capi.Context(32, 24, LEVELS)
    raw8 = np.zeros((24, 32), np.uint8)
    raw16 = np.zeros((24, 32), np.uint16)
    ERR_ARG, ERR_STATE = -1, -3
    e = C.c_float(0)

    def frame(raw, bpp=None):
        return L.ldso_b200_undistort_frame(ctx.ctx, 0, None if raw is None else raw.ctypes.data_as(C.c_void_p),
                                           raw.itemsize if bpp is None else bpp, 1.0, 1.0, C.byref(e))
    assert frame(raw8) == ERR_STATE          # before any set_undistort
    rx = np.zeros(32 * 24, np.float32)
    G8, G16 = np.arange(256, dtype=np.float32), np.arange(65536, dtype=np.float32)
    vinv = np.ones(40 * 30, np.float32)
    f = lambda a: None if a is None else a.ctypes.data_as(capi.c_fp)  # noqa: E731

    def calib(wOrg=40, hOrg=30, w=32, h=24, remapX=rx, remapY=rx, G=G8, vig=vinv, mode=2, use_exposure=1):
        c = capi.UndistortCalibC(wOrg, hOrg, w, h, f(remapX), f(remapY), f(G), 0 if G is None else G.size, f(vig), mode, use_exposure)
        return L.ldso_b200_set_undistort(ctx.ctx, C.byref(c))
    assert calib(w=64) == ERR_ARG                     # rectified size other than the context's
    assert calib(remapY=None) == ERR_ARG              # one remap table missing
    assert calib(remapX=None, remapY=None) == ERR_ARG     # passthrough with wOrg x hOrg != w x h
    assert calib(G=np.zeros(100, np.float32)) == ERR_ARG  # g_entries not 256 / 65536
    assert calib(mode=3) == ERR_ARG
    assert calib(vig=None) == ERR_ARG                 # mode 2 with G but no vignette
    assert frame(raw8) == ERR_STATE                   # none of the above installed a calibration
    assert calib(G=None, vig=None) == 0               # no valid calibration: the factor path, no vignette needed
    assert calib(G=None, vig=None, mode=1) == 0
    assert calib() == 0
    raw_big8 = np.zeros((30, 40), np.uint8)
    raw_big16 = np.zeros((30, 40), np.uint16)
    assert frame(raw_big16) == ERR_ARG                # 16-bit frame with a 256-entry G
    assert frame(raw_big8, bpp=3) == ERR_ARG
    assert frame(None, bpp=1) == ERR_ARG
    assert frame(raw_big8) == 0
    assert calib(G=G16) == 0 and frame(raw_big16) == 0
    assert calib(remapX=None, remapY=None, wOrg=32, hOrg=24, G=G16, vig=np.ones(32 * 24, np.float32), use_exposure=0) == 0
    assert frame(raw16) == 0 and e.value == 1.0       # use_exposure off: exposure time 1
    assert frame(raw8) == 0
    ctx.synchronize()
    ctx.close()
    with pytest.raises(ValueError):
        c2 = capi.Context(32, 24, LEVELS)
        c2.set_undistort(40, 30, rx[:10], rx, G8, vinv)
