"""ctypes binding of the C ABI in include/ldso_b200.h (libldso_b200.so, built in-tree by ldso_b200.build).

This is plumbing only: it marshals numpy arrays into the `extern "C"` entry points. All arithmetic of the hot path
runs in the sm_90a kernels of ldso_b200/csrc; there is no CPU fallback — if the library or a CUDA device is missing
every call raises.
"""
from __future__ import annotations

import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LDSO_B200_LIB") or os.path.join(_HERE, "lib", "libldso_b200.so")   # env override: development A/B builds

MAX_FRAMES = 8
RES_IN, RES_OOB, RES_OUTLIER = 0, 1, 2

c_fp = C.POINTER(C.c_float)
c_dp = C.POINTER(C.c_double)
c_ip = C.POINTER(C.c_int32)
c_bp = C.POINTER(C.c_uint8)


class Settings(C.Structure):
    _fields_ = [(n, C.c_float) for n in (
        "huberTH", "outlierTHSumComponent", "affineOptModeA", "affineOptModeB", "idepthFixPrior", "initialTransPrior",
        "initialRotPrior", "initialAffAPrior", "initialAffBPrior", "initialCalibHessian", "frameEnergyTHN",
        "frameEnergyTHFacMedian", "frameEnergyTHConstWeight", "overallEnergyTHWeight", "coarseCutoffTH",
        "thOptIterations")] + [("solverModeDelta", C.c_double), ("margWeightFac", C.c_float)] + [(n, C.c_float) for n in (
        "maxPixSearch", "outlierTH", "trace_stepsize", "trace_GNThreshold", "trace_extraSlackOnTH", "trace_slackInterval",
        "trace_minImprovementFactor")] + [("minTraceTestRadius", C.c_int32), ("trace_GNIterations", C.c_int32)]


class WindowC(C.Structure):
    _fields_ = [("nPoints", C.c_int), ("nResiduals", C.c_int), ("pt_host", c_ip), ("pt_u", c_fp), ("pt_v", c_fp),
                ("pt_idepth", c_fp), ("pt_idepth_zero", c_fp), ("pt_has_prior", c_bp), ("pt_color", c_fp),
                ("pt_weights", c_fp), ("res_begin", c_ip), ("res_target", c_ip), ("res_state", c_bp),
                ("res_is_linearized", c_bp), ("res_toZeroF", c_fp)]


class ImmatureC(C.Structure):
    _fields_ = [("n", C.c_int), ("u", c_fp), ("v", c_fp), ("host", c_ip), ("color8", c_fp), ("weights8", c_fp), ("gradH4", c_fp),
                ("energyTH", c_fp), ("idepth_min", c_fp), ("idepth_max", c_fp), ("quality", c_fp), ("lastTraceStatus", c_ip),
                ("lastTraceUV2", c_fp), ("lastTracePixelInterval", c_fp)]


class FusedIOC(C.Structure):
    _fields_ = [("image_slot", C.c_int), ("image", c_fp), ("nFrames", C.c_int), ("frames", C.c_void_p), ("calib_value_scaled", c_dp),
                ("calib_value_zero", c_dp), ("window", C.c_void_p), ("first_iteration", C.c_int), ("n_iterations", C.c_int),
                ("lastHS", c_dp), ("lastbS", c_dp), ("lastX", c_dp), ("energy", c_dp), ("canbreak", c_ip), ("pt_idepth", c_fp),
                ("pt_step", c_fp), ("pt_HdiF", c_fp), ("res_state", c_bp), ("res_new_state", c_bp), ("res_energy", c_fp)]


class FinishOutC(C.Structure):
    _fields_ = [("iterations_run", c_ip), ("energy", c_dp), ("rmse", c_fp), ("is_lost", c_ip), ("res_state", c_bp), ("res_dropped", c_bp),
                ("pt_relBS_max", c_fp), ("pt_n_good", c_ip), ("newest_evalR", c_dp), ("newest_evalT", c_dp), ("newest_state_zero", c_dp)]


class FrameStateC(C.Structure):
    _fields_ = [("evalR", C.c_double * 9), ("evalT", C.c_double * 3), ("state_zero", C.c_double * 10),
                ("state", C.c_double * 10), ("ab_exposure", C.c_float), ("frameEnergyTH", C.c_float),
                ("frame_id", C.c_int32), ("image_slot", C.c_int32)]


FRAME_DTYPE = np.dtype([("evalR", "<f8", 9), ("evalT", "<f8", 3), ("state_zero", "<f8", 10), ("state", "<f8", 10),
                        ("ab_exposure", "<f4"), ("frameEnergyTH", "<f4"), ("frame_id", "<i4"), ("image_slot", "<i4")])
assert FRAME_DTYPE.itemsize == C.sizeof(FrameStateC)

class UndistortCalibC(C.Structure):
    _fields_ = [("wOrg", C.c_int), ("hOrg", C.c_int), ("w", C.c_int), ("h", C.c_int), ("remapX", c_fp), ("remapY", c_fp),
                ("G", c_fp), ("g_entries", C.c_int), ("vignetteMapInv", c_fp), ("photometric_mode", C.c_int), ("use_exposure", C.c_int)]


# every symbol include/ldso_b200.h declares (tests check the shared object exports all of them)
SYMBOLS = [
    "ldso_b200_default_settings", "ldso_b200_create", "ldso_b200_destroy", "ldso_b200_last_error", "ldso_b200_set_stream",
    "ldso_b200_synchronize", "ldso_b200_launch_count", "ldso_b200_kernel_times", "ldso_b200_upload_frame", "ldso_b200_make_images",
    "ldso_b200_download_frame_level", "ldso_b200_set_undistort", "ldso_b200_undistort_frame", "ldso_b200_set_window", "ldso_b200_set_frames", "ldso_b200_set_marg_prior",
    "ldso_b200_get_marg_prior", "ldso_b200_linearize_all", "ldso_b200_apply_res", "ldso_b200_backup_state",
    "ldso_b200_solve_system", "ldso_b200_get_system", "ldso_b200_do_step", "ldso_b200_marginalize_points", "ldso_b200_marginalize_frame", "ldso_b200_calc_energies", "ldso_b200_accumulate", "ldso_b200_select_activation", "ldso_b200_init_calc_res", "ldso_b200_optimize_begin",
    "ldso_b200_gn_iterations", "ldso_b200_gn_iterations_until", "ldso_b200_get_iterations_run", "ldso_b200_get_until_form",
    "ldso_b200_optimize_iteration_budget", "ldso_b200_optimize_from_host_until", "ldso_b200_optimize_from_host_until_submit",
    "ldso_b200_optimize_from_host_until_wait", "ldso_b200_optimize_finish", "ldso_b200_get_finish",
    "ldso_b200_optimize_from_host_full", "ldso_b200_optimize_from_host_full_submit", "ldso_b200_optimize_from_host_full_wait", "ldso_b200_optimize_from_host", "ldso_b200_optimize_from_host_submit", "ldso_b200_optimize_from_host_wait", "ldso_b200_reduce_buffer", "ldso_b200_set_shard", "ldso_b200_gn_phase_a",
    "ldso_b200_gn_phase_b", "ldso_b200_peer_export", "ldso_b200_peer_connect", "ldso_b200_peer_error", "ldso_b200_prefetch_results", "ldso_b200_get_energy", "ldso_b200_get_last_solution", "ldso_b200_get_points",
    "ldso_b200_get_residuals", "ldso_b200_get_frames", "ldso_b200_get_nullspace_projector", "ldso_b200_immature_init",
    "ldso_b200_trace_immature", "ldso_b200_optimize_immature", "ldso_b200_tracker_make_k",
    "ldso_b200_tracker_set_ref_level", "ldso_b200_tracker_make_coarse_depth", "ldso_b200_tracker_get_ref_level",
    "ldso_b200_tracker_set_frames", "ldso_b200_tracker_eval", "ldso_b200_tracker_track", "ldso_b200_tracker_track_batch", "ldso_b200_posegraph_optimize",
]

_lib = None


def load():
    """Load libldso_b200.so (raises if it has not been built: there is nothing to fall back to)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run `python -m ldso_b200.build` (nvcc, sm_90a). "
                               "ldso_b200 has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        L.ldso_b200_create.restype = C.c_void_p
        L.ldso_b200_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(Settings)]
        L.ldso_b200_destroy.argtypes = [C.c_void_p]
        L.ldso_b200_last_error.restype = C.c_char_p
        L.ldso_b200_last_error.argtypes = [C.c_void_p]
        L.ldso_b200_launch_count.restype = C.c_longlong
        L.ldso_b200_launch_count.argtypes = [C.c_void_p]
        L.ldso_b200_set_stream.argtypes = [C.c_void_p, C.c_void_p]
        L.ldso_b200_set_undistort.argtypes = [C.c_void_p, C.POINTER(UndistortCalibC)]
        L.ldso_b200_undistort_frame.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_float, c_fp]
        for name in SYMBOLS:
            fn = getattr(L, name)
            if name not in ("ldso_b200_create", "ldso_b200_destroy", "ldso_b200_last_error", "ldso_b200_launch_count",
                            "ldso_b200_default_settings", "ldso_b200_set_stream"):
                fn.restype = C.c_int
        _lib = L
    return _lib


UNTIL_FORMS = {0: "host", 1: "graph+pdl", 2: "graph"}     # LDSO_B200_UNTIL_*


def optimize_iteration_budget(nF, max_its=6) -> int:
    """FullSystem::optimize's iteration budget for a window of nF keyframes (0 below 2, 15 below 4, else max_its =
    setting_maxOptIterations)."""
    r = load().ldso_b200_optimize_iteration_budget(int(nF), int(max_its))
    if r < 0:
        raise Error(f"ldso_b200_optimize_iteration_budget({nF}, {max_its}) failed: {r}")
    return r


def default_settings() -> Settings:
    s = Settings()
    load().ldso_b200_default_settings(C.byref(s))
    return s


def _f(a):
    return None if a is None else a.ctypes.data_as(c_fp)


def _d(a):
    return None if a is None else a.ctypes.data_as(c_dp)


def _i(a):
    return None if a is None else a.ctypes.data_as(c_ip)


def _b(a):
    return None if a is None else a.ctypes.data_as(c_bp)


class Error(RuntimeError):
    pass


class Context:
    """One ldso_b200 context = one GPU's device-resident keyframe window + coarse tracker."""

    def __init__(self, w, h, levels, device=0, settings: Settings | None = None):
        self.L = load()
        self.w, self.h, self.levels = int(w), int(h), int(levels)
        self.ctx = self.L.ldso_b200_create(int(device), self.w, self.h, self.levels, C.byref(settings) if settings is not None else None)
        if not self.ctx:
            raise Error("ldso_b200_create failed: no usable CUDA device (ldso_b200 has no CPU fallback)")
        self.ctx = C.c_void_p(self.ctx)
        self.nF = 0
        self.nP = 0
        self.nR = 0

    def close(self):
        if getattr(self, "ctx", None):
            self.L.ldso_b200_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc):
        if rc != 0:
            raise Error(f"ldso_b200 error {rc}: {self.L.ldso_b200_last_error(self.ctx).decode()}")

    @property
    def n(self):
        return 8 * self.nF + 4

    # ---- plumbing
    def set_stream(self, cuda_stream_ptr: int):
        self._chk(self.L.ldso_b200_set_stream(self.ctx, C.c_void_p(cuda_stream_ptr)))

    def synchronize(self):
        self._chk(self.L.ldso_b200_synchronize(self.ctx))

    def kernel_times(self, enable):
        """enable=True: start per-kernel event timing; enable=False: stop, return avg us of (k1, k2a, k2b, k3, k2r)."""
        out = (C.c_double * 5)()
        self._chk(self.L.ldso_b200_kernel_times(self.ctx, int(bool(enable)), out))
        return dict(zip(("k1", "k2a", "k2b", "k3", "k2r"), list(out)))

    def launch_count(self) -> int:
        return int(self.L.ldso_b200_launch_count(self.ctx))

    # ---- images
    def upload_frame(self, slot, pyramid):
        lv = [np.ascontiguousarray(p, np.float32) for p in pyramid]
        arr = (c_fp * len(lv))(*[_f(p) for p in lv])
        self._chk(self.L.ldso_b200_upload_frame(self.ctx, int(slot), arr, len(lv)))

    def make_images(self, slot, color):
        color = np.ascontiguousarray(color, np.float32)
        assert color.shape == (self.h, self.w)
        self._chk(self.L.ldso_b200_make_images(self.ctx, int(slot), _f(color)))

    def download_frame_level(self, slot, lvl):
        out = np.zeros((self.h >> lvl, self.w >> lvl, 3), np.float32)
        self._chk(self.L.ldso_b200_download_frame_level(self.ctx, int(slot), int(lvl), _f(out)))
        return out

    # ---- raw camera frames (undistortion on the device)
    def set_undistort(self, wOrg, hOrg, remapX=None, remapY=None, G=None, vignetteMapInv=None, photometric_mode=2, use_exposure=True):
        """ldso_b200_set_undistort with LDSO's Undistort tables: remapX / remapY (h x w, None = passthrough), G (256 or 65536
        entries, None = no valid photometric calibration), vignetteMapInv (hOrg x wOrg), setting_photometricCalibration and
        setting_useExposure. The arrays are copied to the device before this returns."""
        arrs = {}
        for name, a, n in (("remapX", remapX, self.w * self.h), ("remapY", remapY, self.w * self.h), ("G", G, None),
                           ("vignetteMapInv", vignetteMapInv, int(wOrg) * int(hOrg))):
            if a is None:
                continue
            a = np.ascontiguousarray(a, np.float32).reshape(-1)
            if n is not None and a.size != n:
                raise ValueError(f"{name} has {a.size} entries, expected {n}")
            arrs[name] = a
        c = UndistortCalibC(int(wOrg), int(hOrg), self.w, self.h, _f(arrs.get("remapX")), _f(arrs.get("remapY")), _f(arrs.get("G")),
                            int(arrs["G"].size) if "G" in arrs else 0, _f(arrs.get("vignetteMapInv")), int(photometric_mode),
                            int(bool(use_exposure)))
        self._chk(self.L.ldso_b200_set_undistort(self.ctx, C.byref(c)))
        self._ud_size = (int(hOrg), int(wOrg))

    def undistort_frame(self, slot, raw, exposure, factor=1.0) -> float:
        """ldso_b200_undistort_frame: one raw uint8 / uint16 frame (hOrg x wOrg) -> rectified irradiance -> slot's pyramid.
        Returns the frame's exposure time as processFrame sets it (exposure, or 1 without use_exposure)."""
        raw = np.ascontiguousarray(raw)
        if raw.dtype not in (np.uint8, np.uint16):
            raise ValueError("raw must be uint8 or uint16")
        if getattr(self, "_ud_size", None) is not None and raw.size != self._ud_size[0] * self._ud_size[1]:
            raise ValueError(f"raw has {raw.size} pixels, expected {self._ud_size[0]} x {self._ud_size[1]}")
        e = C.c_float(0)
        self._keep_raw = raw      # valid until the next synchronising call
        self._chk(self.L.ldso_b200_undistort_frame(self.ctx, int(slot), raw.ctypes.data_as(C.c_void_p), raw.itemsize, float(exposure),
                                                   float(factor), C.byref(e)))
        return float(e.value)

    # ---- window
    def set_frames(self, Rcw, tcw, state_zero, state, ab_exposure, frame_id, slots, K_scaled, K_zero=None,
                   frame_energy_th=None):
        nF = len(Rcw)
        arr = np.zeros(nF, FRAME_DTYPE)          # same layout as ldso_b200_frame_state
        arr["evalR"] = np.asarray(Rcw, np.float64).reshape(nF, 9)
        arr["evalT"] = np.asarray(tcw, np.float64).reshape(nF, 3)
        arr["state_zero"] = np.asarray(state_zero, np.float64).reshape(nF, 10)
        arr["state"] = np.asarray(state, np.float64).reshape(nF, 10)
        arr["ab_exposure"] = np.asarray(ab_exposure, np.float32)
        arr["frameEnergyTH"] = 8 * 8 * 8 if frame_energy_th is None else np.asarray(frame_energy_th, np.float32)
        arr["frame_id"] = np.asarray(frame_id, np.int32)
        arr["image_slot"] = np.asarray(slots, np.int32)
        Ks = np.ascontiguousarray(K_scaled, np.float64)
        if K_zero is None:   # CalibHessian ctor: value_zero = value = SCALE_*_INVERSE * value_scaled
            K_zero = Ks * np.float64(np.float32(1.0) / np.float32(50.0))
        Kz = np.ascontiguousarray(K_zero, np.float64)
        self._chk(self.L.ldso_b200_set_frames(self.ctx, nF, arr.ctypes.data_as(C.POINTER(FrameStateC)), _d(Ks), _d(Kz)))
        self.nF = nF

    def set_window(self, pt_host, pt_u, pt_v, pt_idepth, pt_idepth_zero, pt_has_prior, pt_color, pt_weights, res_begin,
                   res_target, res_state=None, res_is_linearized=None, res_toZeroF=None):
        keep = dict(
            pt_host=np.ascontiguousarray(pt_host, np.int32), pt_u=np.ascontiguousarray(pt_u, np.float32),
            pt_v=np.ascontiguousarray(pt_v, np.float32), pt_idepth=np.ascontiguousarray(pt_idepth, np.float32),
            pt_idepth_zero=np.ascontiguousarray(pt_idepth_zero, np.float32),
            pt_has_prior=np.ascontiguousarray(pt_has_prior, np.uint8), pt_color=np.ascontiguousarray(pt_color, np.float32),
            pt_weights=np.ascontiguousarray(pt_weights, np.float32), res_begin=np.ascontiguousarray(res_begin, np.int32),
            res_target=np.ascontiguousarray(res_target, np.int32))
        w = WindowC()
        w.nPoints = int(keep["pt_host"].shape[0])
        w.nResiduals = int(keep["res_target"].shape[0])
        w.pt_host = _i(keep["pt_host"]); w.pt_u = _f(keep["pt_u"]); w.pt_v = _f(keep["pt_v"])
        w.pt_idepth = _f(keep["pt_idepth"]); w.pt_idepth_zero = _f(keep["pt_idepth_zero"])
        w.pt_has_prior = _b(keep["pt_has_prior"]); w.pt_color = _f(keep["pt_color"]); w.pt_weights = _f(keep["pt_weights"])
        w.res_begin = _i(keep["res_begin"]); w.res_target = _i(keep["res_target"])
        if res_state is not None:
            keep["res_state"] = np.ascontiguousarray(res_state, np.uint8); w.res_state = _b(keep["res_state"])
        if res_is_linearized is not None:
            keep["lin"] = np.ascontiguousarray(res_is_linearized, np.uint8); w.res_is_linearized = _b(keep["lin"])
        if res_toZeroF is not None:
            keep["rtz"] = np.ascontiguousarray(res_toZeroF, np.float32); w.res_toZeroF = _f(keep["rtz"])
        self._chk(self.L.ldso_b200_set_window(self.ctx, C.byref(w)))
        self.nP, self.nR = w.nPoints, w.nResiduals

    def load_synth_window(self, win, upload_images=True):
        """Convenience: push a ldso_b200.synth.Window (images, frames, points, residuals)."""
        if upload_images:
            for i in range(win.nF):
                self.upload_frame(i, win.pyramids[i])
        self.set_frames(win.Rcw, win.tcw, win.state_zero, win.state, win.ab_exposure, win.frame_id, list(range(win.nF)), win.K)
        self.set_window(win.pt_host, win.pt_u, win.pt_v, win.pt_idepth, win.pt_idepth_zero, win.pt_has_prior,
                        win.pt_color, win.pt_weights, win.res_begin, win.res_target)

    def set_marg_prior(self, HM=None, bM=None):
        HMc = None if HM is None else np.asfortranarray(HM, np.float64)
        bMc = None if bM is None else np.ascontiguousarray(bM, np.float64)
        self._chk(self.L.ldso_b200_set_marg_prior(self.ctx, _d(HMc), _d(bMc)))

    # ---- piecewise
    def linearize_all(self, fix=False, flags=1):
        e = C.c_double()
        self._chk(self.L.ldso_b200_linearize_all(self.ctx, int(fix), int(flags), C.byref(e)))
        return e.value

    def apply_res(self):
        self._chk(self.L.ldso_b200_apply_res(self.ctx))

    def backup_state(self):
        self._chk(self.L.ldso_b200_backup_state(self.ctx))

    def solve_system(self, iteration):
        n = self.n
        HS = np.zeros((n, n), np.float64, order="F")
        bS = np.zeros(n)
        X = np.zeros(n)
        self._chk(self.L.ldso_b200_solve_system(self.ctx, int(iteration), _d(HS), _d(bS), _d(X)))
        return HS, bS, X

    def do_step(self):
        cb = C.c_int()
        self._chk(self.L.ldso_b200_do_step(self.ctx, C.byref(cb)))
        return bool(cb.value)

    def marginalize_points(self, idx, prior_fac=600.0 * 600.0):
        idx = np.ascontiguousarray(idx, np.int32)
        r = C.c_int()
        self._chk(self.L.ldso_b200_marginalize_points(self.ctx, int(idx.shape[0]), _i(idx), C.c_float(prior_fac), C.byref(r)))
        return r.value

    def marginalize_frame(self, idx):
        """EnergyFunctional::marginalizeFrame's prior algebra on the device; returns the shrunken (HM, bM)."""
        nd = C.c_int()
        self._chk(self.L.ldso_b200_marginalize_frame(self.ctx, int(idx), C.byref(nd)))
        return self.marg_prior(nd.value)

    def accumulate(self, mode, idx=None, shift_prior=True):
        """addPoint<mode> + stitchDouble(usePrior=False) and the Schur addPoint + stitchDouble over the points idx (None = all)."""
        n = self.n
        out = dict(HA=np.zeros((n, n), np.float64, order="F"), bA=np.zeros(n), Hsc=np.zeros((n, n), np.float64, order="F"), bsc=np.zeros(n))
        r = C.c_int()
        ip = None if idx is None else np.ascontiguousarray(idx, np.int32)
        self._chk(self.L.ldso_b200_accumulate(self.ctx, int(mode), 0 if ip is None else len(ip), None if ip is None else ip.ctypes.data_as(C.POINTER(C.c_int32)),
                                              int(bool(shift_prior)), _d(out["HA"]), _d(out["bA"]), _d(out["Hsc"]), _d(out["bsc"]), C.byref(r)))
        out["nres"] = r.value
        return out

    def calc_energies(self):
        """(calcLEnergyF_MT, calcMEnergyF) at the current state."""
        el, em = C.c_double(), C.c_double()
        self._chk(self.L.ldso_b200_calc_energies(self.ctx, C.byref(el), C.byref(em)))
        return el.value, em.value

    def marg_prior(self, n=None):
        n = self.n if n is None else n
        HM = np.zeros((n, n), np.float64, order="F")
        bM = np.zeros(n)
        self._chk(self.L.ldso_b200_get_marg_prior(self.ctx, _d(HM), _d(bM)))
        return HM, bM

    # ---- fused loop
    def optimize_begin(self, want_energy=True):
        if not want_energy:     # fully asynchronous
            self._chk(self.L.ldso_b200_optimize_begin(self.ctx, None))
            return None
        e = C.c_double()
        self._chk(self.L.ldso_b200_optimize_begin(self.ctx, C.byref(e)))
        return e.value

    def gn_iterations(self, first, n):
        self._chk(self.L.ldso_b200_gn_iterations(self.ctx, int(first), int(n)))

    def gn_iterations_until(self, first, max_its, min_its=1):
        """At most max_its bodies from iteration `first`, stopping after the body whose canbreak fired at iteration >= min_its
        (FullSystem::optimize's exit). Asynchronous; iterations_run() gives the count."""
        self._chk(self.L.ldso_b200_gn_iterations_until(self.ctx, int(first), int(max_its), int(min_its)))

    def iterations_run(self) -> int:
        n = C.c_int()
        self._chk(self.L.ldso_b200_get_iterations_run(self.ctx, C.byref(n)))
        return n.value

    def until_form(self) -> str:
        """'graph+pdl', 'graph' (conditional WHILE node) or 'host' (host-driven): the form of the last gn_iterations_until."""
        f = C.c_int()
        self._chk(self.L.ldso_b200_get_until_form(self.ctx, C.byref(f)))
        return UNTIL_FORMS[f.value]

    def optimize_finish(self):
        """The end of FullSystem::optimize (FullSystem.cc:833-863) on the device: the newest frame's new evaluation point, the
        adjoints and pair records, linearizeAll(true) with its per-point bookkeeping, the RMSE. Asynchronous; finish_results()
        reads it back. Afterwards the window entry points need set_window, the solve entry points also set_frames."""
        self._chk(self.L.ldso_b200_optimize_finish(self.ctx))

    def finish_results(self):
        """What ldso_b200_get_finish returns, as a dict of arrays."""
        out = _finish_arrays(self.nP, self.nR)
        self._chk(self.L.ldso_b200_get_finish(self.ctx, *_finish_ptrs(out)))
        return _finish_scalars(out)

    def reduce_buffer(self):
        p = C.c_void_p()
        n = C.c_size_t()
        self._chk(self.L.ldso_b200_reduce_buffer(self.ctx, C.byref(p), C.byref(n)))
        return p.value, n.value

    def set_shard(self, offset, total):
        self._chk(self.L.ldso_b200_set_shard(self.ctx, int(offset), int(total)))

    def peer_export(self) -> bytes:
        h = (C.c_ubyte * 64)()
        self._chk(self.L.ldso_b200_peer_export(self.ctx, h))
        return bytes(h)

    def peer_connect(self, rank, world, handles):
        """handles: list of `world` 64-byte IPC handles (peer_export of every rank, in rank order)."""
        blob = b"".join(handles)
        assert len(blob) == 64 * world
        buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        self._chk(self.L.ldso_b200_peer_connect(self.ctx, int(rank), int(world), buf))

    def peer_error(self) -> int:
        e = C.c_int()
        self._chk(self.L.ldso_b200_peer_error(self.ctx, C.byref(e)))
        return e.value

    def gn_phase_a(self, iteration):
        self._chk(self.L.ldso_b200_gn_phase_a(self.ctx, int(iteration)))

    def gn_phase_b(self):
        self._chk(self.L.ldso_b200_gn_phase_b(self.ctx))

    # ---- read-back
    def energy(self):
        e = C.c_double()
        cb = C.c_int()
        self._chk(self.L.ldso_b200_get_energy(self.ctx, C.byref(e), C.byref(cb)))
        return e.value, bool(cb.value)

    def last_solution(self):
        n = self.n
        HS = np.zeros((n, n), np.float64, order="F")
        bS = np.zeros(n)
        X = np.zeros(n)
        self._chk(self.L.ldso_b200_get_last_solution(self.ctx, _d(HS), _d(bS), _d(X)))
        return dict(lastHS=HS, lastbS=bS, lastX=X)

    def system(self):
        n = self.n
        out = dict(HA=np.zeros((n, n), np.float64, order="F"), bA=np.zeros(n), Hsc=np.zeros((n, n), np.float64, order="F"),
                   bsc=np.zeros(n))
        r = C.c_int()
        self._chk(self.L.ldso_b200_get_system(self.ctx, _d(out["HA"]), _d(out["bA"]), _d(out["Hsc"]), _d(out["bsc"]), C.byref(r)))
        out["resInA"] = r.value
        return out

    def points(self):
        nP = self.nP
        keys = ("idepth", "idepth_zero", "step", "HdiF", "bdSumF", "Hdd_accAF", "bd_accAF")
        out = {k: np.zeros(nP, np.float32) for k in keys}
        out["Hcd_accAF"] = np.zeros((nP, 4), np.float32)
        self._chk(self.L.ldso_b200_get_points(self.ctx, *[_f(out[k]) for k in keys], _f(out["Hcd_accAF"])))
        return out

    def residuals(self, with_J=True):
        nR = self.nR
        out = dict(state_state=np.zeros(nR, np.uint8), state_NewState=np.zeros(nR, np.uint8),
                   state_energy=np.zeros(nR, np.float32), state_NewEnergy=np.zeros(nR, np.float32),
                   state_NewEnergyWithOutlier=np.zeros(nR, np.float32), isActive=np.zeros(nR, np.uint8),
                   JpJdF=np.zeros((nR, 8), np.float32))
        if with_J:
            out.update(J=np.zeros((nR, 74), np.float32), projectedTo=np.zeros((nR, 8, 2), np.float32),
                       centerProjectedTo=np.zeros((nR, 3), np.float32))
        self._chk(self.L.ldso_b200_get_residuals(
            self.ctx, _b(out["state_state"]), _b(out["state_NewState"]), _f(out["state_energy"]), _f(out["state_NewEnergy"]),
            _f(out["state_NewEnergyWithOutlier"]), _b(out["isActive"]), _f(out["JpJdF"]), _f(out.get("J")),
            _f(out.get("projectedTo")), _f(out.get("centerProjectedTo"))))
        return out

    def residuals_light(self):
        """States, activity and centerProjectedTo only (no Jacobians, no per-pixel projections): what setCoarseTrackingRef reads."""
        nR = self.nR
        out = dict(state_state=np.zeros(nR, np.uint8), isActive=np.zeros(nR, np.uint8), centerProjectedTo=np.zeros((nR, 3), np.float32))
        self._chk(self.L.ldso_b200_get_residuals(self.ctx, _b(out["state_state"]), None, None, None, None, _b(out["isActive"]), None, None, None,
                                                 _f(out["centerProjectedTo"])))
        return out

    def prefetch_results(self):
        self._chk(self.L.ldso_b200_prefetch_results(self.ctx))

    def frames(self):
        nF = self.nF
        out = dict(state=np.zeros((nF, 10)), step=np.zeros((nF, 10)), frameEnergyTH=np.zeros(nF, np.float32),
                   precalc=np.zeros((nF * nF, 40), np.float32), adHost=np.zeros((nF * nF, 8, 8)),
                   adTarget=np.zeros((nF * nF, 8, 8)), adHTdeltaF=np.zeros((nF * nF, 8), np.float32), calib_value=np.zeros(4))
        self._chk(self.L.ldso_b200_get_frames(self.ctx, _d(out["state"]), _d(out["step"]), _f(out["frameEnergyTH"]),
                                              _f(out["precalc"]), _d(out["adHost"]), _d(out["adTarget"]), _f(out["adHTdeltaF"]),
                                              _d(out["calib_value"])))
        return out

    def nullspace_projector(self):
        n = self.n
        P = np.zeros((n, n), np.float64, order="F")
        self._chk(self.L.ldso_b200_get_nullspace_projector(self.ctx, _d(P)))
        return P

    # ---- tracker
    # ---- immature points
    def immature_init(self, host_slot, u, v):
        """ImmaturePoint's constructor for candidates (u, v) of the keyframe in image slot host_slot."""
        u = np.ascontiguousarray(u, np.float32); v = np.ascontiguousarray(v, np.float32)
        n = u.shape[0]
        out = dict(color=np.zeros((n, 8), np.float32), weights=np.zeros((n, 8), np.float32), gradH=np.zeros((n, 4), np.float32),
                   energyTH=np.zeros(n, np.float32))
        self._chk(self.L.ldso_b200_immature_init(self.ctx, int(host_slot), n, _f(u), _f(v), _f(out["color"]), _f(out["weights"]),
                                                 _f(out["gradH"]), _f(out["energyTH"])))
        return out

    def trace_immature(self, new_slot, pts: dict, KRKi, Kt, aff):
        """One traceNewCoarse pass. pts: dict of arrays u, v, host, color, weights, gradH, energyTH, idepth_min, idepth_max, quality,
        status, uv, interval (the last six are updated in place). KRKi (nH,3,3), Kt (nH,3), aff (nH,2) per host."""
        f32 = lambda k: np.ascontiguousarray(pts[k], np.float32)
        for k in ("idepth_min", "idepth_max", "quality", "uv", "interval"):
            assert pts[k].dtype == np.float32 and pts[k].flags.c_contiguous
        assert pts["status"].dtype == np.int32 and pts["status"].flags.c_contiguous
        keep = dict(u=f32("u"), v=f32("v"), host=np.ascontiguousarray(pts["host"], np.int32), color=f32("color"), weights=f32("weights"),
                    gradH=f32("gradH"), energyTH=f32("energyTH"), K=np.ascontiguousarray(KRKi, np.float32),
                    t=np.ascontiguousarray(Kt, np.float32), a=np.ascontiguousarray(aff, np.float32))
        p = ImmatureC()
        p.n = int(keep["u"].shape[0])
        p.u = _f(keep["u"]); p.v = _f(keep["v"]); p.host = _i(keep["host"]); p.color8 = _f(keep["color"]); p.weights8 = _f(keep["weights"])
        p.gradH4 = _f(keep["gradH"]); p.energyTH = _f(keep["energyTH"]); p.idepth_min = _f(pts["idepth_min"]); p.idepth_max = _f(pts["idepth_max"])
        p.quality = _f(pts["quality"]); p.lastTraceStatus = _i(pts["status"]); p.lastTraceUV2 = _f(pts["uv"])
        p.lastTracePixelInterval = _f(pts["interval"])
        self._chk(self.L.ldso_b200_trace_immature(self.ctx, int(new_slot), C.byref(p), int(keep["K"].shape[0]), _f(keep["K"]), _f(keep["t"]),
                                                  _f(keep["a"])))

    def optimize_immature(self, u, v, host, idepth_min, idepth_max, color, weights, energyTH, min_obs=1):
        """FullSystem::optimizeImmaturePoint for every candidate against the device-resident frames: (ok, idepth, res_state[n, nF])."""
        f32 = lambda a: np.ascontiguousarray(a, np.float32)
        u, v, imin, imax, col, wts, eth = map(f32, (u, v, idepth_min, idepth_max, color, weights, energyTH))
        host = np.ascontiguousarray(host, np.int32)
        n = u.shape[0]
        ok = np.zeros(n, np.int32); idepth = np.zeros(n, np.float32); states = np.zeros((n, max(self.nF, 1)), np.uint8)
        self._chk(self.L.ldso_b200_optimize_immature(self.ctx, n, _f(u), _f(v), _i(host), _f(imin), _f(imax), _f(col), _f(wts), _f(eth), int(min_obs),
                                                     _i(ok), _f(idepth), _b(states)))
        return ok, idepth, states

    def select_activation(self, newest, current_min_act_dist, u, v, host, idepth_min, idepth_max, status, interval, quality, my_type,
                          frame_flagged=None, min_trace_quality=3.0, want_map=False):
        """FullSystem::activatePointsMT's selection loop over the device-resident window: action per candidate (0 stays immature,
        1 activate, 2 delete) and, if asked, the level-1 distance map as the loop leaves it."""
        f32 = lambda a: np.ascontiguousarray(a, np.float32)
        u, v, imin, imax, itv, q, mt = map(f32, (u, v, idepth_min, idepth_max, interval, quality, my_type))
        host = np.ascontiguousarray(host, np.int32); status = np.ascontiguousarray(status, np.int32)
        n = u.shape[0]
        flagged = np.zeros(max(self.nF, 1), np.uint8) if frame_flagged is None else np.ascontiguousarray(frame_flagged, np.uint8)
        action = np.zeros(n, np.uint8)
        dmap = np.zeros((self.h >> 1, self.w >> 1), np.float32) if want_map else None
        self._chk(self.L.ldso_b200_select_activation(self.ctx, int(newest), C.c_float(current_min_act_dist), C.c_float(min_trace_quality), n, _f(u), _f(v),
                                                     _i(host), _f(imin), _f(imax), _i(status), _f(itv), _f(q), _f(mt), _b(flagged), _b(action),
                                                     _f(dmap) if want_map else None))
        return (action, dmap) if want_map else action

    def init_calc_res(self, first_slot, new_slot, lvl, R, t, tlog3, aff_a, aff_b, K4, u, v, idepth_new, iR, isGood, energy2, outlierTH,
                      alphaK=2.5 * 2.5, alphaW=150.0 * 150.0, couplingWeight=1.0):
        """EXPERIMENTAL: CoarseInitializer::calcResAndGS for the points of one pyramid level (see include/ldso_b200.h)."""
        f32 = lambda a: np.ascontiguousarray(a, np.float32)
        u, v, idn, iR, e2, oth = map(f32, (u, v, idepth_new, iR, energy2, outlierTH))
        good = np.ascontiguousarray(isGood, np.uint8)
        n = u.shape[0]
        R = np.ascontiguousarray(R, np.float64); t = np.ascontiguousarray(t, np.float64); tl = np.ascontiguousarray(tlog3, np.float64)
        out = dict(isGood_new=np.zeros(n, np.uint8), energy_new=np.zeros((n, 2), np.float32), maxstep=np.zeros(n, np.float32),
                   lastHessian_new=np.zeros(n, np.float32), Jb=np.zeros((n, 10), np.float32), H=np.zeros((8, 8), np.float32), b=np.zeros(8, np.float32),
                   Hsc=np.zeros((8, 8), np.float32), bsc=np.zeros(8, np.float32), res=np.zeros(3, np.float32))
        self._chk(self.L.ldso_b200_init_calc_res(self.ctx, int(first_slot), int(new_slot), int(lvl), _d(R), _d(t), _d(tl), C.c_float(aff_a), C.c_float(aff_b),
                                                 C.c_float(K4[0]), C.c_float(K4[1]), C.c_float(K4[2]), C.c_float(K4[3]), n, _f(u), _f(v), _f(idn), _f(iR),
                                                 _b(good), _f(e2), _f(oth), C.c_float(alphaK), C.c_float(alphaW), C.c_float(couplingWeight),
                                                 _b(out["isGood_new"]), _f(out["energy_new"]), _f(out["maxstep"]), _f(out["lastHessian_new"]), _f(out["Jb"]),
                                                 _f(out["H"]), _f(out["b"]), _f(out["Hsc"]), _f(out["bsc"]), _f(out["res"])))
        return out

    def tracker_make_k(self, fx, fy, cx, cy):
        self._chk(self.L.ldso_b200_tracker_make_k(self.ctx, C.c_float(fx), C.c_float(fy), C.c_float(cx), C.c_float(cy)))

    def tracker_set_ref_level(self, lvl, u, v, idepth, color):
        a = [np.ascontiguousarray(x, np.float32) for x in (u, v, idepth, color)]
        self._chk(self.L.ldso_b200_tracker_set_ref_level(self.ctx, int(lvl), int(a[0].shape[0]), *[_f(x) for x in a]))

    def tracker_make_coarse_depth(self, ref_slot, cpt, HdiF):
        cpt = np.ascontiguousarray(cpt, np.float32)
        hd = np.ascontiguousarray(HdiF, np.float32)
        self._chk(self.L.ldso_b200_tracker_make_coarse_depth(self.ctx, int(ref_slot), int(hd.shape[0]), _f(cpt), _f(hd)))

    def tracker_get_ref_level(self, lvl):
        n = C.c_int()
        self._chk(self.L.ldso_b200_tracker_get_ref_level(self.ctx, int(lvl), C.byref(n), None, None, None, None))
        a = [np.zeros(n.value, np.float32) for _ in range(4)]
        self._chk(self.L.ldso_b200_tracker_get_ref_level(self.ctx, int(lvl), C.byref(n), *[_f(x) for x in a]))
        return a

    def tracker_set_frames(self, ref_a, ref_b, ref_exposure, new_slot, new_exposure):
        self._chk(self.L.ldso_b200_tracker_set_frames(self.ctx, C.c_float(ref_a), C.c_float(ref_b), C.c_float(ref_exposure),
                                                      int(new_slot), C.c_float(new_exposure)))

    def tracker_eval(self, lvl, R, t, aff_a, aff_b, cutoff, with_H=True):
        R = np.ascontiguousarray(R, np.float64)
        t = np.ascontiguousarray(t, np.float64)
        res = np.zeros(6)
        H = np.zeros((8, 8))
        b = np.zeros(8)
        self._chk(self.L.ldso_b200_tracker_eval(self.ctx, int(lvl), _d(R), _d(t), C.c_float(aff_a), C.c_float(aff_b),
                                                C.c_float(cutoff), _d(res), _d(H) if with_H else None, _d(b) if with_H else None))
        return res, H, b

    def tracker_track(self, R, t, aff_a, aff_b, coarsest, min_res=None):
        R = np.array(R, np.float64, order="C")
        t = np.array(t, np.float64)
        a = C.c_float(aff_a)
        b = C.c_float(aff_b)
        mr = np.full(5, np.nan) if min_res is None else np.ascontiguousarray(min_res, np.float64)
        lr = np.zeros(5)
        lf = np.zeros(3)
        ok = C.c_int()
        self._chk(self.L.ldso_b200_tracker_track(self.ctx, _d(R), _d(t), C.byref(a), C.byref(b), int(coarsest), _d(mr), _d(lr),
                                                 _d(lf), C.byref(ok)))
        return bool(ok.value), R, t, a.value, b.value, lr, lf


    def _tracker_track_batch(self, R, t, aff, coarsest):
        """n hypotheses side by side: R (n,3,3), t (n,3), aff (n,2) -> dict of per-hypothesis results."""
        R = np.ascontiguousarray(R, np.float64); t = np.ascontiguousarray(t, np.float64); aff = np.ascontiguousarray(aff, np.float32)
        n = R.shape[0]
        out = dict(R=np.zeros((n, 3, 3)), t=np.zeros((n, 3)), aff=np.zeros((n, 2), np.float32), lastResiduals=np.zeros((n, 5)),
                   lastFlowIndicators=np.zeros((n, 3)), ok=np.zeros(n, np.int32))
        self._chk(self.L.ldso_b200_tracker_track_batch(self.ctx, n, _d(R), _d(t), _f(aff), int(coarsest), _d(out["R"]), _d(out["t"]), _f(out["aff"]),
                                                       _d(out["lastResiduals"]), _d(out["lastFlowIndicators"]), _i(out["ok"])))
        return out


    def _posegraph_optimize(self, q, t, ei, ej, mq, mt, info, fixed, iterations=25, pcg_tol=1e-10, pcg_max_iter=2000):
        """Sim(3) pose graph Gauss-Newton on the device; returns (q, t, chi2[iterations + 1], CG iterations spent)."""
        q = np.ascontiguousarray(q, np.float64).copy(); t = np.ascontiguousarray(t, np.float64).copy()
        ei = np.ascontiguousarray(ei, np.int32); ej = np.ascontiguousarray(ej, np.int32)
        mq = np.ascontiguousarray(mq, np.float64); mt = np.ascontiguousarray(mt, np.float64); info = np.ascontiguousarray(info, np.float64)
        chi = np.zeros(iterations + 1); ncg = C.c_int()
        self._chk(self.L.ldso_b200_posegraph_optimize(self.ctx, len(q), _d(q), _d(t), len(ei), _i(ei), _i(ej), _d(mq), _d(mt), _d(info), int(fixed),
                                                      int(iterations), C.c_double(pcg_tol), int(pcg_max_iter), _d(chi), C.byref(ncg)))
        return q, t, chi, ncg.value


Context.tracker_track_batch = Context._tracker_track_batch
Context.posegraph_optimize = Context._posegraph_optimize


def _finish_arrays(nP, nR):
    return dict(energy=np.zeros(1), rmse=np.zeros(1, np.float32), is_lost=np.zeros(1, np.int32), res_state=np.zeros(nR, np.uint8),
                res_dropped=np.zeros(nR, np.uint8), pt_relBS_max=np.zeros(nP, np.float32), pt_n_good=np.zeros(nP, np.int32),
                newest_evalR=np.zeros((3, 3)), newest_evalT=np.zeros(3), newest_state_zero=np.zeros(10))


def _finish_ptrs(o):
    return (_d(o["energy"]), _f(o["rmse"]), _i(o["is_lost"]), _b(o["res_state"]), _b(o["res_dropped"]), _f(o["pt_relBS_max"]),
            _i(o["pt_n_good"]), _d(o["newest_evalR"]), _d(o["newest_evalT"]), _d(o["newest_state_zero"]))


def _finish_scalars(o):
    o = dict(o)
    o["energy"], o["rmse"], o["is_lost"] = float(o["energy"][0]), float(o["rmse"][0]), bool(o["is_lost"][0])
    return o


class StepIO:
    """Persistent host buffers + pre-built C argument blocks for one window, the way a C++ caller holds them: every
    call below is the bare C-ABI call on memory allocated once (no per-call numpy allocation or dtype conversion).
    Used by bench.py's end-to-end leg."""

    def __init__(self, ctx: Context, win, pinned_alloc=None):
        self.ctx, self.L, self.h = ctx, ctx.L, ctx.ctx
        nF, nP, nR = win.nF, win.nP, win.nR
        self.nF, self.nP, self.nR = nF, nP, nR
        alloc = pinned_alloc or (lambda a: a)
        k = self.keep = {}
        # ---- inputs
        k["color"] = alloc(np.ascontiguousarray(win.pyramids[nF - 1][0][:, :, 0], np.float32))
        fr = np.zeros(nF, FRAME_DTYPE)
        fr["evalR"] = np.asarray(win.Rcw, np.float64).reshape(nF, 9); fr["evalT"] = np.asarray(win.tcw, np.float64).reshape(nF, 3)
        fr["state_zero"] = np.asarray(win.state_zero, np.float64).reshape(nF, 10); fr["state"] = np.asarray(win.state, np.float64).reshape(nF, 10)
        fr["ab_exposure"] = np.asarray(win.ab_exposure, np.float32); fr["frameEnergyTH"] = 8 * 8 * 8
        fr["frame_id"] = np.asarray(win.frame_id, np.int32); fr["image_slot"] = np.arange(nF, dtype=np.int32)
        k["frames"] = fr
        k["Ks"] = np.ascontiguousarray(win.K, np.float64)
        k["Kz"] = np.ascontiguousarray(k["Ks"] * np.float64(np.float32(1.0) / np.float32(50.0)))
        for name, dt in (("pt_host", np.int32), ("pt_u", np.float32), ("pt_v", np.float32), ("pt_idepth", np.float32),
                         ("pt_idepth_zero", np.float32), ("pt_has_prior", np.uint8), ("pt_color", np.float32),
                         ("pt_weights", np.float32), ("res_begin", np.int32), ("res_target", np.int32)):
            k[name] = alloc(np.ascontiguousarray(getattr(win, name), dt))
        w = self.w = WindowC()
        w.nPoints, w.nResiduals = nP, nR
        w.pt_host = _i(k["pt_host"]); w.pt_u = _f(k["pt_u"]); w.pt_v = _f(k["pt_v"]); w.pt_idepth = _f(k["pt_idepth"])
        w.pt_idepth_zero = _f(k["pt_idepth_zero"]); w.pt_has_prior = _b(k["pt_has_prior"]); w.pt_color = _f(k["pt_color"])
        w.pt_weights = _f(k["pt_weights"]); w.res_begin = _i(k["res_begin"]); w.res_target = _i(k["res_target"])
        self._wref = C.byref(w)
        self._color, self._frames = _f(k["color"]), fr.ctypes.data_as(C.POINTER(FrameStateC))
        self._Ks, self._Kz = _d(k["Ks"]), _d(k["Kz"])
        # ---- outputs
        n = 8 * nF + 4
        o = self.out = dict(lastHS=np.zeros((n, n), np.float64, order="F"), lastbS=np.zeros(n), lastX=np.zeros(n),
                            idepth=np.zeros(nP, np.float32), step=np.zeros(nP, np.float32), HdiF=np.zeros(nP, np.float32),
                            state_state=np.zeros(nR, np.uint8), state_NewState=np.zeros(nR, np.uint8),
                            state_energy=np.zeros(nR, np.float32))
        self._sol = (_d(o["lastHS"]), _d(o["lastbS"]), _d(o["lastX"]))
        self._pts = (_f(o["idepth"]), None, _f(o["step"]), _f(o["HdiF"]), None, None, None, None)
        self._res = (_b(o["state_state"]), _b(o["state_NewState"]), _f(o["state_energy"]), None, None, None, None, None, None, None)
        self.h2d_bytes = (k["color"].nbytes + nF * (9 + 3 + 10 + 10) * 8 + 8 * 8 +
                          sum(k[x].nbytes for x in ("pt_host", "pt_u", "pt_v", "pt_idepth", "pt_idepth_zero", "pt_has_prior",
                                                    "pt_color", "pt_weights", "res_begin", "res_target")))
        self.d2h_bytes = sum(v.nbytes for v in o.values())

    def submit(self, iteration=0, n_iterations=1):
        """ldso_b200_optimize_from_host_submit: queue the whole step, do not wait."""
        self._prep(iteration, n_iterations)
        self.ctx._chk(self.L.ldso_b200_optimize_from_host_submit(self.h, C.byref(self._io)))

    def wait(self):
        """ldso_b200_optimize_from_host_wait: block until the submitted step is done, outputs filled."""
        self.ctx._chk(self.L.ldso_b200_optimize_from_host_wait(self.h, C.byref(self._io)))
        self.ctx.nF, self.ctx.nP, self.ctx.nR = self.nF, self.nP, self.nR
        return self.out

    def fused(self, iteration=0, n_iterations=1):
        """The same step as upload() + step() + download(), as ONE C-ABI call (ldso_b200_optimize_from_host)."""
        self._prep(iteration, n_iterations)
        self.ctx._chk(self.L.ldso_b200_optimize_from_host(self.h, C.byref(self._io)))
        self.ctx.nF, self.ctx.nP, self.ctx.nR = self.nF, self.nP, self.nR
        return self.out

    def submit_until(self, iteration=0, max_iterations=6, min_iterations=1):
        """ldso_b200_optimize_from_host_until_submit: the step with FullSystem::optimize's exit, not waited for."""
        self._prep(iteration, max_iterations)
        self.ctx._chk(self.L.ldso_b200_optimize_from_host_until_submit(self.h, C.byref(self._io), int(min_iterations)))

    def wait_until(self):
        """ldso_b200_optimize_from_host_until_wait: outputs filled, self.iterations_run = bodies run."""
        n = C.c_int()
        self.ctx._chk(self.L.ldso_b200_optimize_from_host_until_wait(self.h, C.byref(self._io), C.byref(n)))
        self.ctx.nF, self.ctx.nP, self.ctx.nR = self.nF, self.nP, self.nR
        self.iterations_run = n.value
        return self.out

    def fused_until(self, iteration=0, max_iterations=6, min_iterations=1):
        """ldso_b200_optimize_from_host_until: the whole step with the exit as ONE call; self.iterations_run = bodies run."""
        self._prep(iteration, max_iterations)
        n = C.c_int()
        self.ctx._chk(self.L.ldso_b200_optimize_from_host_until(self.h, C.byref(self._io), int(min_iterations), C.byref(n)))
        self.ctx.nF, self.ctx.nP, self.ctx.nR = self.nF, self.nP, self.nR
        self.iterations_run = n.value
        return self.out

    def _finish_out(self):
        if not hasattr(self, "_fo"):
            self.finish = _finish_arrays(self.nP, self.nR)
            self._fin_n = np.zeros(1, np.int32)
            self._fo = FinishOutC(_i(self._fin_n), *_finish_ptrs(self.finish))
        return C.byref(self._fo)

    def _finished(self):
        self.ctx.nF, self.ctx.nP, self.ctx.nR = self.nF, self.nP, self.nR
        self.iterations_run = int(self._fin_n[0])
        return self.out, _finish_scalars(self.finish)

    def submit_full(self, iteration=0, max_iterations=6, min_iterations=1):
        """ldso_b200_optimize_from_host_full_submit: the step with the exit and the finish, not waited for."""
        self._prep(iteration, max_iterations)
        self.ctx._chk(self.L.ldso_b200_optimize_from_host_full_submit(self.h, C.byref(self._io), int(min_iterations)))

    def wait_full(self):
        """ldso_b200_optimize_from_host_full_wait: (loop outputs, finish results)."""
        self.ctx._chk(self.L.ldso_b200_optimize_from_host_full_wait(self.h, C.byref(self._io), self._finish_out()))
        return self._finished()

    def fused_full(self, iteration=0, max_iterations=6, min_iterations=1):
        """ldso_b200_optimize_from_host_full: one keyframe's whole FullSystem::optimize as ONE call: (loop outputs, finish results)."""
        self._prep(iteration, max_iterations)
        self.ctx._chk(self.L.ldso_b200_optimize_from_host_full(self.h, C.byref(self._io), int(min_iterations), self._finish_out()))
        return self._finished()

    def scalars(self):
        """(energy, canbreak) the last fused / submitted step returned"""
        return float(self._scal[0][0]), bool(self._scal[1][0])

    def _prep(self, iteration, n_iterations):
        if not hasattr(self, "_io"):
            io = self._io = FusedIOC()
            o = self.out
            self._scal = (np.zeros(1), np.zeros(1, np.int32))
            io.image_slot = self.nF - 1; io.image = self._color; io.nFrames = self.nF
            io.frames = C.cast(self._frames, C.c_void_p); io.calib_value_scaled = self._Ks; io.calib_value_zero = self._Kz
            io.window = C.cast(C.pointer(self.w), C.c_void_p)
            io.lastHS, io.lastbS, io.lastX = self._sol
            io.energy = _d(self._scal[0]); io.canbreak = _i(self._scal[1])
            io.pt_idepth = _f(o["idepth"]); io.pt_step = _f(o["step"]); io.pt_HdiF = _f(o["HdiF"])
            io.res_state = _b(o["state_state"]); io.res_new_state = _b(o["state_NewState"]); io.res_energy = _f(o["state_energy"])
        self._io.first_iteration = int(iteration); self._io.n_iterations = int(n_iterations)

    def upload(self):
        """newest keyframe's raw image (+ device makeImages), frame states, the whole window"""
        L, h, chk = self.L, self.h, self.ctx._chk
        # the two asynchronous uploads first; make_images blocks until the caller's image buffer has been consumed
        chk(L.ldso_b200_set_window(h, self._wref))
        chk(L.ldso_b200_set_frames(h, self.nF, self._frames, self._Ks, self._Kz))
        chk(L.ldso_b200_make_images(h, self.nF - 1, self._color))
        self.ctx.nF, self.ctx.nP, self.ctx.nR = self.nF, self.nP, self.nR

    def step(self, iteration=0):
        """optimize() prologue + one Gauss-Newton iteration; the result read-back is queued behind it"""
        L, h, chk = self.L, self.h, self.ctx._chk
        chk(L.ldso_b200_optimize_begin(h, None))
        chk(L.ldso_b200_gn_iterations(h, int(iteration), 1))
        chk(L.ldso_b200_prefetch_results(h))

    def download(self):
        """solution (lastHS, lastbS, lastX), point idepth/step/HdiF, residual states + energies"""
        L, h, chk = self.L, self.h, self.ctx._chk
        chk(L.ldso_b200_get_last_solution(h, *self._sol))
        chk(L.ldso_b200_get_points(h, *self._pts))
        chk(L.ldso_b200_get_residuals(h, *self._res))
        return self.out
