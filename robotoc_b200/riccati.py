"""Host-side mirror of the reference's Riccati classes, calling the CUDA library through its C ABI.

  RiccatiRecursion          <-> robotoc/include/robotoc/riccati/riccati_recursion.hpp:26-119
  UnconstrRiccatiRecursion  <-> robotoc/include/robotoc/riccati/unconstr_riccati_recursion.hpp

Same method names and argument meaning; the per-stage containers (KKTMatrix, KKTResidual, RiccatiFactorization,
Direction, aligned_vector<LQRPolicy>) are the packed numpy arrays described by robotoc_b200.layout.Layout,
with a leading batch axis (many independent OCPs per call).  Errors follow the reference's conventions:
argument errors raise ValueError (std::invalid_argument / std::out_of_range), everything else RuntimeError.
"""
import ctypes

import numpy as np

from . import _lib
from .layout import Dims, Layout, ULayout

KKT, RIC, FACT, DIR, DX0 = 0, 1, 2, 3, 4


def _check(rc, msg_fn, what):
    if rc == 0:
        return
    msg = msg_fn()
    if rc == 1:
        raise ValueError(f"[{what}] invalid argument: {msg}")
    raise RuntimeError(f"[{what}] error {rc}: {msg}")


def _vp(a):
    if a is None:
        return None
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"], "packed arrays must be C-contiguous float64"
    return a.ctypes.data_as(ctypes.c_void_p)


class RiccatiRecursion:
    """RiccatiRecursion(ocp, max_dts0) -- riccati_recursion.hpp:35.  `dims`, `n_grid_max` (= N+1+reserved events)
    and `batch` play the role of the OCP argument."""

    def __init__(self, dims: Dims, n_grid_max: int, batch: int, max_dts0: float = 0.1, device: int = 0):
        if max_dts0 <= 0:
            raise ValueError("[RiccatiRecursion] invalid argument: 'max_dts0' must be positive!")
        self._lib = _lib.lib()
        self.dims, self.batch, self.n_grid_max = dims, batch, n_grid_max
        self.layout = Layout(dims)
        self._max_dts0 = float(max_dts0)
        self._h = ctypes.c_void_p()
        cd = dims.c()
        rc = self._lib.rbt_create(ctypes.byref(cd), n_grid_max, batch, device, ctypes.byref(self._h))
        if rc != 0:
            msg = self._lib.rbt_last_error(self._h).decode() if self._h else "unsupported dimensions or bad sizes"
            if self._h:
                self._lib.rbt_destroy(self._h)
                self._h = None
            _check(rc, lambda: msg, "RiccatiRecursion")
        self.n_grid = 0
        self._ctrl = None

    def close(self):
        if getattr(self, "_h", None):
            self._lib.rbt_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _err(self):
        return self._lib.rbt_last_error(self._h).decode()

    # -- reference API ------------------------------------------------------------------------------------
    def setRegularization(self, max_dts0: float):
        """riccati_recursion.hpp:58"""
        if max_dts0 <= 0:
            raise ValueError("[RiccatiRecursion] invalid argument: 'max_dts0' must be positive!")
        self._max_dts0 = float(max_dts0)
        if self._ctrl is not None:
            self.setTimeDiscretization(self._ctrl)

    def setTimeDiscretization(self, ctrl):
        """The TimeDiscretization argument of backward/forwardRiccatiRecursion, as a ctypes rbt_stage_ctrl array."""
        n = len(ctrl)
        _check(self._lib.rbt_set_schedule(self._h, ctrl, n, self._max_dts0), self._err, "RiccatiRecursion")
        self._ctrl, self.n_grid = ctrl, n

    def backwardRiccatiRecursion(self, kkt=None, write_fact=False, stream=None):
        """riccati_recursion.cpp:32-80.  `kkt` (host, [batch, n_grid, k_stride]) is uploaded when given; otherwise the
        device-resident KKT buffer (rbt_dev_ptr) is used as is."""
        if kkt is not None:
            self._shape(kkt, self.layout.k_stride)
            _check(self._lib.rbt_upload(self._h, KKT, _vp(kkt), stream), self._err, "RiccatiRecursion")
        _check(self._lib.rbt_riccati_backward(self._h, int(write_fact), stream), self._err, "RiccatiRecursion")

    def forwardRiccatiRecursion(self, dx0=None, stream=None):
        """riccati_recursion.cpp:83-131; dx0 = d[0].dx for every OCP ([batch, nx])."""
        if dx0 is not None:
            if dx0.shape != (self.batch, self.dims.nx):
                raise ValueError("[RiccatiRecursion] invalid argument: dx0 must be [batch, nx]")
            _check(self._lib.rbt_upload(self._h, DX0, _vp(dx0), stream), self._err, "RiccatiRecursion")
        _check(self._lib.rbt_riccati_forward(self._h, stream), self._err, "RiccatiRecursion")

    def getRiccatiFactorization(self, stream=None):
        return self._get(RIC, self.layout.r_stride, stream)

    def getLQRPolicy(self, stream=None):
        """riccati_recursion.hpp:104 -- K (row-major nu x nx) and k per stage, as views into the Riccati records."""
        ric = self.getRiccatiFactorization(stream)
        L, d = self.layout, self.dims
        K = ric[..., L.r_K:L.r_K + d.nu * d.nx].reshape(self.batch, self.n_grid, d.nu, d.nx)
        k = ric[..., L.r_k:L.r_k + d.nu]
        return K, k

    def getFactorizedKKT(self, stream=None):
        return self._get(FACT, self.layout.f_stride, stream)

    def getDirection(self, stream=None):
        return self._get(DIR, self.layout.d_stride, stream)

    def solve_host(self, kkt, dx0, want_ric=True, want_dir=True, stream=None):
        """One C-ABI call with host buffers (H2D, backward, forward, D2H): rbt_riccati_solve_host."""
        self._shape(kkt, self.layout.k_stride)
        ric = np.empty((self.batch, self.n_grid, self.layout.r_stride)) if want_ric else None
        d = np.empty((self.batch, self.n_grid, self.layout.d_stride)) if want_dir else None
        _check(self._lib.rbt_riccati_solve_host(self._h, _vp(kkt), _vp(dx0), _vp(ric), _vp(d), stream), self._err,
               "RiccatiRecursion")
        self.synchronize(stream)
        return ric, d

    def info(self, stream=None):
        flags = np.zeros(self.batch, dtype=np.int32)
        _check(self._lib.rbt_download_info(self._h, flags.ctypes.data_as(ctypes.c_void_p), stream), self._err,
               "RiccatiRecursion")
        self.synchronize(stream)
        return flags

    def checkInfo(self, stream=None):
        """Raises RuntimeError (RBT_ERR_NUMERIC) if a factorization of the last condense / backward sweep failed -- where
        the reference asserts llt_.info() == Eigen::Success (riccati_factorizer.cpp:50,64).  Returns None otherwise."""
        first = ctypes.c_int(-1)
        _check(self._lib.rbt_check_info(self._h, ctypes.byref(first), stream), self._err, "RiccatiRecursion")

    def synchronize(self, stream=None):
        _check(self._lib.rbt_sync(self._h, stream), self._err, "RiccatiRecursion")

    def dev_ptr(self, which):
        return self._lib.rbt_dev_ptr(self._h, which)

    def bind_buffer(self, which, dev_ptr):
        """Use a caller-owned device buffer (e.g. a torch tensor's data_ptr()) for `which`; None restores the own one."""
        _check(self._lib.rbt_bind_buffer(self._h, which, dev_ptr), self._err, "RiccatiRecursion")

    def buf_doubles(self, which):
        return int(self._lib.rbt_buf_doubles(self._h, which))

    def launch_count(self):
        return int(self._lib.rbt_launch_count(self._h))

    # -- helpers ------------------------------------------------------------------------------------------
    def _shape(self, a, stride):
        if a.shape != (self.batch, self.n_grid, stride):
            raise ValueError(f"[RiccatiRecursion] invalid argument: expected shape {(self.batch, self.n_grid, stride)}, "
                             f"got {a.shape}")

    def _get(self, which, stride, stream):
        out = np.empty((self.batch, self.n_grid, stride))
        _check(self._lib.rbt_download(self._h, which, _vp(out), stream), self._err, "RiccatiRecursion")
        self.synchronize(stream)
        return out


class UnconstrRiccatiRecursion:
    """UnconstrRiccatiRecursion(ocp) -- unconstr_riccati_recursion.cpp:9-16 (N stages, dt = T/N)."""

    def __init__(self, nv: int, N: int, dt: float, batch: int, device: int = 0):
        if N <= 0:
            raise ValueError("[UnconstrRiccatiRecursion] invalid argument: 'N' must be positive!")
        if dt <= 0:
            raise ValueError("[UnconstrRiccatiRecursion] invalid argument: 'dt' must be positive!")
        self._lib = _lib.lib()
        self.nv, self.N, self.dt, self.batch = nv, N, float(dt), batch
        self.layout = ULayout(nv)
        self._h = ctypes.c_void_p()
        rc = self._lib.rbt_unconstr_create(nv, N, dt, batch, device, ctypes.byref(self._h))
        if rc != 0:
            msg = self._lib.rbt_unconstr_last_error(self._h).decode() if self._h else "unsupported nv or bad sizes"
            if self._h:
                self._lib.rbt_unconstr_destroy(self._h)
                self._h = None
            _check(rc, lambda: msg, "UnconstrRiccatiRecursion")

    def close(self):
        if getattr(self, "_h", None):
            self._lib.rbt_unconstr_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _err(self):
        return self._lib.rbt_unconstr_last_error(self._h).decode()

    def backwardRiccatiRecursion(self, kkt=None, write_fact=False, stream=None):
        """unconstr_riccati_recursion.cpp:26-35"""
        if kkt is not None:
            if kkt.shape != (self.batch, self.N + 1, self.layout.k_stride):
                raise ValueError("[UnconstrRiccatiRecursion] invalid argument: kkt shape")
            _check(self._lib.rbt_unconstr_upload(self._h, KKT, _vp(kkt), stream), self._err, "UnconstrRiccatiRecursion")
        _check(self._lib.rbt_unconstr_backward(self._h, int(write_fact), stream), self._err, "UnconstrRiccatiRecursion")

    def forwardRiccatiRecursion(self, dx0=None, stream=None):
        """unconstr_riccati_recursion.cpp:37-46"""
        if dx0 is not None:
            if dx0.shape != (self.batch, 2 * self.nv):
                raise ValueError("[UnconstrRiccatiRecursion] invalid argument: dx0 must be [batch, nx]")
            _check(self._lib.rbt_unconstr_upload(self._h, DX0, _vp(dx0), stream), self._err, "UnconstrRiccatiRecursion")
        _check(self._lib.rbt_unconstr_forward(self._h, stream), self._err, "UnconstrRiccatiRecursion")

    def _get(self, which, stride, stream=None):
        out = np.empty((self.batch, self.N + 1, stride))
        _check(self._lib.rbt_unconstr_download(self._h, which, _vp(out), stream), self._err, "UnconstrRiccatiRecursion")
        self.synchronize(stream)
        return out

    def getRiccatiFactorization(self, stream=None):
        return self._get(RIC, self.layout.r_stride, stream)

    def getLQRPolicy(self, stream=None):
        ric = self.getRiccatiFactorization(stream)
        L, nv = self.layout, self.nv
        K = ric[..., L.r_K:L.r_K + nv * 2 * nv].reshape(self.batch, self.N + 1, nv, 2 * nv)
        return K, ric[..., L.r_k:L.r_k + nv]

    def getFactorizedKKT(self, stream=None):
        return self._get(FACT, self.layout.f_stride, stream)

    def getDirection(self, stream=None):
        return self._get(DIR, self.layout.d_stride, stream)

    def solve_host(self, kkt, dx0, want_ric=True, want_dir=True, stream=None):
        ric = np.empty((self.batch, self.N + 1, self.layout.r_stride)) if want_ric else None
        d = np.empty((self.batch, self.N + 1, self.layout.d_stride)) if want_dir else None
        _check(self._lib.rbt_unconstr_solve_host(self._h, _vp(kkt), _vp(dx0), _vp(ric), _vp(d), stream), self._err,
               "UnconstrRiccatiRecursion")
        self.synchronize(stream)
        return ric, d

    def info(self, stream=None):
        flags = np.zeros(self.batch, dtype=np.int32)
        _check(self._lib.rbt_unconstr_download_info(self._h, flags.ctypes.data_as(ctypes.c_void_p), stream), self._err,
               "UnconstrRiccatiRecursion")
        self.synchronize(stream)
        return flags

    def synchronize(self, stream=None):
        _check(self._lib.rbt_unconstr_sync(self._h, stream), self._err, "UnconstrRiccatiRecursion")

    def launch_count(self):
        return int(self._lib.rbt_unconstr_launch_count(self._h))
