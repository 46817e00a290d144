"""`ProjectedProcessEngine`: the Python face of the C-ABI (one context = one GPU).

Mirrors the reference seam `ProjectedGaussianProcessHelper` (commons/ProjectedGaussianProcessHelper.scala):
  getMatrixKmnKnmAndVectorKmny(experts, activeSet)  ->  begin / accumulate* / finish
  getMagicVector(kernel, G, b, ...)                 ->  magic()
and `GaussianProjectedProcessRawPredictor.predict` (commons/GaussianProcessCommons.scala:121-125) -> predict().
Error codes are mapped back to the reference's exception types."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as N
from .kernels import Kernel


class NotPositiveDefiniteException(Exception):
    """ProjectedGaussianProcessHelper.scala:9-11."""


class TrainingVectorsNotInitializedException(Exception):
    """kernel/Kernel.scala:116-117 (raised here for call-order violations)."""


class MatrixSingularException(Exception):
    """breeze MatrixSingularException (commons/util/logDetAndInv.scala:27-28)."""


class SgpError(RuntimeError):
    pass


class OperandRangeError(SgpError):
    """SGP_E_RANGE: the int8 path cannot represent these coordinates (rerun in SGP_PREC_F64), or a k-means distance to
    the nearest centre is beyond the fp32 range after the data's prescale."""


def is_cuda_tensor(x) -> bool:
    """A CUDA torch tensor (checked without importing torch: the package has no hard torch dependency)."""
    return type(x).__module__.partition(".")[0] == "torch" and bool(getattr(x, "is_cuda", False))


def device_tensor(X, device: int, what: str, dtype=None):
    """A CUDA torch tensor as the library reads it on cuda:`device`: float32 and float64 as given (or `dtype` when given),
    other dtypes converted to float64, contiguous.  Synchronises torch's current stream, so that whatever torch still has
    queued for the tensor is written before the library's stream reads it.  ValueError for a tensor on another device."""
    import torch
    if X.device.type != "cuda" or X.device.index != device:
        raise ValueError("%s: the tensor is on %s, the model on cuda:%d" % (what, X.device, device))
    if dtype is not None:
        X = X.to(dtype)
    elif X.dtype not in (torch.float32, torch.float64):
        X = X.to(torch.float64)
    X = X.contiguous()
    torch.cuda.current_stream(X.device).synchronize()
    return X


def device_fit_data(X, y, device: int, what: str):
    """The (X, y) of a fit from a CUDA tensor X: ValueError, before anything runs on the device, for X on another device
    than cuda:`device` or not n x d, and for y on another device than X or not n entries.  y may be a host vector; it
    becomes a CUDA float64 vector.  X keeps its dtype (`device_tensor` converts it where the library reads it)."""
    import torch
    if X.device.type != "cuda" or X.device.index != device:
        raise ValueError("%s: X is on %s, the estimator on cuda:%d" % (what, X.device, device))
    if X.ndim != 2:
        raise ValueError("%s: X must be n x d" % what)
    if isinstance(y, torch.Tensor):
        if y.device != X.device:
            raise ValueError("%s: y is on %s, X on %s" % (what, y.device, X.device))
        y = y.to(torch.float64)
    else:
        y = torch.as_tensor(np.asarray(y, dtype=np.float64), device=X.device)
    if y.ndim != 1 or len(y) != len(X):
        raise ValueError("%s: y must hold one label per row of X (%d), not shape %s" % (what, len(X), tuple(y.shape)))
    return X, y


def take_rows(X, idx):
    """X[idx] on X's side: a numpy array, or a CUDA tensor gathered on the device (nothing crosses PCIe but idx)."""
    if is_cuda_tensor(X):
        import torch
        return X[torch.as_tensor(np.asarray(idx, dtype=np.int64), device=X.device)]
    return np.asarray(X)[idx]


def rows_to_host(X, idx):
    """X[idx] as a float64 host array: for a CUDA tensor only these rows cross PCIe."""
    if is_cuda_tensor(X):
        import torch
        return take_rows(X, idx).to(torch.float64).cpu().numpy()
    return np.asarray(np.asarray(X)[idx], dtype=np.float64)


def host_copy(x):
    """An explicit float64 host copy of a CUDA tensor, for the algorithms that run on the host; host arrays pass as they
    are."""
    if is_cuda_tensor(x):
        return np.asarray(x.cpu().numpy(), dtype=np.float64)
    return x


def _rows(X):
    """Points as the library reads them: float32 stays as it is (no copy when already contiguous), anything else becomes
    float64; C-contiguous."""
    X = np.asarray(X)
    return np.ascontiguousarray(X if X.dtype == np.float32 else np.asarray(X, dtype=np.float64))


def _make_desc(kernel: Kernel, d: int):
    terms = kernel.flatten()
    arr = (N.KernelTerm * len(terms))()
    keep = []
    for i, t in enumerate(terms):
        arr[i].type = t["type"]
        arr[i].scale = t["scale"]
        arr[i].sigma = t.get("sigma", 0.0)
        if t["type"] == N.SGP_TERM_ARD:
            beta = np.ascontiguousarray(t["beta"], dtype=np.float64)
            if len(beta) != d:
                raise ValueError("ARDRBFKernel has %d betas but the data has %d features" % (len(beta), d))
            keep.append(beta)
            arr[i].beta = beta.ctypes.data_as(C.POINTER(C.c_double))
    desc = N.KernelDesc(len(terms), 0, arr)
    return desc, (arr, keep)


class ProjectedProcessEngine:
    def __init__(self, device: int = 0):
        self._lib = N.load()
        self._h = C.c_void_p()
        rc = self._lib.sgp_ctx_create(C.byref(self._h), device)
        if rc != N.SGP_OK:
            raise SgpError("sgp_ctx_create failed (%d): %s" % (rc, self._lib.sgp_last_error(None).decode()))
        self.m = self.d = 0
        self._device = device
        self._has_comm = False

    # ---- a small per-device pool: creating a context costs ~20 ms (streams, cuBLAS, cuSOLVER) and a fresh context
    #      re-allocates every grow-only workspace; an estimator that fits repeatedly gets its contexts back from here ----
    _idle = {}
    _IDLE_MAX = 4

    @classmethod
    def acquire(cls, device: int = 0):
        """An idle context of the pool, or a new one.  Estimators fit from several threads at once (one Spark task each):
        the pool is popped without a check-then-pop window, so two threads never get the same context and a thread
        that finds the pool emptied under it creates its own."""
        try:
            eng = cls._idle.get(device, []).pop()
        except IndexError:
            return cls(device)
        eng.set_precision(N.SGP_PREC_AUTO)
        return eng

    def release(self):
        """Hand the context back to the pool (or destroy it when the pool is full or it carries a communicator)."""
        if not self._h:
            return
        pool = ProjectedProcessEngine._idle.setdefault(self._device, [])
        if self._has_comm or len(pool) >= ProjectedProcessEngine._IDLE_MAX:
            self.close()
        else:
            pool.append(self)

    def close(self):
        if self._h:
            self._lib.sgp_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc == N.SGP_OK:
            return
        msg = self._lib.sgp_last_error(self._h).decode()
        if rc == N.SGP_E_NOT_PD:
            raise NotPositiveDefiniteException(msg)
        if rc == N.SGP_E_STATE:
            raise TrainingVectorsNotInitializedException(msg)
        if rc == N.SGP_E_SINGULAR:
            raise MatrixSingularException(msg)
        if rc == N.SGP_E_BADARG:
            raise ValueError(msg)
        if rc == N.SGP_E_RANGE:
            raise OperandRangeError(msg)
        raise SgpError("sgp error %d: %s" % (rc, msg))

    # ---- configuration ---------------------------------------------------------------------------
    def set_precision(self, mode: int):
        self._check(self._lib.sgp_set_precision(self._h, mode))

    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(N.SGP_UNIQUE_ID_BYTES)
        rc = N.load().sgp_comm_unique_id(buf)
        if rc != N.SGP_OK:
            raise SgpError("sgp_comm_unique_id failed")
        return buf.raw

    def comm_init(self, unique_id: bytes, rank: int, nranks: int):
        buf = C.create_string_buffer(unique_id, N.SGP_UNIQUE_ID_BYTES)
        self._check(self._lib.sgp_comm_init(self._h, buf, rank, nranks))
        self._has_comm = True

    # ---- getMatrixKmnKnmAndVectorKmny ---------------------------------------------------------------
    def begin(self, kernel: Kernel, active_set):
        Z = np.ascontiguousarray(active_set, dtype=np.float64)
        if Z.ndim != 2:
            raise ValueError("activeSet must be m x d")
        self.m, self.d = Z.shape
        desc, keep = _make_desc(kernel, self.d)
        self._check(self._lib.sgp_stats_begin(self._h, C.byref(desc), N.ptr(Z), self.m, self.d))
        del keep

    def accumulate(self, X, y):
        """One shard of points in host memory.  X: n x d (float32 or float64), y: n."""
        X = _rows(X)
        y =np.ascontiguousarray(y, dtype=np.float64)
        if X.ndim != 2 or X.shape[1] != self.d or len(y) != len(X):
            raise ValueError("shard shape mismatch")
        self._check(self._lib.sgp_stats_accumulate(self._h, N.ptr(X), int(X.dtype == np.float32), N.ptr(y), len(X)))

    def accumulate_ptr(self, x_ptr: int, x_is_f32: bool, y_ptr: int, n: int, device: bool):
        fn = self._lib.sgp_stats_accumulate_device if device else self._lib.sgp_stats_accumulate
        self._check(fn(self._h, C.c_void_p(x_ptr), int(x_is_f32), C.c_void_p(y_ptr), n))

    def finish(self, copy_out: bool = True):
        if not copy_out:
            self._check(self._lib.sgp_stats_finish(self._h, None, None))
            return None, None
        G = np.empty((self.m, self.m))
        b = np.empty(self.m)
        self._check(self._lib.sgp_stats_finish(self._h, N.ptr(G), N.ptr(b)))
        return G, b

    def sync(self):
        self._check(self._lib.sgp_sync(self._h))

    def statistics(self, kernel: Kernel, active_set, X, y, shard_points: int = 1 << 22):
        """`getMatrixKmnKnmAndVectorKmny` over host data in shards (PGPH:23 broadcast, PGPH:25-35 seqOp over shards), or
        over a CUDA tensor X (and y) in one `sgp_stats_accumulate_device` call: the library cuts its own launch windows,
        so shard_points applies to host data only.  When the int8 path reports SGP_E_RANGE (coordinates outside its
        operand range, or AUTO's magnitude budget exceeded over the whole window) the pass is repeated on the fp64 DMMA
        kernel -- still on the GPU."""
        if is_cuda_tensor(X):
            import torch
            X = device_tensor(X, self._device, "statistics")
            y = device_tensor(y, self._device, "statistics", torch.float64)
            if X.ndim != 2 or y.shape != (len(X),):
                raise ValueError("statistics: X must be n x d and y n entries")

        def run():
            self.begin(kernel, active_set)
            if is_cuda_tensor(X):
                if X.shape[1] != self.d:
                    raise ValueError("shard shape mismatch")
                self.accumulate_ptr(X.data_ptr(), X.dtype == torch.float32, y.data_ptr(), len(X), device=True)
            else:
                for s in range(0, len(X), shard_points):
                    self.accumulate(X[s:s + shard_points], y[s:s + shard_points])
            return self.finish()
        try:
            return run()
        except OperandRangeError:
            # the int8 Gram refused the shard (coordinates outside its operand range, or scaled norms above AUTO's budget:
            # tiny kernel values, where its fixed-point elements are not parity-grade): the fp64 DMMA kernel takes anything
            self.set_precision(N.SGP_PREC_F64)
            return run()

    # ---- the BCM hyper-parameter objective (GPR:55-68 over all experts, GPC:73-78) ----------------------------------
    def experts_upload(self, X, y, offsets):
        """Experts packed expert-major: expert e owns rows offsets[e]..offsets[e+1]-1."""
        X = np.ascontiguousarray(X, dtype=np.float64)
        y = np.ascontiguousarray(y, dtype=np.float64)
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        self._check(self._lib.sgp_experts_upload(self._h, N.ptr(X), N.ptr(y), N.ptr(off), len(off) - 1, X.shape[1]))
        self._experts_d = X.shape[1]

    def _device_xy(self, X, y, what):
        """(X, y) of a device entry: X as `device_tensor` reads it, y float64, each with its pointer."""
        import torch
        X = device_tensor(X, self._device, what)
        y = device_tensor(y, self._device, what, torch.float64)
        return X, y, C.c_void_p(X.data_ptr()), C.c_void_p(y.data_ptr()), int(X.dtype == torch.float32)

    def experts_upload_grouped(self, X, y, dataset_size_for_expert: int):
        """Groups the points into experts ON THE DEVICE (GPC:26-31: point i -> expert i % E) while they stream in; X may be
        float32 or float64, row-major as given.  A CUDA tensor X (and y) is read in place
        (`sgp_experts_upload_grouped_device`): the same experts, bit for bit.  Returns the number of experts."""
        if is_cuda_tensor(X):
            X, y, px, py, f32 = self._device_xy(X, y, "experts_upload_grouped")
            self._check(self._lib.sgp_experts_upload_grouped_device(self._h, px, f32, py, len(X), X.shape[1],
                                                                    int(dataset_size_for_expert)))
        else:
            X = _rows(X)
            y =np.ascontiguousarray(y, dtype=np.float64)
            self._check(self._lib.sgp_experts_upload_grouped(self._h, N.ptr(X), int(X.dtype == np.float32), N.ptr(y),
                                                             len(X), X.shape[1], int(dataset_size_for_expert)))
        self._experts_d = X.shape[1]
        return int(np.floor(len(X) / dataset_size_for_expert + 0.5))

    def experts_upload_strided(self, X, y, n_experts: int):
        """Groups CUDA tensor rows into n_experts experts on the device, row i -> expert i % n_experts
        (`sgp_experts_upload_strided_device`): a data-parallel fit's rank uploads its block of the global experts with it,
        its rows in global row order.  Returns n_experts."""
        X, y, px, py, f32 = self._device_xy(X, y, "experts_upload_strided")
        if X.ndim != 2 or y.shape != (len(X),):
            raise ValueError("experts_upload_strided: X must be n x d and y n entries")
        self._check(self._lib.sgp_experts_upload_strided_device(self._h, px, f32, py, len(X), X.shape[1], int(n_experts)))
        self._experts_d = X.shape[1]
        return int(n_experts)

    def _descriptors(self, kernel: Kernel, d: int = None):
        """(kernel desc, hyper-parameter descriptors, their count, the buffers both point into) for d features (default:
        the uploaded experts')."""
        desc, keep = _make_desc(kernel, self._experts_d if d is None else d)
        hd = kernel.hyper_descriptors()
        arr = (N.Hyper * max(len(hd), 1))()
        coefs = []
        for i, h in enumerate(hd):
            arr[i].kind = h["kind"]
            arr[i].term = h.get("term", 0)
            arr[i].dim = h.get("dim", 0)
            arr[i].value = h.get("value", 0.0)
            if h["kind"] == N.SGP_HYPER_SCALE:
                cf = np.zeros(desc.n_terms)
                for t, v in h["coef"].items():
                    cf[t] = v
                coefs.append(cf)
                arr[i].coef = cf.ctypes.data_as(C.POINTER(C.c_double))
        return desc, arr, len(hd), (keep, coefs)

    def _objective(self, fn, kernel: Kernel, *args):
        """Runs one per-expert objective of the library over the uploaded experts: (value, gradient w.r.t.
        kernel.getHyperparameters())."""
        desc, arr, nh, keep = self._descriptors(kernel)
        val = C.c_double()
        grad = np.zeros(max(nh, 1))
        self._check(fn(self._h, C.byref(desc), arr, nh, *args, C.byref(val), N.ptr(grad)))
        del keep
        return val.value, grad[:nh]

    def laplace_nll(self, kernel: Kernel, tol: float):
        """Binary classification: (-log Z summed over experts, its gradient).  Updates the device-resident latent
        modes f of the uploaded experts (warm start), as GaussianProcessClassifier.likelihoodAndGradient does."""
        return self._objective(self._lib.sgp_laplace_nll, kernel, float(tol))

    def laplace_nll_any_size(self, kernel: Kernel, tol: float):
        """`laplace_nll` for experts of any size (`sgp_laplace_nll_any_size`): the same launch and bits while the largest
        expert fits on chip (117 points), the global-memory kernel above."""
        return self._objective(self._lib.sgp_laplace_nll_any_size, kernel, float(tol))

    def last_laplace_path(self) -> int:
        """Which kernel the last Laplace objective ran: 0 on chip, 1 global memory, -1 none yet."""
        return int(self._lib.sgp_last_laplace_path(self._h))

    def experts_upload_folds(self, X, y, fold_of, n_folds: int, dataset_size_for_expert: int):
        """Uploads the training set of every fold of a k-fold split (`sgp_experts_upload_folds`): set k holds the points
        with fold_of != k in index order, grouped into experts as `experts_upload_grouped` groups them.  X may be float32
        or float64; a CUDA tensor X (and y) is read in place (`sgp_experts_upload_folds_device`), fold_of stays a host
        array.  Returns the number of experts of each set."""
        folds = np.ascontiguousarray(fold_of, dtype=np.int32)
        if is_cuda_tensor(X):
            X, y, px, py, f32 = self._device_xy(X, y, "experts_upload_folds")
            fn = self._lib.sgp_experts_upload_folds_device
        else:
            X = _rows(X)
            y =np.ascontiguousarray(y, dtype=np.float64)
            px, py, f32, fn = N.ptr(X), N.ptr(y), int(X.dtype == np.float32), self._lib.sgp_experts_upload_folds
        if X.ndim != 2 or len(y) != len(X) or folds.shape != (len(X),):
            raise ValueError("experts_upload_folds: X must be n x d, y and fold_of n entries")
        self._check(fn(self._h, px, f32, py, len(X), X.shape[1], N.ptr(folds), int(n_folds), int(dataset_size_for_expert)))
        self._experts_d = X.shape[1]
        n_k = len(X) - np.bincount(folds, minlength=int(n_folds))
        return np.floor(n_k / dataset_size_for_expert + 0.5).astype(np.int64)

    def experts_upload_fold_sets(self, X, y, set_rows, set_experts):
        """Uploads training sets given as blocks of CUDA tensor rows (`sgp_experts_upload_fold_sets_device`): block k is
        the next set_rows[k] rows, grouped row i -> expert i % set_experts[k], and becomes fold set k, as
        `experts_upload_folds` stores its sets.  A data-parallel model selection's rank uploads its block of every training
        set's experts with it.  Returns set_experts as an int64 array."""
        X, y, px, py, f32 = self._device_xy(X, y, "experts_upload_fold_sets")
        rows = np.ascontiguousarray(set_rows, dtype=np.int64)
        experts = np.ascontiguousarray(set_experts, dtype=np.int64)
        if X.ndim != 2 or y.shape != (len(X),) or rows.ndim != 1 or experts.shape != rows.shape \
                or int(rows.sum()) != len(X):
            raise ValueError("experts_upload_fold_sets: X must be n x d, y n entries, and set_rows sum to n")
        self._check(self._lib.sgp_experts_upload_fold_sets_device(self._h, px, f32, py, N.ptr(rows), N.ptr(experts),
                                                                  len(rows), X.shape[1]))
        self._experts_d = X.shape[1]
        return experts

    def _batched_objective(self, fn, head, kernels, tail=()):
        """Runs one batched per-expert objective of the library, `fn(ctx, *head, descs, hypers, n_hypers, *tail, values,
        gradients)`, with one evaluation per kernel.  Returns (values [n_eval], gradients [n_eval x n_hypers])."""
        descs = (N.KernelDesc * len(kernels))()
        keep, hyp, nh = [], None, None
        for i, k in enumerate(kernels):
            desc, arr, n_i, kp = self._descriptors(k)
            if nh is None:
                nh = n_i
                hyp = (N.Hyper * max(len(kernels) * nh, 1))()
            elif n_i != nh:
                raise ValueError("every slot needs the same hyper-parameter layout")
            descs[i] = desc
            for j in range(nh):
                hyp[i * nh + j] = arr[j]
            keep.append(kp)
        vals = np.zeros(len(kernels))
        grads = np.zeros((len(kernels), max(nh, 1)))
        self._check(fn(self._h, *head, descs, hyp, nh, *tail, N.ptr(vals), N.ptr(grads)))
        del keep
        return vals, np.ascontiguousarray(grads[:, :nh])

    def bcm_nll_folds(self, sets, kernels):
        """The BCM objective of each listed fold set at its own kernels[i], all in one launch (`sgp_bcm_nll_folds`) over
        the last `experts_upload_folds`.  A set may be listed several times.  Returns (values [n_eval], gradients
        [n_eval x n_hypers])."""
        st = np.ascontiguousarray(sets, dtype=np.int32)
        if st.ndim != 1 or len(st) == 0 or len(st) != len(kernels):
            raise ValueError("bcm_nll_folds: one kernel per listed set")
        return self._batched_objective(self._lib.sgp_bcm_nll_folds, (N.ptr(st), len(st)), kernels)

    def bcm_nll_slots(self, kernels):
        """The BCM objective of the last `experts_upload_grouped` at each of kernels, all in one launch
        (`sgp_bcm_nll_slots`): slot i is `bcm_nll(kernels[i])`, bit for bit.  Returns (values [n_eval], gradients
        [n_eval x n_hypers])."""
        if len(kernels) == 0:
            raise ValueError("bcm_nll_slots: at least one kernel")
        return self._batched_objective(self._lib.sgp_bcm_nll_slots, (len(kernels),), kernels)

    def laplace_nll_classes(self, n_classes: int, classes, kernels, tol: float):
        """One-vs-rest over uploaded class indices: the binary Laplace objective of each listed class c (labels y == c)
        at its own kernels[i], all in one launch (`sgp_laplace_nll_classes`).  Returns (values [n_eval], gradients
        [n_eval x n_hypers]); each class's device-resident modes warm-start its next evaluation."""
        return self._laplace_classes(self._lib.sgp_laplace_nll_classes, n_classes, classes, kernels, tol)

    def laplace_nll_classes_any_size(self, n_classes: int, classes, kernels, tol: float):
        """`laplace_nll_classes` for experts of any size (`sgp_laplace_nll_classes_any_size`)."""
        return self._laplace_classes(self._lib.sgp_laplace_nll_classes_any_size, n_classes, classes, kernels, tol)

    def _laplace_classes(self, fn, n_classes, classes, kernels, tol):
        cls = np.ascontiguousarray(classes, dtype=np.int32)
        if cls.ndim != 1 or len(cls) == 0 or len(cls) != len(kernels):
            raise ValueError("laplace_nll_classes: one kernel per listed class")
        return self._batched_objective(fn, (int(n_classes), N.ptr(cls), len(cls)), kernels, (float(tol),))

    def laplace_nll_slots_any_size(self, n_mode_slots: int, mode_slots, classes, kernels, tol: float):
        """Param-map slots (`sgp_laplace_nll_slots_any_size`): listed slot i evaluates the binary Laplace objective of the
        labels (y == classes[i]) at kernels[i], warm-started from and writing the modes of mode slot mode_slots[i], all in
        one launch.  Classes may repeat; mode slots are distinct in [0, n_mode_slots).  Returns (values [n_eval],
        gradients [n_eval x n_hypers])."""
        modes = np.ascontiguousarray(mode_slots, dtype=np.int32)
        cls = np.ascontiguousarray(classes, dtype=np.int32)
        if modes.ndim != 1 or len(modes) == 0 or cls.shape != modes.shape or len(modes) != len(kernels):
            raise ValueError("laplace_nll_slots_any_size: one class and one kernel per listed mode slot")
        return self._batched_objective(self._lib.sgp_laplace_nll_slots_any_size,
                                       (int(n_mode_slots), N.ptr(modes), N.ptr(cls), len(modes)), kernels, (float(tol),))

    def laplace_nll_fold_slots_any_size(self, n_mode_slots: int, mode_slots, sets, classes, kernels, tol: float):
        """Fold slots over the last `experts_upload_folds` (`sgp_laplace_nll_fold_slots_any_size`): listed slot i evaluates
        the binary Laplace objective of training set sets[i] with the labels (y == classes[i]) at kernels[i], warm-started
        from and writing the modes of mode slot mode_slots[i].  Sets and classes may repeat; mode slots are distinct in
        [0, n_mode_slots).  Each slot equals `laplace_nll_any_size` on a grouped upload of that set alone, bit for bit.
        Returns (values [n_eval], gradients [n_eval x n_hypers])."""
        modes = np.ascontiguousarray(mode_slots, dtype=np.int32)
        st = np.ascontiguousarray(sets, dtype=np.int32)
        cls = np.ascontiguousarray(classes, dtype=np.int32)
        if modes.ndim != 1 or len(modes) == 0 or st.shape != modes.shape or cls.shape != modes.shape \
                or len(modes) != len(kernels):
            raise ValueError("laplace_nll_fold_slots_any_size: one set, class and kernel per listed mode slot")
        return self._batched_objective(self._lib.sgp_laplace_nll_fold_slots_any_size,
                                       (int(n_mode_slots), N.ptr(modes), N.ptr(st), N.ptr(cls), len(modes)), kernels,
                                       (float(tol),))

    def experts_f_fold_slot(self, set_: int, slot: int, n: int):
        """Mode slot `slot`'s latent modes on fold set `set_` of n training rows, after `laplace_nll_fold_slots_any_size`
        (the set's packed expert-major order)."""
        return self._modes(self._lib.sgp_experts_get_f_fold_slot, n, int(set_), int(slot))

    def experts_f_fold_slot_rows(self, set_: int, slot: int, n: int):
        """`experts_f_fold_slot` in the set's training-row order as a CUDA float64 tensor on this context's device,
        ungrouped on the device (`sgp_experts_get_f_fold_rows_device`)."""
        import torch
        f = torch.empty(n, dtype=torch.float64, device="cuda:%d" % self._device)
        self._check(self._lib.sgp_experts_get_f_fold_rows_device(self._h, int(set_), int(slot), C.c_void_p(f.data_ptr())))
        return f

    def _modes(self, fn, n: int, *which):
        """n latent modes (packed expert-major order) read back by `fn(ctx, *which, out)`."""
        f = np.empty(n)
        self._check(fn(self._h, *which, N.ptr(f)))
        return f

    def experts_f_slot(self, slot: int, n: int):
        """Mode slot `slot`'s latent modes after `laplace_nll_slots_any_size` (packed expert-major order)."""
        return self._modes(self._lib.sgp_experts_get_f_slot, n, int(slot))

    def experts_f_class(self, cls: int, n: int):
        """Class cls's latent modes after `laplace_nll_classes` (packed expert-major order)."""
        return self._modes(self._lib.sgp_experts_get_f_class, n, int(cls))

    def experts_f(self, n: int):
        return self._modes(self._lib.sgp_experts_get_f, n)

    def experts_modes(self, store: int, index: int, n: int):
        """The n modes of one store (N.SGP_MODES_BINARY / _CLASS / _SLOT, index: the class or mode slot), packed
        expert-major, in host memory."""
        if store == N.SGP_MODES_CLASS:
            return self.experts_f_class(index, n)
        if store == N.SGP_MODES_SLOT:
            return self.experts_f_slot(index, n)
        return self.experts_f(n)

    def experts_modes_rows(self, store: int, index: int, n: int):
        """`experts_modes` in ROW order as a CUDA float64 tensor on this context's device, ungrouped on the device
        (`sgp_experts_get_f_rows_device`): the modes never leave it.  Needs a grouped upload of n points."""
        import torch
        f = torch.empty(n, dtype=torch.float64, device="cuda:%d" % self._device)
        self._check(self._lib.sgp_experts_get_f_rows_device(self._h, int(store), int(index), C.c_void_p(f.data_ptr())))
        return f

    def bcm_nll(self, kernel: Kernel):
        """(sum over experts of 1/2 y'K^-1 y + 1/2 log|K|, gradient w.r.t. kernel.getHyperparameters())."""
        return self._objective(self._lib.sgp_bcm_nll, kernel)

    # ---- getMagicVector -------------------------------------------------------------------------------
    def magic(self, G=None, b=None, copy_out: bool = True):
        mv = np.empty(self.m) if copy_out else None
        mm = np.empty((self.m, self.m)) if copy_out else None
        if G is not None:
            G = np.ascontiguousarray(G, dtype=np.float64)
            b = np.ascontiguousarray(b, dtype=np.float64)
        self._check(self._lib.sgp_magic(self._h, N.ptr(G) if G is not None else None,
                                        N.ptr(b) if b is not None else None,
                                        N.ptr(mv) if copy_out else None, N.ptr(mm) if copy_out else None))
        return mv, mm

    # ---- predict --------------------------------------------------------------------------------------
    def set_magic(self, vector, matrix):
        """Installs a caller-supplied (vector, matrix) for `predict`:  mean = k.v,  var = selfKernel + k M k^T
        (the per-point quadratic forms of the greedy active-set provider, ActiveSetProvider.scala:109-113)."""
        v = np.ascontiguousarray(vector, dtype=np.float64)
        M = np.ascontiguousarray(matrix, dtype=np.float64)
        if v.shape != (self.m,) or M.shape != (self.m, self.m):
            raise ValueError("set_magic: vector must be m, matrix m x m")
        self._check(self._lib.sgp_set_magic(self._h, N.ptr(v), N.ptr(M)))

    def predict(self, X, with_variance: bool = True):
        X = np.ascontiguousarray(X, dtype=np.float64)
        if X.ndim == 1:
            X = X[None, :]
        mean = np.empty(len(X))
        var = np.empty(len(X)) if with_variance else None
        self._check(self._lib.sgp_predict(self._h, N.ptr(X), len(X), N.ptr(mean),
                                          N.ptr(var) if with_variance else None))
        return mean, var

    def predict_device(self, x_ptr: int, x_is_f32: bool, n: int, mean_ptr: int, var_ptr: int = 0):
        """`sgp_predict_device` on device pointers (var_ptr 0: mean only); asynchronous on the context's stream (`sync`)."""
        self._check(self._lib.sgp_predict_device(self._h, C.c_void_p(x_ptr), int(x_is_f32), n, C.c_void_p(mean_ptr),
                                                 C.c_void_p(var_ptr) if var_ptr else None))

    def predict_tensor(self, X, with_variance: bool = True):
        """`predict` for a CUDA torch tensor on this context's device (n x d or d; float32 is read as it is, other dtypes
        are converted to float64): (mean, var or None) as CUDA float64 tensors of n entries, without a host round trip."""
        import torch
        X = device_tensor(X, self._device, "predict")       # X may still be written on torch's stream
        if X.ndim == 1:
            X = X[None, :]
        if X.ndim != 2 or X.shape[1] != self.d:
            raise ValueError("predict: features must be n x %d" % self.d)
        n = X.shape[0]
        mean = torch.empty(n, dtype=torch.float64, device=X.device)
        var = torch.empty(n, dtype=torch.float64, device=X.device) if with_variance else None
        self.predict_device(X.data_ptr(), X.dtype == torch.float32, n, mean.data_ptr(),
                            var.data_ptr() if var is not None else 0)
        self.sync()
        return mean, var

    def predict_probability(self, X, nodes: int = 100, with_mean_var: bool = False):
        """`sgp_predict_probability`: (p, mean, var) for n x d or d host features, p the probability of class 1 averaged
        over the latent posterior N(mean, var) with the `nodes`-node Gauss-Hermite rule (GPML eq. 3.25, as
        commons/util/Integrator.scala computes it, a negative variance taken as 0); mean and var are those of `predict`,
        bit for bit, or None unless with_mean_var."""
        X = np.ascontiguousarray(X, dtype=np.float64)
        if X.ndim == 1:
            X = X[None, :]
        p = np.empty(len(X))
        mean, var = (np.empty(len(X)), np.empty(len(X))) if with_mean_var else (None, None)
        self._check(self._lib.sgp_predict_probability(self._h, N.ptr(X), len(X), int(nodes), N.ptr(p),
                                                      N.ptr(mean) if with_mean_var else None,
                                                      N.ptr(var) if with_mean_var else None))
        return p, mean, var

    def predict_probability_device(self, x_ptr: int, x_is_f32: bool, n: int, nodes: int, p_ptr: int, mean_ptr: int = 0,
                                   var_ptr: int = 0):
        """`sgp_predict_probability_device` on device pointers (mean_ptr, var_ptr 0: not returned); asynchronous on the
        context's stream (`sync`)."""
        self._check(self._lib.sgp_predict_probability_device(
            self._h, C.c_void_p(x_ptr), int(x_is_f32), n, int(nodes), C.c_void_p(p_ptr),
            C.c_void_p(mean_ptr) if mean_ptr else None, C.c_void_p(var_ptr) if var_ptr else None))

    def predict_probability_tensor(self, X, nodes: int = 100, with_mean_var: bool = False):
        """`predict_probability` for a CUDA torch tensor on this context's device (n x d or d; float32 is read as it is,
        other dtypes are converted to float64): (p, mean, var) as CUDA float64 tensors of n entries (mean and var None
        unless with_mean_var), without a host round trip."""
        import torch
        X = device_tensor(X, self._device, "predict_probability")
        if X.ndim == 1:
            X = X[None, :]
        if X.ndim != 2 or X.shape[1] != self.d:
            raise ValueError("predict_probability: features must be n x %d" % self.d)
        n = X.shape[0]
        new = lambda: torch.empty(n, dtype=torch.float64, device=X.device)
        p = new()
        mean, var = (new(), new()) if with_mean_var else (None, None)
        self.predict_probability_device(X.data_ptr(), X.dtype == torch.float32, n, nodes, p.data_ptr(),
                                        mean.data_ptr() if with_mean_var else 0, var.data_ptr() if with_mean_var else 0)
        self.sync()
        return p, mean, var

    @staticmethod
    def gauss_hermite_rule(n: int):
        """`sgp_gauss_hermite_rule`: the n-node Gauss-Hermite (nodes, weights) for the weight exp(-x^2), 1 <= n <= 256."""
        lib = N.load()
        x, w = np.empty(max(n, 0)), np.empty(max(n, 0))
        if lib.sgp_gauss_hermite_rule(int(n), N.ptr(x), N.ptr(w)) != N.SGP_OK:
            raise ValueError(lib.sgp_last_error(None).decode())
        return x, w

    def cross_kernel(self, X):
        """kernel.crossKernel(test) with the active set as training vectors: len(test) x m."""
        X = np.ascontiguousarray(X, dtype=np.float64)
        if X.ndim == 1:
            X = X[None, :]
        K = np.empty((len(X), self.m))
        self._check(self._lib.sgp_cross_kernel(self._h, N.ptr(X), len(X), N.ptr(K)))
        return K

    def kernel_eval(self, kernel: Kernel, A, B=None, derivatives: bool = False):
        """The kernel's matrix on the given vectors (`sgp_kernel_eval`; `sgp_kernel_eval_device` for CUDA tensors on this
        context's device, read in place): crossKernel K = k(A, B) (n x m), or with B None the training kernel k(A, A)
        with the Eye terms on the diagonal.  Returns (K, dK): dK [n_hypers x n x m] in kernel.getHyperparameters() order
        with derivatives, else None.  A may be float32; B is read as float64.  Host arrays give numpy arrays, CUDA
        tensors CUDA float64 tensors."""
        on_device = is_cuda_tensor(A)
        if on_device:
            import torch
            A = device_tensor(A, self._device, "kernel_eval")
            B = None if B is None else device_tensor(B, self._device, "kernel_eval", torch.float64)
            f32 = int(A.dtype == torch.float32)
        else:
            A = _rows(A)
            B = None if B is None else np.ascontiguousarray(B, dtype=np.float64)
            f32 = int(A.dtype == np.float32)
        if A.ndim != 2 or (B is not None and (B.ndim != 2 or B.shape[1] != A.shape[1])):
            raise ValueError("kernel_eval: A must be n x d and B m x d")
        n, d = A.shape
        m = n if B is None else B.shape[0]
        desc, arr, nh, keep = self._descriptors(kernel, d)
        mode = N.SGP_KEVAL_TRAINING if B is None else N.SGP_KEVAL_CROSS
        shape_dk = (nh if derivatives else 0, n, m)
        if on_device:
            K = torch.empty((n, m), dtype=torch.float64, device=A.device)
            dK = torch.empty(shape_dk, dtype=torch.float64, device=A.device)
            ptr = lambda t: C.c_void_p(t.data_ptr())
            fn = self._lib.sgp_kernel_eval_device
        else:
            K, dK = np.empty((n, m)), np.empty(shape_dk)
            ptr, fn = N.ptr, self._lib.sgp_kernel_eval
        self._check(fn(self._h, C.byref(desc), arr, nh, ptr(A), f32, n, None if B is None else ptr(B), m, d, mode, ptr(K),
                       ptr(dK) if shape_dk[0] > 0 else None))
        if on_device:
            self.sync()
        del keep
        return K, (dK if derivatives else None)

    def greedy_active_set(self, kernel: Kernel, X, y, n_experts: int, first_index: int, m_target: int):
        """Row indices of the points GreedilyOptimizingActiveSetProvider selects (ActiveSetProvider.scala:58-139), computed
        with rank-1 updates on the device (`sgp_greedy_active_set`): O(n m) per round instead of a statistics pass.  A
        CUDA tensor X (and y) is converted to float64 on the device and read in place (`sgp_greedy_active_set_device`)."""
        if is_cuda_tensor(X):
            import torch
            X = device_tensor(X, self._device, "greedy_active_set", torch.float64)
            y = device_tensor(y, self._device, "greedy_active_set", torch.float64)
            px, py, fn = C.c_void_p(X.data_ptr()), C.c_void_p(y.data_ptr()), self._lib.sgp_greedy_active_set_device
        else:
            X = np.ascontiguousarray(X, dtype=np.float64)
            y = np.ascontiguousarray(y, dtype=np.float64)
            px, py, fn = N.ptr(X), N.ptr(y), self._lib.sgp_greedy_active_set
        desc, keep = _make_desc(kernel, X.shape[1])
        idx = np.empty(int(m_target), dtype=np.int64)
        self._check(fn(self._h, C.byref(desc), px, py, len(X), X.shape[1], int(n_experts), int(first_index),
                       int(m_target), N.ptr(idx)))
        del keep
        return idx

    def kmeans(self, X, k: int, max_iter: int = 20, tol: float = 1e-4, seed: int = 0, init_centers=None):
        """Spark 3.1 MLlib KMeans (k-means|| seeding, Lloyd iterations) on the device (`sgp_kmeans`): returns
        (centres [k_out x d] fp64, labels [n] int32, iterations, cost).  X: n x d, float32 (used without a copy) or
        float64.  init_centers (k x d) replaces the seeding, as mllib's setInitialModel.  A CUDA tensor X is read in place
        (`sgp_kmeans_device`): the same outputs, bit for bit."""
        if is_cuda_tensor(X):
            import torch
            X = device_tensor(X, self._device, "kmeans")
            px, f32, fn = C.c_void_p(X.data_ptr()), int(X.dtype == torch.float32), self._lib.sgp_kmeans_device
        else:
            X = _rows(X)
            px, f32, fn = N.ptr(X), int(X.dtype == np.float32), self._lib.sgp_kmeans
        if X.ndim != 2:
            raise ValueError("X must be n x d")
        n, d = X.shape
        k = int(k)
        init = None
        if init_centers is not None:
            init = np.ascontiguousarray(init_centers, dtype=np.float64)
            if init.shape != (k, d):
                raise ValueError("init_centers must be k x d")
        centres = np.empty((max(k, 1), max(d, 1)))
        labels = np.empty(max(n, 1), dtype=np.int32)
        k_out, iters, cost = C.c_int32(), C.c_int32(), C.c_double()
        seed = C.c_int64(int(seed) & 0xFFFFFFFFFFFFFFFF).value
        self._check(fn(self._h, px, f32, n, d, k, int(max_iter), float(tol), seed, N.ptr(init) if init is not None else None,
                       N.ptr(centres), C.byref(k_out), N.ptr(labels), C.byref(iters), C.byref(cost)))
        return np.ascontiguousarray(centres[:k_out.value]), labels[:n], iters.value, cost.value

    def kmeans_sharded(self, X, offset: int, n_total: int, k: int, max_iter: int = 20, tol: float = 1e-4, seed: int = 0,
                       init_centers=None, d: int = None):
        """`kmeans` on the concatenation of every rank's rows over this context's communicator (`sgp_kmeans_sharded`;
        `sgp_kmeans_sharded_device` for a CUDA tensor X): this rank holds the global rows [offset, offset + len(X)) of
        n_total.  Every rank gets the same (centres, iterations, cost) and the labels of its own rows.  X may be empty
        (0 x d; give d when X has no shape)."""
        if is_cuda_tensor(X):
            import torch
            X = device_tensor(X, self._device, "kmeans_sharded")
            px, f32, fn = C.c_void_p(X.data_ptr() if len(X) else None), int(X.dtype == torch.float32), \
                self._lib.sgp_kmeans_sharded_device
        else:
            X = _rows(X)
            px, f32, fn = (N.ptr(X) if len(X) else None), int(X.dtype == np.float32), self._lib.sgp_kmeans_sharded
        if X.ndim != 2:
            raise ValueError("X must be n x d")
        n, d = len(X), int(X.shape[1] if d is None else d)
        k = int(k)
        init = None
        if init_centers is not None:
            init = np.ascontiguousarray(init_centers, dtype=np.float64)
            if init.shape != (k, d):
                raise ValueError("init_centers must be k x d")
        centres = np.empty((max(k, 1), max(d, 1)))
        labels = np.empty(max(n, 1), dtype=np.int32)
        k_out, iters, cost = C.c_int32(), C.c_int32(), C.c_double()
        seed = C.c_int64(int(seed) & 0xFFFFFFFFFFFFFFFF).value
        self._check(fn(self._h, px, f32, n, int(offset), int(n_total), d, k, int(max_iter), float(tol), seed,
                       N.ptr(init) if init is not None else None, N.ptr(centres), C.byref(k_out), N.ptr(labels),
                       C.byref(iters), C.byref(cost)))
        return np.ascontiguousarray(centres[:k_out.value]), labels[:n], iters.value, cost.value

    def column_sums(self, X, center=None):
        """fp64 sums over the rows of a CUDA tensor X (n x d, on this context's device, read in place; float32 as it is,
        other dtypes as float64) in the library's fixed order (`sgp_column_sums_device`): sum_i x_ik per column, or with
        `center` (d values) sum_i (x_ik - center_k)^2.  Returns a host array of d values."""
        import torch
        X = device_tensor(X, self._device, "column_sums")
        if X.ndim != 2:
            raise ValueError("column_sums: X must be n x d")
        n, d = X.shape
        c = None if center is None else np.ascontiguousarray(center, dtype=np.float64)
        if c is not None and c.shape != (d,):
            raise ValueError("column_sums: center must hold %d values" % d)
        out = np.empty(d)
        self._check(self._lib.sgp_column_sums_device(self._h, C.c_void_p(X.data_ptr() if n else None),
                                                     int(X.dtype == torch.float32), n, d,
                                                     N.ptr(c) if c is not None else None, N.ptr(out)))
        return out

    def scale_apply(self, X, mean, sd):
        """(x_ik - mean_k) / sd_k for a CUDA tensor X (n x d, on this context's device) as a CUDA float64 n x d tensor on
        X's device (`sgp_scale_apply_device`): every element is the host formula's on the same mean and sd."""
        import torch
        X = device_tensor(X, self._device, "scale_apply")
        if X.ndim != 2:
            raise ValueError("scale_apply: X must be n x d")
        n, d = X.shape
        mean, sd = (np.ascontiguousarray(v, dtype=np.float64) for v in (mean, sd))
        if mean.shape != (d,) or sd.shape != (d,):
            raise ValueError("scale_apply: mean and sd must hold %d values each" % d)
        Y = torch.empty((n, d), dtype=torch.float64, device=X.device)
        self._check(self._lib.sgp_scale_apply_device(self._h, C.c_void_p(X.data_ptr() if n else None),
                                                     int(X.dtype == torch.float32), n, d, N.ptr(mean), N.ptr(sd),
                                                     C.c_void_p(Y.data_ptr() if n else None)))
        self.sync()
        return Y

    def kmn_sweep(self, X):
        """fp32 K[i][j] = k(x_i, z_j) (n x m) through the tensor-core sweep kernel (one non-Eye term, d <= 32)."""
        X = _rows(X)
        K =np.empty((len(X), self.m), dtype=np.float32)
        self._check(self._lib.sgp_kmn_sweep(self._h, N.ptr(X), int(X.dtype == np.float32), len(X), N.ptr(K)))
        return K

    def kmn_sweep_device(self, x_ptr: int, x_is_f32: bool, n: int, k_ptr: int):
        self._check(self._lib.sgp_kmn_sweep_device(self._h, C.c_void_p(x_ptr), int(x_is_f32), n, C.c_void_p(k_ptr)))

    def debug_i8_tile(self):
        """Arms (first call) / reads back the SGP_PREC_I8 debug dump: (T [128x64] fp32, words [128x64] uint32)."""
        T = np.zeros((128, 64), dtype=np.float32)
        w = np.zeros((128, 64), dtype=np.uint32)
        self._check(self._lib.sgp_debug_i8_tile(self._h, N.ptr(T), N.ptr(w)))
        return T, w

    # ---- introspection ---------------------------------------------------------------------------------
    def last_path(self) -> int:
        """SGP_PREC_F64 / SGP_PREC_F64_STRICT / SGP_PREC_I8: the kernel the last statistics launch ran."""
        return int(self._lib.sgp_last_path(self._h))

    def last_bcm_path(self) -> int:
        """0: on-chip Cholesky objective kernel; 1: global-memory LU path (large experts / not positive definite)."""
        return int(self._lib.sgp_last_bcm_path(self._h))

    def last_tail_path(self) -> int:
        """1: the tail ran on Cholesky factors (PD check included); 0: the reference's dsyevd + LU sequence; -1: never ran."""
        return int(self._lib.sgp_last_tail_path(self._h))

    def launch_count(self) -> int:
        return int(self._lib.sgp_launch_count(self._h))

    def event_record(self, slot: int):
        self._check(self._lib.sgp_event_record(self._h, slot))

    def event_elapsed_ms(self, a: int, b: int) -> float:
        ms = C.c_double()
        self._check(self._lib.sgp_event_elapsed_ms(self._h, a, b, C.byref(ms)))
        return ms.value

    def gram_kernel_time(self):
        ms = C.c_double()
        n = C.c_int64()
        self._check(self._lib.sgp_gram_kernel_time(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value
