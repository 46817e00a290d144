"""Data-parallel `fit` of `GaussianProcessRegression`, the binary `GaussianProcessClassifier` and `OneVsRest` over a
torch.distributed process group: one process per GPU, each passing its own shard, every rank returning the model of the
concatenation of the shards in rank order (DESIGN.md section 5).

The reference's cluster steps, one by one:
  * `groupForExperts` (GPC:26-31): E = round(N / datasetSizeForExpert) over all N rows, expert e holds the global rows
    e, e + E, ...  Rank r owns the experts [r E // R, (r + 1) E // R); every row moves to its expert's owner in one
    all-to-all, and the rows a rank receives, in global row order, are grouped on its device row i -> expert i % E_r
    (`sgp_experts_upload_strided_device`), which makes each expert the single-GPU upload's, row for row.
  * `optimizeHypers` (GPC:66-92): every rank runs the same L-BFGS-B on the reducing objective entries
    (`sgp_bcm_nll`, `sgp_laplace_nll_any_size`, and for one-vs-rest `sgp_laplace_nll_classes_any_size` over the classes
    in lock step), which all-reduce [value; gradient] and the status words, so every rank sees the same bits and takes
    the same steps.  The classifiers' latent modes stay with their expert's owner.
  * `getMatrixKmnKnmAndVectorKmny` (PGPH:20-36): each rank accumulates its rows -- the regression its own shard, the
    classifiers their experts' rows with each slot's modes as labels -- and `sgp_stats_finish` all-reduces G and b and
    the int8 status, so AUTO's fall-back to fp64 is taken on every rank together.

A rank that returns before a collective leaves its peers blocked in it.  So before the first collective every rank
states the refusals it can compute (its data, the global sizes), the ranks exchange them, and if any rank would refuse,
every rank raises the same exception.  The SGP_E_NOMEM checks depend on each rank's free memory and are not agreed.

The model selectors over a group (`selection`, `Selection`) reuse these steps with several training sets: one
`ShardPlan` per set, one all-to-all that moves each row once per set it belongs to (`exchange_sets`), and one gather of
the ranks' validation labels and predictions, so that every rank scores the same arrays.

`scale` standardises every rank's shard with the mean and standard deviation of the concatenation: two all-reduces of
d + 1 and d values after the agreement, no rows moved.

`engine_factory` is the context class (a test passes a stand-in)."""
from __future__ import annotations

import numpy as np

from . import _native as N
from .engine import ProjectedProcessEngine, is_cuda_tensor, rows_to_host
from .hyperopt import each, fit_data, fit_slots, optimize_hypers, own_context, produce, slot_modes, slot_objective

# per-expert point limits of the library: the BCM LU path (sgp_bcm_nll) and the global-memory Laplace kernel
BCM_MAX_EXPERT_POINTS = 46340
LAPLACE_MAX_EXPERT_POINTS = 46336

_EXCEPTIONS = {e.__name__: e for e in (ValueError, RuntimeError, TypeError, ZeroDivisionError)}


class ShardPlan:
    """Where every row and expert lives, from the ranks' shard sizes in rank order (the same on every rank)."""

    def __init__(self, sizes, rank: int, dataset_size_for_expert: int):
        self.sizes = np.asarray(sizes, dtype=np.int64)
        self.R, self.rank = len(self.sizes), int(rank)
        self.offsets = np.concatenate([[0], np.cumsum(self.sizes)]).astype(np.int64)
        self.N = int(self.offsets[-1])
        self.E = int(np.floor(self.N / dataset_size_for_expert + 0.5))       # Math.round(N / n_e), GPC:27
        # rank r owns the experts [first[r], first[r + 1])
        self.first = np.array([r * self.E // self.R for r in range(self.R + 1)], dtype=np.int64)

    @property
    def offset(self) -> int:
        return int(self.offsets[self.rank])

    @property
    def local_experts(self) -> int:
        return int(self.first[self.rank + 1] - self.first[self.rank])

    def owner(self, rows):
        """The rank owning each global row's expert."""
        return np.searchsorted(self.first, np.asarray(rows) % self.E, side="right") - 1

    def destinations(self, r: int = None):
        """The destination rank of each row of rank r's shard (default: this rank)."""
        r = self.rank if r is None else r
        return self.owner(np.arange(self.offsets[r], self.offsets[r + 1]))

    def send_counts(self):
        return np.bincount(self.destinations(), minlength=self.R).astype(np.int64)

    def recv_counts(self):
        return np.array([int((self.destinations(s) == self.rank).sum()) for s in range(self.R)], dtype=np.int64)

    def expert_rows(self):
        """The global rows this rank receives, in the order it receives them (global row order)."""
        e0, e1 = self.first[self.rank], self.first[self.rank + 1]
        g = np.arange(self.N)
        return g[(g % self.E >= e0) & (g % self.E < e1)]

    def local_order(self):
        """The expert-major order of the received rows (expert e0 + q holds rows q, q + E_r, ...): the permutation the
        strided upload applies."""
        n, E = int(self.recv_counts().sum()), self.local_experts
        return np.concatenate([np.arange(q, n, E) for q in range(E)]) if E > 0 else np.arange(0)


def _dist():
    import torch.distributed as dist
    return dist


def group_refusal(plan: ShardPlan, infos, classifier: bool, experts: bool):
    """The refusal every rank takes, from every rank's agreement entry (n, d, dtype, local refusal[, largest label]) and
    the plan, or None: the first rank's own refusal, then a disagreement of the ranks' shapes or dtypes, then the expert
    grouping's limits (only when the fit groups experts).  Returns (exception class name, message)."""
    for r, info in enumerate(infos):
        if info[3] is not None:
            return info[3][0], "rank %d: %s" % (r, info[3][1])
    ds = sorted({i[1] for i in infos if i[0] > 0} or {infos[0][1]})
    if len(ds) > 1:
        return "ValueError", "the ranks' shards have different numbers of features: %s" % ds
    dtypes = sorted({i[2] for i in infos if i[0] > 0})
    if len(dtypes) > 1:
        return "ValueError", "the ranks' shards have different dtypes: %s" % ", ".join(dtypes)
    if plan.N == 0:
        return "ValueError", "every rank's shard is empty"
    if not experts:
        return None
    return expert_refusal(plan, classifier)


def expert_refusal(plan: ShardPlan, classifier: bool):
    """The expert grouping's limits over the plan's ranks, or None: no expert, fewer experts than ranks, or an expert above
    the BCM / Laplace point limit.  Returns (exception class name, message)."""
    if plan.E <= 0:
        return "ZeroDivisionError", "numberOfExperts == 0 (N < datasetSizeForExpert / 2)"
    if plan.E < plan.R:
        return "ValueError", ("%d experts for %d ranks: every rank needs at least one expert (lower datasetSizeForExpert "
                              "or use fewer ranks)" % (plan.E, plan.R))
    largest = -(-plan.N // plan.E)
    limit = LAPLACE_MAX_EXPERT_POINTS if classifier else BCM_MAX_EXPERT_POINTS
    if largest > limit:
        return "ValueError", "datasetSizeForExpert above %d: the largest expert holds %d points" % (limit, largest)
    return None


def num_classes(infos):
    """One-vs-rest's numClasses of the concatenation from every rank's agreement entry: one more than the largest label
    of any rank (an empty shard, or a fit without class labels, sends -1)."""
    return max(i[4] for i in infos) + 1


def agree(group, n: int, d: int, dtype: str, err, dataset_size_for_expert: int, classifier: bool, experts: bool,
          top: int = -1):
    """The agreement step, the fit's first collective: every rank's (n, d, dtype, refusal, largest label top) to every
    rank.  Raises the agreed refusal on every rank; else returns (the plan, the agreed dtype, the agreed number of
    features: those of the non-empty shards, which an empty shard takes whatever its own shape, `num_classes`)."""
    dist = _dist()
    infos = [None] * dist.get_world_size(group)
    dist.all_gather_object(infos, (int(n), int(d), str(dtype), err, int(top)), group=group)
    plan = ShardPlan([i[0] for i in infos], dist.get_rank(group), dataset_size_for_expert)
    verdict = group_refusal(plan, infos, classifier, experts)
    if verdict is not None:
        raise _EXCEPTIONS.get(verdict[0], RuntimeError)(verdict[1])
    first = next(i for i in infos if i[0] > 0)
    return plan, first[2], first[1], num_classes(infos)


def exchange(plan: ShardPlan, X, y, group):
    """Moves every row of the shard (torch tensors X n x d, y n, on the group's device) to its expert's owner in one
    all-to-all of the rows' bytes with y appended.  Returns (X, y) of the rows this rank owns, in global row order."""
    return exchange_sets([plan], [None], X, y, group)[:2]


def exchange_sets(plans, members, X, y, group):
    """`exchange` of several training sets in one all-to-all: set k holds this rank's rows where the host bool mask
    members[k] is set (None: every row), in row order, and plans[k] is its `ShardPlan` over the ranks' rows of the set.
    A row moves once per set it belongs to, to the owner of its expert in that set.  Each rank sends its rows ordered by
    (destination, set, row) and orders what it receives by (set, source rank, row): global row order within each set.
    Returns (X, y, rows): the rows this rank owns, set after set, and rows[k], the size of set k's block."""
    import torch
    dist = _dist()
    d, es = X.shape[1], X.element_size()
    R, S = plans[0].R, len(plans)
    local = [np.arange(len(X)) if m is None else np.flatnonzero(m) for m in members]
    dest = np.concatenate([p.destinations() for p in plans]).astype(np.int64)
    setof = np.concatenate([np.full(len(i), k, dtype=np.int64) for k, i in enumerate(local)])
    order = np.argsort(dest * S + setof, kind="stable")
    src = torch.as_tensor(np.concatenate(local)[order], device=X.device)
    rows = torch.empty((0, d * es + 8), dtype=torch.uint8, device=X.device)
    if len(src):
        rows = torch.cat([X.contiguous().view(torch.uint8).reshape(len(X), d * es),
                          y.reshape(len(y), 1).to(torch.float64).view(torch.uint8)], dim=1)[src].contiguous()
    send = np.bincount(dest, minlength=R).astype(np.int64)
    # counts[s, k]: the rows of set k that rank s sends here
    counts = np.array([[int((p.destinations(s) == p.rank).sum()) for p in plans] for s in range(R)], dtype=np.int64)
    recv = counts.sum(axis=1)
    out = torch.empty((int(recv.sum()), d * es + 8), dtype=torch.uint8, device=X.device)
    dist.all_to_all_single(out, rows, recv.tolist(), send.tolist(), group=group)
    if S > 1 and len(out):
        at = np.concatenate([[0], np.cumsum(counts.ravel())]).reshape(-1)[:-1].reshape(R, S)
        out = out[torch.as_tensor(np.concatenate([np.arange(at[s, k], at[s, k] + counts[s, k])
                                                  for k in range(S) for s in range(R)]), device=X.device)]
    set_rows = counts.sum(axis=0)
    if len(out) == 0:
        return X.new_empty((0, d)), y.new_empty(0, dtype=torch.float64), set_rows
    Xr = out[:, :d * es].contiguous().view(X.dtype).reshape(len(out), d)
    yr = out[:, d * es:].contiguous().view(torch.float64).reshape(len(out))
    return Xr, yr, set_rows


def gather_rows(plan: ShardPlan, X, idx, group, device):
    """The global rows idx of the concatenation as a float64 host array on every rank: the owners contribute the rows
    (`rows_to_host`, the single-GPU provider's conversion) and the rows' bit patterns are summed as int64 (exact: every
    other rank adds zero)."""
    import torch
    dist = _dist()
    idx = np.asarray(idx, dtype=np.int64)
    lo, hi = plan.offset, plan.offset + int(plan.sizes[plan.rank])
    mine = (idx >= lo) & (idx < hi)
    out = np.zeros((len(idx), X.shape[1]), dtype=np.int64)
    if mine.any():
        out[mine] = np.ascontiguousarray(rows_to_host(X, idx[mine] - lo)).view(np.int64)
    t = torch.as_tensor(out, device=device)
    dist.all_reduce(t, group=group)
    return t.cpu().numpy().view(np.float64)


def active_set(gp, plan: ShardPlan, eng, X, theta, group, device):
    """The active set of the concatenation, the same on every rank: the random provider's single-GPU draw over N
    (gathered from the owners), the explicit provider's rows, or the sharded GPU K-means."""
    from .regression import KMeansActiveSetProvider, _RandomActiveSetProvider
    provider = gp._activeSetProvider
    if type(provider) is _RandomActiveSetProvider:
        rng = np.random.default_rng(gp._seed)
        idx = rng.choice(plan.N, size=min(gp._activeSetSize, plan.N), replace=False)
        return gather_rows(plan, X, idx, group, device)
    if type(provider) is KMeansActiveSetProvider:
        centres, _, _, _ = eng.kmeans_sharded(X, plan.offset, plan.N, int(gp._activeSetSize), max_iter=provider.maxIter,
                                              tol=1e-4, seed=int(gp._seed), d=X.shape[1])
        return centres
    return provider(gp._activeSetSize, X, None, gp.getKernel, theta, gp._seed, gp=gp)


def check_provider(provider):
    """ValueError for a provider that cannot run over a process group (its configuration is the same on every rank, so
    every rank raises, before any collective).  Only the three classes themselves are accepted, not subclasses: a
    provider called on one rank's shard could give every rank a different active set, and the all-reduced statistics
    would then sum over different active sets."""
    from .regression import ExplicitActiveSetProvider, KMeansActiveSetProvider, _RandomActiveSetProvider
    if type(provider) is KMeansActiveSetProvider and not provider.on_gpu:
        raise ValueError("a fit over a process group needs KMeansActiveSetProvider(on_gpu=True): scikit-learn's K-means "
                         "runs on one host's points")
    if type(provider) not in (_RandomActiveSetProvider, ExplicitActiveSetProvider, KMeansActiveSetProvider):
        raise ValueError("%s cannot run over a process group: use the random, explicit or GPU K-means provider"
                         % type(provider).__name__)


# One context with a communicator per (member ranks, device, context class), kept for the process's lifetime: the fits
# over a group reuse it instead of making a communicator each (the models get contexts of their own).  Every rank of
# the group makes the same sequence of fits, so every rank finds or makes its entry at the same fit.
_COMM_ENGINES = {}


def comm_engine(group, device_index: int, device, engine_factory):
    """The group's context with a communicator on device_index, made (and its communicator attached) at first use."""
    dist = _dist()
    key = (tuple(dist.get_process_group_ranks(group)), device_index, engine_factory)
    eng = _COMM_ENGINES.get(key)
    if eng is None:
        eng = engine_factory(device_index)
        try:
            attach_communicator(eng, group, device)
        except BaseException:
            eng.close()
            raise
        _COMM_ENGINES[key] = eng
    return key, eng


def attach_communicator(eng, group, device):
    """One NCCL communicator of the group's ranks on eng: rank 0 makes the id, the group broadcasts it."""
    dist = _dist()
    obj = [eng.comm_unique_id() if dist.get_rank(group) == 0 else None]
    dist.broadcast_object_list(obj, src=dist.get_global_rank(group, 0), group=group, device=device)
    eng.comm_init(obj[0], dist.get_rank(group), dist.get_world_size(group))


def _local_data(X, y, device: int, kind: str, what: str):
    """The shard as the single-GPU fit reads it (`fit_data`), with the labels checked for the classifiers.  Returns (X, y,
    the largest label: one-vs-rest's, -1 for an empty shard and for the other fits)."""
    X, y = fit_data(X, y, device, what, keep_float32=kind == "regression")
    if X.ndim != 2 or y.ndim != 1 or len(y) != len(X):
        raise ValueError("%s: X must be n x d and y n entries" % what)
    top = -1
    if kind == "binary":
        from .classification import assert_labels_are_01
        assert_labels_are_01(y)
    elif kind == "classes" and len(y):
        from .classification import one_vs_rest_labels
        y, top = one_vs_rest_labels(y)
        top -= 1
    return X, y, top


def _tensor(a, device, dtype=None):
    import torch
    t = a if is_cuda_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
    t = t.to(device)
    return t if dtype is None else t.to(dtype)


def fit(gp, X, y, hyperparameters, classifier: bool, engine_factory=ProjectedProcessEngine):
    """The data-parallel fit of gp (a GaussianProcessRegression or binary GaussianProcessClassifier with a process
    group) on this rank's shard (`group_fit`).  Returns the model's `Fitted` slot."""
    models, record = group_fit(gp, X, y, hyperparameters, "binary" if classifier else "regression", engine_factory)
    if record is not None and record["slots"] is not None:
        gp.last_objective = dict(record["slots"][0], launches=record["launches"])
    return models[0]


def group_fit(gp, X, y, hyperparameters, kind: str, engine_factory=ProjectedProcessEngine):
    """The data-parallel fit over gp's process group on this rank's shard.  kind: "regression", "binary" (gp a binary
    GaussianProcessClassifier) or "classes" (one-vs-rest over gp: y holds class indices, numClasses agreed by the ranks,
    and hyperparameters, if given, numClasses x n_hypers).  The fit runs on the group's context with a communicator
    (`comm_engine`); each model gets a context of its own holding its active set and magic pair (`own_context`).
    Returns (per slot -- the one model, or one per class -- its `Fitted` value, with the latent modes of this rank's
    expert rows for the classifiers, the Laplace fit record of `fit_slots` or None for the regression).  Fits over one group must
    not run concurrently."""
    import contextlib

    import torch
    dist = _dist()
    group = gp._process_group
    what = "OneVsRest.fit" if kind == "classes" else "%s.fit" % type(gp).__name__
    classifier = kind != "regression"
    check_provider(gp._activeSetProvider)
    nccl = dist.get_backend(group) == "nccl"
    device = torch.device("cuda", gp._device) if nccl else torch.device("cpu")
    with torch.cuda.device(gp._device) if nccl else contextlib.nullcontext():
        experts = classifier or (hyperparameters is None and gp._maxIter > 0)
        err, n, d, dtype, top = None, 0, -1, "", -1
        try:
            X, y, top = _local_data(X, y, gp._device, kind, what)
            n, d, dtype = len(X), X.shape[1], str(X.dtype).replace("torch.", "")
        except (ValueError, TypeError, RuntimeError) as e:
            err = (type(e).__name__, str(e))
        plan, dtype, d, n_classes = agree(group, n, d, dtype, err, gp._datasetSizeForExpert, classifier, experts, top)
        if len(X) == 0:                                     # an empty shard takes the agreed dtype and width
            X = np.empty((0, d), dtype=np.float32 if dtype == "float32" else np.float64)
            y = np.empty(0)
        key, eng = comm_engine(group, gp._device, device, engine_factory)
        try:
            slots, record = _fit(gp, plan, eng, X, y, hyperparameters, kind, n_classes, dtype, group, device)
        except BaseException:
            # a failure after a collective may leave the ranks out of step: the communicator is not reused
            _COMM_ENGINES.pop(key, None)
            eng.close()
            raise
        return [own_context(fitted, gp._device, engine_factory) for fitted in slots], record


def _fit(gp, plan, eng, X, y, hyperparameters, kind, n_classes, dtype, group, device):
    """The fit on the group's context: each slot's `Fitted` value and the Laplace fit record.  Each slot's
    model has the active set of the concatenation and the statistics all-reduced over the group: of this rank's shard
    for the regression, of its expert rows with the slot's modes as labels for the classifiers."""
    import torch
    eng.set_precision(N.SGP_PREC_AUTO)                      # as on a freshly acquired context
    exchanged = lambda: exchange(plan, _tensor(X, device, getattr(torch, dtype)), _tensor(y, device, torch.float64), group)
    x0 = gp.getKernel().getHyperparameters()
    if kind == "regression":
        if hyperparameters is not None:
            theta = hyperparameters
        elif gp._maxIter > 0:
            Xe, ye = exchanged()
            eng.experts_upload_strided(Xe, ye, plan.local_experts)
            theta = optimize_hypers(gp, eng, plan.E)
        else:
            theta = x0
        theta = np.asarray(theta, dtype=np.float64)
        return [produce(gp, eng, X, y, theta, active_set(gp, plan, eng, X, theta, group, device))], None
    # the Laplace fit of one slot (the binary classifier) or of every class (one-vs-rest), as `laplace_fit` on one GPU
    if kind == "binary":
        store, n_slots, entry = N.SGP_MODES_BINARY, 1, each(lambda k: eng.laplace_nll_any_size(k, gp._tol))
        given = None if hyperparameters is None else [np.asarray(hyperparameters, dtype=np.float64)]
    else:
        store, n_slots = N.SGP_MODES_CLASS, n_classes
        entry = lambda classes, kernels: eng.laplace_nll_classes_any_size(n_classes, classes, kernels, gp._tol)
        given = None if hyperparameters is None else \
            np.array(hyperparameters, dtype=np.float64).reshape(n_classes, len(x0))
    Xe, ye = exchanged()
    eng.experts_upload_strided(Xe, ye, plan.local_experts)
    thetas, record = fit_slots(eng, gp, slot_objective([gp] * n_slots, entry), [x0] * n_slots, given, laplace=True)
    n_e = len(Xe)
    if not is_cuda_tensor(X):
        Xe = Xe.cpu().numpy()
    slots = []
    for i, theta in enumerate(thetas):
        f = slot_modes(eng, is_cuda_tensor(X), n_e, plan.local_experts, store, i)
        slots.append(produce(gp, eng, Xe, f, theta, active_set(gp, plan, eng, X, theta, group, device))._replace(latent=f))
    return slots, record


# ---- feature scaling over the group (`utils.scale` with a process group) --------------------------------------------
def scale(X, group, engine_factory=ProjectedProcessEngine.acquire):
    """`utils.scale` of this rank's shard X (a host array or a CUDA tensor, n x d, possibly empty) with the mean and
    standard deviation of the concatenation of every rank's shard, as the reference's `reduce`s over the whole RDD give
    them.  The agreement step comes first (as `agree`: the number of features, the dtype and every rank's own refusal;
    every rank raises the same exception, before any context exists, also when every shard is empty).  Then every rank
    sums its column-sum partials [S; n] over the group in one all-reduce, computes the same mean, and sums its centred
    squares Q in a second one (`utils.moments`).  No rows move.  Each rank returns its own rows scaled: a CUDA float64
    tensor for a CUDA shard, a host float64 array for a host shard (staged through the rank's current CUDA device)."""
    import contextlib

    import torch

    from .utils import moments
    dist = _dist()
    on_device = is_cuda_tensor(X)
    index = X.device.index if on_device else (torch.cuda.current_device() if torch.cuda.is_available() else 0)
    nccl = dist.get_backend(group) == "nccl"
    device = torch.device("cuda", index) if nccl else torch.device("cpu")
    with torch.cuda.device(index) if nccl else contextlib.nullcontext():
        err, n, d, dtype = None, 0, -1, ""
        try:
            if not on_device:
                X = np.asarray(X)
                X = np.ascontiguousarray(X if X.dtype == np.float32 else X.astype(np.float64))
            if X.ndim != 2:
                raise ValueError("scale: X must be n x d")
            n, d, dtype = len(X), X.shape[1], str(X.dtype).replace("torch.", "")
        except (ValueError, TypeError, RuntimeError) as e:
            err = (type(e).__name__, str(e))
        d = agree(group, n, d, dtype, err, 1, False, False)[2]
        if len(X) == 0:                                     # an empty shard takes the agreed width
            X = torch.empty((0, d), dtype=torch.float64, device=X.device) if on_device else np.empty((0, d))
        Xd = X if on_device else _tensor(X, torch.device("cuda", index) if torch.cuda.is_available() else "cpu")

        def total(v):
            t = torch.as_tensor(v, dtype=torch.float64, device=device)
            dist.all_reduce(t, group=group)
            return t.cpu().numpy()

        eng = engine_factory(index)
        try:
            mean, sd = moments(eng, Xd, total)
            Y = eng.scale_apply(Xd, mean, sd)
        finally:
            eng.release()
        return Y if on_device else Y.cpu().numpy()


# ---- model selection over the group (`tuning.CrossValidator` / `TrainValidationSplit` with a process group) ----------
def set_refusal(N: int, sizes, n_es, classifier: bool, validation):
    """The refusal of a selection's training sets over N rows from every rank's rows in every set (sizes, R x n_sets), or
    None: validation(N, N_k per set) names an empty validation side (the plain selector's message, or None), then for
    every datasetSizeForExpert in n_es (the maps whose fit groups experts) and every set, `expert_refusal` of the set's
    plan, named by set.  Returns (exception class name, message)."""
    sizes = np.asarray(sizes, dtype=np.int64)
    message = validation(int(N), sizes.sum(axis=0))
    if message is not None:
        return "ValueError", message
    for n_e in sorted(set(n_es)):
        for k in range(sizes.shape[1]):
            verdict = expert_refusal(ShardPlan(sizes[:, k], 0, n_e), classifier)
            if verdict is not None:
                return verdict[0], "training set %d: %s" % (k, verdict[1])
    return None


def selection_refusal(infos, classifier: bool, n_es, validation):
    """The refusal of a model selection over the group from every rank's entry (n, d, dtype, refusal, largest label, rows
    per set, largest label per set), or None: `group_refusal` without experts, then `set_refusal`."""
    plan = ShardPlan([i[0] for i in infos], 0, 1)
    verdict = group_refusal(plan, infos, classifier, False)
    if verdict is None:
        verdict = set_refusal(plan.N, [i[5] for i in infos], n_es, classifier, validation)
    return verdict


class Selection:
    """A model selection's side of the group, for the selectors' drivers (`tuning`): the group's context with a
    communicator, this rank's rows of every training set (members[k], a host bool mask of its shard) and every rank's
    count of them (sizes, R x n_sets), the sets regrouped across ranks for the slot fits, the fold models over the set
    plans, and the gathered validation arrays.  classes[k]: one-vs-rest's C_k of set k (the maximum label over ranks
    plus one)."""

    def __init__(self, group, device, eng, X, y, members, sizes, classes):
        self.group, self.device, self.eng = group, device, eng
        self.X, self.y, self.members = X, y, members
        self.sizes, self.classes = np.asarray(sizes, dtype=np.int64), classes
        self.rank = _dist().get_rank(group)
        self.on_device = is_cuda_tensor(X)
        self._blocks = {}

    def plan(self, k: int, dataset_size_for_expert: int = 1) -> ShardPlan:
        return ShardPlan(self.sizes[:, k], self.rank, dataset_size_for_expert)

    def context(self, device):
        import contextlib
        return contextlib.nullcontext(self.eng)

    def gather(self, v):
        """Every rank's v (its validation rows' labels or predictions) as one host float64 array, in rank order: global
        row order."""
        dist = _dist()
        parts = [None] * dist.get_world_size(self.group)
        dist.all_gather_object(parts, np.asarray(v.cpu().numpy() if is_cuda_tensor(v) else v, dtype=np.float64),
                               group=self.group)
        return np.concatenate(parts)

    def blocks(self, dataset_size_for_expert: int):
        """(X, y, rows, local experts) of this rank's experts of every training set (`exchange_sets`), kept per
        datasetSizeForExpert for the fold models."""
        import torch
        n_e = int(dataset_size_for_expert)
        if n_e not in self._blocks:
            plans = [self.plan(k, n_e) for k in range(len(self.members))]
            X = _tensor(self.X, self.device, getattr(torch, str(self.X.dtype).replace("torch.", "")))
            Xe, ye, rows = exchange_sets(plans, self.members, X, _tensor(self.y, self.device, torch.float64), self.group)
            self._blocks[n_e] = (Xe, ye, rows, [p.local_experts for p in plans], [p.E for p in plans])
        return self._blocks[n_e]

    def upload_sets(self, eng, dataset_size_for_expert: int):
        """Uploads this rank's experts of every training set (`experts_upload_fold_sets`).  Returns (rows, experts) per
        set."""
        Xe, ye, rows, experts, _ = self.blocks(dataset_size_for_expert)
        eng.experts_upload_fold_sets(Xe, ye, rows, experts)
        return rows, experts

    def set_classes(self, ovr: bool):
        """C_k of every training set: the agreed one-vs-rest counts, or 1 for the binary classifier (the labels were
        checked before the agreement)."""
        return list(self.classes) if ovr else [1] * len(self.members)

    def upload_training(self, eng, dataset_size_for_expert: int, Xt=None, yt=None, laplace: bool = False):
        """Uploads this rank's experts of the one training set (`experts_upload_strided`) in place of the training rows
        (Xt, yt).  Returns (rows, local experts, the set's number of experts)."""
        Xe, ye, rows, experts, E = self.blocks(dataset_size_for_expert)
        eng.experts_upload_strided(Xe, ye, experts[0])
        return int(rows[0]), experts[0], E[0]

    def validate(self, est, k: int, Xt, yt, Xv, theta):
        """The regression's fold model of set k at theta (its own set-k rows Xt, yt, the active set of the set) on the
        group's context, and its gathered validation predictions.  Returns (predictions, magic vector)."""
        fitted = produce(est, self.eng, Xt, yt, theta,
                         active_set(est, self.plan(k), self.eng, Xt, theta, self.group, self.device))
        return self.gather(self.latent_mean(self.eng, Xv)), fitted.magic_vector

    def fold_model(self, gp, eng, k: int, Xt, f, theta):
        """The classifier's model of set k at theta on the group's context: the statistics of this rank's set-k expert
        rows with the slot's modes f as labels, the active set of the set over its own set-k rows Xt."""
        Xe, _, rows, _, _ = self.blocks(gp._datasetSizeForExpert)
        lo = int(np.sum(rows[:k]))
        Xk = Xe[lo:lo + int(rows[k])]
        if not self.on_device:
            Xk = Xk.cpu().numpy()
        return produce(gp, eng, Xk, f, theta, active_set(gp, self.plan(k), eng, Xt, theta, self.group, self.device))

    @staticmethod
    def latent_mean(eng, Xv):
        """The latent mean of the model eng holds at this rank's validation rows (host float64; none on a rank without
        any)."""
        if len(Xv) == 0:
            return np.empty(0)
        if is_cuda_tensor(Xv):
            return eng.predict_tensor(Xv, with_variance=False)[0].cpu().numpy().astype(np.float64)
        return eng.predict(Xv, with_variance=False)[0]


def selection(gp, estimators, kind: str, X, y, split, what: str, validation, engine_factory=ProjectedProcessEngine):
    """The set-up of a model selection over gp's process group on this rank's shard, as a context manager yielding a
    `Selection`.  gp: the estimator with the group (the wrapped classifier of one-vs-rest); estimators: one per param map
    (their providers and datasetSizeForExpert are checked); kind as in `group_fit`.  split(n, offset) -> the host bool
    masks of the rank's rows in each training set, the rank's rows being the global rows [offset, offset + n)
    (ValueError for a bad given split).  validation(N, N_k) -> the plain selector's message for an empty validation
    side, or None.
    Two collectives come before any context: the shard sizes (the seeded splits number the rows globally), then the
    agreement, after which every rank raises the same exception for any rank's refusal.  A failure after the agreement
    drops the communicator context, as `group_fit` does."""
    import contextlib

    import torch
    dist = _dist()
    group = gp._process_group
    classifier = kind != "regression"
    nccl = dist.get_backend(group) == "nccl"
    device = torch.device("cuda", gp._device) if nccl else torch.device("cpu")
    R, rank = dist.get_world_size(group), dist.get_rank(group)
    n_es = [e._datasetSizeForExpert for e in estimators if classifier or e._maxIter > 0]

    @contextlib.contextmanager
    def run():
        with torch.cuda.device(gp._device) if nccl else contextlib.nullcontext():
            err, n, d, dtype, top, Xl, yl = None, 0, -1, "", -1, X, y
            try:
                for e in estimators:
                    check_provider(e._activeSetProvider)
                Xl, yl, top = _local_data(X, y, gp._device, kind, what)
                n, d, dtype = len(Xl), Xl.shape[1], str(Xl.dtype).replace("torch.", "")
            except (ValueError, TypeError, RuntimeError) as e:
                err = (type(e).__name__, str(e))
            counts = [None] * R
            dist.all_gather_object(counts, int(n), group=group)
            members, rows, tops = [], [], []
            if err is None:
                try:
                    members = split(n, int(sum(counts[:rank])))
                    rows = [int(np.count_nonzero(m)) for m in members]
                    yh = np.asarray(yl.cpu().numpy() if is_cuda_tensor(yl) else yl)
                    tops = [int(yh[m].max()) if kind == "classes" and m.any() else -1 for m in members]
                except ValueError as e:
                    err = (type(e).__name__, str(e))
            infos = [None] * R
            dist.all_gather_object(infos, (int(n), int(d), str(dtype), err, int(top), rows, tops), group=group)
            verdict = selection_refusal(infos, classifier, n_es, validation)
            if verdict is not None:
                raise _EXCEPTIONS.get(verdict[0], RuntimeError)(verdict[1])
            first = next(i for i in infos if i[0] > 0)
            if n == 0:                                      # an empty shard takes the agreed dtype and width
                Xl = np.empty((0, first[1]), dtype=np.float32 if first[2] == "float32" else np.float64)
                yl = np.empty(0)
                members = [np.zeros(0, dtype=bool) for _ in first[5]]
            sizes = np.array([i[5] if i[0] > 0 else [0] * len(first[5]) for i in infos], dtype=np.int64)
            classes = [max(i[6][k] if i[0] > 0 else -1 for i in infos) + 1 for k in range(len(first[5]))]
            key, eng = comm_engine(group, gp._device, device, engine_factory)
            try:
                yield Selection(group, device, eng, Xl, yl, members, sizes, classes)
            except BaseException:
                # a failure after a collective may leave the ranks out of step: the communicator is not reused
                if _COMM_ENGINES.get(key) is eng:
                    _COMM_ENGINES.pop(key)
                    eng.close()
                raise

    return run()
