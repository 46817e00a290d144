"""Host-side rules that let several contexts run side by side on one device, each from its own thread (no GPU needed).

The dynamic shared-memory cap, read from the sources: cudaFuncAttributeMaxDynamicSharedMemorySize is one value per kernel per device, shared by every context of the process on
that device.  A launcher that set it to its own call's plan size would race with a context on another thread launching
the same kernel with a larger plan (that launch is refused with cudaErrorInvalidValue).  Whether a run on the GPU hits
that window is a matter of timing, so the rule is checked here: the attribute is set in one helper only, to one value
that does not depend on the call.

The per-device pool of idle contexts, which estimators fitting from several threads draw from at once."""
import os
import re
import threading

from spark_gp_b200.engine import ProjectedProcessEngine

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "spark_gp_b200", "csrc")
ATTRIBUTE_NAMES = ("cudaFuncAttributeMaxDynamicSharedMemorySize", "CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES")


def _code(path):
    """The source without its comments (a comment may name the attribute)."""
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def _sources():
    return {f: _code(os.path.join(CSRC, f)) for f in sorted(os.listdir(CSRC))
            if f.endswith((".cu", ".cuh", ".h", ".cpp", ".hpp"))}


def _helper_body(internal):
    m = re.search(r"inline cudaError_t allow_dynamic_smem\(const void\* fn\) \{(.*?)\n\}", internal, re.S)
    assert m, "sgp_internal.h: allow_dynamic_smem(const void* fn) not found"
    return m.group(1)


def test_dynamic_smem_attribute_set_only_in_helper():
    """Every opt-in to dynamic shared memory in csrc/ goes through allow_dynamic_smem: the attribute's name appears in
    that helper's body and nowhere else in the code."""
    sources = _sources()
    assert "sgp_internal.h" in sources and len(sources) > 10
    body = _helper_body(sources["sgp_internal.h"])
    outside = []
    for f, code in sources.items():
        if f == "sgp_internal.h":
            code = code.replace(body, "")
        for name in ATTRIBUTE_NAMES:
            outside += ["%s:%d" % (f, code[:m.start()].count("\n") + 1) for m in re.finditer(name, code)]
    assert not outside, "the dynamic shared-memory cap is set outside allow_dynamic_smem at %s" % ", ".join(outside)
    assert body.count("cudaFuncAttributeMaxDynamicSharedMemorySize") == 1


def test_dynamic_smem_cap_is_one_value_per_kernel():
    """The helper takes the kernel alone and sets the opt-in maximum less the kernel's static shared memory (both
    properties of the function): no argument of the call can reach the cap."""
    body = _helper_body(_code(os.path.join(CSRC, "sgp_internal.h")))
    call = re.fullmatch(r"\s*cudaFuncAttributes a;\s*const cudaError_t e = cudaFuncGetAttributes\(&a, fn\);\s*"
                        r"if \(e != cudaSuccess\) return e;\s*"
                        r"return cudaFuncSetAttribute\(fn, cudaFuncAttributeMaxDynamicSharedMemorySize,\s*"
                        r"static_cast<int>\(kSmemOptInMax - a\.sharedSizeBytes\)\);\s*", body)
    assert call, "allow_dynamic_smem must set the cap from the kernel alone, not from a size of the call:\n%s" % body


def test_every_large_smem_launcher_uses_helper():
    """The launchers whose kernels take more than 48 KiB of dynamic shared memory each opt in through the helper (a
    missing opt-in fails every such launch, so this pins the list the rule covers)."""
    sources = _sources()
    calls = {f: code.count("allow_dynamic_smem(") for f, code in sources.items() if f != "sgp_internal.h"}
    assert {f: n for f, n in calls.items() if n} == {"bcm_nll.cu": 2, "gram_f64.cu": 2, "gram_i8_wgmma.cu": 3,
                                                     "kmn_sweep.cu": 1, "laplace.cu": 1, "predict.cu": 1}


class _StandIn(ProjectedProcessEngine):
    """A pooled context without a device: only the pool's bookkeeping runs."""
    _idle = {}
    created = []

    def __init__(self, device=0):
        self._h, self._device, self._has_comm = 1, device, False
        _StandIn.created.append(self)

    def set_precision(self, mode):
        pass

    def close(self):
        self._h = None


class _EmptiedList(list):
    """A pool another thread empties between this thread's look at it and its pop."""

    def __bool__(self):
        return True


def test_pool_emptied_under_acquire_creates_a_context():
    _StandIn._idle, _StandIn.created = {0: _EmptiedList()}, []
    eng = _StandIn.acquire(0)
    assert _StandIn.created == [eng]


def test_pool_hands_each_idle_context_to_one_thread():
    _StandIn.created = []
    idle = [_StandIn(0) for _ in range(3)]
    _StandIn._idle = {0: list(idle)}
    got, start = [None] * 8, threading.Barrier(8)

    def take(i):
        start.wait()
        got[i] = _StandIn.acquire(0)

    ts = [threading.Thread(target=take, args=(i,)) for i in range(8)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert len({id(e) for e in got}) == 8 and all(any(e is g for g in got) for e in idle)
    assert len(_StandIn.created) == 3 + 5 and not _StandIn._idle[0]
