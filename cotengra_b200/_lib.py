"""ctypes binding of ``libctgb200.so`` (the C-ABI in ``include/ctg_b200.h``).

The library is built in-tree by ``__graft_entry__.build()`` /
``cotengra_b200/csrc/build.sh``.  There is deliberately no fallback: if the
shared object is missing or exports the wrong ABI, importing the compute path
fails loudly.
"""

from __future__ import annotations

import ctypes as C
import os

from . import lowering

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libctgb200.so")

# every symbol include/ctg_b200.h declares
EXPORTS = (
    "ctgb_abi_version",
    "ctgb_desc_words",
    "ctgb_single_desc_words",
    "ctgb_last_error",
    "ctgb_device_info",
    "ctgb_contract_pair",
    "ctgb_reduce_single",
    "ctgb_plan_create",
    "ctgb_plan_set_chunk_desc",
    "ctgb_plan_set_scale_slots",
    "ctgb_plan_set_accumulator",
    "ctgb_plan_destroy",
    "ctgb_plan_workspace_bytes",
    "ctgb_plan_launches_per_slice",
    "ctgb_plan_strip_modes",
    "ctgb_plan_execute",
    "ctgb_plan_execute_host",
    "ctgb_launch_count",
    "ctgb_tensor_map_launches",
    "ctgb_plan_profile",
    "ctgb_plan_profile_read",
    "ctgb_probe_fp64_peaks",
    "ctgb_tc05_launch_config",
    "ctgb_dmmastream_launch_config",
    "ctgb_absorb_root",
    "ctgb_contract_pair2",
    "ctgb_plan_execute_jvp",
    "ctgb_plan_execute_jvp_stripped",
    "ctgb_plan_set_tangent_scale_slots",
)
TC05_LAUNCH_FIELDS = ("b_stat", "nb", "sa", "grid", "smem", "tm_rank", "bulk", "chunk_steps", "chunks")
DMMASTREAM_LAUNCH_FIELDS = ("nj", "rows", "grid")


class CtgbTensor(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("input_index", C.c_int32),
        ("offset", C.c_int64),
        ("nbytes", C.c_int64),
        ("n_sliced", C.c_int32),
        ("slice_pos", C.POINTER(C.c_int32)),
        ("slice_stride", C.POINTER(C.c_int64)),
    ]


class CtgbNode(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("a", C.c_int32),
        ("b", C.c_int32),
        ("c", C.c_int32),
        ("phase", C.c_int32),
        ("zero_fill", C.c_int32),
        ("is_root", C.c_int32),
        ("desc", C.POINTER(C.c_int64)),
    ]


class CtgbPlanDesc(C.Structure):
    _fields_ = [
        ("dtype", C.c_int32),
        ("n_inputs", C.c_int32),
        ("n_tensors", C.c_int32),
        ("tensors", C.POINTER(CtgbTensor)),
        ("n_nodes", C.c_int32),
        ("nodes", C.POINTER(CtgbNode)),
        ("n_sliced", C.c_int32),
        ("slice_radix", C.POINTER(C.c_int64)),
        ("slice_project", C.POINTER(C.c_int64)),
        ("slice_out_stride", C.POINTER(C.c_int64)),
        ("out_elements", C.c_int64),
        ("workspace_bytes", C.c_int64),
        ("persistent_bytes", C.c_int64),
        ("strip_exponent", C.c_int32),
        ("cotangent_offset", C.c_int64),
    ]


_lib = None

_ERRORS = {1: ValueError, 2: NotImplementedError, 3: RuntimeError, 4: MemoryError}


def load():
    """Load (once) and type the library."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import "
            "__graft_entry__ as g; g.build()'` (nvcc, sm_90a). cotengra_b200 "
            "has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name in EXPORTS:
        if not hasattr(lib, name):
            raise ImportError(f"{LIB_PATH} does not export {name}")
    lib.ctgb_last_error.restype = C.c_char_p
    lib.ctgb_launch_count.restype = C.c_int64
    lib.ctgb_tensor_map_launches.restype = C.c_int64
    lib.ctgb_plan_workspace_bytes.restype = C.c_size_t
    lib.ctgb_plan_workspace_bytes.argtypes = [C.c_void_p]
    lib.ctgb_plan_launches_per_slice.restype = C.c_int64
    lib.ctgb_plan_launches_per_slice.argtypes = [C.c_void_p]
    lib.ctgb_plan_strip_modes.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int]
    lib.ctgb_device_info.argtypes = [
        C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_size_t)
    ]
    lib.ctgb_contract_pair.argtypes = [C.c_void_p] * 5
    lib.ctgb_reduce_single.argtypes = [C.c_void_p] * 4
    lib.ctgb_absorb_root.argtypes = [C.c_void_p] * 6
    lib.ctgb_contract_pair2.argtypes = [C.c_void_p] * 7
    lib.ctgb_plan_execute_jvp.argtypes = [
        C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p,
        C.c_void_p, C.c_size_t, C.c_int64, C.c_int64, C.c_int64, C.c_void_p,
    ]
    lib.ctgb_plan_execute_jvp_stripped.argtypes = [
        C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_void_p,
        C.c_void_p, C.c_size_t, C.c_int64, C.c_int64, C.c_int64, C.c_void_p,
    ]
    lib.ctgb_plan_set_tangent_scale_slots.argtypes = [
        C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int]
    lib.ctgb_plan_create.argtypes = [C.POINTER(CtgbPlanDesc), C.POINTER(C.c_void_p)]
    lib.ctgb_plan_set_chunk_desc.argtypes = [C.c_void_p, C.c_void_p]
    lib.ctgb_plan_set_scale_slots.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int]
    lib.ctgb_plan_set_accumulator.argtypes = [C.c_void_p, C.c_int32]
    lib.ctgb_plan_destroy.argtypes = [C.c_void_p]
    lib.ctgb_plan_destroy.restype = None
    lib.ctgb_plan_execute.argtypes = [
        C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p),
        C.c_void_p, C.c_size_t, C.c_int64, C.c_int64, C.c_int64, C.c_void_p,
    ]
    lib.ctgb_plan_execute_host.argtypes = [
        C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_void_p,
        C.POINTER(C.c_double), C.c_void_p, C.c_size_t, C.c_int64, C.c_int64,
        C.c_int64, C.c_void_p,
    ]
    lib.ctgb_plan_profile.argtypes = [C.c_void_p, C.c_int]
    lib.ctgb_plan_profile_read.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int]
    lib.ctgb_probe_fp64_peaks.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_void_p]
    lib.ctgb_tc05_launch_config.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_uint64,
                                            C.POINTER(C.c_int64), C.c_int]
    lib.ctgb_dmmastream_launch_config.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int64), C.c_int]
    if lib.ctgb_abi_version() != 2:
        raise ImportError("libctgb200.so: ABI version mismatch")
    if lib.ctgb_desc_words() != lowering.DESC_WORDS:
        raise ImportError("libctgb200.so: pair descriptor layout mismatch")
    if lib.ctgb_single_desc_words() != lowering.SDESC_WORDS:
        raise ImportError("libctgb200.so: single descriptor layout mismatch")
    _lib = lib
    return lib


def check(rc):
    if rc:
        msg = load().ctgb_last_error().decode()
        raise _ERRORS.get(rc, RuntimeError)(f"ctgb error {rc}: {msg}")


def device_info():
    lib = load()
    sm, ma, mi, sh = C.c_int(), C.c_int(), C.c_int(), C.c_size_t()
    check(lib.ctgb_device_info(C.byref(sm), C.byref(ma), C.byref(mi), C.byref(sh)))
    return {"sm_count": sm.value, "cc": (ma.value, mi.value), "smem_optin": sh.value}


def probe_fp64_peaks(stream=0):
    lib = load()
    a, b = C.c_double(), C.c_double()
    check(lib.ctgb_probe_fp64_peaks(C.byref(a), C.byref(b), stream))
    return {"dmma_tflops": a.value, "dfma_tflops": b.value}


def launch_count() -> int:
    return int(load().ctgb_launch_count())


def tensor_map_launches() -> int:
    """wgmma launches so far whose A tiles were fetched by tensor-map TMA."""
    return int(load().ctgb_tensor_map_launches())


def tc05_launch_config(words, a_addr, sms, smem_optin) -> dict:
    """The launch-time choices of the wgmma kernel for descriptor ``words`` (int64 numpy array) with
    A at device address ``a_addr`` on a device with ``sms`` SMs and ``smem_optin`` bytes of opt-in
    shared memory (include/ctg_b200.h).  Needs no device."""
    import numpy as np

    w = np.ascontiguousarray(words, dtype=np.int64)
    out = (C.c_int64 * len(TC05_LAUNCH_FIELDS))()
    check(load().ctgb_tc05_launch_config(w.ctypes.data, int(a_addr), int(sms), int(smem_optin), out,
                                         len(TC05_LAUNCH_FIELDS)))
    return dict(zip(TC05_LAUNCH_FIELDS, (int(x) for x in out)))


def dmmastream_launch_config(words, sms) -> dict:
    """The DMMA stream kernel's instantiation (``nj`` column fragments, ``rows`` per warp block) and
    grid for descriptor ``words`` on a device with ``sms`` SMs (include/ctg_b200.h).  Needs no device."""
    import numpy as np

    w = np.ascontiguousarray(words, dtype=np.int64)
    out = (C.c_int64 * len(DMMASTREAM_LAUNCH_FIELDS))()
    check(load().ctgb_dmmastream_launch_config(w.ctypes.data, int(sms), out, len(DMMASTREAM_LAUNCH_FIELDS)))
    return dict(zip(DMMASTREAM_LAUNCH_FIELDS, (int(x) for x in out)))
