"""ctypes binding of libb200sv.so (include/b200sv.h).  No CPU fallback: a missing library is a hard error."""
from __future__ import annotations

import ctypes
import os
import subprocess
from ctypes import POINTER, c_char_p, c_double, c_int, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200SV_LIB selects another build of the same library (to A/B-time two builds in one session); default = the in-tree product
LIB_PATH = os.environ.get("B200SV_LIB") or os.path.join(_HERE, "libb200sv.so")
CSRC = os.path.join(_HERE, "csrc")
SOURCES = ["b200sv.cu", "fused.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "-shared", "-cudart", "static"]

B200SV_OK, B200SV_EINVAL, B200SV_ENOMEM, B200SV_ECUDA, B200SV_ESTATE = 0, -1, -2, -3, -4


class Stats(ctypes.Structure):
    _fields_ = [("gates_submitted", c_uint64), ("kernel_launches", c_uint64), ("fused_sweeps", c_uint64),
                ("fused_gates", c_uint64), ("single_launches", c_uint64), ("bytes_swept", c_uint64),
                ("pull_sweeps", c_uint64)]


# name -> (argtypes)  — every symbol include/b200sv.h declares; tests/test_abi.py checks the two stay in sync
H = c_void_p
SIGNATURES = {
    "b200sv_abi_version": [],
    "b200sv_device_count": [POINTER(c_int)],
    "b200sv_device_info": [c_int, POINTER(c_uint64), POINTER(c_uint64), POINTER(c_int)],
    "b200sv_can_access_peer": [c_int, c_int, POINTER(c_int)],
    "b200sv_create": [c_int, c_int, c_int, POINTER(H)],
    "b200sv_destroy": [H],
    "b200sv_clone": [H, POINTER(H)],
    "b200sv_qubit_count": [H, POINTER(c_int)],
    "b200sv_precision": [H, POINTER(c_int)],
    "b200sv_device": [H, POINTER(c_int)],
    "b200sv_set_device": [H, c_int],
    "b200sv_device_ptr": [H, POINTER(c_void_p)],
    "b200sv_create_external": [c_int, c_int, c_int, c_void_p, POINTER(H)],
    "b200sv_rebind_external": [H, c_void_p],
    "b200sv_set_stream": [H, c_void_p, c_int],
    "b200sv_set_permutation": [H, c_uint64, c_double, c_double],
    "b200sv_zero": [H],
    "b200sv_is_zero": [H, POINTER(c_int)],
    "b200sv_set_state": [H, c_void_p],
    "b200sv_get_state": [H, c_void_p],
    "b200sv_get_probs": [H, c_void_p],
    "b200sv_get_page": [H, c_void_p, c_uint64, c_uint64],
    "b200sv_set_page": [H, c_void_p, c_uint64, c_uint64],
    "b200sv_copy_page": [H, H, c_uint64, c_uint64, c_uint64],
    "b200sv_shuffle": [H, H],
    "b200sv_copy_state": [H, H],
    "b200sv_get_amplitude": [H, c_uint64, POINTER(c_double), POINTER(c_double)],
    "b200sv_set_amplitude": [H, c_uint64, c_double, c_double],
    "b200sv_apply2x2": [H, c_uint64, c_uint64, POINTER(c_double), c_int, POINTER(c_uint64), c_double, c_double,
                        POINTER(c_double)],
    "b200sv_apply_gates": [H, c_int, POINTER(c_uint64), POINTER(c_uint64), POINTER(c_uint64), POINTER(c_double)],
    "b200sv_xmask": [H, c_uint64],
    "b200sv_phase_parity": [H, c_double, c_uint64],
    "b200sv_phase_root_n_mask": [H, c_int, c_uint64],
    "b200sv_uniform_parity_rz": [H, c_uint64, c_uint64, c_double],
    "b200sv_uniformly_controlled": [H, c_int, POINTER(c_int), c_int, POINTER(c_double), c_int, POINTER(c_uint64),
                                    c_uint64, c_double],
    "b200sv_apply_m": [H, c_uint64, c_uint64, c_double, c_double],
    "b200sv_collapse_parity": [H, c_uint64, c_int, POINTER(c_double)],
    "b200sv_prob_mask": [H, c_uint64, c_uint64, POINTER(c_double)],
    "b200sv_prob_parity": [H, c_uint64, POINTER(c_double)],
    "b200sv_prob_mask_all": [H, c_uint64, c_void_p],
    "b200sv_norm": [H, c_double, POINTER(c_double)],
    "b200sv_normalize": [H, c_double, c_double, c_double],
    "b200sv_inner": [H, H, POINTER(c_double), POINTER(c_double)],
    "b200sv_expectation": [H, c_int, c_int, POINTER(c_double)],
    "b200sv_moments_bits": [H, c_int, POINTER(c_int), POINTER(c_uint64), c_uint64, c_double, POINTER(c_double)],
    "b200sv_moments_floats": [H, c_int, POINTER(c_int), POINTER(c_double), c_double, POINTER(c_double)],
    "b200sv_expectation_pauli": [H, c_uint64, c_uint64, POINTER(c_double)],
    "b200sv_reduced_density_matrix": [H, c_int, POINTER(c_int), POINTER(c_double)],
    "b200sv_highest_prob": [H, POINTER(c_uint64)],
    "b200sv_sample": [H, c_double, POINTER(c_uint64)],
    "b200sv_sample_many": [H, c_int, POINTER(c_double), POINTER(c_uint64)],
    "b200sv_compose": [H, H, c_int],
    "b200sv_decompose": [H, c_int, c_int, H],
    "b200sv_dispose_perm": [H, c_int, c_int, c_uint64],
    "b200sv_alloc_page": [c_int, c_uint64, POINTER(c_void_p)],
    "b200sv_free_page": [c_int, c_void_p],
    "b200sv_ipc_export": [c_int, c_void_p, c_void_p],
    "b200sv_ipc_import": [c_int, c_void_p, POINTER(c_void_p)],
    "b200sv_ipc_release": [c_int, c_void_p],
    "b200sv_exchange_scatter": [H, c_int, POINTER(c_int), c_int, POINTER(c_void_p)],
    "b200sv_exchange_pull": [H, c_int, POINTER(c_int), c_int, POINTER(c_void_p), c_void_p],
    "b200sv_rol": [H, c_int, c_int, c_int],
    "b200sv_inc": [H, c_uint64, c_int, c_int, c_uint64],
    "b200sv_incdecc": [H, c_uint64, c_int, c_int, c_int],
    "b200sv_incs": [H, c_uint64, c_int, c_int, c_int],
    "b200sv_incdecsc": [H, c_uint64, c_int, c_int, c_int, c_int],
    "b200sv_muldiv": [H, c_int, c_uint64, c_int, c_int, c_int, c_uint64],
    "b200sv_modnout": [H, c_int, c_uint64, c_uint64, c_int, c_int, c_int, c_uint64],
    "b200sv_indexed": [H, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_char_p],
    "b200sv_hash": [H, c_int, c_int, c_char_p],
    "b200sv_phase_flip_if_less": [H, c_uint64, c_int, c_int, c_int],
    "b200sv_flush": [H],
    "b200sv_finish": [H],
    "b200sv_set_fusion": [H, c_int],
    "b200sv_emulate_fused": [c_int, c_int, c_int, POINTER(c_uint64), POINTER(c_uint64), POINTER(c_uint64), POINTER(c_double),
                             c_void_p],
    "b200sv_plan_gates": [c_int, c_int, c_int, POINTER(c_uint64), POINTER(c_uint64), POINTER(c_uint64), POINTER(c_double),
                          POINTER(c_int), POINTER(c_int), POINTER(c_int)],
    "b200sv_emulate_fused_pull": [c_int, c_int, c_int, POINTER(c_uint64), POINTER(c_uint64), POINTER(c_uint64), POINTER(c_double),
                                  c_int, POINTER(c_int), c_int, POINTER(c_void_p), c_void_p],
    "b200sv_get_stats": [H, POINTER(Stats)],
    "b200sv_reset_stats": [H],
    "b200sv_timer_begin": [H],
    "b200sv_timer_end": [H, POINTER(c_double)],
    "b200sv_flush_l2": [H, c_uint64],
}

_lib = None


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile libb200sv.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h", ".inl"))]
    deps.append(os.path.join(_HERE, "..", "include", "b200sv.h"))
    if not force and os.path.exists(LIB_PATH):
        newest = max(os.path.getmtime(d) for d in deps if os.path.exists(d))
        if os.path.getmtime(LIB_PATH) >= newest:
            return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + srcs + ["-o", LIB_PATH]
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True)
    return LIB_PATH


def load():
    """dlopen the library (building it first if the source tree is newer and nvcc exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("qrack_b200: %s is missing — run `python -c 'import __graft_entry__ as g; g.build()'`. "
                           "There is no CPU fallback for the engine." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, args in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = c_int
    lib.b200sv_last_error.argtypes = []
    lib.b200sv_last_error.restype = c_char_p
    _lib = lib
    return lib


def check(lib, rc: int):
    if rc == B200SV_OK:
        return
    msg = lib.b200sv_last_error().decode("utf-8", "replace")
    if rc == B200SV_EINVAL:
        raise ValueError(msg)  # reference: std::invalid_argument
    if rc == B200SV_ENOMEM:
        raise MemoryError(msg)  # reference: Qrack::bad_alloc
    raise RuntimeError("b200sv error %d: %s" % (rc, msg))


def create(lib, device: int, n_qubits: int, precision: int, external_ptr: int = 0):
    h = c_void_p()
    if external_ptr:
        check(lib, lib.b200sv_create_external(device, n_qubits, precision, c_void_p(external_ptr), ctypes.byref(h)))
    else:
        check(lib, lib.b200sv_create(device, n_qubits, precision, ctypes.byref(h)))
    return h
