"""ctypes binding of libissue_emb_b200.so (C ABI: include/issue_emb_b200.h).

There is deliberately NO fallback: if the CUDA library is missing or cannot be loaded this module raises, and
every entry point fails when no sm_90 (H100) device is present.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libissue_emb_b200.so"

IE_OK, IE_ERR_INVALID, IE_ERR_CUDA, IE_ERR_OOM, IE_ERR_STATE, IE_ERR_TOKEN = 0, -1, -2, -3, -4, -5
IE_FLAG_DEVICE_PTRS = 1
IE_MAX_BATCH = 3072          # upper bound; a handle's own limit is ie_encoder_max_batch() (1280 by default)
IE_CFG_ACCURATE_GATES, IE_CFG_FP32, IE_CFG_F32_GX = 1, 2, 4
IE_KNN_COSINE, IE_KNN_EUCLIDEAN = 0, 1


class ie_config(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("emb_sz", C.c_int32), ("n_hid", C.c_int32), ("vocab_sz", C.c_int32),
                ("pad_idx", C.c_int32), ("device", C.c_int32), ("flags", C.c_int32)]


# name -> (restype, argtypes); must list every symbol declared in include/issue_emb_b200.h
PROTOTYPES = {
    "ie_version": (C.c_int, []),
    "ie_last_error": (C.c_char_p, []),
    "ie_encoder_create": (C.c_int, [C.POINTER(ie_config), C.POINTER(C.c_void_p)]),
    "ie_encoder_destroy": (None, [C.c_void_p]),
    "ie_encoder_load_embedding": (C.c_int, [C.c_void_p, C.c_void_p]),
    "ie_encoder_load_layer": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ie_encoder_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                    C.c_void_p]),
    "ie_encoder_raw_features": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                          C.c_void_p]),
    "ie_encoder_launch_count": (C.c_int64, [C.c_void_p]),
    "ie_encoder_max_batch": (C.c_int32, [C.c_void_p]),
    "ie_debug_workspace_bytes": (C.c_int64, [C.c_void_p]),
    "ie_encoder_check_errors": (C.c_int, [C.c_void_p]),
    "ie_encoder_last_phase_ms": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32]),
    "ie_encoder_last_phase_mhz": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32]),
    "ie_debug_seq_trace": (C.c_int64, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]),
    "ie_mlp_create": (C.c_int, [C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_void_p)]),
    "ie_mlp_load_layer": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "ie_mlp_predict_proba": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "ie_mlp_destroy": (None, [C.c_void_p]),
    "ie_pr_thresholds": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "ie_debug_gemm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                C.c_void_p, C.c_int32]),
    "ie_debug_gemm_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_int32, C.c_int32, C.c_void_p, C.c_int32]),
    "ie_debug_gemm_frag": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                     C.c_int32, C.c_void_p, C.c_int32]),
    "ie_debug_epilogue_layout": (C.c_int64, [C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "ie_debug_gates": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "ie_debug_layer_states": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                        C.c_void_p]),
    "ie_knn_create": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
    "ie_knn_destroy": (None, [C.c_void_p]),
    "ie_knn_add": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "ie_knn_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                C.c_void_p]),
    "ie_knn_check_errors": (C.c_int, [C.c_void_p]),
    "ie_debug_knn_shortlist": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "ie_mlp_train_create": (C.c_int, [C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_void_p)]),
    "ie_mlp_train_destroy": (None, [C.c_void_p]),
    "ie_mlp_train_set_layer": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "ie_mlp_train_get_layer": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "ie_mlp_train_set_data": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64]),
    "ie_mlp_train_epoch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_double, C.c_double,
                                     C.c_double, C.c_double, C.c_void_p]),
    "ie_mlp_train_validation_proba": (C.c_int, [C.c_void_p, C.c_void_p]),
    "ie_mlp_train_snapshot": (C.c_int, [C.c_void_p, C.c_int32]),
    "ie_mlp_train_launch_count": (C.c_int64, [C.c_void_p]),
    "ie_mlp_train_last_epoch_ms": (C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
    "ie_debug_mlp_train_step": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_int64, C.POINTER(C.c_double)]),
    "ie_mlp_group_capacity": (C.c_int, [C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_double,
                                        C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "ie_mlp_group_create": (C.c_int, [C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32,
                                      C.POINTER(C.c_void_p)]),
    "ie_mlp_group_destroy": (None, [C.c_void_p]),
    "ie_mlp_group_set_data": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]),
    "ie_mlp_group_set_layer": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "ie_mlp_group_get_layer": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "ie_mlp_group_set_hyper": (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_double]),
    "ie_mlp_group_set_validation": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]),
    "ie_mlp_group_epoch": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p]),
    "ie_mlp_group_validation_proba": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "ie_mlp_group_snapshot": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "ie_mlp_group_launch_count": (C.c_int64, [C.c_void_p]),
    "ie_mlp_group_last_epoch_ms": (C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
    "ie_clas_window": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]),
    "ie_clas_create": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_void_p)]),
    "ie_clas_destroy": (None, [C.c_void_p]),
    "ie_clas_load_stage": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double,
                                     C.c_void_p, C.c_void_p]),
    "ie_clas_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_void_p, C.c_int32, C.c_void_p]),
    "ie_clas_pool": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                               C.c_int32, C.c_void_p]),
    "ie_clas_check_errors": (C.c_int, [C.c_void_p]),
    "ie_clas_launch_count": (C.c_int64, [C.c_void_p]),
    "ie_lm_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "ie_lm_destroy": (None, [C.c_void_p]),
    "ie_lm_load_decoder": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "ie_lm_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_int32, C.c_void_p]),
    "ie_lm_check_errors": (C.c_int, [C.c_void_p]),
    "ie_lm_launch_count": (C.c_int64, [C.c_void_p]),
    "ie_debug_lm_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                     C.c_void_p]),
    "ie_gen_state_create": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]),
    "ie_gen_state_destroy": (None, [C.c_void_p]),
    "ie_gen_state_reset": (C.c_int, [C.c_void_p]),
    "ie_gen_topk": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                   C.c_void_p, C.c_int32, C.c_void_p]),
    "ie_gen_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_double,
                                     C.c_double, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "ie_gen_select": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "ie_gen_beam_select": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                    C.c_void_p]),
    "ie_gen_state_export": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "ie_debug_gen_topk": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_int32]),
    "ie_debug_gen_sample": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_double, C.c_double,
                                     C.c_void_p, C.c_void_p, C.c_int32]),
}

_lib = None


def build(verbose: bool = False) -> Path:
    """Compile the CUDA sources for sm_90a (nvcc cross-compiles without a GPU)."""
    r = subprocess.run(["make", "-C", str(_PKG / "csrc"), "-j8"], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout[-4000:])
        print(r.stderr[-4000:])
    if r.returncode != 0:
        raise RuntimeError("building libissue_emb_b200.so failed")
    return LIB_PATH


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        if os.environ.get("IE_B200_NO_AUTOBUILD"):
            raise ImportError(f"{LIB_PATH} is missing (run `python -c 'import __graft_entry__ as g; g.build()'`)")
        build()
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def _debug_gemm(a, b, bias=None, act: int = 0, out_type: int = 0, segs: int = 1, device: int = 0):
    """Test hook ``ie_debug_gemm_ex``: act(a [M,K] @ b [N,K]^T + bias) through the library's wgmma GEMM, stored as f32
    (out_type 0), bf16 (1) or fp16 (2) and returned widened to float32 (M, N); segs 3 = split-bf16 operands."""
    import numpy as np
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    (M, K), N = a.shape, b.shape[0]
    if b.shape[1] != K:
        raise ValueError(f"a {a.shape} and b {b.shape} disagree on K")
    bias_p = None
    if bias is not None:
        bias = np.ascontiguousarray(bias, dtype=np.float32)
        if bias.shape != (N,):
            raise ValueError(f"bias {bias.shape} != ({N},)")
        bias_p = bias.ctypes.data
    d = np.empty((M, N), dtype=np.float32)
    check(load().ie_debug_gemm_ex(a.ctypes.data, b.ctypes.data, bias_p, M, N, K, act, out_type, segs, d.ctypes.data,
                                  device))
    return d


GATE_FNS = ("sigmoid_fast", "tanh_fast", "sigmoid_acc", "tanh_acc", "sigmoid_ieee", "tanh_ieee")
CELL_FNS = {"fast": 6, "exp": 7, "ieee": 8}
# the language-model decoder's ex2.approx.ftz and logf (csrc/lm.cu), text generation's expf (csrc/lm_gen.cu)
LM_MATH_FNS = {"lm_ex2": 9, "lm_log": 10, "lm_expf": 11}


def _debug_gates(fn, x):
    """Test hook ``ie_debug_gates`` on CUDA float32 tensors.  fn a name of GATE_FNS or LM_MATH_FNS: f(x) elementwise,
    same shape.  fn 'lm_pow' (text generation's powf): x [2, n] planes (x, y) -> [n] powf(x, y).  fn 'cell_fast' |
    'cell_exp' | 'cell_ieee': x [5, n] planes (zi, zf, zg, zo, c_prev) -> [2, n] (c_new, h)."""
    import torch
    x = x.contiguous()
    if x.dtype != torch.float32 or not x.is_cuda:
        raise ValueError("ie_debug_gates takes a CUDA float32 tensor")
    if fn in GATE_FNS or fn in LM_MATH_FNS:
        code = GATE_FNS.index(fn) if fn in GATE_FNS else LM_MATH_FNS[fn]
        n, out = x.numel(), torch.empty_like(x)
    elif fn == "lm_pow":
        if x.dim() != 2 or x.shape[0] != 2:
            raise ValueError(f"powf input {tuple(x.shape)} must be [2, n]")
        code, n = 12, x.shape[1]
        out = torch.empty(n, dtype=torch.float32, device=x.device)
    else:
        code = CELL_FNS[fn.removeprefix("cell_")]
        if x.dim() != 2 or x.shape[0] != 5:
            raise ValueError(f"cell input {tuple(x.shape)} must be [5, n]")
        n, out = x.shape[1], torch.empty(2, x.shape[1], dtype=torch.float32, device=x.device)
    stream = torch.cuda.current_stream(x.device).cuda_stream
    check(load().ie_debug_gates(code, x.data_ptr(), out.data_ptr(), n, x.device.index, stream))
    return out


def check(rc: int) -> None:
    """Map C error codes to the exceptions the reference's callers expect (SURVEY.md section 8b):
    RuntimeError for CUDA failures / OOM (so the batch-halving loop of
    py/code_intelligence/inference.py:214-223 still works), ValueError for bad shapes / token ids."""
    if rc == IE_OK:
        return
    msg = (load().ie_last_error() or b"").decode("utf-8", "replace")
    if rc in (IE_ERR_INVALID, IE_ERR_TOKEN):
        raise ValueError(msg)
    if rc == IE_ERR_OOM:
        raise RuntimeError("CUDA out of memory. " + msg)
    raise RuntimeError(msg)
