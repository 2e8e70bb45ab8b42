"""ctypes binding of ``csrc/libl2o_b200.so`` (C-ABI declared in ``include/l2o_b200.h``).

There is deliberately NO fallback: if the shared library is missing or a call fails, this module
raises.  The product path never routes through ``oracle/`` or plain PyTorch math.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.environ.get("L2O_LIB") or os.path.join(CSRC, "libl2o_b200.so")  # L2O_LIB: A/B-test an alternative build
INCLUDE = os.path.join(_ROOT, "include")

L2O_OK, L2O_E_INVALID, L2O_E_UNSUPPORTED, L2O_E_CUDA, L2O_E_NOMEM = 0, -1, -2, -3, -4
PRE_IDENTITY, PRE_LOGSIGN, PRE_FC = 0, 1, 2
OPT_NONE, OPT_RASTRIGIN_SEP, OPT_QUADRATIC_DIAG, OPT_QUADRATIC_BATCH = 0, 1, 2, 3
ENGINE_AUTO, ENGINE_FFMA, ENGINE_TC = 0, 1, 2

# every symbol include/l2o_b200.h declares (tests check the .so exports all of them)
EXPORTS = [
    "l2o_net_create", "l2o_net_destroy", "l2o_net_set_engine", "l2o_theta_count", "l2o_state_floats", "l2o_workspace_bytes",
    "l2o_step", "l2o_unroll_fwd", "l2o_unroll_bwd", "l2o_unroll_bwd_carry", "l2o_tc_fwd_variant", "l2o_tc_weight_image", "l2o_adam_step", "l2o_log_and_sign", "l2o_lasso_grad",
    "l2o_confocal_grad", "l2o_mnist_grad", "l2o_mnist_conv_workspace_bytes", "l2o_mnist_conv_workspace_layout",
    "l2o_mnist_conv_grad", "l2o_cifar_conv_workspace_bytes", "l2o_cifar_conv_workspace_layout", "l2o_cifar_conv_grad",
    "l2o_nas_workspace_bytes", "l2o_nas_workspace_layout", "l2o_nas_grad",
    "l2o_dense_create", "l2o_dense_destroy", "l2o_dense_theta_count", "l2o_dense_state_floats", "l2o_dense_step",
    "l2o_dense_unroll_bwd",
    "l2o_launch_count", "l2o_status_string", "l2o_last_cuda_error", "l2o_version",
    "l2o_hrnn_create", "l2o_hrnn_destroy", "l2o_hrnn_theta_count", "l2o_hrnn_state_floats", "l2o_hrnn_coords",
    "l2o_hrnn_workspace_bytes", "l2o_hrnn_init_state", "l2o_hrnn_prepare", "l2o_hrnn_step",
    "l2o_hrnn_set_global_sizes", "l2o_hrnn_prepare_local", "l2o_hrnn_prepare_finish",
    "l2o_hrnn_step_local", "l2o_hrnn_step_finish", "l2o_hrnn_coord_bwd", "l2o_hrnn_workspace_layout",
    "l2o_crnn_theta_count", "l2o_crnn_state_floats", "l2o_crnn_step", "l2o_crnn_bwd",
    "l2o_tadam_theta_count", "l2o_tadam_state_floats", "l2o_tadam_step", "l2o_tadam_bwd", "l2o_lrsgd_step",
    "l2o_lrsgd_bwd",
    "l2o_ista_workspace_bytes", "l2o_ista_fwd", "l2o_ista_bwd", "l2o_ista_loss_grad",
    "l2o_minimax_theta_count", "l2o_minimax_image_floats", "l2o_minimax_image", "l2o_minimax_workspace_bytes",
    "l2o_minimax_fwd", "l2o_minimax_bwd",
    "l2o_zoo_value_grad", "l2o_zoo_hvp", "l2o_zoo_hess_form",
]


class NetDesc(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("hidden", C.c_int32 * 2), ("preprocess", C.c_int32),
                ("n_in", C.c_int32), ("fc_dim", C.c_int32), ("logsign_k", C.c_float), ("scale", C.c_float),
                ("tanh_output", C.c_int32)]


_fp = C.c_void_p


class StepArgs(C.Structure):
    _fields_ = [("n", C.c_int64), ("theta", _fp), ("in0", _fp), ("in1", _fp), ("m", _fp), ("v", _fp),
                ("beta1", C.c_float), ("beta2", C.c_float), ("p", C.c_float), ("state_in", _fp),
                ("state_out", _fp), ("x", _fp), ("delta", _fp), ("feat_out", _fp), ("step_ptr", _fp), ("t_offset", C.c_int32),
                ("reuse_weights", C.c_int32)]


class UnrollArgs(C.Structure):
    _fields_ = [("n", C.c_int64), ("T", C.c_int32), ("theta", _fp), ("in_seq", _fp), ("opt_kind", C.c_int32),
                ("opt_a", _fp), ("opt_b", _fp), ("opt_alpha", C.c_float), ("opt_fscale", C.c_float), ("x", _fp),
                ("state", _fp), ("ckpt", _fp), ("m", _fp), ("v", _fp), ("beta1", C.c_float), ("beta2", C.c_float),
                ("step0", C.c_int32), ("g_rec", _fp), ("feat_rec", _fp), ("fx", _fp), ("delta_seq", _fp),
                ("labels", _fp), ("imit_loss", _fp), ("n_total", C.c_int64), ("opt_group", C.c_int32)]


class BwdArgs(C.Structure):
    _fields_ = [("n", C.c_int64), ("T", C.c_int32), ("theta", _fp), ("in_seq", _fp), ("ckpt", _fp), ("g_rec", _fp),
                ("labels", _fp), ("n_total", C.c_int64), ("dtheta", _fp), ("delta_seq", _fp), ("scratch", _fp)]


class BwdCarry(C.Structure):
    _fields_ = [("d_state", _fp), ("lam", _fp)]


class LassoArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("m", C.c_int32), ("n", C.c_int32), ("A", _fp), ("y", _fp), ("x", _fp),
                ("scale", _fp), ("l1", C.c_float), ("g", _fp), ("f", _fp)]


class ConfocalArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_points", C.c_int32), ("roi", C.c_int32 * 3), ("x", _fp), ("sim", _fp),
                ("scale", _fp), ("g", _fp), ("f", _fp)]


class MnistArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_examples", C.c_int32), ("n_layers", C.c_int32), ("hidden", C.c_int32 * 4),
                ("activation", C.c_int32), ("seed", C.c_uint64), ("counter", _fp), ("images", _fp), ("labels", _fp),
                ("x", _fp), ("scale", _fp), ("g", _fp), ("f", _fp), ("idx_out", _fp)]


MNIST_INPUT, MNIST_CLASSES, MNIST_MAX_HIDDEN, MNIST_MAX_WIDTH, MNIST_MAX_BATCH = 784, 10, 4, 64, 1024
MNIST_SIGMOID, MNIST_RELU = 0, 1


class MnistConvArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_examples", C.c_int32), ("seed", C.c_uint64), ("counter", _fp),
                ("images", _fp), ("labels", _fp), ("x", _fp), ("scale", _fp), ("g", _fp), ("f", _fp), ("idx_out", _fp),
                ("workspace", _fp), ("workspace_bytes", C.c_size_t)]


MNIST_CONV_COORDS, MNIST_CONV_MAX_BATCH, MNIST_CONV_LAYOUT = 18122, 1024, 4


class CifarConvArgs(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_examples", C.c_int32), ("seed", C.c_uint64), ("counter", _fp),
                ("images", _fp), ("labels", _fp), ("x", _fp), ("scale", _fp), ("g", _fp), ("f", _fp), ("idx_out", _fp),
                ("workspace", _fp), ("workspace_bytes", C.c_size_t)]


CIFAR_INPUT = 3 * 32 * 32
CIFAR_CONV_COORDS, CIFAR_CONV_MAX_BATCH, CIFAR_CONV_LAYOUT = 13610, 1024, 4


class NasArgs(C.Structure):
    _fields_ = CifarConvArgs._fields_


NAS_COORDS, NAS_MAX_BATCH, NAS_LAYOUT = 7578, 1024, 6


class DenseDesc(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("hidden", C.c_int32 * 2), ("n_in", C.c_int32), ("preprocess", C.c_int32),
                ("logsign_k", C.c_float), ("n_out", C.c_int32), ("scale", C.c_float), ("tanh_output", C.c_int32)]


class DenseStepArgs(C.Structure):
    _fields_ = [("rows", C.c_int64), ("theta", _fp), ("in_", _fp), ("state_in", _fp), ("state_out", _fp), ("x", _fp),
                ("delta", _fp)]


class DenseBwdArgs(C.Structure):
    _fields_ = [("rows", C.c_int64), ("T", C.c_int32), ("theta", _fp), ("in_seq", _fp), ("ckpt", _fp), ("g_rec", _fp),
                ("labels", _fp), ("n_total", C.c_int64), ("dtheta", _fp)]


class HrnnArgs(C.Structure):
    _fields_ = [("theta", _fp), ("x", _fp), ("g", _fp), ("state", _fp), ("layer", _fp), ("global_", _fp),
                ("workspace", _fp), ("update", _fp)]


class HrnnBwdArgs(C.Structure):
    _fields_ = [("theta", _fp), ("state_old", _fp), ("g", _fp), ("bias0", _fp), ("zero_flag", _fp), ("mean_log_lr", _fp),
                ("d_state_new", _fp), ("d_upd", _fp), ("d_sums", _fp), ("d_state_old", _fp), ("d_theta", _fp),
                ("d_bias0", _fp), ("d_mean_log_lr", _fp), ("d_g", _fp)]


class CrnnStepArgs(C.Structure):
    _fields_ = [("n", C.c_int64), ("theta", _fp), ("g", _fp), ("state_in", _fp), ("state_out", _fp), ("x", _fp),
                ("update", _fp)]


class CrnnBwdArgs(C.Structure):
    _fields_ = [("n", C.c_int64), ("theta", _fp), ("g", _fp), ("state_old", _fp), ("d_state_new", _fp),
                ("d_update", _fp), ("d_state_old", _fp), ("d_theta", _fp), ("d_g", _fp)]


class TadamStepArgs(C.Structure):
    _fields_ = [("n", C.c_int64), ("theta", _fp), ("g", _fp), ("state_in", _fp), ("state_out", _fp), ("x", _fp),
                ("update", _fp)]


class TadamBwdArgs(C.Structure):
    _fields_ = [("n", C.c_int64), ("theta", _fp), ("g", _fp), ("state_old", _fp), ("d_state_new", _fp),
                ("d_update", _fp), ("d_state_old", _fp), ("d_theta", _fp), ("d_g", _fp)]


class LrsgdStepArgs(C.Structure):
    _fields_ = [("n", C.c_int64), ("rates", _fp), ("n_steps", C.c_int32), ("itr", _fp), ("g", _fp), ("x", _fp),
                ("update", _fp)]


class LrsgdBwdArgs(C.Structure):
    _fields_ = [("n", C.c_int64), ("rates", _fp), ("n_steps", C.c_int32), ("itr", _fp), ("g", _fp),
                ("d_update", _fp), ("d_rates", _fp), ("d_g", _fp)]


class IstaArgs(C.Structure):
    _fields_ = [("form", C.c_int32), ("batch", C.c_int32), ("m", C.c_int32), ("n", C.c_int32),
                ("num_layers", C.c_int32), ("k0", C.c_int32), ("k1", C.c_int32), ("share_W", C.c_int32),
                ("A", _fp), ("B1", _fp), ("W", _fp), ("theta", _fp), ("step", _fp), ("ss_rank", _fp), ("y", _fp),
                ("ldy", C.c_int64), ("x_in", _fp), ("xs", _fp), ("zs", _fp), ("rs", _fp), ("sel", _fp),
                ("W2", _fp), ("s2_in", _fp), ("rowrec", _fp)]


class IstaGrads(C.Structure):
    _fields_ = [("d_xk", _fp), ("d_x_in", _fp), ("dW", _fp), ("dB1", _fp), ("dtheta", _fp), ("dstep", _fp),
                ("gscale", _fp), ("scratch", _fp), ("dW2", _fp), ("d_s2", _fp), ("d_s2_in", _fp)]


class IstaLossArgs(C.Structure):
    _fields_ = [("task", C.c_int32), ("batch", C.c_int32), ("m", C.c_int32), ("n", C.c_int32), ("A", _fp),
                ("y", _fp), ("ldy", C.c_int64), ("x_true", _fp), ("ldx", C.c_int64), ("x", _fp), ("lam", C.c_float),
                ("d_x", _fp), ("loss", _fp)]


class MinimaxArgs(C.Structure):
    _fields_ = [("loss", C.c_int32), ("batch", C.c_int32), ("dim", C.c_int32), ("hidden", C.c_int32),
                ("t0", C.c_int32), ("t1", C.c_int32), ("warm_end", C.c_int32), ("out_mul", C.c_float),
                ("rescale", C.c_float), ("lr", _fp), ("theta", _fp), ("image", _fp), ("data", _fp), ("u", _fp),
                ("v", _fp), ("state", _fp), ("traj", _fp), ("ckpt", _fp), ("dl", _fp), ("lval", _fp)]


class MinimaxGrads(C.Structure):
    _fields_ = [("coef", _fp), ("weight", _fp), ("dtheta", _fp), ("scratch", _fp)]


class ZooArgs(C.Structure):
    _fields_ = [("family", C.c_int32), ("n", C.c_int32), ("rows", C.c_int32), ("p0", C.c_float), ("x", _fp),
                ("v", _fp), ("A", _fp), ("y", _fp), ("c", _fp), ("f", _fp), ("out", _fp)]


class ZooFormArgs(C.Structure):
    _fields_ = [("base", ZooArgs), ("k", C.c_int32), ("U", _fp), ("V", _fp), ("q", _fp)]


ZOO_MAX_N = 4096
ZOO_MAX_PAIRS = 10
ZOO_FAMILIES = ["QUADRATIC", "LASSO", "RASTRIGIN", "BOWL", "NORM", "PROJECTION_QUADRATIC", "SUM_OF_QUADRATICS",
                "OUTWARD_SNAKE", "ISOTROPIC_QUADRATIC", "DEPENDENCY_CHAIN", "MIN_MAX_WELL", "ROSENBROCK", "SADDLE",
                "LOGSUMEXP", "ACKLEY", "BEALE", "BOOTH", "STYBLINSKI_TANG", "MATYAS", "BRANIN", "MICHALEWICZ"]
ZOO = {name: i for i, name in enumerate(ZOO_FAMILIES)}   # the L2O_ZOO_* family ids


class L2OError(RuntimeError):
    pass


ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]   # H100 (Hopper); the kernels use wgmma / TMA (sm_90a only)
NVCC_FLAGS = ARCH + ["-std=c++17", "-O3", "-lineinfo", "-I" + INCLUDE, "-I" + CSRC, "-Xcompiler", "-fPIC"]
OBJ_DIR = os.path.join(_ROOT, "build", "obj")


def translation_units():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cu")]


def sources():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h"))] + \
           [os.path.join(INCLUDE, "l2o_b200.h")]


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA translation unit in-tree for sm_90a (nvcc cross-compiles without a GPU) and link
    ``libl2o_b200.so``.  Objects are rebuilt only when a source/header is newer."""
    from concurrent.futures import ThreadPoolExecutor
    os.makedirs(OBJ_DIR, exist_ok=True)
    newest_hdr = max(os.path.getmtime(p) for p in sources() if not p.endswith(".cu"))
    jobs = []
    for tu in translation_units():
        obj = os.path.join(OBJ_DIR, os.path.basename(tu)[:-3] + ".o")
        stale = force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(tu), newest_hdr)
        jobs.append((tu, obj, stale))

    def compile_one(job):
        tu, obj, stale = job
        if not stale:
            return None
        cmd = ["nvcc"] + NVCC_FLAGS + ["-c", "-o", obj, tu]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise L2OError("nvcc failed for %s:\n%s%s" % (tu, r.stdout, r.stderr))
        return obj

    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        rebuilt = [o for o in ex.map(compile_one, jobs) if o]
    objs = [j[1] for j in jobs]
    if rebuilt or not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < max(os.path.getmtime(o) for o in objs):
        cmd = ["nvcc"] + ARCH + ["-shared", "-o", LIB_PATH] + objs
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise L2OError("link failed:\n" + r.stdout + r.stderr)
    return LIB_PATH


_lib = None


def lib():
    """Load the shared library (fails loudly if it was never built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise L2OError(f"{LIB_PATH} not found - run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no CPU/PyTorch fallback)")
    L = C.CDLL(LIB_PATH)
    L.l2o_net_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(NetDesc)]
    L.l2o_net_create.restype = C.c_int
    L.l2o_net_destroy.argtypes = [C.c_void_p]
    L.l2o_net_destroy.restype = None
    L.l2o_net_set_engine.argtypes = [C.c_void_p, C.c_int32]
    L.l2o_net_set_engine.restype = C.c_int
    L.l2o_theta_count.argtypes = [C.c_void_p]
    L.l2o_theta_count.restype = C.c_int64
    L.l2o_state_floats.argtypes = [C.c_void_p]
    L.l2o_state_floats.restype = C.c_int64
    L.l2o_workspace_bytes.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    L.l2o_workspace_bytes.restype = C.c_int
    L.l2o_step.argtypes = [C.c_void_p, C.POINTER(StepArgs), C.c_void_p]
    L.l2o_step.restype = C.c_int
    L.l2o_unroll_fwd.argtypes = [C.c_void_p, C.POINTER(UnrollArgs), C.c_void_p]
    L.l2o_unroll_fwd.restype = C.c_int
    L.l2o_unroll_bwd.argtypes = [C.c_void_p, C.POINTER(BwdArgs), C.c_void_p]
    L.l2o_unroll_bwd.restype = C.c_int
    L.l2o_unroll_bwd_carry.argtypes = [C.c_void_p, C.POINTER(BwdArgs), C.POINTER(BwdCarry), C.c_void_p]
    L.l2o_unroll_bwd_carry.restype = C.c_int
    L.l2o_tc_fwd_variant.argtypes = [C.c_void_p, C.POINTER(UnrollArgs)]
    L.l2o_tc_fwd_variant.restype = C.c_int
    L.l2o_tc_weight_image.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    L.l2o_tc_weight_image.restype = C.c_int64
    L.l2o_adam_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float,
                                C.c_float, C.c_float, C.c_float, C.c_void_p]
    L.l2o_adam_step.restype = C.c_int
    L.l2o_log_and_sign.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p]
    L.l2o_log_and_sign.restype = C.c_int
    L.l2o_lasso_grad.argtypes = [C.POINTER(LassoArgs), C.c_void_p]
    L.l2o_lasso_grad.restype = C.c_int
    L.l2o_confocal_grad.argtypes = [C.POINTER(ConfocalArgs), C.c_void_p]
    L.l2o_confocal_grad.restype = C.c_int
    L.l2o_mnist_grad.argtypes = [C.POINTER(MnistArgs), C.c_void_p]
    L.l2o_mnist_grad.restype = C.c_int
    L.l2o_mnist_conv_workspace_bytes.argtypes = [C.c_int32]
    L.l2o_mnist_conv_workspace_bytes.restype = C.c_int64
    L.l2o_mnist_conv_workspace_layout.argtypes = [C.c_int32, C.POINTER(C.c_int64)]
    L.l2o_mnist_conv_workspace_layout.restype = C.c_int
    L.l2o_mnist_conv_grad.argtypes = [C.POINTER(MnistConvArgs), C.c_void_p]
    L.l2o_mnist_conv_grad.restype = C.c_int
    L.l2o_cifar_conv_workspace_bytes.argtypes = [C.c_int32]
    L.l2o_cifar_conv_workspace_bytes.restype = C.c_int64
    L.l2o_cifar_conv_workspace_layout.argtypes = [C.c_int32, C.POINTER(C.c_int64)]
    L.l2o_cifar_conv_workspace_layout.restype = C.c_int
    L.l2o_cifar_conv_grad.argtypes = [C.POINTER(CifarConvArgs), C.c_void_p]
    L.l2o_cifar_conv_grad.restype = C.c_int
    L.l2o_nas_workspace_bytes.argtypes = [C.c_int32]
    L.l2o_nas_workspace_bytes.restype = C.c_int64
    L.l2o_nas_workspace_layout.argtypes = [C.c_int32, C.POINTER(C.c_int64)]
    L.l2o_nas_workspace_layout.restype = C.c_int
    L.l2o_nas_grad.argtypes = [C.POINTER(NasArgs), C.c_void_p]
    L.l2o_nas_grad.restype = C.c_int
    L.l2o_dense_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(DenseDesc)]
    L.l2o_dense_create.restype = C.c_int
    L.l2o_dense_destroy.argtypes = [C.c_void_p]
    L.l2o_dense_destroy.restype = None
    for name in ("l2o_dense_theta_count", "l2o_dense_state_floats"):
        getattr(L, name).argtypes = [C.c_void_p]
        getattr(L, name).restype = C.c_int64
    L.l2o_dense_step.argtypes = [C.c_void_p, C.POINTER(DenseStepArgs), C.c_void_p]
    L.l2o_dense_step.restype = C.c_int
    L.l2o_dense_unroll_bwd.argtypes = [C.c_void_p, C.POINTER(DenseBwdArgs), C.c_void_p]
    L.l2o_dense_unroll_bwd.restype = C.c_int
    L.l2o_launch_count.argtypes = []
    L.l2o_launch_count.restype = C.c_int64
    L.l2o_hrnn_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32]
    L.l2o_hrnn_create.restype = C.c_int
    L.l2o_hrnn_destroy.argtypes = [C.c_void_p]
    L.l2o_hrnn_destroy.restype = None
    L.l2o_hrnn_theta_count.argtypes = []
    L.l2o_hrnn_theta_count.restype = C.c_int64
    L.l2o_hrnn_state_floats.argtypes = []
    L.l2o_hrnn_state_floats.restype = C.c_int64
    for name in ("l2o_hrnn_coords", "l2o_hrnn_workspace_bytes"):
        getattr(L, name).argtypes = [C.c_void_p]
        getattr(L, name).restype = C.c_int64
    L.l2o_hrnn_set_global_sizes.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    L.l2o_hrnn_set_global_sizes.restype = C.c_int
    L.l2o_hrnn_coord_bwd.argtypes = [C.c_void_p, C.POINTER(HrnnBwdArgs), C.c_void_p]
    L.l2o_hrnn_coord_bwd.restype = C.c_int
    L.l2o_hrnn_workspace_layout.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    L.l2o_hrnn_workspace_layout.restype = C.c_int
    for name in ("l2o_hrnn_init_state", "l2o_hrnn_prepare", "l2o_hrnn_step", "l2o_hrnn_prepare_local",
                 "l2o_hrnn_prepare_finish", "l2o_hrnn_step_local", "l2o_hrnn_step_finish"):
        getattr(L, name).argtypes = [C.c_void_p, C.POINTER(HrnnArgs), C.c_void_p]
        getattr(L, name).restype = C.c_int
    for name in ("l2o_crnn_theta_count", "l2o_crnn_state_floats"):
        getattr(L, name).argtypes = []
        getattr(L, name).restype = C.c_int64
    L.l2o_crnn_step.argtypes = [C.POINTER(CrnnStepArgs), C.c_void_p]
    L.l2o_crnn_step.restype = C.c_int
    L.l2o_crnn_bwd.argtypes = [C.POINTER(CrnnBwdArgs), C.c_void_p]
    L.l2o_crnn_bwd.restype = C.c_int
    for name in ("l2o_tadam_theta_count", "l2o_tadam_state_floats"):
        getattr(L, name).argtypes = []
        getattr(L, name).restype = C.c_int64
    for name, args in (("l2o_tadam_step", TadamStepArgs), ("l2o_tadam_bwd", TadamBwdArgs),
                       ("l2o_lrsgd_step", LrsgdStepArgs), ("l2o_lrsgd_bwd", LrsgdBwdArgs)):
        getattr(L, name).argtypes = [C.POINTER(args), C.c_void_p]
        getattr(L, name).restype = C.c_int
    L.l2o_ista_workspace_bytes.argtypes = [C.POINTER(IstaArgs), C.POINTER(C.c_size_t)]
    L.l2o_ista_fwd.argtypes = [C.POINTER(IstaArgs), C.c_void_p]
    L.l2o_ista_bwd.argtypes = [C.POINTER(IstaArgs), C.POINTER(IstaGrads), C.c_void_p]
    L.l2o_ista_loss_grad.argtypes = [C.POINTER(IstaLossArgs), C.c_void_p]
    for name in ("l2o_ista_workspace_bytes", "l2o_ista_fwd", "l2o_ista_bwd", "l2o_ista_loss_grad"):
        getattr(L, name).restype = C.c_int
    for name in ("l2o_minimax_theta_count", "l2o_minimax_image_floats"):
        getattr(L, name).argtypes = [C.c_int32]
        getattr(L, name).restype = C.c_int64
    L.l2o_minimax_image.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    L.l2o_minimax_workspace_bytes.argtypes = [C.POINTER(MinimaxArgs), C.POINTER(C.c_size_t)]
    L.l2o_minimax_fwd.argtypes = [C.POINTER(MinimaxArgs), C.c_void_p]
    L.l2o_minimax_bwd.argtypes = [C.POINTER(MinimaxArgs), C.POINTER(MinimaxGrads), C.c_void_p]
    for name in ("l2o_minimax_image", "l2o_minimax_workspace_bytes", "l2o_minimax_fwd", "l2o_minimax_bwd"):
        getattr(L, name).restype = C.c_int
    for name in ("l2o_zoo_value_grad", "l2o_zoo_hvp"):
        getattr(L, name).argtypes = [C.POINTER(ZooArgs), C.c_void_p]
        getattr(L, name).restype = C.c_int
    L.l2o_zoo_hess_form.argtypes = [C.POINTER(ZooFormArgs), C.c_void_p]
    L.l2o_zoo_hess_form.restype = C.c_int
    for name in ("l2o_status_string", "l2o_last_cuda_error", "l2o_version"):
        getattr(L, name).restype = C.c_char_p
    L.l2o_status_string.argtypes = [C.c_int]
    _lib = L
    return L


def check(rc: int, what: str):
    if rc != L2O_OK:
        L = lib()
        msg = L.l2o_status_string(rc).decode()
        if rc == L2O_E_CUDA:
            msg += ": " + L.l2o_last_cuda_error().decode()
        raise L2OError(f"{what} failed: {msg} ({rc})")
