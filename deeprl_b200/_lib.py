"""ctypes binding of ``libb2rl.so`` (C ABI declared in ``include/b2rl.h``).

The library is the product: there is NO CPU / eager fallback.  If the shared object is missing or a
symbol cannot be resolved the import of any device-side component fails loudly with the build command.
PyTorch is used for device memory and streams only: every call receives raw ``data_ptr()`` addresses
and ``torch.cuda.current_stream().cuda_stream``.
"""
import ctypes
import os
import subprocess
import sys

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(CSRC, "libb2rl.so")
SOURCES = ["core.cu", "replay.cu", "sumtree.cu", "losses.cu", "onpolicy.cu", "optim.cu", "dense.cu", "gemm.cu", "pack.cu", "head.cu", "tail.cu", "disthead.cu", "actor.cu", "ppo_persistent.cu", "a2c.cu", "dist_dqn.cu", "rainbow.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]

c_p, c_i32, c_i64, c_u64, c_f32, c_f64 = (ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64,
                                          ctypes.c_float, ctypes.c_double)

# name -> argtypes, in the order of include/b2rl.h
SIGNATURES = {
    "b2rl_replay_feed": [c_p, c_p, c_p, c_p, c_p, c_i64, c_p, c_p, c_p, c_p, c_i32, c_i32, c_p],
    "b2rl_replay_select_uniform": [c_p, c_p, c_i32, c_u64, c_i32, c_i32, c_i32, c_p, c_p, c_p],
    "b2rl_replay_select_uniform_scalars": [c_p, c_p, c_i32, c_u64, c_i32, c_i32, c_i32, c_p, c_p, c_p, c_p, c_p, c_f64, c_p,
                                           c_p, c_p, c_p],
    "b2rl_replay_gather": [c_p, c_p, c_p, c_p, c_i64, c_i64, c_p, c_i32, c_i32, c_i32, c_f64, c_p, c_i32, c_i32, c_i32,
                           c_p, c_p, c_p, c_p, c_p, c_p],
    "b2rl_sumtree_add": [c_p, c_p, c_i64, c_p, c_p, c_i32, c_p, c_p],
    "b2rl_sumtree_sample": [c_p, c_p, c_i64, c_p, c_p, c_p, c_u64, c_i32, c_i32, c_i32, c_p, c_p, c_p, c_p, c_p],
    "b2rl_sumtree_get": [c_p, c_p, c_i64, c_p, c_i32, c_p, c_p, c_p],
    "b2rl_sumtree_update": [c_p, c_p, c_i64, c_p, c_p, c_i32, c_p, c_p, c_p],
    "b2rl_dqn_loss": [c_p, c_p, c_p, c_p, c_p, c_p, c_f32, c_i32, c_i32, c_p, c_f32, c_f32, c_f32, c_p, c_p, c_p, c_p,
                      c_p, c_p],
    "b2rl_c51_loss": [c_p, c_p, c_p, c_p, c_p, c_p, c_f32, c_f32, c_f32, c_i32, c_i32, c_i32, c_p, c_f32, c_f32, c_f32,
                      c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    "b2rl_qr_loss": [c_p, c_p, c_p, c_p, c_p, c_f32, c_f32, c_i32, c_i32, c_i32, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    "b2rl_nstep_q_loss_ctas": [c_i32],
    "b2rl_nstep_q_loss": [c_p, c_p, c_p, c_p, c_p, c_f32, c_i32, c_i32, c_i32, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    "b2rl_gae": [c_p, c_p, c_p, c_f32, c_f32, c_i32, c_i32, c_i32, c_i32, c_p, c_p, c_p],
    "b2rl_normalize_advantage": [c_p, c_i32, c_p],
    "b2rl_ppo_loss": [c_p, c_p, c_p, c_p, c_p, c_p, c_f32, c_f32, c_i32, c_p, c_p, c_p, c_p, c_p],
    "b2rl_a2c_loss": [c_p, c_p, c_p, c_p, c_p, c_f32, c_f32, c_i32, c_p, c_p, c_p, c_p, c_p],
    "b2rl_ppo_rollout_prep": [c_p, c_p, c_p, c_p, c_f32, c_f32, c_i32, c_i32, c_i32, c_i32, c_p, c_p, c_p, c_p],
    "b2rl_ppo_cat_loss_ctas": [c_i32],
    "b2rl_ppo_cat_loss": [c_p, c_p, c_p, c_p, c_p, c_p, c_f32, c_f32, c_i32, c_i32, c_p, c_p, c_p, c_p, c_p],
    "b2rl_a2c_rollout_loss_ctas": [c_i32],
    "b2rl_a2c_rollout_loss": [c_p, c_p, c_p, c_p, c_f32, c_f32, c_i32, c_f32, c_f32, c_i32, c_i32, c_i32, c_p, c_p, c_p, c_p, c_p,
                              c_p, c_p],
    "b2rl_bias_act_bf16": [c_p, c_p, c_i64, c_i32, c_i32, c_p],
    "b2rl_bias_act_f32_to_bf16": [c_p, c_p, c_p, c_i64, c_i32, c_i32, c_p],
    "b2rl_act_bwd_bias_grad_bf16": [c_p, c_p, c_i64, c_i32, c_i32, c_p, c_p, c_p, c_p, c_i32, c_i32, c_i32, c_p],
    "b2rl_set_cta_budget": [c_i32],
    "b2rl_last_grid_ctas": [c_p],
    "b2rl_conv_gemm_bf16": [c_i32, c_p, c_i64, c_i32, c_p, c_i32, c_i32, c_i32, c_i32, c_i32, c_p, c_i64, c_p, c_i32, c_i32,
                            c_i32, c_i32, c_i32, c_i32, c_i32, c_p],
    "b2rl_conv_gemm_dual_bf16": [c_p, c_p, c_i64, c_i32, c_p, c_p, c_i32, c_i32, c_i32, c_i32, c_i32, c_p, c_p, c_i64, c_p, c_p,
                                 c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_p],
    "b2rl_gemm_dual_bf16": [c_p, c_p, c_i64, c_p, c_p, c_i64, c_p, c_p, c_i64, c_i32, c_i32, c_i32, c_p, c_p, c_i32, c_i32,
                            c_i32, c_p],
    "b2rl_conv_gemm_bwd_bf16": [c_p, c_i64, c_i32, c_p, c_i32, c_i32, c_i32, c_i32, c_p, c_i64, c_i32, c_i32, c_i32, c_p, c_i32, c_p],
    "b2rl_gemm_bwd_bf16": [c_p, c_i64, c_p, c_i32, c_i64, c_p, c_i64, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_p, c_i32, c_p],
    "b2rl_gemm_bf16": [c_p, c_i32, c_i64, c_p, c_i32, c_i64, c_p, c_i64, c_i32, c_i32, c_i32, c_p, c_i32, c_i32, c_i32, c_i32,
                       c_p],
    "b2rl_conv1_u8_fwd": [c_p, c_i64, c_p, c_i32, c_i64, c_i32, c_i32, c_i32, c_p, c_i32, c_p, c_i64, c_p, c_i32, c_i32, c_i32, c_p],
    "b2rl_conv1_u8_wgrad_partials": [c_p, c_i64, c_p, c_i32, c_i64, c_i32, c_i32, c_i32, c_p, c_i32, c_p, c_p, c_p],
    "b2rl_conv1_wgrad_partials": [c_p, c_i64, c_i32, c_p, c_i32, c_p, c_p, c_p],
    "b2rl_conv1_u8_fwd_pair": [c_p, c_i64, c_p, c_i32, c_i64, c_i32, c_i32, c_i32, c_p, c_p, c_p, c_p, c_i64, c_p, c_p, c_i32,
                               c_i32, c_i32, c_p],
    "b2rl_conv1_set_phase_clocks": [c_p],
    "b2rl_gemm_splitk_bf16": [c_p, c_i64, c_p, c_i64, c_p, c_i64, c_i32, c_i32, c_i32, c_p, c_i32, c_i32, c_i32, c_p],
    "b2rl_nature_pack_weights": [c_p, c_p, c_p, c_p, c_i32, c_i32, c_f32, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    "b2rl_nature_unpack_grads": [c_p] * 8 + [c_i32, c_i32, c_f32] + [c_p] * 8 + [c_i32, c_i32, c_i32, c_p],
    "b2rl_conv_taps_wgrad_partials": [c_p, c_i64, c_i32, c_p, c_i32, c_i32, c_i32, c_i32, c_p, c_p, c_p],
    "b2rl_head_fwd": [c_p, c_p, c_p, c_p, c_p, c_i32, c_i32, c_i32, c_p, c_p],
    "b2rl_head_bwd": [c_p, c_p, c_p, c_p, c_i32, c_i32, c_i32, c_p, c_p, c_p, c_p, c_p, c_p],
    "b2rl_head_bwd_relu": [c_p, c_p, c_p, c_p, c_i32, c_i32, c_i32, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    "b2rl_ac_head_fwd": [c_p, c_p, c_p, c_p, c_p, c_i32, c_i32, c_i32, c_p, c_u64, c_p, c_p, c_p, c_p],
    "b2rl_head_bwd_geff_relu": [c_p, c_p, c_p, c_p, c_i32, c_i32, c_i32, c_p, c_p, c_p, c_p, c_p, c_p, c_p],
    "b2rl_nature_grad_reduce": [c_p, c_i32, c_p, c_i32, c_p, c_i32, c_p, c_i32, c_p, c_p, c_p, c_p, c_p, c_i32, c_i32, c_f32, c_p,
                                c_p, c_p, c_p, c_f32, c_f32, c_p],
    "b2rl_nature_fused_opt": [c_p, c_i32, c_p, c_p, c_p, c_p, c_i32, c_f32, c_f32, c_f32, c_f32, c_f32, c_f32, c_p, c_i32, c_p,
                              c_p, c_i32, c_i32, c_f32, c_p, c_p, c_p, c_p, c_p, c_p, c_i32, c_p, c_p],
    "b2rl_nature_fused_opt_lr": [c_p, c_i32, c_p, c_p, c_p, c_p, c_i32, c_f32, c_p, c_f32, c_f32, c_f32, c_f32, c_f32, c_p, c_i32,
                                 c_p, c_p, c_i32, c_i32, c_f32, c_p, c_p, c_p, c_p, c_p, c_p, c_i32, c_p, c_p],
    "b2rl_gaussian_actor_step": [c_p, c_p, c_p, c_p, c_i32, c_f64, c_f64] + [c_p] * 13 + [c_i32] * 5 + [c_p, c_u64, c_p, c_p] + [c_p] * 6 + [c_p],
    "b2rl_ppo_set_phase_clocks": [c_p],
    "b2rl_ppo_minibatch_updates": [c_p] * 5 + [c_i32] * 5 + [c_p, c_i32] + [c_p] * 10 + [c_f32] * 11 + [c_p, c_p],
    "b2rl_ppo_minibatch_updates_dp": ([c_p] * 5 + [c_i32] * 5 + [c_p, c_i32] + [c_p] * 10 + [c_f32] * 11 + [c_p]
                                      + [c_i32] * 5 + [c_p, c_i64, c_i64, c_p, c_i32, c_p]),
    "b2rl_a2c_smem_bytes": [c_i32] * 8,
    "b2rl_a2c_actor_step": [c_i32, c_i32, c_i32, c_p, c_f64, c_p, c_p] + [c_i32] * 5 + [c_p, c_p, c_p, c_u64, c_p, c_p],
    "b2rl_a2c_update": [c_i32, c_i32, c_i32] + [c_p] * 4 + [c_i32] * 6 + [c_p] * 5 + [c_f32] * 3 + [c_i32] + [c_f32] * 2
                       + [c_i32] + [c_f32] * 3 + [c_p, c_p],
    "b2rl_nstep_dqn_smem_bytes": [c_i32] * 6,
    "b2rl_nstep_dqn_actor_step": [c_i32, c_p, c_f64, c_p, c_p] + [c_i32] * 5 + [c_f32, c_p, c_p, c_p, c_u64, c_p, c_p],
    "b2rl_nstep_dqn_update": ([c_i32] + [c_p] * 4 + [c_i32] * 6 + [c_p, c_p, c_i32] + [c_p] * 4 + [c_f32] * 3 + [c_i32]
                              + [c_f32] * 2 + [c_p, c_p]),
    "b2rl_dqn_replay_smem_bytes": [c_i32] * 7,
    "b2rl_dqn_replay_update": ([c_i32, c_i32, c_p, c_p, c_i32, c_f64, c_p, c_p, c_p] + [c_i32] * 5 + [c_p] * 6 + [c_f32] * 3
                               + [c_i32, c_f32, c_i32, c_f32, c_p] + [c_f32] * 3 + [c_p] * 4),
    "b2rl_dist_dqn_smem_bytes": [c_i32] * 8,
    "b2rl_dist_dqn_actor_step": [c_i32, c_i32, c_p, c_f64, c_p, c_p] + [c_i32] * 6 + [c_f64, c_f64, c_f32, c_p, c_p, c_u64, c_p,
                                                                                       c_p],
    "b2rl_dist_dqn_replay_update": ([c_i32, c_i32, c_p, c_p, c_i32, c_f64, c_p, c_p, c_p] + [c_i32] * 6 + [c_p] * 6
                                    + [c_f32] * 3 + [c_i32, c_f32, c_i32, c_f64, c_f64, c_f32, c_p] + [c_f32] * 3 + [c_p] * 4),
    "b2rl_rainbow_smem_bytes": [c_i32] * 8,
    "b2rl_rainbow_actor_step": [c_i32, c_i32, c_p, c_f64, c_p, c_p] + [c_i32] * 6 + [c_f64, c_f64, c_f32, c_p, c_p, c_u64, c_p,
                                                                                      c_f32, c_p, c_p, c_p, c_p],
    "b2rl_rainbow_replay_update": ([c_i32, c_i32, c_p, c_p, c_i32, c_f64, c_p, c_p, c_p] + [c_i32] * 6 + [c_p] * 6
                                   + [c_f32] * 3 + [c_i32, c_f32, c_i32, c_f64, c_f64, c_f32, c_p] + [c_f32] * 3 + [c_p] * 3
                                   + [c_u64, c_f32] + [c_p] * 5),
    "b2rl_ipc_alloc": [c_i64, c_p],
    "b2rl_ipc_get_handle": [c_p, c_p],
    "b2rl_ipc_open_handle": [c_p, c_p],
    "b2rl_ipc_close": [c_p],
    "b2rl_ipc_free": [c_p],
    "b2rl_peer_access_ok": [c_i32, c_i32, c_p],
    "b2rl_dist_softmax": [c_p, c_i32, c_i32, c_p, c_p, c_p],
    "b2rl_dist_head_bwd_prep": [c_p, c_p, c_i32, c_i32, c_i32, c_p, c_i32, c_p, c_p],
    "b2rl_grad_norm": [c_p, c_i64, c_f32, c_f32, c_p, c_p],
    "b2rl_dqn_head_fused": [c_p] * 14 + [c_f32, c_i32, c_i32, c_i32, c_p, c_f32, c_p, c_f32, c_f32] + [c_p] * 12,
    "b2rl_dqn_head_two": [c_p] * 14 + [c_f32, c_i32, c_i32, c_i32, c_p, c_f32, c_p, c_f32, c_f32] + [c_p] * 13,
    "b2rl_clip_rmsprop": [c_p, c_p, c_p, c_p, c_i64, c_f32, c_f32, c_f32, c_f32, c_i32, c_f32, c_p, c_p, c_p],
    "b2rl_clip_adam": [c_p, c_p, c_p, c_p, c_i64, c_f32, c_f32, c_f32, c_f32, c_f32, c_p, c_f32, c_p, c_p, c_p],
    "b2rl_clip_adam_gated": [c_p, c_p, c_p, c_p, c_i64, c_f32, c_f32, c_f32, c_f32, c_f32, c_p, c_f32, c_p, c_p, c_p, c_f32, c_p],
}

U8, F16, BF16, F32 = 0, 1, 2, 3
DTYPE_CODE = {torch.uint8: U8, torch.float16: F16, torch.bfloat16: BF16, torch.float32: F32}


class BwdEpilogue(ctypes.Structure):
    """``b2rl_bwd_epilogue`` of include/b2rl.h: ReLU-gradient mask, bias-gradient accumulator, scatter-map channel count."""
    _fields_ = [("mask", c_p), ("mask_ld", c_i64), ("dbias", c_p), ("dbias_mod", c_i32), ("sub_c", c_i32)]


def bwd_epilogue(mask, dbias, dbias_mod, sub_c=0):
    e = BwdEpilogue(ctypes.c_void_p(mask.data_ptr()), int(mask.stride(0)), ctypes.c_void_p(dbias.data_ptr()), int(dbias_mod),
                    int(sub_c))
    return e


class B2RLError(RuntimeError):
    pass


def build(verbose=False):
    """Compile csrc/*.cu into csrc/libb2rl.so for sm_90a (nvcc cross-compiles without a GPU)."""
    cmd = ["nvcc"] + NVCC_FLAGS + ["-o", LIB_PATH] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    subprocess.run(cmd, check=True, cwd=CSRC)
    return LIB_PATH


def _stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h", ".inc"))]
    deps.append(os.path.join(os.path.dirname(_HERE), "include", "b2rl.h"))
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B2RLError("libb2rl.so is not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(nvcc -gencode arch=compute_90a,code=sm_90a); there is no CPU fallback")
        L = ctypes.CDLL(LIB_PATH)
        L.b2rl_version.restype = ctypes.c_int
        L.b2rl_last_error.restype = ctypes.c_char_p
        L.b2rl_launch_count.restype = ctypes.c_int64
        L.b2rl_ppo_minibatch_smem_bytes.restype = ctypes.c_int64
        L.b2rl_ppo_minibatch_smem_bytes.argtypes = [ctypes.c_int32] * 5
        L.b2rl_ppo_dp_region_bytes.restype = ctypes.c_int64
        L.b2rl_ppo_dp_region_bytes.argtypes = [ctypes.c_int32] * 2
        L.b2rl_reset_launch_count.restype = None
        for name, args in SIGNATURES.items():
            fn = getattr(L, name)          # AttributeError here = header / library mismatch: fail loudly
            fn.argtypes = args
            fn.restype = ctypes.c_int
        L.b2rl_a2c_smem_bytes.restype = ctypes.c_int64       # (a size, not a status)
        L.b2rl_nstep_dqn_smem_bytes.restype = ctypes.c_int64
        L.b2rl_dqn_replay_smem_bytes.restype = ctypes.c_int64
        L.b2rl_dist_dqn_smem_bytes.restype = ctypes.c_int64
        L.b2rl_rainbow_smem_bytes.restype = ctypes.c_int64
        _lib = L
    return _lib


def ptr(t):
    """Device address of a tensor (None -> NULL)."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def call(name, *args):
    L = lib()
    rc = getattr(L, name)(*args)
    if rc != 0:
        raise B2RLError("%s failed (%d): %s" % (name, rc, L.b2rl_last_error().decode()))


def set_conv_slab(on):
    """Forward / dgrad convolution GEMMs: 2 = slab kernel (default), 0 = per-tap operand loads (csrc/gemm.cu)."""
    L = lib()
    L.b2rl_set_conv_slab.restype = None
    L.b2rl_set_conv_slab.argtypes = [ctypes.c_int32]
    L.b2rl_set_conv_slab(int(on))
    global CONV_SLAB
    CONV_SLAB = int(on)


CONV_SLAB = 2


def set_pdl(on):
    """Programmatic dependent launch of the per-update kernels (csrc/common.cuh); on by default."""
    L = lib()
    L.b2rl_set_pdl.restype = None
    L.b2rl_set_pdl.argtypes = [ctypes.c_int32]
    L.b2rl_set_pdl(int(on))


def launch_count():
    return int(lib().b2rl_launch_count())


def reset_launch_count():
    lib().b2rl_reset_launch_count()


def require_cuda(device):
    device = torch.device(device)
    if device.type != "cuda":
        raise B2RLError("the replay / loss kernels live in HBM and run on sm_90a: select a CUDA device "
                        "(select_device(0)); there is no CPU fallback")
    return device
