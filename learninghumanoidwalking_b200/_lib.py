"""ctypes binding of liblhw_b200.so (include/lhw_b200.h).  No fallback: if the CUDA library is missing the
import of any product module that needs it raises — the hot path never silently runs on the CPU."""
from __future__ import annotations

import ctypes
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
# LHW_B200_LIB points the binding at another build of the same library (tools/ab_variants.py times candidate kernels that way);
# it is still a CUDA build of include/lhw_b200.h and still mandatory
LIB_PATH = os.environ.get("LHW_B200_LIB") or os.path.join(_PKG, "liblhw_b200.so")

c_void_p, c_int, c_uint32, c_float, c_ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32, ctypes.c_float, ctypes.c_longlong

# name -> (restype, argtypes); mirrors include/lhw_b200.h one to one
SIGNATURES = {
    "lhw_version": (c_int, []),
    "lhw_last_error": (ctypes.c_char_p, []),
    "lhw_sim_create": (c_int, [ctypes.POINTER(c_void_p), c_void_p, c_int, c_int, c_int]),
    "lhw_sim_destroy": (c_int, [c_void_p]),
    "lhw_sim_state_reals": (c_int, [c_void_p]),
    "lhw_sim_state_ints": (c_int, [c_void_p]),
    "lhw_sim_obs_dim": (c_int, [c_void_p]),
    "lhw_sim_act_dim": (c_int, [c_void_p]),
    "lhw_sim_smem_bytes_per_env": (c_int, [c_void_p]),
    "lhw_sim_precision": (c_int, [c_void_p]),
    "lhw_sim_device": (c_int, [c_void_p]),
    "lhw_sim_reset": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, c_int, c_void_p, c_void_p]),
    "lhw_sim_step": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, c_int, c_int,
                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "lhw_sim_bind": (c_int, [c_void_p, c_void_p]),
    "lhw_sim_set_step_height": (c_int, [c_void_p, ctypes.c_double]),
    "lhw_sim_render": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int] + [ctypes.c_double] * 7
                       + [c_void_p, c_void_p]),
    "lhw_sim_eval_words": (c_int, []),
    "lhw_sim_eval_accumulate": (c_int, [c_void_p] * 3 + [c_int] + [c_void_p] * 5),
    "lhw_sim_push": (c_int, [c_void_p] * 3 + [c_int, c_uint32, c_uint32, c_void_p, ctypes.c_double, c_int, c_void_p, c_void_p]),
    "lhw_sim_set_command": (c_int, [c_void_p] * 3 + [c_int] + [c_void_p] * 4),
    "lhw_sim_command_words": (c_int, []),
    "lhw_sim_command_accumulate": (c_int, [c_void_p] * 2 + [c_int] + [c_void_p] * 3),
    "lhw_sim_footstep_limits": (c_int, [c_void_p] * 3),
    "lhw_sim_reset_footsteps": (c_int, [c_void_p] * 3 + [c_int, c_uint32, c_uint32, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "lhw_sim_reset_stairs": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, c_int, c_void_p, c_void_p,
                                     c_int, c_void_p]),
    "lhw_sim_step_stairs": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, c_int, c_int,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                    c_void_p]),
    "lhw_sim_step_delay": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, c_int, c_int,
                                   c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_int, c_void_p]),
    "lhw_sim_draw_delay": (c_int, [c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, c_int, c_void_p, c_void_p]),
    "lhw_sim_step_payload": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, c_int, c_int,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_int, c_void_p]),
    "lhw_sim_draw_payload": (c_int, [c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, ctypes.c_double, ctypes.c_double, c_void_p,
                                     c_void_p]),
    "lhw_sim_step_motor": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, c_int, c_int,
                                   c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "lhw_sim_draw_motor": (c_int, [c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, ctypes.c_double, c_void_p, c_void_p]),
    "lhw_sim_sense": (c_int, [c_void_p, c_void_p, c_int, c_uint32, c_uint32, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p,
                              c_void_p, c_void_p]),
    "lhw_launch_count": (c_ll, []),
    "lhw_gae": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_float, c_void_p,
                        c_void_p]),
    "lhw_gae_partial_words": (c_int, [c_int]),
    "lhw_adv_stats_from_gae": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "lhw_adv_stats_words": (c_int, []),
    "lhw_adv_stats": (c_int, [c_void_p, c_void_p, c_void_p, c_ll, c_void_p]),
    "lhw_adv_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_ll, c_float, c_void_p]),
    "lhw_ppo_loss_partial_words": (c_int, [c_int]),
    "lhw_ppo_loss": (c_int, [c_void_p] * 8 + [c_int, c_int, c_float, c_float, c_float] + [c_void_p] * 7),
    "lhw_ppo_loss_imitation": (c_int, [c_void_p] * 10 + [c_int, c_int, c_float, c_float, c_float, c_float] + [c_void_p] * 7),
    "lhw_gather_minibatch": (c_int, [c_void_p] * 9 + [c_int, c_int, c_int, c_void_p]),
    "lhw_grad_sumsq": (c_int, [c_void_p, c_void_p, c_ll, c_float, c_void_p]),
    "lhw_linear_wgrad_workspace_floats": (c_ll, [c_int, c_int, c_int]),
    "lhw_linear_wgrad": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "lhw_comm_last_error": (ctypes.c_char_p, []),
    "lhw_comm_handle_size": (c_int, []),
    "lhw_comm_create": (c_int, [ctypes.POINTER(c_void_p), c_ll, c_int, c_int, c_int]),
    "lhw_comm_grad_ptr": (c_void_p, [c_void_p]),
    "lhw_comm_size": (c_ll, [c_void_p]),
    "lhw_comm_device": (c_int, [c_void_p]),
    "lhw_comm_export": (c_int, [c_void_p, c_void_p]),
    "lhw_comm_import": (c_int, [c_void_p, c_void_p]),
    "lhw_comm_destroy": (c_int, [c_void_p]),
    "lhw_fused_allreduce_clip_adam": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_ll, c_float, c_float,
                                              c_float, c_float, c_float, c_void_p]),
    "lhw_comm_status": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "lhw_comm_set_step": (c_int, [c_void_p, c_int, c_void_p]),
    "lhw_fused_allreduce_clip_adam_adaptive": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_ll, c_void_p, c_void_p,
                                                       ctypes.c_double, c_float, c_float, c_float, c_float, c_void_p]),
    "lhw_comm_lr_ptr": (c_void_p, [c_void_p]),
    "lhw_comm_get_lr": (c_int, [c_void_p, c_void_p, c_void_p]),
    "lhw_comm_set_lr": (c_int, [c_void_p, ctypes.c_double, c_void_p]),
    "lhw_clip_adam_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_float, c_float, c_float,
                                  c_float, c_float, c_float, c_void_p]),
    "lhw_clip_adam": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_float, c_float, c_float,
                              c_float, c_float, c_float, c_void_p]),
}

_lib = None


class LhwError(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LhwError(
                f"{LIB_PATH} is missing: the CUDA extension has not been built (python -m learninghumanoidwalking_b200.build "
                "or __graft_entry__.build()). There is no CPU fallback for the rollout / PPO data path.")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


TORCH_LIB_PATH = os.path.join(_PKG, "liblhw_b200_torch.so")
_ops = None


def ops():
    """torch.ops.lhw — the same entry points registered through PyTorch's C++ extension ABI (csrc/torch_ops.cpp): every call
    checks device / dtype / shape of its tensors before it reaches the C-ABI, and takes the current stream itself.  This is the
    path the product uses; like the C-ABI library it is mandatory (no fallback).  The only exception is LHW_B200_LIB (the A/B
    harness timing another build of the C-ABI library): liblhw_b200_torch.so is linked against the in-tree library, so the
    harness binds the candidate with ctypes instead (use_torch_ops() is False)."""
    global _ops
    if _ops is None:
        import torch
        if not os.path.exists(TORCH_LIB_PATH):
            raise LhwError(f"{TORCH_LIB_PATH} is missing: build the extension (python -m learninghumanoidwalking_b200.build). "
                           "There is no fallback for the torch.ops.lhw entry points.")
        lib()      # the C-ABI library first: the op library resolves its symbols from it
        torch.ops.load_library(TORCH_LIB_PATH)
        _ops = torch.ops.lhw
    return _ops


def use_torch_ops() -> bool:
    return not os.environ.get("LHW_B200_LIB") and os.environ.get("LHW_TORCH_OPS", "1") != "0"


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        raise LhwError(f"{what} failed (rc={rc}): {lib().lhw_last_error().decode(errors='replace')}")


def ptr(t) -> int | None:
    """Device pointer of a torch tensor (None passes NULL)."""
    return None if t is None else t.data_ptr()


def current_stream_ptr() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream
