"""PeerComm — host side of the fused NVLink exchange step (csrc/comm_kernels.cu, include/lhw_b200.h).

Owns the IPC-exported flat gradient buffer of this rank, exchanges the CUDA IPC handles through torch.distributed
(the only thing the process group is used for here) and maps the peers' buffers.  The modules' .grad tensors are
views of `grad` so autograd writes straight into peer-visible memory; lhw_fused_allreduce_clip_adam then does
all-reduce + clip + Adam for actor and critic in three graph-capturable launches.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch
import torch.distributed as dist

from .. import _lib


class _CudaArray:
    def __init__(self, ptr: int, n: int):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3, "strides": None}


class PeerComm:
    def __init__(self, n_floats: int, device: torch.device):
        L = _lib.lib()
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank() if self.world > 1 else 0
        self.n = int(n_floats)
        h = ctypes.c_void_p()
        rc = L.lhw_comm_create(ctypes.byref(h), self.n, self.rank, self.world, device.index)
        if rc:
            raise _lib.LhwError(f"lhw_comm_create failed: {L.lhw_comm_last_error().decode()}")
        self._h = h
        self._keep = _CudaArray(L.lhw_comm_grad_ptr(h), self.n)
        with torch.cuda.device(device):
            self.grad = torch.as_tensor(self._keep, device=device)
        assert self.grad.data_ptr() == L.lhw_comm_grad_ptr(h)
        if self.world > 1:
            hs = L.lhw_comm_handle_size()
            blob = ctypes.create_string_buffer(hs)
            if L.lhw_comm_export(h, blob):
                raise _lib.LhwError(f"lhw_comm_export failed: {L.lhw_comm_last_error().decode()}")
            mine = torch.from_numpy(np.frombuffer(blob.raw, dtype=np.uint8).copy()).to(device)
            allh = [torch.empty_like(mine) for _ in range(self.world)]
            dist.all_gather(allh, mine)
            packed = torch.cat(allh).cpu().numpy().tobytes()
            if L.lhw_comm_import(h, packed):
                raise _lib.LhwError(f"lhw_comm_import failed: {L.lhw_comm_last_error().decode()}")
            dist.barrier()

    def fused_step(self, param, exp_avg, exp_avg_sq, n_actor, lr, betas, eps, max_norm):
        """All-reduce (peer memory) + clip x2 + Adam x2: three plain launches on the current stream, capturable into a CUDA graph
        (the Adam step number and the barrier epoch live in device memory)."""
        _lib.ops().fused_exchange(self._h.value, param, exp_avg, exp_avg_sq, int(n_actor), lr, betas[0], betas[1], eps, max_norm)

    def fused_step_adaptive(self, param, exp_avg, exp_avg_sq, n_actor, kl, desired_kl, betas, eps, max_norm):
        """fused_step with the KL-adaptive rate (DESIGN.md §7.3): kl is this rank's minibatch KL (one float32 device scalar); the
        rate is self.lr, in device memory, updated from the ranks' mean KL before this step's Adam update uses it."""
        _lib.ops().fused_exchange_adaptive(self._h.value, param, exp_avg, exp_avg_sq, int(n_actor), kl, self.lr, float(desired_kl),
                                           betas[0], betas[1], eps, max_norm)

    @property
    def lr(self) -> torch.Tensor:
        """The adaptive schedule's float64 rate word of this comm, as a [1] device tensor."""
        if getattr(self, "_lr", None) is None:
            L = _lib.lib()
            ptr = L.lhw_comm_lr_ptr(self._h)
            arr = _CudaArray(ptr, 1)
            arr.__cuda_array_interface__["typestr"] = "<f8"
            self._lr_keep = arr
            self._lr = torch.as_tensor(arr, device=self.grad.device)
            assert self._lr.data_ptr() == ptr
        return self._lr

    def get_lr(self) -> float:
        """The device rate (synchronises the current stream)."""
        v = ctypes.c_double(0.0)
        if _lib.lib().lhw_comm_get_lr(self._h, ctypes.byref(v), _lib.current_stream_ptr()):
            raise _lib.LhwError(f"lhw_comm_get_lr failed: {_lib.lib().lhw_comm_last_error().decode()}")
        return v.value

    def set_lr(self, lr: float):
        if _lib.lib().lhw_comm_set_lr(self._h, float(lr), _lib.current_stream_ptr()):
            raise _lib.LhwError(f"lhw_comm_set_lr failed: {_lib.lib().lhw_comm_last_error().decode()}")

    def status(self):
        """(completed Adam steps, (actor grad norm, critic grad norm) of the last step); raises if a peer did not arrive at the
        gradient exchange within the spin limit (the kernels carry on with partial sums rather than hang the GPU).
        Synchronises the current stream: call once per iteration, not per step."""
        L = _lib.lib()
        err, steps, norms = ctypes.c_int(0), ctypes.c_int(0), (ctypes.c_float * 2)()
        rc = L.lhw_comm_status(self._h, ctypes.byref(err), ctypes.byref(steps), norms, _lib.current_stream_ptr())
        if rc:
            raise _lib.LhwError(f"gradient exchange failed on rank {self.rank}: {L.lhw_comm_last_error().decode()}")
        return steps.value, (norms[0], norms[1])

    def set_step(self, adam_steps: int):
        if _lib.lib().lhw_comm_set_step(self._h, int(adam_steps), _lib.current_stream_ptr()):
            raise _lib.LhwError(f"lhw_comm_set_step failed: {_lib.lib().lhw_comm_last_error().decode()}")

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lr = None
            _lib.lib().lhw_comm_destroy(self._h)
            self._h = ctypes.c_void_p()
