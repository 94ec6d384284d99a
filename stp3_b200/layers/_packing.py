"""Lazy, checkpoint-aware weight packing shared by the drop-in modules.

The modules keep the reference's parameter tree (so Lightning checkpoints load with strict=True) and derive the
folded / packed tensors the CUDA kernels consume the first time forward() runs in eval mode; the cache is rebuilt
whenever a parameter or buffer was modified in place (load_state_dict, optimizer step) or moved to another device.
"""
import torch
import torch.nn as nn


class PackedModule(nn.Module):
    def _signature(self):
        sig = []
        for t in list(self.parameters()) + list(self.buffers()):
            sig.append((t.data_ptr(), t._version, str(t.device)))
        return tuple(sig)

    def packed(self):
        sig = self._signature()
        cache = self.__dict__.get("_packed_cache")
        if cache is None or cache[0] != sig:
            with torch.no_grad():
                cache = (sig, self._pack())
            self.__dict__["_packed_cache"] = cache
        return cache[1]

    def _pack(self):
        raise NotImplementedError

    def _require_eval(self):
        if self.training:
            raise NotImplementedError(
                f"{type(self).__name__}: the sm_90a path implements the inference forward (eval-mode BatchNorm "
                "folded into the tensor-core kernels); call .eval() -- training through this module is SURVEY.md row f2")
