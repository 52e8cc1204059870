"""Device-side caches are not model state.

The modules keep ctypes structs holding raw device pointers (`_packed`), scratch buffers (`_workspace`), precomputed
conditioning (`_trajectory`) and captured CUDA graphs (`_graphs`).  ctypes objects with pointers cannot be pickled, and a
copy must not alias another instance's buffers, so `copy.deepcopy(model)` (the EMA pattern of train.py:95-97),
`pickle` and `torch.save(model)` see these attributes as empty; they are rebuilt on the next call.
"""
from __future__ import annotations

import torch


class DeviceCacheMixin:
    _CACHE_ATTRS = {"_packed": None, "_packed_key": None, "_workspace": None, "_trajectory": None, "_graphs": None,
                    "_frozen": None, "_train_backend": None, "_train_operands": None, "_packed_enc": None}

    def __getstate__(self):
        state = dict(self.__dict__)
        for k, empty in self._CACHE_ATTRS.items():
            if k in state:
                state[k] = empty
        return state

    def _aligned_workspace(self, need: int, device) -> int:
        """Device address of `need` bytes of scratch on a 1024-byte boundary, inside `_workspace` (reallocated when it is too
        small or on another device)."""
        ws = self._workspace
        if ws is None or ws.numel() < need + 1024 or ws.device != device:
            ws = self._workspace = torch.empty(need + 1024, dtype=torch.uint8, device=device)
        return (ws.data_ptr() + 1023) // 1024 * 1024
