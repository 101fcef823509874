"""`EMA` -- the reference's exponential moving average of the weights (scripts/train.py:81-119, `train.py --ema`), on
the library's multi-tensor kernels (csrc/ema.cu).

The averages live in one flat float32 buffer; each named parameter's average is a view of its slice (16-byte aligned),
so the addresses are stable for CUDA graphs and `state_dict()` returns the reference's keys.  One launch updates every
parameter, `ema = ema * factor + p * (1 - factor)` rounded exactly as torch rounds that float32 expression; the first
call for a parameter clones it instead, decided on the device (a per-parameter `initialised` flag) so that a
GraphedTrainer can capture the update (`GraphedTrainer(..., ema=ema)`).  Memory: one float32 copy of the parameters.
"""
import math
from typing import Any, Dict

import torch

from . import _lib, engine, ops

_ALIGN = 4          # float32 elements: every slice of the flat buffer starts 16-byte aligned (the kernel's float4 path)


class EMA:
    """scripts/train.py:81-119, with the same hook signatures as model.WarmupCallback / BetaWarmupCallback."""

    def __init__(self, factor: float = .999) -> None:
        self.factor = factor
        self._module = None
        self._pending: Dict[str, Any] = {}      # load_state_dict before the first update: applied when binding
        self._extra: Dict[str, Any] = {}        # loaded names the module does not have (kept, as dict.update does)
        self._graphed = False                   # a GraphedTrainer launches the update inside its graphs

    # ------------------------------------------------------------------ binding to a module
    def _bind(self, module) -> None:
        """Allocate the flat buffer, the flags and the kernel table for `module`'s parameters (once), or check that
        `module` is the bound one and that none of its parameters was replaced by a new tensor."""
        if self._module is not None:
            if module is not self._module:
                raise RuntimeError("EMA: bound to another module (one EMA averages one model)")
            named = list(module.named_parameters())
            if [n for n, _ in named] != self._names or [p.data_ptr() for _, p in named] != self._ptrs:
                raise RuntimeError("EMA: the module's parameters changed (a parameter was replaced by a new tensor, or "
                                   "added / removed) since the averages were allocated; update parameters in place")
            return
        named = list(module.named_parameters())
        if not named:
            raise RuntimeError("EMA: the module has no parameters")
        device = named[0][1].device
        for n, p in named:
            if p.dtype != torch.float32 or p.device != device or not p.is_contiguous():
                raise RuntimeError(f"EMA: parameter {n} is not a contiguous float32 tensor on {device}")
        offsets, total = [], 0
        for _, p in named:
            offsets.append(total)
            total += -(-p.numel() // _ALIGN) * _ALIGN
        self.flat = torch.zeros(total, dtype=torch.float32, device=device)
        self._names = [n for n, _ in named]
        self._ptrs = [p.data_ptr() for _, p in named]
        self._params = [p for _, p in named]
        self._views = {n: self.flat[o:o + p.numel()].view_as(p) for (n, p), o in zip(named, offsets)}
        self._index = {n: i for i, n in enumerate(self._names)}
        # [initialised flag per parameter | completion ticket of the update launch]
        self._state = torch.zeros(len(named) + 1, dtype=torch.int32, device=device)
        self._table = None
        if device.type == "cuda":
            chunk = ops.ema_chunk_elems()
            chunks = [math.ceil(p.numel() / chunk) for p in self._params]
            chunk0 = [0]
            for c in chunks:
                chunk0.append(chunk0[-1] + c)
            self._n_chunks = chunk0[-1]
            rows = self._ptrs + [v.data_ptr() for v in self._views.values()] + [p.numel() for p in self._params] + chunk0
            self._table = torch.tensor(rows, dtype=torch.int64).to(device)
        self._module = module
        pending, self._pending = self._pending, {}
        self.load_state_dict(pending)

    def _launch_update(self) -> None:
        self._require_device()
        ops.ema_update(self._table, len(self._names), self._n_chunks, self._state, self.factor)

    def _launch_swap(self) -> None:
        self._require_device()
        ops.ema_swap(self._table, len(self._names), self._n_chunks)

    def _require_device(self) -> None:
        if self._table is None:
            raise _lib.RaveB200Error("EMA: the parameters are not on a CUDA device (rave_b200 has no CPU path)")

    def _has_weights(self) -> bool:
        if self._module is None:
            return bool(self._pending or self._extra)
        return bool(self._extra) or bool(self._state[:-1].any().item())

    # ------------------------------------------------------------------ the reference's callback interface
    def on_train_batch_end(self, trainer, pl_module, outputs, batch, batch_idx) -> None:
        """One update launch over every parameter of `pl_module` (discriminator included, on every step kind)."""
        if self._graphed:
            raise RuntimeError("EMA: this EMA is updated inside a GraphedTrainer's graphs (GraphedTrainer(..., ema=)); "
                               "calling on_train_batch_end as well would average twice per step")
        self._bind(pl_module)
        self._launch_update()

    def swap_weights(self, module) -> None:
        """Exchange the module's parameters and the averages in place; a second swap restores both.  The engine's
        prepared weights (the tap-major cache and a GraphedTrainer's static layouts) are rebuilt from the new values."""
        self._bind(module)
        self._launch_swap()
        from .graphs import _refresh_static_after_load
        engine.invalidate_prepared()
        _refresh_static_after_load(module, None)

    def on_validation_epoch_start(self, trainer, pl_module) -> None:
        if self._has_weights():
            self.swap_weights(pl_module)
        else:
            print("no ema weights available")

    def on_validation_epoch_end(self, trainer, pl_module) -> None:
        if self._has_weights():
            self.swap_weights(pl_module)
        else:
            print("no ema weights available")

    def state_dict(self) -> Dict[str, Any]:
        """Parameter name -> average (views of the flat buffer), for the parameters averaged or loaded so far."""
        if self._module is None:
            return {**self._extra, **self._pending}
        flags = self._state[:-1].tolist()
        return {**self._extra, **{n: self._views[n] for n, f in zip(self._names, flags) if f}}

    def load_state_dict(self, state_dict: Dict[str, Any]) -> None:
        """dict.update semantics: the names in `state_dict` take its values (copied into the flat buffer in place and
        marked initialised, so the next update averages them), the others keep theirs."""
        if self._module is None:
            self._pending.update(state_dict)
            return
        loaded = []
        with torch.no_grad():
            for n, v in state_dict.items():
                if n in self._views:
                    self._views[n].copy_(v)
                    loaded.append(self._index[n])
                else:
                    self._extra[n] = v
        if loaded:
            self._state[torch.tensor(loaded, dtype=torch.long, device=self._state.device)] = 1
