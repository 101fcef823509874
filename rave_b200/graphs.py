"""Whole-step CUDA graphs: the phase-2 training step is ~1.3k kernel launches (ours + the loss
arithmetic + Adam); issued from Python that is tens of milliseconds of host time, several times the
GPU time of the bf16 step.  `GraphedTrainer` captures the generator step and the discriminator step of
`RAVE.train_body` once (after eager warm-up; in phase 1 only the generator step) and replays them, so the step costs its GPU time.

Replay-safe because train_body has no host-side decisions or syncs, the optimisers are `capturable`
(lr and step counters live on the device; LinearLR updates the lr tensor in place between replays) and
every buffer the library kernels see is allocated from the graph's private pool (tensor maps bake the
addresses at capture).  Host-side scalars that a schedule may move are read from device memory:
`beta_factor` (BetaWarmupCallback) lives in `model._beta_dev`, refreshed before every replay; the loss
weights (`model.weights`) and the valid-signal crop (`model.receptive_field`) are constants of the captured graph --
changing them needs a new GraphedTrainer.

The eager warm-up the capture needs (lazy state, cuFFT plans, kernel attributes) performs real optimiser
updates; parameters, buffers and optimiser state are snapshotted before it and restored afterwards, so
constructing a GraphedTrainer does not move the model.
"""
import copy
from typing import Dict, Optional

import torch

from . import _lib, engine


def _encoder_is_frozen(model) -> bool:
    from .blocks import VariationalEncoder, WasserteinEncoder
    enc = model.encoder
    # compute_losses sets the encoder's own flag from model.warmed_up before every forward; a SphericalEncoder ignores
    # it and keeps training in phase 2
    return isinstance(enc, (VariationalEncoder, WasserteinEncoder)) and bool(model.warmed_up)


def _refresh_static_after_load(m, keys):
    if getattr(m, "_static_disc_prep", False):
        engine.refresh_static_prep(m.discriminator)
    if getattr(m, "_static_enc_prep", False):
        engine.refresh_static_prep(m.encoder)


class GraphedTrainer:
    def __init__(self, model, example_batch: torch.Tensor, grad_hook=None, warmup_steps: int = 3):
        if not example_batch.is_cuda:
            raise RuntimeError("GraphedTrainer needs a CUDA batch")
        self.model = model
        self.grad_hook = grad_hook
        self.x_static = example_batch.clone()
        model.optimizers(capturable=True)
        # phase 2 captures a G-step and a D-step; phase 1 (no discriminator in the loop) only the G-step
        self.phase2 = bool(model.warmed_up)
        kinds = (True, False) if self.phase2 else (False,)
        self._weights_at_capture = dict(model.weights)
        # the valid-signal crop of the multiband loss is baked in at capture too (validation_epoch_end sets it once)
        self._receptive_field_at_capture = model._receptive_field_host()
        model._beta_dev = torch.tensor(float(model.beta_factor), dtype=torch.float32, device=example_batch.device)
        gen_opt, dis_opt = model.optimizers()
        # the discriminator only changes in D-steps: its prepared weights become persistent buffers, rewritten in place
        # after the discriminator's optimiser step (inside the D-step graph) instead of being rebuilt by every replay
        self.static_prep = engine.precision() == "bf16"
        # phase 2 of a VariationalEncoder model: the encoder output is detached (rave/blocks.py:739-743), no gradient
        # ever reaches the encoder, Adam skips it -- its prepared weights are constants of the captured graphs too
        self.static_encoder = bool(self.static_prep and _encoder_is_frozen(model))
        if self.static_prep:
            engine.enable_static_prep(model.discriminator)
            model._static_disc_prep = True
            if self.static_encoder:
                engine.enable_static_prep(model.encoder)
                model._static_enc_prep = True
            if not getattr(model, "_static_prep_hook", None):
                model._static_prep_hook = model.register_load_state_dict_post_hook(_refresh_static_after_load)
        snap_tensors = [(t, t.detach().clone()) for t in list(model.parameters()) + list(model.buffers())]
        snap_opt = [(o, copy.deepcopy(o.state_dict())) for o in (gen_opt, dis_opt)]
        self.graphs: Dict[bool, torch.cuda.CUDAGraph] = {}
        self.outputs: Dict[bool, Dict[str, torch.Tensor]] = {}
        self.launches: Dict[bool, int] = {}      # library kernel launches recorded in each graph
        # eager warm-up on a side stream: lazy state (Adam moments, cuFFT plans, PQMF tables, kernel
        # attributes, tensor-map entry point) must exist before capture
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for i in range(warmup_steps):
                for is_dis in kinds:
                    model.train_body(self.x_static, is_dis, None, grad_hook)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        pool = None
        for is_dis in kinds:
            g = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count()
            # thread_local: other threads (NCCL watchdog, samplers) may touch CUDA while we capture
            with torch.cuda.graph(g, pool=pool, capture_error_mode="thread_local"):
                logs = model.train_body(self.x_static, is_dis, None, grad_hook)
                out = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in logs.items()}
            pool = g.pool()
            self.launches[is_dis] = _lib.launch_count() - n0
            self.graphs[is_dis] = g
            self.outputs[is_dis] = out
        # undo the warm-up updates: parameters / buffers back to their values, optimiser state back to what it was
        # (moments the warm-up created lazily are zeroed IN PLACE: the graphs hold their addresses)
        with torch.no_grad():
            for t, v in snap_tensors:
                t.copy_(v)
            for opt, sd in snap_opt:
                old = {}
                for g_new, g_old in zip(opt.param_groups, sd["param_groups"]):
                    for p, idx in zip(g_new["params"], g_old["params"]):
                        old[p] = sd["state"].get(idx)
                    st_old = g_old.get("step")
                    if torch.is_tensor(g_new.get("step")):
                        g_new["step"].copy_(st_old) if torch.is_tensor(st_old) else g_new["step"].zero_()
                for p, st in opt.state.items():
                    for k, v in st.items():
                        if torch.is_tensor(v):
                            o = old.get(p)
                            v.copy_(o[k]) if (o is not None and k in o) else v.zero_()
        engine.invalidate_prepared()
        if self.static_prep:
            engine.refresh_static_prep(model.discriminator)      # the restore above moved the parameters
            if self.static_encoder:
                engine.refresh_static_prep(model.encoder)

    def step(self, batch: torch.Tensor, batch_idx: int):
        """Same contract as RAVE.training_step: returns the logged scalars (device tensors)."""
        is_dis = self.model.is_discriminator_step(batch_idx)
        if bool(self.model.warmed_up) != self.phase2:
            raise RuntimeError(f"GraphedTrainer: captured phase-{2 if self.phase2 else 1} steps but model.warmed_up is "
                               f"{bool(self.model.warmed_up)}; build a new GraphedTrainer")
        if self.model.weights != self._weights_at_capture:
            raise RuntimeError("GraphedTrainer: model.weights changed after capture (the loss weights are constants of "
                               "the captured graphs); build a new GraphedTrainer")
        if self.model._receptive_field_host() != self._receptive_field_at_capture:
            raise RuntimeError("GraphedTrainer: model.receptive_field changed after capture (the valid-signal crop is a "
                               "constant of the captured graphs); build a new GraphedTrainer")
        self.model._beta_dev.fill_(float(self.model.beta_factor))
        self.x_static.copy_(batch, non_blocking=True)
        self.graphs[is_dis].replay()
        engine.invalidate_prepared()       # parameters changed without bumping their autograd versions
        self.outputs[is_dis]["beta_factor"] = self.model.beta_factor
        self.model.logged = self.outputs[is_dis]
        return self.outputs[is_dis]
