"""`RAVE` -- the caller of the hot path (rave/model.py:133-511), without pytorch-lightning.

`__init__`, `encode`, `decode`, `forward`, `split_features`, `configure_optimizers` and
`training_step` keep the reference's signatures and arithmetic (including quirk D1, the loss
weights applied twice, rave/model.py:397,410-411).  Work whose result the reference discards is
not computed (SURVEY.md 3.1 / quirk D2): the D-step does not back-propagate into the generator,
the G-step does not accumulate discriminator weight gradients, and `x_raw` gets no gradient --
parameter updates are identical.  `reg.item()` (quirk D7, a host sync per step) is replaced by
adding the (possibly zero) KL term unconditionally: same value, no sync.
"""
import math
from typing import Callable, Dict, Iterable, Optional

import contextlib

import torch
import torch.nn as nn

from . import blocks, core

_default_loss_weights = {
    "audio_distance": 1.,
    "multiband_audio_distance": 1.,
    "adversarial": 1.,
    "feature_matching": 20,
}


def _pqmf_encode(pqmf, x: torch.Tensor):
    """rave/model.py:116-122."""
    batch_size = x.shape[:-2]
    x_multiband = x.reshape(-1, 1, x.shape[-1])
    x_multiband = pqmf(x_multiband)
    return x_multiband.reshape(*batch_size, -1, x_multiband.shape[-1])


def _pqmf_decode(pqmf, x: torch.Tensor, batch_size: Iterable[int], n_channels: int):
    """rave/model.py:125-130."""
    x = x.reshape(x.shape[0] * n_channels, -1, x.shape[-1])
    x = pqmf.inverse(x)
    return x.reshape(*batch_size, n_channels, -1)


class WarmupCallback:
    """rave/model.py:45-61."""

    def __init__(self) -> None:
        self.state = {"training_steps": 0}

    def on_train_batch_start(self, trainer, pl_module, batch, batch_idx) -> None:
        if self.state["training_steps"] >= pl_module.warmup:
            pl_module.warmed_up = True
        self.state["training_steps"] += 1

    def state_dict(self):
        return self.state.copy()

    def load_state_dict(self, state_dict):
        self.state.update(state_dict)


class BetaWarmupCallback:
    """rave/model.py:78-113."""

    def __init__(self, initial_value: float = .2, target_value: float = .2, warmup_len: int = 1,
                 log: bool = True) -> None:
        self.state = {"training_steps": 0}
        self.warmup_len = warmup_len
        self.initial_value = initial_value
        self.target_value = target_value
        self.log_warmup = log

    def on_train_batch_start(self, trainer, pl_module, batch, batch_idx) -> None:
        self.state["training_steps"] += 1
        if self.state["training_steps"] >= self.warmup_len:
            pl_module.beta_factor = self.target_value
            return
        warmup_ratio = self.state["training_steps"] / self.warmup_len
        if self.log_warmup:
            beta = math.log(self.initial_value) * (1 - warmup_ratio) + math.log(self.target_value) * warmup_ratio
            pl_module.beta_factor = math.exp(beta)
        else:
            beta = warmup_ratio * (self.target_value - self.initial_value) + self.initial_value
            pl_module.beta_factor = min(beta, self.target_value)

    def state_dict(self):
        return self.state.copy()

    def load_state_dict(self, state_dict):
        self.state.update(state_dict)


class RAVE(nn.Module):

    def __init__(self, latent_size, sampling_rate, encoder, decoder, discriminator, phase_1_duration,
                 gan_loss, valid_signal_crop, feature_matching_fun, num_skipped_features,
                 audio_distance: Callable[[], nn.Module],
                 multiband_audio_distance: Callable[[], nn.Module], n_bands: int = 16, balancer=None,
                 weights: Optional[Dict[str, float]] = None, warmup_quantize: Optional[int] = None,
                 pqmf: Optional[Callable[[], nn.Module]] = None, spectrogram: Optional[Callable] = None,
                 update_discriminator_every: int = 2, n_channels: int = 1, input_mode: str = "pqmf",
                 output_mode: str = "pqmf", audio_monitor_epochs: int = 1,
                 enable_pqmf_encode: Optional[bool] = None, enable_pqmf_decode: Optional[bool] = None,
                 is_mel_input: Optional[bool] = None, loss_weights=None):
        super().__init__()
        self.pqmf = pqmf(n_channels=n_channels)
        self.spectrogram = spectrogram
        assert input_mode in ["pqmf", "mel", "raw"]
        assert output_mode in ["raw", "pqmf"]
        self.input_mode = input_mode
        self.output_mode = output_mode
        if (enable_pqmf_encode is not None) or (enable_pqmf_decode is not None):
            self.input_mode = "pqmf" if enable_pqmf_encode else "raw"
            self.output_mode = "pqmf" if enable_pqmf_decode else "raw"
        if is_mel_input is not None:
            self.input_mode = "mel"
        if loss_weights is not None:
            weights = loss_weights
        assert weights is not None, "RAVE model requires either weights or loss_weights (depreciated) keyword"

        self.encoder = encoder(n_channels=n_channels)
        self.decoder = decoder(n_channels=n_channels)
        self.discriminator = discriminator(n_channels=n_channels)
        self.audio_distance = audio_distance()
        self.multiband_audio_distance = multiband_audio_distance()
        self.gan_loss = gan_loss

        self.register_buffer("latent_pca", torch.eye(latent_size))
        self.register_buffer("latent_mean", torch.zeros(latent_size))
        self.register_buffer("fidelity", torch.zeros(latent_size))
        self.latent_size = latent_size
        self.automatic_optimization = False

        self.warmup = phase_1_duration
        self.warmup_quantize = warmup_quantize
        # the reference aliases and mutates the module-global dict (quirk D1); a copy gives the
        # same values without the cross-instance side effect
        self.weights = dict(_default_loss_weights)
        self.weights.update(weights)
        self.warmed_up = False

        self.sr = sampling_rate
        self.valid_signal_crop = valid_signal_crop
        self.n_channels = n_channels
        self.feature_matching_fun = feature_matching_fun
        self.num_skipped_features = num_skipped_features
        self.update_discriminator_every = update_discriminator_every
        self.eval_number = 0
        self.beta_factor = 1.
        self.integrator = None
        self.register_buffer("receptive_field", torch.tensor([0, 0]).long())
        self.audio_monitor_epochs = audio_monitor_epochs

        self._optimizers = None
        self._scheduler = None
        self.logged: Dict[str, torch.Tensor] = {}

    def _receptive_field_host(self):
        """Host copy of the `receptive_field` buffer (read once: no device->host sync per step)."""
        ver = self.receptive_field._version          # bumped by load_state_dict / any in-place write to the buffer
        hit = getattr(self, "_rf_host", None)
        if hit is None or hit[0] != ver or hit[1] is not self.receptive_field:
            hit = self._rf_host = (ver, self.receptive_field, tuple(int(v) for v in self.receptive_field.tolist()))
        return hit[2]

    def set_receptive_field(self, left: int, right: int):
        """What validation_epoch_end does in the reference (rave/model.py:446-453)."""
        self.receptive_field[0] = left
        self.receptive_field[1] = right
        self._rf_host = (self.receptive_field._version, self.receptive_field, (int(left), int(right)))

    # ------------------------------------------------------------------ optimisers
    def configure_optimizers(self, capturable: bool = False):
        """rave/model.py:226-236.  `capturable=True` keeps lr / step counters on the device so that the
        whole step can be replayed from a CUDA graph (rave_b200/graphs.py); same Adam arithmetic."""
        gen_p = list(self.encoder.parameters()) + list(self.decoder.parameters())
        dis_p = list(self.discriminator.parameters())
        if gen_p[0].is_cuda:
            # multi-tensor Adam kernel, lr / step counter on the device: graph-replayable either way
            from .optim import FusedAdam
            gen_opt = FusedAdam(gen_p, 1e-3, (.5, .9))
            dis_opt = FusedAdam(dis_p, 1e-4, (.5, .9))
        elif capturable:
            dev = gen_p[0].device
            gen_opt = torch.optim.Adam(gen_p, torch.tensor(1e-3, device=dev), (.5, .9), capturable=True)
            dis_opt = torch.optim.Adam(dis_p, torch.tensor(1e-4, device=dev), (.5, .9), capturable=True)
        else:
            gen_opt = torch.optim.Adam(gen_p, 1e-3, (.5, .9))
            dis_opt = torch.optim.Adam(dis_p, 1e-4, (.5, .9))
        sched = torch.optim.lr_scheduler.LinearLR(gen_opt, start_factor=1.0, end_factor=0.1,
                                                  total_iters=self.warmup)
        return ({"optimizer": gen_opt, "lr_scheduler": {"scheduler": sched}}, {"optimizer": dis_opt})

    def optimizers(self, capturable: bool = False):
        if self._optimizers is None:
            g, d = self.configure_optimizers(capturable)
            self._optimizers = (g["optimizer"], d["optimizer"])
            self._scheduler = g["lr_scheduler"]["scheduler"]
        return self._optimizers

    def lr_schedulers(self):
        self.optimizers()
        return self._scheduler

    def log(self, name, value):
        self.logged[name] = value.detach() if torch.is_tensor(value) else value

    def log_dict(self, d):
        for k, v in d.items():
            self.log(k, v)

    # ------------------------------------------------------------------ inference path
    def encode(self, x, return_mb: bool = False):
        x_enc = x
        if self.input_mode == "pqmf":
            x_enc = _pqmf_encode(self.pqmf, x_enc)
        elif self.input_mode == "mel":
            x_enc = self.spectrogram.encode_log1p(x)          # rave/model.py:238-242
        z = self.encoder(x_enc)
        if return_mb:
            if self.input_mode == "pqmf":
                return z, x_enc
            # quirk D9 (SURVEY.md): the reference analyses x_enc, i.e. the mel spectrogram in mel mode, which its own
            # multiband distance cannot take; the multiband target is the PQMF analysis of the waveform
            return z, _pqmf_encode(self.pqmf, x if self.input_mode == "mel" else x_enc)
        return z

    def decode(self, z):
        batch_size = z.shape[:-2]
        y = self.decoder(z)
        if self.output_mode == "pqmf":
            y = _pqmf_decode(self.pqmf, y, batch_size=batch_size, n_channels=self.n_channels)
        return y

    def forward(self, x):
        z = self.encode(x, return_mb=False)
        z = self.encoder.reparametrize(z)[0]
        return self.decode(z)

    def update_adain(self, learn_target: bool = False, learn_source: bool = False, reset_target: bool = False,
                     reset_source: bool = False) -> int:
        """Style transfer of a model with AdaIN layers (v3): learn the target statistics over target audio
        (`learn_target=True`), then the source statistics (`learn_source=True`; the transfer already applies in those
        calls), then `update_adain()` to transfer with the statistics frozen; `reset_*` forget them.  Eval mode only
        (AdaIN is the identity in training).  Returns the number of AdaIN layers (0 without any): blocks.update_adain."""
        return blocks.update_adain(self, learn_target, learn_source, reset_target, reset_source)

    def on_train_batch_end(self, outputs=None, batch=None, batch_idx=None) -> None:
        self.lr_schedulers().step()

    def split_features(self, features):
        feature_real, feature_fake = [], []
        for scale in features:
            true, fake = zip(*map(lambda x: torch.split(x, x.shape[0] // 2, 0), scale))
            feature_real.append(true)
            feature_fake.append(fake)
        return feature_real, feature_fake

    # ------------------------------------------------------------------ training step
    def compute_losses(self, x_raw, is_dis_step: bool, eps: Optional[torch.Tensor] = None):
        """Forward part of training_step (rave/model.py:292-399).  Returns (loss_gen dict, loss_dis,
        aux)."""
        batch_size = x_raw.shape[:-2]
        if getattr(self, "_static_enc_prep", False) and not self.warmed_up:
            # back in phase 1 after a GraphedTrainer froze the encoder's prepared weights: the encoder trains again
            from . import engine
            engine.disable_static_prep(self.encoder)
            self._static_enc_prep = False
        self.encoder.set_warmed_up(self.warmed_up)
        self.decoder.set_warmed_up(self.warmed_up)

        z, x_multiband = self.encode(x_raw, return_mb=True)
        if eps is not None:
            z, reg = self.encoder.reparametrize(z, eps)[:2]
        else:
            z, reg = self.encoder.reparametrize(z)[:2]

        y = self.decoder(z)
        if self.output_mode == "pqmf":
            y_multiband = y
            y_raw = _pqmf_decode(self.pqmf, y, batch_size=batch_size, n_channels=self.n_channels)
        else:
            y_raw = y
            y_multiband = _pqmf_encode(self.pqmf, y)
        y_raw = y_raw[..., :x_raw.shape[-1]]
        y_multiband = y_multiband[..., :x_multiband.shape[-1]]

        if self.valid_signal_crop:
            left_rf, right_rf = self._receptive_field_host()
            if left_rf + right_rf:
                dim = x_multiband.shape[1]                      # core.valid_signal_crop, host-side ints
                x_multiband = x_multiband[..., left_rf // dim:]
                y_multiband = y_multiband[..., left_rf // dim:]
                if right_rf:
                    x_multiband = x_multiband[..., :-right_rf // dim]
                    y_multiband = y_multiband[..., :-right_rf // dim]

        # The spectral losses (20 STFTs + their small kernels) and the discriminator chains only share their inputs:
        # the former go to a side stream so that they fill the holes between the discriminator's persistent kernels
        # (autograd replays each part's backward on its own stream).
        from . import discriminator
        side = None
        if y_raw.is_cuda and self.warmed_up and discriminator.DISC_STREAMS > 1:
            if getattr(self, "_loss_stream", None) is None:
                self._loss_stream = torch.cuda.Stream()
            side = self._loss_stream
            cur = torch.cuda.current_stream()
            side.wait_stream(cur)
            for t in (x_multiband, y_multiband, x_raw, y_raw):
                t.record_stream(side)
        distances = {}
        with torch.cuda.stream(side) if side is not None else contextlib.nullcontext():
            for k, v in self.multiband_audio_distance(x_multiband, y_multiband).items():
                distances[f"multiband_{k}"] = self.weights["multiband_audio_distance"] * v
            for k, v in self.audio_distance(x_raw, y_raw).items():
                distances[f"fullband_{k}"] = self.weights["audio_distance"] * v

        feature_matching_distance = 0.
        fused = None
        if self.warmed_up:
            y_d = y_raw.detach() if is_dis_step else y_raw     # quirk D2: discarded gradients
            xy = torch.cat([x_raw, y_d], 0)
            fused = self._fused_feature_matching(xy, fake_grad_only=not is_dis_step)
        if fused is not None:
            feature_matching_distance, loss_dis, loss_adv, pred_real, pred_fake = fused
        elif self.warmed_up:
            from . import engine
            # generator step: the discriminator is frozen and only the fake half's input gradient is used -> its
            # engine chains run their backward on the fake rows only
            with engine.fake_rows_only(not is_dis_step):
                features = self.discriminator(xy)
            feature_real, feature_fake = self.split_features(features)
            loss_dis = 0
            loss_adv = 0
            pred_real = 0
            pred_fake = 0
            # Features that are views of a dense channel-last buffer holding [real; fake] (the Descript discriminator on
            # the engine) are matched on that buffer: one pass, gradient written in the buffer's own layout.
            kw = getattr(self.feature_matching_fun, "keywords", None)
            on_bases = (kw is not None and getattr(self.feature_matching_fun, "func", None) is core.mean_difference
                        and kw.get("norm", "L1") == "L1")
            skip = self.num_skipped_features
            # features whose two L1 sums came out of their own activation pass (ops.leaky_fm): all of them are turned
            # into terms by ONE stacked division + weighted sum (a Descript discriminator has ~100 such features:
            # one scalar division, one addition and their backward launches each, otherwise)
            tapped = []
            for scale, scale_real, scale_fake in zip(features, feature_real, feature_fake):
                terms = []
                n_terms = len(scale[skip:])
                for full, real, fake in zip(scale[skip:], scale_real[skip:], scale_fake[skip:]):
                    base = getattr(full, "_cl_base", None) if on_bases else None
                    st = getattr(full, "_fm_stats", None) if on_bases else None
                    if st is not None:
                        tapped.append((st, real.numel(), 1.0 / (n_terms * len(feature_real))))
                    elif base is not None:
                        terms.append(core.mean_difference_halves(base, real.numel(), bool(kw.get("relative", False))))
                    else:
                        terms.append(self.feature_matching_fun(real, fake))
                if terms:
                    feature_matching_distance = feature_matching_distance + sum(terms) / (n_terms * len(feature_real))
                _dis, _adv = self.gan_loss(scale_real[-1], scale_fake[-1])
                pred_real = pred_real + scale_real[-1].mean()
                pred_fake = pred_fake + scale_fake[-1].mean()
                loss_dis = loss_dis + _dis
                loss_adv = loss_adv + _adv
            if tapped:
                feature_matching_distance = feature_matching_distance + core.stacked_l1_terms(
                    tapped, bool(kw.get("relative", False)))
        else:
            # device zeros (not host tensors copied over: a phase-1 step is captured by GraphedTrainer too)
            pred_real = x_raw.new_zeros(())
            pred_fake = x_raw.new_zeros(())
            loss_dis = x_raw.new_zeros(())
            loss_adv = x_raw.new_zeros(())

        if side is not None:
            torch.cuda.current_stream().wait_stream(side)
            for v in distances.values():
                v.record_stream(torch.cuda.current_stream())
        loss_gen = {}
        loss_gen.update(distances)
        # schedule-driven scalar: a captured graph reads it from device memory (GraphedTrainer refreshes the tensor
        # before every replay), eager steps use the Python float as the reference does
        beta_dev = getattr(self, "_beta_dev", None)
        if beta_dev is not None and not (reg.is_cuda and torch.cuda.is_current_stream_capturing()):
            beta_dev = None
        loss_gen["regularization"] = reg * (beta_dev if beta_dev is not None else self.beta_factor)
        if self.warmed_up:
            loss_gen["feature_matching"] = self.weights["feature_matching"] * feature_matching_distance
            loss_gen["adversarial"] = self.weights["adversarial"] * loss_adv
        aux = dict(pred_real=pred_real, pred_fake=pred_fake, y_raw=y_raw, z=z)
        return loss_gen, loss_dis, aux

    def _fused_feature_matching(self, xy, fake_grad_only: bool = False):
        """The discrimination block (rave/model.py:348-379) without materialising the hidden features:
        in bf16 mode every ConvNet returns, per hidden layer, (sum|h_r - h_f|, sum|h_r|) computed by the
        engine from its own operand stream, plus the score tensor.  Same arithmetic as
        core.mean_difference(norm='L1', relative=...) averaged like the reference."""
        disc = self.discriminator
        kw = getattr(self.feature_matching_fun, "keywords", None)
        if kw is None or getattr(self.feature_matching_fun, "func", None) is not core.mean_difference:
            return None
        if kw.get("norm", "L1") != "L1" or not hasattr(disc, "supports_fused_fm") or not disc.supports_fused_fm(xy):
            return None
        relative = bool(kw.get("relative", False))
        skip = self.num_skipped_features
        fm_total, loss_dis, loss_adv, pred_real, pred_fake = 0., 0., 0., 0., 0.
        nets = disc.forward_fm(xy, fake_grad_only=fake_grad_only)
        tail = self._fused_tail(nets, relative, skip)
        if tail is not None:
            return tail
        for stats, counts, score, _, _ in nets:
            half = score.shape[0] // 2
            s_real, s_fake = score[:half], score[half:]
            terms = []
            for i in range(skip, len(counts)):
                if relative:
                    terms.append(stats[i, 0] / stats[i, 1])
                else:
                    terms.append(stats[i, 0] / counts[i])
            if skip <= len(counts):                       # the score itself is the last "feature"
                terms.append(self.feature_matching_fun(s_real, s_fake))
            fm_total = fm_total + sum(terms) / len(terms)
            _dis, _adv = self.gan_loss(s_real, s_fake)
            pred_real = pred_real + s_real.mean()
            pred_fake = pred_fake + s_fake.mean()
            loss_dis = loss_dis + _dis
            loss_adv = loss_adv + _adv
        return fm_total / len(nets), loss_dis, loss_adv, pred_real, pred_fake

    def _fused_tail(self, nets, relative: bool, skip: int):
        """Vectorised loss assembly from the per-ConvNet statistics (hinge GAN, equal depths): a dozen launches
        instead of ~40 scalar ATen launches per ConvNet in each direction.  Same arithmetic as the loop in
        _fused_feature_matching / rave/model.py:348-379."""
        if self.gan_loss is not core.hinge_gan:
            return None
        depths = {len(counts) for _, counts, _, _, _ in nets}
        if len(depths) != 1 or any(n_score <= 0 for *_, n_score in nets):
            return None
        nh = depths.pop()
        if skip > nh:
            return None
        dev = nets[0][0].device
        key = (tuple(tuple(c) for _, c, _, _, _ in nets), tuple(n for *_, n in nets))
        consts = self._fm_consts.get(key) if hasattr(self, "_fm_consts") else None
        if consts is None:
            if torch.cuda.is_available() and dev.type == "cuda" and torch.cuda.is_current_stream_capturing():
                raise RuntimeError("fused loss tail: run one eager step before capturing a CUDA graph")
            inv_counts = torch.tensor([[1.0 / c for c in cs] for cs in key[0]], dtype=torch.float32,
                                      device=dev).reshape(len(nets), nh)
            inv_ns = torch.tensor([1.0 / n for n in key[1]], dtype=torch.float32, device=dev)
            if not hasattr(self, "_fm_consts"):
                self._fm_consts = {}
            consts = self._fm_consts[key] = (inv_counts, inv_ns)
        inv_counts, inv_ns = consts
        S = torch.stack([st for st, _, _, _, _ in nets])            # [N, nh, 2]
        T = torch.stack([ss for _, _, _, ss, _ in nets])            # [N, 3, 2]
        score_term = (T[:, 0, 0] / T[:, 0, 1]) if relative else (T[:, 0, 0] * inv_ns)
        if skip < nh:
            hidden = (S[:, skip:, 0] / S[:, skip:, 1]) if relative else (S[:, skip:, 0] * inv_counts[:, skip:])
            terms = torch.cat([hidden, score_term[:, None]], 1)
        else:
            terms = score_term[:, None]
        fm_total = terms.mean(1).sum() / len(nets)
        loss_dis = ((T[:, 1, 0] + T[:, 1, 1]) * inv_ns).sum()
        means = (T[:, 2, :] * inv_ns[:, None]).sum(0)                # (pred_real, pred_fake)
        return fm_total, loss_dis, -means[1], means[0], means[1]

    def is_discriminator_step(self, batch_idx: int) -> bool:
        return (not (batch_idx % self.update_discriminator_every)) and self.warmed_up

    def training_step(self, batch, batch_idx, eps: Optional[torch.Tensor] = None, grad_hook=None):
        """rave/model.py:288-424.  `grad_hook(params)` (optional) runs between backward and the
        optimiser step: the data-parallel gradient all-reduce plugs in there (rave_b200/ddp.py)."""
        x_raw = batch
        is_dis = self.is_discriminator_step(batch_idx)
        return self.train_body(x_raw, is_dis, eps, grad_hook)

    def train_body(self, x_raw, is_dis: bool, eps: Optional[torch.Tensor] = None, grad_hook=None):
        """Everything `training_step` does for one batch once the step kind is known (no host-side
        decisions, no device->host sync: capturable in a CUDA graph)."""
        gen_opt, dis_opt = self.optimizers()
        dis_params = [p for p in self.discriminator.parameters()]
        for p in dis_params:                       # G-step: no discriminator wgrad (discarded work)
            p.requires_grad_(is_dis)

        loss_gen, loss_dis, aux = self.compute_losses(x_raw, is_dis, eps)

        if is_dis:
            dis_opt.zero_grad(set_to_none=True)
            loss_dis.backward()
            if grad_hook is not None:
                grad_hook(dis_params)
            dis_opt.step()
            if getattr(self, "_static_disc_prep", False):
                # GraphedTrainer keeps the discriminator's prepared (weight-normalised, tap-major bf16) weights in
                # persistent buffers: rewrite them now that the parameters moved (engine.enable_static_prep)
                from . import engine
                engine.refresh_static_prep(self.discriminator)
        else:
            gen_opt.zero_grad(set_to_none=True)
            loss_gen_value = 0.
            for k, v in loss_gen.items():
                loss_gen_value = loss_gen_value + v * self.weights.get(k, 1.)
            loss_gen_value.backward()
            if grad_hook is not None:
                grad_hook([p for g in gen_opt.param_groups for p in g["params"]])
            gen_opt.step()

        self.log("beta_factor", self.beta_factor)
        if self.warmed_up:
            self.log("loss_dis", loss_dis)
            self.log("pred_real", aux["pred_real"].mean())
            self.log("pred_fake", aux["pred_fake"].mean())
        self.log_dict(loss_gen)
        return self.logged

    # ------------------------------------------------------------------ validation
    def validation_step(self, x, batch_idx, eps: Optional[torch.Tensor] = None):
        """rave/model.py:426-444: reconstruct one validation batch and log `validation`, the full-band spectral
        distance (the fused spectral kernels).  Returns (cat([x, y], -1), posterior mean [B, D, L] or None), the
        mean for a VariationalEncoder only.  `eps` injects the reparametrisation noise as in training_step."""
        with torch.no_grad():
            z = self.encode(x)
            if isinstance(self.encoder, blocks.VariationalEncoder):
                mean = torch.split(z, z.shape[1] // 2, 1)[0]
            else:
                mean = None
            z = (self.encoder.reparametrize(z, eps) if eps is not None else self.encoder.reparametrize(z))[0]
            y = self.decode(z)
            distance = self.audio_distance(x, y)
            self.log("validation", sum(distance.values()))
            return torch.cat([x, y], -1), mean

    def validation_epoch_end(self, out):
        """rave/model.py:446-495 without the audio logging: probe the receptive field once (it turns on the
        valid-signal crop of training_step), then, in phase 1 of a VariationalEncoder model, fit the latent PCA
        (`latent_mean`, `latent_pca`, `fidelity`, read by the prior) on this epoch's posterior means and log
        fidelity_{0.8,0.9,0.95,0.99}.  Other encoders only get the receptive field, as in the reference."""
        if not sum(self._receptive_field_host()):
            self.set_receptive_field(*core.get_rave_receptive_field(self, n_channels=self.n_channels))
        if not len(out):
            return
        if not self.warmed_up and isinstance(self.encoder, blocks.VariationalEncoder):
            latent_mean, components, fidelity = core.latent_analysis([mean for _, mean in out], self.latent_size)
            with torch.no_grad():
                self.latent_mean.copy_(latent_mean)
                self.latent_pca.copy_(components)
                self.fidelity.copy_(fidelity)
            for p in (.8, .9, .95, .99):
                self.log(f"fidelity_{p}", (fidelity > p).to(torch.uint8).argmax().float())
        self.eval_number += 1
