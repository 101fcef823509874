"""rave/prior/model.py: `Prior` / `VariationalPrior` with the reference's constructor, sub-modules and `state_dict`, and
a training step that runs as one autograd node on the library's kernels.

Training step (`training_step`), with D = latent_size, R = resolution, T' = T - D + 1 frames:
  1. frozen encode: `pretrained_vae.encode` in eval mode, forward only, on the existing chains;
  2. ops.prior_latent_classes: reparametrise, centre, PCA, DiagonalShift and QuantizedNormal.encode in one pass, written
     as int32 classes [B, T', D].  The stacked one-hot of the reference (R·D channels) is never built;
  3. _PriorStepFn: pre_net as a gather of weight columns (ops.prior_embed_fwd), the residual blocks on the conv engine
     with the gated unit in between (ops.gate_fwd), post_net.0, and the grouped head fused with the cross-entropy
     against the next frame's classes (ops.prior_head_ce_fwd); the backward runs the same plan in reverse.
In bf16 mode (`rave_b200.set_precision("bf16")`) the convs are wgmma launches on channel-last bf16 operands with fp32
residual and skip streams; in fp32 mode the same plan runs on the CUDA-core parity kernels in [B, C, T] fp32.
Sampling (`sample`) is one library call (ops.prior_sample) with cached per-block state; `decode_classes` turns classes
into audio through one kernel (ops.prior_classes_to_latent) and the RAVE decoder.  `generate` is the reference's dense
loop.
"""
import copy
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib, cc, engine, ops
from .core import DiagonalShift, QuantizedNormal
from .residual_block import ResidualBlock

SLOPE = 0.2       # nn.LeakyReLU(.2) of pre_net and post_net


class _ConvPlan:
    """The conv launches of the step: bf16 wgmma engine on channel-last operands (cl) or fp32 parity kernels on [B, C, T]
    (operand and fp32 stream are then the same tensor).  Every conv is stride 1 with left padding only, so input and
    output have the same T."""

    def __init__(self, cl: bool):
        self.cl = cl

    def conv(self, x, w, b, dil=1, pad_l=0, res=None, want_f32=True, want_op=False):
        Cout, Cin, K = w.shape
        if not self.cl:
            B, _, T = x.shape
            y = torch.empty(B, Cout, T, dtype=torch.float32, device=x.device)
            ops._gather(x, w, b, res, y, K, 1, dil, pad_l, Cin * K, K, ops.ACT_NONE, 0.0, None)
            return y, y
        return ops.conv1d_tc(x, ops.weight_to_tapmajor_bf16(w), bias=b, res_cl=res, dil=dil, pad=(pad_l, 0),
                             Lout=x.shape[1], want_f32=want_f32, want_act=want_op)

    def dgrad(self, dy, w, dil=1, pad_l=0, res=None, want_f32=True, want_op=False):
        """Input gradient (+ res) of conv(x, w) from its output gradient operand dy."""
        Cout, Cin, K = w.shape
        if not self.cl:
            B, _, T = dy.shape
            dx = torch.empty(B, Cin, T, dtype=torch.float32, device=dy.device)
            ops._scatter(dy, w, None, res, dx, K, 1, dil, pad_l, K, Cin * K, ops.ACT_NONE, 0.0, None)
            return dx, dx
        # stride 1: the transposed taps, reversed, read rows t + k·dil - ((K-1)·dil - pad_l)
        wt = ops.weight_to_tapmajor_bf16(w, transpose=True, flip=True)
        return ops.conv1d_tc(dy, wt, res_cl=res, dil=dil, pad=((K - 1) * dil - pad_l, pad_l), Lout=dy.shape[1],
                             want_f32=want_f32, want_act=want_op)

    def wgrad(self, dy, x, w, dil=1, pad_l=0):
        """(dw like w, dbias) from the output gradient operand dy and the input operand x."""
        Cout, Cin, K = w.shape
        if not self.cl:
            dw = torch.empty_like(w)
            ops._wgrad(dy, x, dw, K, 1, dil, pad_l, Cin * K, K, ops.ACT_NONE, ops.ACT_NONE, 0.0, None)
            return dw, dy.sum((0, 2))
        dwt = ops.conv1d_tc_wgrad(dy, x, K, 1, dil, pad_l)
        return ops.tapmajor_to_weight(dwt), ops.colsum_bf16(dy, dy.shape[1], Cout)


def _split_params(params, n_layers):
    pre = params[0:2]
    res = [params[2 + 6 * i: 8 + 6 * i] for i in range(n_layers)]
    post = params[2 + 6 * n_layers:]
    return pre, res, post


def _step_forward(cls, params, dilations, cl):
    """Loss of the step and what its backward needs."""
    plan = _ConvPlan(cl)
    n = len(dilations)
    (we, be), layers, (w0, b0, wh, bh) = _split_params(params, n)
    x_f32, x_op = ops.prior_embed_fwd(cls, we, be, cl, SLOPE)
    res_f32, res_op = x_f32, (x_op if cl else x_f32)
    saved = {"x0": res_op, "layers": []}
    skp = skp_op = None
    for i, (wd, bd, wr, br, ws, bs) in enumerate(layers):
        dil = dilations[i]
        pad = (wd.shape[-1] - 1) * dil
        h = plan.conv(res_op, wd, bd, dil, pad, want_f32=False, want_op=True)[1]
        g = ops.gate_fwd(h, cl)
        last = i == n - 1
        skp, skp_op = plan.conv(g, ws, bs, res=skp, want_op=last)
        saved["layers"].append((res_op, h, g))
        if not last:          # the last block's residual output is unused (rave/prior/model.py:104-110)
            res_f32, res_op = plan.conv(g, wr, br, res=res_f32, want_op=True)
    p = plan.conv(skp_op, w0, b0, want_f32=False, want_op=True)[1]
    loss = ops.prior_head_ce_fwd(p, wh, bh, cls, cl, SLOPE)
    saved.update(skp_op=skp_op, p=p)
    return loss, saved


def _step_backward(cls, params, dilations, cl, saved, gloss):
    plan = _ConvPlan(cl)
    n = len(dilations)
    (we, be), layers, (w0, b0, wh, bh) = _split_params(params, n)
    dp, dwh, dbh = ops.prior_head_ce_bwd(saved["p"], wh, bh, cls, gloss, cl, SLOPE)
    dskp = plan.dgrad(dp, w0, want_f32=False, want_op=True)[1]
    dw0, db0 = plan.wgrad(dp, saved["skp_op"], w0)
    grads = [None] * (6 * n)
    dres_f32 = dres_op = None
    for i in reversed(range(n)):
        wd, bd, wr, br, ws, bs = layers[i]
        x_op, h, g = saved["layers"][i]
        dil = dilations[i]
        pad = (wd.shape[-1] - 1) * dil
        dg = plan.dgrad(dskp, ws)[0]
        if dres_op is not None:
            dg = plan.dgrad(dres_op, wr, res=dg)[0]
        dh = ops.gate_bwd(dg, h, cl)
        dx_f32, dx_op = plan.dgrad(dh, wd, dil, pad, res=dres_f32, want_op=i > 0)
        grads[6 * i: 6 * i + 2] = plan.wgrad(dh, x_op, wd, dil, pad)
        if dres_op is not None:
            grads[6 * i + 2: 6 * i + 4] = plan.wgrad(dres_op, g, wr)
        grads[6 * i + 4: 6 * i + 6] = plan.wgrad(dskp, g, ws)
        dres_f32, dres_op = dx_f32, dx_op
    dwe, dbe = ops.prior_embed_wgrad(cls, dres_f32, saved["x0"], tuple(we.shape), cl, SLOPE)
    return [dwe, dbe] + grads + [dw0, db0, dwh, dbh]


class _PriorStepFn(torch.autograd.Function):
    """Prior forward + cross-entropy as one autograd node over the trained parameters (pre_net, residuals, post_net,
    in `Prior._trained_parameters` order).  The last block's rconv gets no gradient (None), as in the reference."""

    @staticmethod
    def forward(ctx, cls, dilations, cl, *params):
        loss, saved = _step_forward(cls, params, dilations, cl)
        ctx.cls, ctx.dilations, ctx.cl, ctx.saved = cls, dilations, cl, saved
        ctx.params = params
        return loss

    @staticmethod
    def backward(ctx, gloss):
        grads = _step_backward(ctx.cls, ctx.params, ctx.dilations, ctx.cl, ctx.saved, gloss.contiguous())
        ctx.saved = None
        return (None, None, None, *grads)


class Prior(nn.Module):

    def __init__(self, resolution, res_size, skp_size, kernel_size, cycle_size,
                 n_layers, pretrained_vae=None, fidelity=None, n_channels=1, latent_size=None, sr=44100):
        super().__init__()

        self.diagonal_shift = DiagonalShift()
        self.quantized_normal = QuantizedNormal(resolution)

        self.synth = pretrained_vae
        self.sr = sr

        if latent_size is not None:
            self.latent_size = 2**math.ceil(math.log2(latent_size))
        elif fidelity is not None:
            assert pretrained_vae, "giving fidelity keyword needs the pretrained_vae keyword to be given"
            latent_size = int(torch.where(pretrained_vae.fidelity > fidelity)[0][0])
            self.latent_size = 2**math.ceil(math.log2(latent_size))
        else:
            raise RuntimeError('please init Prior with either fidelity or latent_size keywords')

        self.pre_net = nn.Sequential(
            cc.Conv1d(resolution * self.latent_size, res_size, kernel_size,
                      padding=cc.get_padding(kernel_size, mode="causal"), groups=self.latent_size, bias=True),
            nn.LeakyReLU(SLOPE),
        )
        self.residuals = nn.ModuleList([
            ResidualBlock(res_size, skp_size, kernel_size, 2**(i % cycle_size)) for i in range(n_layers)
        ])
        self.post_net = nn.Sequential(
            cc.Conv1d(skp_size, skp_size, 1, bias=True),
            nn.LeakyReLU(SLOPE),
            cc.Conv1d(skp_size, resolution * self.latent_size, 1, groups=self.latent_size, bias=True),
        )

        self.n_channels = n_channels
        self.val_idx = 0
        self.cycle_size = cycle_size
        self.dilations = tuple(2**(i % cycle_size) for i in range(n_layers))
        rf = (kernel_size - 1) * sum(2**(np.arange(n_layers) % cycle_size)) + 1
        if pretrained_vae is not None:
            ratio = self.get_model_ratio()
            self.min_receptive_field = 2**math.ceil(math.log2(rf * ratio))
        self._optimizer = None
        self.logged = {}

    def get_model_ratio(self):
        """Samples per latent frame, from the model's configuration (no encode): the product of the encoder's conv
        strides times the PQMF band count (pqmf input) or the mel hop (mel input).  2048 for v2."""
        ratio = 1
        for m in self.synth.encoder.modules():
            if isinstance(m, nn.Conv1d):
                ratio *= m.stride[0]
        mode = getattr(self.synth, "input_mode", "pqmf")
        if mode == "pqmf":
            ratio *= self.synth.pqmf.hk.shape[0]
        elif mode == "mel":
            ratio *= self.synth.spectrogram.hop_length
        return ratio

    def _trained_parameters(self):
        return list(self.pre_net.parameters()) + list(self.residuals.parameters()) + list(self.post_net.parameters())

    def configure_optimizers(self):
        p = self._trained_parameters()
        if p[0].is_cuda:
            from ..optim import FusedAdam
            return FusedAdam(p, lr=1e-4)
        return torch.optim.Adam(p, lr=1e-4)

    def optimizers(self):
        if self._optimizer is None:
            self._optimizer = self.configure_optimizers()
        return self._optimizer

    def log(self, name, value):
        self.logged[name] = value.detach() if torch.is_tensor(value) else value

    @torch.no_grad()
    def encode(self, x, eps=None):
        self.synth.eval()
        z = self.synth.encode(x)
        z = self.post_process_latent(z, eps)
        return z

    @torch.no_grad()
    def decode(self, z):
        self.synth.eval()
        z = self.pre_process_latent(z)
        return self.synth.decode(z)

    def forward(self, x):
        """Dense forward on the stacked one-hot [B, R·D, T] (generation); the training step never builds it."""
        res = self.pre_net(x)
        skp = torch.tensor(0.).to(x)
        for layer in self.residuals:
            res, skp = layer(res, skp)
        x = self.post_net(skp)
        return x

    @torch.no_grad()
    def generate(self, x, argmax: bool = False):
        for i in range(x.shape[-1] - 1):
            start = i if cc.USE_BUFFER_CONV else None
            pred = self.forward(x[..., start:i + 1])
            if not cc.USE_BUFFER_CONV:
                pred = pred[..., -1:]
            pred = self.post_process_prediction(pred, argmax=argmax)
            x[..., i + 1:i + 2] = pred
        return x

    @torch.no_grad()
    def sample(self, prefix, n_frames: int, argmax: bool = False, uniform=None, return_logits: bool = False):
        """Cached autoregressive sampling: int32 classes [B, n_frames, D] that continue the int32 prefix [B, P, D]
        (1 <= P <= n_frames, B <= 64), plus the logits [B, n_frames - 1, D, R] of every step if `return_logits`.

        Step i reads frame i and writes frame i + 1 (the prefix's while i + 1 < P), like `generate`, but each step costs
        one frame of work: every block keeps the inputs its dilated conv still needs, and the whole loop is one
        library call (csrc/prior_sample.cu).  A class is the first argmax, or the first class whose running softmax
        probability exceeds the uniform draw u = uniform[b, i + 1, d]: the same distribution as the reference's
        `torch.multinomial`, whose draws cannot be reproduced bit for bit.  `uniform` [B, n_frames, D] injects the
        draws (frames < P unused); by default they are `torch.rand` on the current CUDA generator.  fp32 kernels in
        both precision modes."""
        if not prefix.is_cuda:
            raise _lib.RaveB200Error("the prior's sampler needs CUDA tensors (there is no CPU path)")
        B, _, D = prefix.shape
        if uniform is None and not argmax:
            uniform = torch.rand(B, n_frames, D, device=prefix.device)
        cls, logits = ops.prior_sample(self._trained_parameters(), self.cycle_size, prefix.to(torch.int32),
                                       uniform, n_frames, self.quantized_normal.resolution, argmax, return_logits)
        return (cls, logits) if return_logits else cls

    @torch.no_grad()
    def decode_classes(self, classes, dither=None, noise=None):
        """Audio of int32 classes [B, T, D]: QuantizedNormal.decode, DiagonalShift.inverse and pre_process_latent in one
        kernel (ops.prior_classes_to_latent), then synth.decode in eval mode.  `dither` [B, T, D] and `noise`
        [B, L - D, T - D + 1] inject the draws; by default they are drawn as the reference draws them, in its order:
        `torch.rand` on the classes' device, then `torch.randn` on the CPU."""
        self.synth.eval()
        B, T, D = classes.shape
        L = self.synth.latent_pca.shape[0]
        if dither is None:
            dither = torch.rand(B, T, D, device=classes.device)
        if noise is None:
            noise = torch.randn(B, L - D, T - D + 1).to(classes.device)
        z = ops.prior_classes_to_latent(classes.to(torch.int32), dither, noise, self.synth.latent_pca,
                                        self.synth.latent_mean, self.quantized_normal.resolution)
        return self.synth.decode(z)

    @torch.no_grad()
    def validation_epoch_end(self, out):
        """The reference's generation: a random first frame (randn_like the encoded first validation batch, shifted and
        quantised), `sample` over the shifted length, `decode_classes`; the audio goes to logged["generation"]."""
        x = torch.randn_like(self.encode(out[0]))
        cls = self.quantized_normal.classes(self.diagonal_shift(x)).permute(0, 2, 1).to(torch.int32)
        cls = self.sample(cls[:, :1].contiguous(), cls.shape[1])
        self.logged["generation"] = self.decode_classes(cls)
        self.val_idx += 1

    def split_classes(self, x):
        # B x D*C x T
        x = x.permute(0, 2, 1)
        x = x.reshape(x.shape[0], x.shape[1], self.latent_size, -1)
        x = x.permute(0, 2, 1, 3)  # B x D x T x C
        return x

    def post_process_prediction(self, x, argmax: bool = False):
        x = self.split_classes(x)
        shape = x.shape[:-1]
        x = x.reshape(-1, x.shape[-1])
        if argmax:
            x = torch.argmax(x, -1)
        else:
            x = torch.softmax(x - torch.logsumexp(x, -1, keepdim=True), -1)
            x = torch.multinomial(x, 1, True).squeeze(-1)
        x = x.reshape(shape[0], shape[1], shape[2])
        x = self.quantized_normal.to_stack_one_hot(x)
        return x

    # ------------------------------------------------------------------ training path
    def latent_classes(self, batch, eps=None):
        """int32 classes [B, T - D + 1, D] of the quantised, diagonally shifted latent of `batch` (one kernel after the
        frozen encode).  `eps` [B, latent channels, T] injects the reparametrisation noise (else drawn like the
        reference's randn_like)."""
        with torch.no_grad():
            self.synth.eval()
            z = self.synth.encode(batch)
            if eps is None:
                eps = torch.randn(z.shape[0], z.shape[1] // 2, z.shape[2], dtype=z.dtype, device=z.device)
            return ops.prior_latent_classes(z, eps, self.synth.latent_mean, self.synth.latent_pca, self.latent_size,
                                            self.quantized_normal.resolution)

    def step_loss(self, cls):
        """Mean cross-entropy of the next frame's classes given the classes (the reference's `latent_prediction`),
        differentiable with respect to the trained parameters."""
        if not cls.is_cuda:
            raise _lib.RaveB200Error("the prior's training step needs CUDA tensors (there is no CPU path)")
        cl = engine.precision() == "bf16"
        return _PriorStepFn.apply(cls, self.dilations, cl, *self._trained_parameters())

    def training_step(self, batch, batch_idx=None, eps=None):
        loss = self.step_loss(self.latent_classes(batch, eps))
        self.log("latent_prediction", loss)
        return loss

    def validation_step(self, batch, batch_idx=None, eps=None):
        with torch.no_grad():
            loss = self.step_loss(self.latent_classes(batch, eps))
        self.log("validation", loss)
        return batch

    def post_process_latent(self, z, eps=None):
        raise NotImplementedError()

    def pre_process_latent(self, z):
        raise NotImplementedError()


class VariationalPrior(Prior):
    """Prior over the PCA latents of a RAVE with a VariationalEncoder (scripts/train_prior.py:103-106)."""

    def __init__(self, *args, **kwargs):
        vae = kwargs.get("pretrained_vae", args[6] if len(args) > 6 else None)
        if vae is not None:
            from ..blocks import VariationalEncoder
            if not isinstance(vae.encoder, VariationalEncoder):
                raise NotImplementedError("prior not implemented for encoder of type %s" % (type(vae.encoder)))
        super().__init__(*args, **kwargs)

    def post_process_latent(self, z, eps=None):
        z = self.synth.encoder.reparametrize(z, eps)[0]
        z = z - self.synth.latent_mean.unsqueeze(-1)
        z = F.conv1d(z, self.synth.latent_pca.unsqueeze(-1))
        z = z[:, :self.latent_size]
        return z

    def pre_process_latent(self, z):
        noise = torch.randn(z.shape[0], self.synth.latent_size - z.shape[1], z.shape[-1]).type_as(z)
        z = torch.cat([z, noise], 1)
        z = F.conv1d(z, self.synth.latent_pca.T.unsqueeze(-1))
        z = z + self.synth.latent_mean.unsqueeze(-1)
        return z


class GraphedPriorTrainer:
    """The whole prior step -- frozen encode, latent classes (noise drawn inside the graph), forward, backward and
    FusedAdam -- captured as one CUDA graph and replayed.  Like graphs.GraphedTrainer, the eager warm-up the capture needs
    runs real updates; parameters, buffers and optimiser state are snapshotted before it and restored afterwards, so
    constructing the trainer does not move the prior.  In bf16 mode the frozen encoder's prepared weights are constants
    of the graph."""

    def __init__(self, prior, example_batch: torch.Tensor, warmup_steps: int = 3):
        if not example_batch.is_cuda:
            raise RuntimeError("GraphedPriorTrainer needs a CUDA batch")
        self.prior = prior
        self.x_static = example_batch.clone()
        opt = prior.optimizers()
        self.static_encoder = engine.precision() == "bf16"
        if self.static_encoder:
            engine.enable_static_prep(prior.synth.encoder)
        snap_tensors = [(t, t.detach().clone()) for t in list(prior.parameters()) + list(prior.buffers())]
        snap_opt = copy.deepcopy(opt.state_dict())
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup_steps):
                self._body()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        n0 = _lib.launch_count()
        with torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
            self.loss = self._body()
        self.launches = _lib.launch_count() - n0
        with torch.no_grad():
            for t, v in snap_tensors:
                t.copy_(v)
            old = {}
            for g_new, g_old in zip(opt.param_groups, snap_opt["param_groups"]):
                for p, idx in zip(g_new["params"], g_old["params"]):
                    old[p] = snap_opt["state"].get(idx)
                st_old = g_old.get("step")
                if torch.is_tensor(g_new.get("step")):
                    g_new["step"].copy_(st_old) if torch.is_tensor(st_old) else g_new["step"].zero_()
            for p, st in opt.state.items():
                for k, v in st.items():
                    if torch.is_tensor(v):
                        o = old.get(p)
                        v.copy_(o[k]) if (o is not None and k in o) else v.zero_()
        engine.invalidate_prepared()
        if self.static_encoder:
            engine.refresh_static_prep(prior.synth.encoder)

    def _body(self):
        prior = self.prior
        params = prior._trained_parameters()
        loss = prior.training_step(self.x_static)
        grads = torch.autograd.grad(loss, params, allow_unused=True)
        for p, g in zip(params, grads):
            p.grad = g
        prior.optimizers().step()
        return loss.detach()

    def step(self, batch: torch.Tensor):
        """One replay on `batch` (same shape as the example batch); returns the loss (device tensor)."""
        self.x_static.copy_(batch, non_blocking=True)
        self.graph.replay()
        engine.invalidate_prepared()
        self.prior.logged = {"latent_prediction": self.loss}
        return self.loss
