"""Restatement of the v3 style transfer in eval mode: AdaptiveInstanceNormalization (rave/blocks.py:863-926) inside
EncoderV2 / GeneratorV2 (rave/blocks.py:514-714), and the export's learn / reset controls (scripts/export.py:213-230).
Pure torch, any dtype (the GPU tests run it in float64 as the arbiter of the bf16 engine).

The statistics live in a dict of the module buffers, keyed like the state_dict ('<layer>.mean_x', ...), and are updated
in place, as the reference's forward does."""
import torch

from oracle import rave_oracle as O

BUFFERS = ("mean_x", "std_x", "mean_y", "std_y", "learn_x", "learn_y", "num_update_x", "num_update_y")
STYLE_SEQUENCE = (   # (update_adain keyword arguments, which input) of tests/golden/style_v3_tiny.pt, in order
    (dict(learn_target=True, reset_target=True, reset_source=True), "target0"),
    (dict(learn_target=True), "target1"),
    (dict(learn_source=True), "source"),
    (dict(), "source"),
    (dict(reset_target=True), "source"),
)


def style_cfg(capacity=16, latent_size=16):
    return O.ArchConfig(capacity=capacity, latent_size=latent_size, ratios=(4, 4, 4, 2), activation="snake", adain=True)


def style_params(shapes, seed):
    """Parameters of the fixture's model, {key: tensor} drawn in sorted key order (whatever order the module lists
    them in): weights N(0, 1 / fan_in) with weight_g = |v| (spectral_oracle.seeded_params) scaled to the variance of
    PyTorch's default initialisation, 1 / (3 fan_in) (at 1 / fan_in the eleven residual Snake units of each chain
    amplify their input several-fold), then every Snake alpha replaced by 0.5 + U[0, 1) from its own generator (alpha
    near 0 would make Snake blow up)."""
    from oracle.spectral_oracle import seeded_params
    shapes = sorted(shapes)
    out = seeded_params(shapes, seed)
    for k in out:
        if k.endswith(("weight", "weight_v", "weight_g")):
            out[k] = out[k] * 3 ** -0.5
    g = torch.Generator().manual_seed(seed + 1)
    for k, s in shapes:
        if k.endswith("alpha"):
            out[k] = 0.5 + torch.rand(tuple(s), generator=g)
    return out


def adain_keys(sd):
    """Prefixes ('encoder.encoder.net.1.', ...) of every AdaIN layer in a state dict, in key order."""
    return sorted({k[:-len("mean_x")] for k in sd if k.endswith(".mean_x")})


def update_adain(st, learn_target=False, learn_source=False, reset_target=False, reset_source=False):
    """ScriptedRAVE.update_adain (scripts/export.py:213-230) on every AdaIN of `st`."""
    for p in adain_keys(st):
        st[p + "learn_x"].zero_()
        st[p + "learn_y"].zero_()
        if learn_target:
            st[p + "learn_y"].add_(1)
        if learn_source:
            st[p + "learn_x"].add_(1)
        for on, s in ((reset_target, "y"), (reset_source, "x")):
            if on:
                st[p + "mean_" + s].zero_()
                st[p + "std_" + s].fill_(1)
                st[p + "num_update_" + s].zero_()


def adain(x, st, p):
    """AdaptiveInstanceNormalization.forward in eval mode (rave/blocks.py:900-926)."""
    bs = x.shape[0]

    def learn(s):
        n = st[p + "num_update_" + s]
        for name, v in (("mean_", x.mean(-1, keepdim=True)), ("std_", x.std(-1, keepdim=True))):
            t = st[p + name + s]
            t[:bs] += (v - t[:bs]) / (n + 1)
        n += 1

    if st[p + "learn_y"].item():
        learn("y")
        return x
    if st[p + "learn_x"].item():
        learn("x")
    if st[p + "num_update_x"].item() and st[p + "num_update_y"].item():
        x = (x - st[p + "mean_x"][:bs]) / (st[p + "std_x"][:bs] + 1e-5)
        x = x * st[p + "std_y"][:bs] + st[p + "mean_y"][:bs]
    return x


def encoder_v3(x, sd, st, cfg, prefix="encoder.encoder."):
    """EncoderV2.forward with eval-mode AdaIN (the raw encoder output: mean and scale, no reparametrisation)."""
    p, k, i = prefix + "net.", cfg.kernel_size, 0
    x = O.conv1d(x, O.wn_weight(sd, f"{p}{i}."), None, pad=O.get_padding(2 * k + 1, mode=cfg.pad_mode))
    i += 1
    C = cfg.capacity
    for r, dil in zip(cfg.ratios, cfg.dilations):
        for d in dil:
            x = adain(x, st, f"{p}{i}.")
            i += 1
            x = O.dilated_unit(x, sd, f"{p}{i}.aligned.branches.0.net.", cfg, C, d)
            i += 1
        x = O._act(x, sd, f"{p}{i}.", cfg)
        i += 1
        x = O.conv1d(x, O.wn_weight(sd, f"{p}{i}."), None, stride=r, pad=O.get_padding(2 * r, r, mode=cfg.pad_mode))
        i += 1
        C *= 2
    x = O._act(x, sd, f"{p}{i}.", cfg)
    i += 1
    return O.conv1d(x, O.wn_weight(sd, f"{p}{i}."), None, pad=O.get_padding(k, mode=cfg.pad_mode))


def generator_v3(z, sd, st, cfg, prefix="decoder."):
    """GeneratorV2.forward with eval-mode AdaIN and amplitude modulation (the multiband output)."""
    p, k, i = prefix + "net.", cfg.kernel_size, 0
    C = 2 ** len(cfg.ratios) * cfg.capacity
    x = O.conv1d(z, O.wn_weight(sd, f"{p}{i}."), None, pad=O.get_padding(k, mode=cfg.pad_mode))
    i += 1
    for r, dil in zip(cfg.ratios[::-1], cfg.dilations[::-1]):
        x = O._act(x, sd, f"{p}{i}.", cfg)
        i += 1
        x = O.conv_transpose1d(x, O.wn_weight(sd, f"{p}{i}."), None, r, r // 2)
        i += 1
        C //= 2
        for d in dil:
            x = adain(x, st, f"{p}{i}.")
            i += 1
            x = O.dilated_unit(x, sd, f"{p}{i}.aligned.branches.0.net.", cfg, C, d)
            i += 1
    x = O._act(x, sd, f"{p}{i}.", cfg)
    i += 1
    x = O.conv1d(x, O.wn_weight(sd, f"{p}{i}."), None, pad=O.get_padding(2 * k + 1, mode=cfg.pad_mode))
    x, amp = x.split(x.shape[1] // 2, 1)
    return torch.tanh(x * torch.sigmoid(amp))


def snapshot(st, B):
    """The fixture's record of the AdaIN buffers: rows [:B] of the statistics, the flags and counters."""
    return {k: (v[:B] if v.dim() == 3 else v).detach().clone() for k, v in st.items()
            if k.rsplit(".", 1)[-1] in BUFFERS}


def run_sequence(sd, inputs, latents, cfg, dtype=torch.float32):
    """STYLE_SEQUENCE on the restatement: per step (encoder output, decoder output, buffer snapshot).  `sd` holds the
    parameters and the initial buffers; `inputs` / `latents` map 'target0' / 'target1' / 'source' to the encoder (PQMF)
    and decoder inputs of that step."""
    sd = {k: v.to(dtype) for k, v in sd.items()}
    st = {k: v.clone() for k, v in sd.items() if k.rsplit(".", 1)[-1] in BUFFERS}
    out = []
    for kw, which in STYLE_SEQUENCE:
        update_adain(st, **kw)
        e = encoder_v3(inputs[which].to(dtype), sd, st, cfg)
        y = generator_v3(latents[which].to(dtype), sd, st, cfg)
        out.append((e, y, snapshot(st, e.shape[0])))
    return out


# the fixture's inputs, regenerated from these seeds by fixture_inputs (only what the reference computed is stored)
AUDIO = {"target0": (301, 0.6), "target1": (302, 0.4), "source": (303, 0.15)}     # (seed, gain) of the audio
LATENT = {"target0": (311, 1.5), "target1": (312, 1.2), "source": (313, 0.5)}    # (seed, gain) of the latent
LATENT_FRAMES = 2


def audio_batch(B, T, seed, gain):
    """One audio batch of the fixture (the encoder sees its PQMF analysis): different gains give different styles."""
    g = torch.Generator().manual_seed(seed)
    return (gain * torch.randn(B, 1, T, generator=g)).clamp(-1, 1)


def latent(B, latent_size, L, seed, gain):
    """One decoder input of the fixture (a fixed latent per style)."""
    return gain * torch.randn(B, latent_size, L, generator=torch.Generator().manual_seed(seed))


def fixture_inputs(B, T, latent_size):
    """({name: encoder input}, {name: decoder input}) of the fixture: the PQMF analysis (the restatement's, pinned
    against the reference's) of seeded audio, and seeded latents of LATENT_FRAMES frames."""
    hk = O.pqmf_design(100, 16)[1]
    inputs = {k: O.pqmf_encode(audio_batch(B, T, seed, gain), hk) for k, (seed, gain) in AUDIO.items()}
    latents = {k: latent(B, latent_size, LATENT_FRAMES, seed, gain) for k, (seed, gain) in LATENT.items()}
    return inputs, latents


def pack(snap):
    """A buffer snapshot as (layout [(key, shape)] in sorted key order, one flat fp32 tensor): one stored tensor per
    step instead of ~180 small ones."""
    keys = sorted(snap)
    return [(k, tuple(snap[k].shape)) for k in keys], torch.cat([snap[k].reshape(-1).float() for k in keys])


def unpack(flat, layout):
    out, o = {}, 0
    for k, shape in layout:
        n = 1
        for d in shape:
            n *= d
        out[k] = flat[o:o + n].reshape(shape)
        o += n
    return out


def load_fixture(path):
    """tests/golden/style_v3_tiny.pt with its inputs regenerated (`inputs`, `latents`) and every step's buffers
    unpacked into a {key: tensor} dict."""
    g = torch.load(path, weights_only=False)
    g["inputs"], g["latents"] = fixture_inputs(g["B"], g["T"], g["latent_size"])
    for step in g["steps"]:
        step["buffers"] = unpack(step["buffers"], g["buffer_layout"])
    return g
