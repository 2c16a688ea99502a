"""
Synthetic LSTM-CRF / transformer models and signals (a utility of the package: no kernel or oracle code in here).

There is no network in the build environment, so the real `dna_r10.4.1_e8.2_400bps_{fast,hac}@v5.0.0`
checkpoints cannot be fetched (`bonito/cli/download.py:31-83`); every test and benchmark uses
seeded random weights of the same architecture (shapes: SURVEY.md Appendix A), stored in the reference's own
on-disk format (`config.toml` + `weights_1.tar`) so the same files drive the reference modules, the oracle
and the native engine.
"""

import os

import numpy as np
import torch

SHAPES = {
    # name: (hidden, state_len)
    "fast": (96, 3),
    "hac": (384, 4),
    "tiny": (96, 3),
    "sup_lstm": (1024, 5),     # dna_r10.4.1@v4.3, the LSTM sup model: the same layer stack at width 1024
}


def model_spec(name="hac", n_lstm=5, stride=6, winlen=19):
    hidden, state_len = SHAPES[name]
    return dict(
        name=name, hidden=hidden, state_len=state_len, n_lstm=n_lstm,
        convs=[(1, 16, 5, 1, 2, "swish"), (16, 16, 5, 1, 2, "swish"), (16, hidden, winlen, stride, winlen // 2, "tanh")],
        reverse=[bool((i + 1) % 2) for i in range(n_lstm)],  # 1,0,1,0,1 as in @v4.3.toml:62-95
        blank_score=2.0, clamp=(-5.0, 5.0), stride=stride,
    )


def v40_spec(n_lstm=5):
    """dna_r10.4.1@v4.0, the R10.4.1 LSTM sup model before v4.3: the v4.3 stack at width 1024 with Clamp(-0.5, 3.5) behind
    each of the three convolutions, conv3 stride 5 with swish, and a Linear 1024 -> 256 (with bias) in front of the head."""
    spec = model_spec("sup_lstm", n_lstm=n_lstm, stride=5)
    spec["convs"][2] = (16, 1024, 19, 5, 9, "swish")
    spec.update(name="sup_lstm_v40", conv_clamp=(-0.5, 3.5), bottleneck=256)
    return spec


def old_style_spec(n_lstm=5, blank_score=2.0):
    """dna_r9.4.1@v3.1: the old-style `[encoder]` (built by rnn_encoder, bonito/crf/model.py:150-162): 1 -> 4 -> 16 stem,
    conv3 k19 stride 5 swish into width 768, LSTMs reversed (n_lstm - i) % 2, LinearCRFEncoder with bias, tanh, scale 5.
    `blank_score=None`: dna_r9.4.1@v3, whose head learns its blank scores ((n_base + 1) * 4^state_len outputs)."""
    return dict(
        name="r9_v3.1" if blank_score is not None else "r9_v3", hidden=768, state_len=5, n_lstm=n_lstm,
        convs=[(1, 4, 5, 1, 2, "swish"), (4, 16, 5, 1, 2, "swish"), (16, 768, 19, 5, 9, "swish")],
        reverse=[bool((n_lstm - i) % 2) for i in range(n_lstm)],
        blank_score=blank_score, clamp=None, stride=5, crf_activation="tanh", crf_scale=5.0, crf_bias=True, old_style=True,
    )


def old_style_config(spec, batchsize=32, chunksize=4000, overlap=500):
    """TOML-equivalent dict of an old-style config (the keys of dna_r9.4.1@v3.1.toml)."""
    enc = dict(stride=spec["convs"][2][3], winlen=spec["convs"][2][2], scale=spec["crf_scale"], features=spec["hidden"],
               rnn_type="lstm", activation=spec["convs"][2][5])
    if spec["blank_score"] is not None:                 # dna_r9.4.1@v3 has no blank_score key: learned blank scores
        enc["blank_score"] = spec["blank_score"]
    if spec["n_lstm"] != 5:
        enc["num_layers"] = spec["n_lstm"]
    return {
        "model": {"package": "bonito.crf"},
        "labels": {"labels": ["N", "A", "C", "G", "T"]},
        "input": {"features": 1},
        "qscore": {"bias": 0.0, "scale": 1.0},
        "encoder": enc,
        "global_norm": {"state_len": spec["state_len"]},
        "basecaller": {"batchsize": batchsize, "chunksize": chunksize, "overlap": overlap},
    }


def model_config(spec, batchnorm=False, batchsize=32, chunksize=3996, overlap=492):
    """TOML-equivalent dict for `Model(config)` (layout of dna_r10.4.1@v4.3.toml, and of @v4.0.toml for specs with
    `conv_clamp` / `bottleneck`; `old_style_config` for old_style specs)."""
    if spec.get("old_style"):
        return old_style_config(spec, batchsize=batchsize, chunksize=chunksize, overlap=overlap)
    sub = []
    for cin, cout, k, s, p, act in spec["convs"]:
        layer = dict(type="convolution", insize=cin, size=cout, bias=True, winlen=k, stride=s, padding=p, activation=act)
        if batchnorm:
            layer["norm"] = "batchnorm"
        sub.append(layer)
        if spec.get("conv_clamp") is not None:
            sub.append(dict(type="clamp", min=spec["conv_clamp"][0], max=spec["conv_clamp"][1]))
    sub.append(dict(type="permute", dims=[2, 0, 1]))
    for i in range(spec["n_lstm"]):
        sub.append(dict(type="lstm", size=spec["hidden"], insize=spec["hidden"], bias=True, reverse=int(spec["reverse"][i])))
    if spec.get("bottleneck") is not None:
        sub.append(dict(type="linear", in_features=spec["hidden"], out_features=spec["bottleneck"]))
    crf = dict(type="linearcrfencoder", insize=spec.get("bottleneck") or spec["hidden"], n_base=4,
               state_len=spec["state_len"], bias=False)
    if spec["blank_score"] is not None:
        crf["blank_score"] = spec["blank_score"]
    if spec.get("crf_activation") is not None:          # old-style head: tanh + scale instead of a Clamp layer
        crf["activation"] = spec["crf_activation"]
    if spec.get("crf_scale") is not None:
        crf["scale"] = spec["crf_scale"]
    sub.append(crf)
    if spec.get("clamp") is not None:
        sub.append(dict(type="clamp", min=spec["clamp"][0], max=spec["clamp"][1]))
    return {
        "model": {"package": "bonito.crf"},
        "labels": {"labels": ["N", "A", "C", "G", "T"]},
        "input": {"features": 1},
        "global_norm": {"state_len": spec["state_len"]},
        "qscore": {"scale": 1.05, "bias": 0.2},
        # picoampere input, standardised with fixed statistics (v4.3+/v5 LSTM configs; SURVEY.md Appendix A)
        "scaling": {"strategy": "pa"},
        "standardisation": {"standardise": 1, "mean": 93.7, "stdev": 23.5},
        "encoder": {"type": "serial", "sublayers": sub},
        "basecaller": {"batchsize": batchsize, "chunksize": chunksize, "overlap": overlap},
    }


def _orthogonal_blocks(rows, cols, block, gen, gain, f64=False):
    w = torch.empty(rows, cols)
    for r in range(0, rows, block):
        g = torch.randn(max(block, cols), max(block, cols), generator=gen)
        q, _ = torch.linalg.qr(g.double() if f64 else g)
        w[r:r + block] = q[:block, :cols].float()
    return w * gain


def make_weights(spec, seed=25, conv_gain=2.5, lstm_gain=1.5, head_gain=6.0, fp16_values=True, qr_f64=False,
                 bottleneck_gain=1.0, blank_gain=0.3, blank_bias=0.4):
    """
    Seeded, non-degenerate weights (oracle naming).  The reference's own init (orthogonal LSTM blocks,
    0.5*truncated-normal input bias, zero state bias: bonito/nn.py:362-390) with gains chosen so that
    decoded sequences vary from chunk to chunk, the +-5 clamp rarely saturates (SURVEY.md hard part H5) and the
    recurrence stays well conditioned (an LSTM gain of 3 makes the stack chaotic: a 1e-3 input perturbation grows to
    O(1) score differences, so no two half-precision implementations could agree; at 1.5 it shrinks).
    With `fp16_values` every tensor is rounded to fp16 (what `model.half()` feeds every implementation).
    `qr_f64=True` factorises the same Gaussian draws in float64: the fp16-rounded weights are then the same on every
    CPU (the float32 QR may round differently elsewhere), for fixtures that store a digest instead of the weights.
    Specs with a `bottleneck` get `linear.weight` / `linear.bias` (drawn after the LSTMs); with `blank_score=None` the head
    has 5 * 4^state_len outputs (learned blank scores) and its blank rows are scaled by `blank_gain` and shifted by
    `blank_bias` (bias, if any): the seeded stacks vary little from frame to frame, and blank rows drawn like the move rows
    give a few states stay scores near the tanh ceiling that the best path never leaves (one or two bases per chunk).
    """
    gen = torch.Generator().manual_seed(seed)
    H = spec["hidden"]
    w = {}
    for i, (cin, cout, k, _, _, _) in enumerate(spec["convs"]):
        fan_in = cin * k
        w[f"conv{i}.weight"] = torch.randn(cout, cin, k, generator=gen) * (conv_gain / fan_in ** 0.5)
        w[f"conv{i}.bias"] = torch.randn(cout, generator=gen) * 0.1
    for i in range(spec["n_lstm"]):
        w[f"lstm{i}.w_ih"] = _orthogonal_blocks(4 * H, H, H, gen, lstm_gain, qr_f64)
        w[f"lstm{i}.w_hh"] = _orthogonal_blocks(4 * H, H, H, gen, lstm_gain, qr_f64)
        w[f"lstm{i}.b_ih"] = 0.5 * torch.randn(4 * H, generator=gen).clamp(-2, 2)
        w[f"lstm{i}.b_hh"] = torch.zeros(4 * H)
    head_in = H
    if spec.get("bottleneck") is not None:
        head_in = spec["bottleneck"]
        w["linear.weight"] = torch.randn(head_in, H, generator=gen) * (bottleneck_gain / H ** 0.5)
        w["linear.bias"] = torch.randn(head_in, generator=gen) * 0.1
    C = 4 ** (spec["state_len"] + 1) if spec["blank_score"] is not None else 5 * 4 ** spec["state_len"]
    w["crf.weight"] = torch.randn(C, head_in, generator=gen) * (head_gain / head_in ** 0.5)
    if spec.get("crf_bias"):                 # old-style heads (LinearCRFEncoder default bias=True)
        w["crf.bias"] = torch.randn(C, generator=gen) * 0.1
    if spec["blank_score"] is None:          # rows [state][stay, m0..m3]
        w["crf.weight"].view(-1, 5, head_in)[:, 0] *= blank_gain
        if "crf.bias" in w:
            w["crf.bias"].view(-1, 5)[:, 0] += blank_bias
    if fp16_values:
        w = {k: v.half().float() for k, v in w.items()}
    return w


def state_dict_from_weights(spec, weights, prefix="encoder."):
    """Oracle naming -> the module tree's state_dict keys (SURVEY.md Appendix A 'State-dict names')."""
    sd = {}
    n_conv = len(spec["convs"])
    per_conv = 2 if spec.get("conv_clamp") is not None else 1     # Convolution [, Clamp]
    for i in range(n_conv):
        sd[f"{prefix}{i * per_conv}.conv.weight"] = weights[f"conv{i}.weight"]
        sd[f"{prefix}{i * per_conv}.conv.bias"] = weights[f"conv{i}.bias"]
    base = n_conv * per_conv + 1  # + Permute
    for i in range(spec["n_lstm"]):
        sd[f"{prefix}{base + i}.rnn.weight_ih_l0"] = weights[f"lstm{i}.w_ih"]
        sd[f"{prefix}{base + i}.rnn.weight_hh_l0"] = weights[f"lstm{i}.w_hh"]
        sd[f"{prefix}{base + i}.rnn.bias_ih_l0"] = weights[f"lstm{i}.b_ih"]
        sd[f"{prefix}{base + i}.rnn.bias_hh_l0"] = weights[f"lstm{i}.b_hh"]
    head = base + spec["n_lstm"]
    if "linear.weight" in weights:
        sd[f"{prefix}{head}.linear.weight"] = weights["linear.weight"]
        sd[f"{prefix}{head}.linear.bias"] = weights["linear.bias"]
        head += 1
    sd[f"{prefix}{head}.linear.weight"] = weights["crf.weight"]
    if "crf.bias" in weights:
        sd[f"{prefix}{head}.linear.bias"] = weights["crf.bias"]
    return sd


def write_model_dir(dirname, spec, weights, **config_kwargs):
    """Write `config.toml` + `weights_1.tar` in the reference's format (bonito/util.py:271-305)."""
    import toml
    os.makedirs(dirname, exist_ok=True)
    with open(os.path.join(dirname, "config.toml"), "w") as fh:
        toml.dump(model_config(spec, **config_kwargs), fh)
    torch.save(state_dict_from_weights(spec, weights), os.path.join(dirname, "weights_1.tar"))
    return dirname


def squiggle(n, length, seed=25, dwell=10.0, noise=0.15):
    """
    Piecewise-constant synthetic nanopore signal, ~N(0,1) after standardisation (SURVEY.md section 8d):
    levels ~ N(0,1) held for geometric dwell times (mean `dwell` samples) plus N(0, noise^2).
    """
    rng = np.random.default_rng(seed)
    out = np.empty((n, length), dtype=np.float32)
    for i in range(n):
        n_levels = int(length / dwell * 2) + 8
        dwells = rng.geometric(1.0 / dwell, size=n_levels)
        levels = rng.standard_normal(n_levels).astype(np.float32)
        sig = np.repeat(levels, dwells)[:length]
        out[i] = sig + noise * rng.standard_normal(length).astype(np.float32)
    return torch.from_numpy(out)[:, None, :]


def gaussian_signal(n, length, seed=25):
    gen = torch.Generator().manual_seed(seed)
    return torch.randn(n, 1, length, generator=gen)


# ---------------------------------------------------------------------------------------------------
# transformer (sup v5.0) shapes: bonito/models/configs/dna_r10.4.1@v5.0.toml
# ---------------------------------------------------------------------------------------------------

def sup_spec(depth=18, d_model=512, nhead=8, dim_feedforward=2048, state_len=5):
    alpha = round((2 * depth) ** 0.25, 7)
    beta = round((8 * depth) ** (-1 / 4), 7)
    return dict(
        name="sup", depth=depth, d_model=d_model, nhead=nhead, dim_feedforward=dim_feedforward, state_len=state_len,
        convs=[(1, 64, 5, 1, 2, "swish"), (64, 64, 5, 1, 2, "swish"), (64, 128, 9, 3, 4, "swish"),
               (128, 128, 9, 2, 4, "swish"), (128, d_model, 5, 2, 2, "swish")],
        alpha=alpha, beta=beta, window=(127, 128), scale=5.0, blank_score=2.0, stride=6,
    )


def sup_config(spec, batchnorm=False, batchsize=32, chunksize=12000, overlap=600):
    convs = []
    for cin, cout, k, s, p, act in spec["convs"]:
        layer = dict(type="convolution", insize=cin, size=cout, bias=True, winlen=k, stride=s, padding=p, activation=act)
        if batchnorm:
            layer["norm"] = "batchnorm"
        convs.append(layer)
    convs.append(dict(type="permute", dims=[0, 2, 1]))
    enc = {
        "type": "namedserial",
        "conv": {"type": "serial", "sublayers": convs},
        "transformer_encoder": {"type": "stack", "depth": spec["depth"], "layer": {
            "type": "transformerencoderlayer", "d_model": spec["d_model"], "nhead": spec["nhead"],
            "dim_feedforward": spec["dim_feedforward"], "deepnorm_alpha": spec["alpha"], "deepnorm_beta": spec["beta"],
            "attn_window": list(spec["window"])}},
        "upsample": {"type": "linearupsample", "d_model": spec["d_model"], "scale_factor": 2},
        "crf": {"type": "linearcrfencoder", "insize": spec["d_model"], "n_base": 4, "state_len": spec["state_len"],
                "bias": False, "scale": spec["scale"], "blank_score": spec["blank_score"], "expand_blanks": True,
                "permute": [1, 0, 2]},
    }
    return {
        "model": {"type": "seqdistmodel", "package": "bonito.transformer",
                  "seqdist": {"state_len": spec["state_len"], "alphabet": ["N", "A", "C", "G", "T"]}, "encoder": enc},
        "qscore": {"scale": 1.05, "bias": 1.3},
        "basecaller": {"batchsize": batchsize, "chunksize": chunksize, "overlap": overlap},
    }


def make_sup_weights(spec, seed=25, conv_gain=1.8, head_gain=0.55, fp16_values=True):
    """Seeded weights with the reference's initialisation scheme (xavier with the DeepNorm beta gain on the value /
    output / feed-forward projections: bonito/transformer/model.py:116-123; RMSNorm weights 1), state-dict names
    relative to `encoder.`."""
    gen = torch.Generator().manual_seed(seed)
    d, ff, beta = spec["d_model"], spec["dim_feedforward"], spec["beta"]
    w = {}
    for i, (cin, cout, k, _, _, _) in enumerate(spec["convs"]):
        w[f"conv.{i}.conv.weight"] = torch.randn(cout, cin, k, generator=gen) * (conv_gain / (cin * k) ** 0.5)
        w[f"conv.{i}.conv.bias"] = torch.randn(cout, generator=gen) * 0.1

    def xavier(rows, cols, gain):
        return torch.randn(rows, cols, generator=gen) * gain * (2.0 / (rows + cols)) ** 0.5

    for l in range(spec["depth"]):
        p = f"transformer_encoder.{l}."
        w[p + "self_attn.Wqkv.weight"] = torch.cat([xavier(2 * d, d, 1.0) * 3.0, xavier(d, d, beta)])
        w[p + "self_attn.out_proj.weight"] = xavier(d, d, beta)
        w[p + "self_attn.out_proj.bias"] = torch.randn(d, generator=gen) * 0.02
        w[p + "ff.fc1.weight"] = xavier(2 * ff, d, beta)
        w[p + "ff.fc2.weight"] = xavier(d, ff, beta)
        w[p + "norm1.weight"] = torch.ones(d)
        w[p + "norm2.weight"] = torch.ones(d)
    w["upsample.linear.weight"] = xavier(2 * d, d, 1.0)
    w["upsample.linear.bias"] = torch.randn(2 * d, generator=gen) * 0.02
    C = 4 ** (spec["state_len"] + 1)
    w["crf.linear.weight"] = torch.randn(C, d, generator=gen) * (head_gain / d ** 0.5)
    if fp16_values:
        w = {k: v.half().float() for k, v in w.items()}
    return w


def sup_state_dict(spec, weights, prefix="encoder."):
    sd = {prefix + k: v for k, v in weights.items()}
    for l in range(spec["depth"]):
        sd[f"{prefix}transformer_encoder.{l}.deepnorm_alpha"] = torch.tensor(spec["alpha"])
    return sd


# ---------------------------------------------------------------------------------------------------
# QuartzNet CTC shapes: dna_r9.4.1@v1 / @v2 (bonito/models/configs/dna_r9.4.1@v1.toml, @v2.toml)
# ---------------------------------------------------------------------------------------------------

QUARTZNET = {
    # name: (activation, [(filters, repeat, kernel, stride, residual, separable)] for C1, B1..B5, C2, C3)
    "v1": ("relu", [(256, 1, 33, 3, False, False), (256, 5, 33, 1, True, True), (256, 5, 39, 1, True, True),
                    (512, 5, 51, 1, True, True), (512, 5, 63, 1, True, True), (512, 5, 75, 1, True, True),
                    (512, 1, 87, 1, False, True), (1024, 1, 1, 1, False, False)]),
    "v2": ("swish", [(344, 1, 9, 3, False, False), (424, 2, 115, 1, True, True), (464, 7, 5, 1, True, True),
                     (456, 4, 123, 1, True, True), (440, 9, 9, 1, True, True), (280, 6, 31, 1, True, True),
                     (384, 1, 67, 1, False, True), (48, 1, 15, 1, False, False)]),
}


def quartznet_spec(name="v1", max_repeat=None):
    """Shapes of dna_r9.4.1@v1 ("v1", relu) or @v2 ("v2", swish); `max_repeat` caps the repeats (reduced test variants)."""
    activation, blocks = QUARTZNET[name]
    if max_repeat is not None:
        blocks = [(f, min(r, max_repeat), k, s, res, sep) for f, r, k, s, res, sep in blocks]
    return dict(name=f"quartznet_{name}", activation=activation, blocks=list(blocks), stride=blocks[0][3])


def quartznet_config(spec, batchsize=64, chunksize=4000, overlap=500, qscore=None):
    """TOML-equivalent dict of a `[[block]]` config (`package = "bonito.ctc"`); `qscore=(scale, bias)` adds a [qscore]."""
    cfg = {
        "model": {"package": "bonito.ctc"},
        "labels": {"labels": ["N", "A", "C", "G", "T"]},
        "input": {"features": 1},
        "encoder": {"activation": spec["activation"]},
        "block": [dict(filters=f, repeat=r, kernel=[k], stride=[s], dilation=[1], dropout=0.0, residual=res, separable=sep)
                  for f, r, k, s, res, sep in spec["blocks"]],
        "basecaller": {"batchsize": batchsize, "chunksize": chunksize, "overlap": overlap},
    }
    if qscore is not None:
        cfg["qscore"] = {"scale": float(qscore[0]), "bias": float(qscore[1])}
    return cfg


def make_quartznet_weights(spec, seed=25, conv_gain=0.5, head_gain=2.0):
    """
    Seeded fp16-representable state dict for `bonito_b200.ctc.model.Model(quartznet_config(spec))`, keyed by the module
    tree's names (the reference's, so it loads there too).  Convolutions ~ N(0, gain^2 / fan_in); every BatchNorm has
    gamma ~ U(0.6, 1.4), beta ~ N(0, 0.1^2), running_mean ~ N(0, 0.2^2) and running_var log-uniform over [0.05, 4], except
    channel 0, whose var is 0.01 with gamma 0.3: there eps = 1e-3 against 1e-5 changes the BatchNorm scale by 5 %.
    Depthwise convolutions have gain 1; pointwise, residual and dense ones `conv_gain`.  The random BatchNorm statistics
    multiply the second moment by E[gamma^2 / var] ~ 4.7, so conv_gain = 0.5 keeps the per-block RMS of both stacks
    between 0.3 and 1 through all 8 blocks (0.7 already grows it ~15x over the stack, 1.6 overflows).  The head is then
    centred and scaled on a seeded calibration read: each class's logit gets mean 0 and standard deviation `head_gain`
    over the frames, so the per-frame argmax moves between all five classes.
    """
    from bonito_b200.ctc.model import Model
    model = Model(quartznet_config(spec))
    gen = torch.Generator().manual_seed(seed)
    out = {}
    for name, t in model.state_dict().items():
        shape = t.shape
        if name.endswith("num_batches_tracked"):
            v = torch.tensor(100, dtype=torch.long)
        elif name.endswith("running_var"):
            u = torch.rand(shape, generator=gen)
            v = torch.exp(np.log(0.05) + u * (np.log(4.0) - np.log(0.05)))
            v[0] = 0.01
        elif name.endswith("running_mean"):
            v = 0.2 * torch.randn(shape, generator=gen)
        elif len(shape) == 1 and name.startswith("encoder") and name.endswith(".weight"):      # BatchNorm gamma
            v = 0.6 + 0.8 * torch.rand(shape, generator=gen)
            v[0] = 0.3
        elif len(shape) == 1 and name.startswith("encoder") and name.endswith(".bias"):        # BatchNorm beta
            v = 0.1 * torch.randn(shape, generator=gen)
        elif name.startswith("decoder") and name.endswith(".bias"):
            v = 0.1 * torch.randn(shape, generator=gen)
        else:                                                                                  # Conv1d weight [out][in][k]
            fan_in = shape[1] * shape[2]
            gain = head_gain if name.startswith("decoder") else 1.0 if "depthwise" in name else conv_gain
            v = torch.randn(shape, generator=gen) * (gain / np.sqrt(fan_in))
        out[name] = v if v.dtype == torch.long else v.to(torch.float16).float()
    # the encoder output has a large per-channel mean shared by every frame (relu / swish after random BatchNorm statistics),
    # which would make one class win everywhere: centre and scale the head on a seeded calibration read instead
    model.load_state_dict(out)
    model.double().eval()          # float64: the calibrated fp16 head must not depend on the CPU's fp32 convolution paths
    with torch.no_grad():
        feats = model.encoder(squiggle(1, 900, seed=seed + 1).double())[0]          # [F, T]
    w = out["decoder.layers.0.weight"][:, :, 0].double()
    logits = w @ feats.double()
    scale = head_gain / logits.std(dim=1, keepdim=True).clamp_min(1e-6)
    w = w * scale
    out["decoder.layers.0.weight"] = w[:, :, None].to(torch.float16).float()
    out["decoder.layers.0.bias"] = (-(w @ feats.double()).mean(dim=1)).to(torch.float16).float()
    return out


def write_quartznet_dir(dirname, spec, state_dict, **config_kwargs):
    """Write `config.toml` + `weights_1.tar` of a QuartzNet CTC model in the reference's format."""
    import toml
    os.makedirs(dirname, exist_ok=True)
    with open(os.path.join(dirname, "config.toml"), "w") as fh:
        toml.dump(quartznet_config(spec, **config_kwargs), fh)
    torch.save(state_dict, os.path.join(dirname, "weights_1.tar"))
    return dirname
