"""dna_r10.4.1@v4.0 (Clamp behind every convolution, conv3 stride 5 swish, Linear 1024 -> 256 in front of the head) and
dna_r9.4.1@v3 (learned blank scores, the learned-blank decode kernel) on the wide LSTM path: the oracle against the reference
fixtures and module tree, the layer-stack parser, the kernels, the engine, the decoder plumbing and the CLI."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _oracle_v40_v3 as X
from oracle import crf_oracle as O
from oracle import reference_shim, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the budgets of test_gpu_lstm_wide.py
TOL_FP16_MAX, TOL_FP16_MEAN = 8.0e-3, 6.0e-4
TOL_FP32_MAX, TOL_FP32_MEAN = 6.0e-2, 3.0e-3

FIXTURES = {"v40": ("forward_sup_lstm_v40.npz", synth.v40_spec), "v3": ("forward_r9_v3.npz",
                                                                          lambda: synth.old_style_spec(blank_score=None))}


def _gold(golden_dir, which):
    from oracle.make_golden import weights_digest
    name, make_spec = FIXTURES[which]
    gold = np.load(os.path.join(golden_dir, name))
    spec = make_spec()
    weights = synth.make_weights(spec, seed=int(gold["seed"]), qr_f64=True)
    if weights_digest(weights) != str(gold["digest"]):
        pytest.skip(f"seeded {which} weights round differently on this CPU: fixture not comparable")
    return gold, spec, weights


def _decode_oracle(scores_ntc, spec, qscale=1.0, qbias=0.0):
    """Oracle decode of native-layout scores: learned blanks for blank_score None, else the fixed blank."""
    if spec["blank_score"] is None:
        return X.decode_native_lb(scores_ntc, spec["state_len"], qscale, qbias)
    return O.decode_native(scores_ntc, spec["state_len"], spec["blank_score"], qscale, qbias)


def _native_layout(scores_tnc, spec):
    """Oracle [T, N, C] -> the engine's [N, T, C] (fixed blank: no blank column; learned blank: all columns)."""
    return scores_tnc.permute(1, 0, 2).contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# CPU: fixtures, reference module tree, seeded weights, layer-stack parser
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", ["v40", "v3"])
def test_oracle_reproduces_the_fixture(golden_dir, which):
    """The CPU oracle (fp32) reproduces the reference module tree's forward (sampled columns within 5e-5) and its
    decode_batch strings exactly."""
    gold, spec, weights = _gold(golden_dir, which)
    x = torch.from_numpy(gold["x"].astype(np.float32))
    with torch.no_grad():
        ref = _native_layout(X.lstm_crf_forward(weights, spec, x), spec)
    cs = int(gold["col_stride"])
    want = torch.from_numpy(gold["scores_ntc"])
    width = 4096 if which == "v40" else 5120
    assert ref.shape == (2, 68, width) and want.shape == (2, 68, -(-width // cs))
    assert torch.allclose(ref[..., ::cs], want, atol=5e-5, rtol=0), (ref[..., ::cs] - want).abs().max().item()
    if which == "v3":
        assert (np.arange(0, width, cs) % 5 == 0).sum() >= 90      # the stored columns include learned blank columns
    _, seq, _, _ = _decode_oracle(ref.numpy(), spec)
    strings = json.loads(str(gold["strings"]))
    assert X.strings(seq) == strings and min(len(s) for s in strings) > 20


@pytest.mark.skipif(not reference_shim.available(), reason="needs the reference checkout")
@pytest.mark.parametrize("which", ["v40", "v3"])
def test_reference_module_tree_matches_the_oracle(which):
    """The reference's own module tree, built from the configs synth writes, agrees with the oracle on the v4.0 stack
    (per-conv clamps, bottleneck) and on the v3 learned-blank head."""
    ref = reference_shim.load()
    spec = synth.v40_spec(n_lstm=2) if which == "v40" else synth.old_style_spec(n_lstm=2, blank_score=None)
    weights = synth.make_weights(spec, seed=7)
    model = ref.crf_model.Model(synth.model_config(spec))
    model.load_state_dict(synth.state_dict_from_weights(spec, weights))
    model.eval()
    x = synth.squiggle(2, 600, seed=8)
    with torch.no_grad():
        got = model.encoder(x)
        want = X.lstm_crf_forward(weights, spec, x, expand_blanks=True)
    assert got.shape == want.shape == (120, 2, 5120)
    assert (got - want).abs().max().item() < 1e-4


def test_model_config_writes_the_v40_layer_order():
    """synth's v4.0 config has the sublayers of dna_r10.4.1@v4.0.toml in its order, and the v3 config no blank_score."""
    cfg = synth.model_config(synth.v40_spec())
    sub = cfg["encoder"]["sublayers"]
    assert [layer["type"] for layer in sub] == ["convolution", "clamp"] * 3 + ["permute"] + ["lstm"] * 5 + [
        "linear", "linearcrfencoder", "clamp"]
    assert [(layer["min"], layer["max"]) for layer in sub[1:6:2]] == [(-0.5, 3.5)] * 3
    assert (sub[4]["stride"], sub[4]["activation"], sub[4]["size"]) == (5, "swish", 1024)
    assert (sub[12]["in_features"], sub[12]["out_features"], sub[13]["insize"]) == (1024, 256, 256)
    assert "blank_score" not in synth.model_config(synth.old_style_spec(blank_score=None))["encoder"]


def test_synthetic_v40_engages_the_conv_clamps():
    """The 3.5 bound of the per-conv clamps engages on a real fraction of the stem and conv3 outputs (swish is never
    below -0.279, so only the upper bound can), and the seeded v4.0 model calls varied sequences."""
    spec = synth.v40_spec(n_lstm=2)
    weights = synth.make_weights(spec, seed=25)
    x = synth.squiggle(4, 1200, seed=3).half().float()
    with torch.no_grad():
        s, feats = X.lstm_crf_forward(weights, spec, x, return_features=True, fp16=True)
    at_hi = {k: float((feats[k] == 3.5).float().mean()) for k in ("conv0", "conv1", "conv2")}
    print("share of outputs at the 3.5 bound", at_hi)
    assert all(v >= 0.03 for v in at_hi.values()), at_hi
    assert all(float(feats[k].max()) == 3.5 and float(feats[k].min()) > -0.28 for k in at_hi)
    _, seq, _, _ = O.decode_native(s.permute(1, 0, 2).numpy(), spec["state_len"], 2.0)
    strings = X.strings(seq)
    assert len(set(strings)) == len(strings) and min(len(t) for t in strings) > 40


def test_learned_blanks_change_the_calls(golden_dir):
    """On the v3 fixture's model the learned blank scores matter: replacing them with 2.0, or with 0, changes the calls."""
    gold, spec, weights = _gold(golden_dir, "v3")
    x = torch.from_numpy(gold["x"].astype(np.float32))
    with torch.no_grad():
        s = _native_layout(X.lstm_crf_forward(weights, spec, x), spec).numpy()
    _, seq, _, _ = X.decode_native_lb(s, spec["state_len"])
    s5 = s.reshape(2, 68, -1, 5)
    blanks = s5[..., 0]
    assert blanks.std(axis=2).mean() > 0.5 and blanks.std(axis=1).mean() > 0.1    # spread across states and frames
    for fixed in (2.0, 0.0):
        _, seq_fixed, _, _ = O.decode_native(s5[..., 1:].reshape(2, 68, -1), spec["state_len"], fixed)
        assert X.strings(seq_fixed) != X.strings(seq)


def test_score_layout():
    from bonito_b200.engine import score_layout
    assert score_layout(4096) == (5, False) and score_layout(5120) == (5, True)
    assert score_layout(256) == (3, False) and score_layout(320) == (3, True) and score_layout(1280, 4) == (4, True)
    for bad in ((4000, None), (5120, 4), (1024, 5)):
        with pytest.raises(ValueError):
            score_layout(*bad)


def _stack(spec):
    from bonito_b200.crf.model import Model
    return list(Model(synth.model_config(spec)).encoder.children())


def test_layer_stack_parser():
    """[Convolution, Clamp?] x 3, Permute, LSTM x L, Linear?, LinearCRFEncoder, Clamp? is accepted; a Clamp or a Linear
    anywhere else is refused."""
    from bonito_b200 import nn as bnn
    from bonito_b200.engine import UnsupportedModel, _parse_stack
    layers = _stack(synth.v40_spec(n_lstm=2))
    convs, conv_clamps, lstms, bottleneck, crf, clamps = _parse_stack(layers)
    assert len(convs) == 3 and all(c is not None for c in conv_clamps) and len(lstms) == 2
    assert isinstance(bottleneck, bnn.Linear) and isinstance(crf, bnn.LinearCRFEncoder) and len(clamps) == 1
    convs, conv_clamps, lstms, bottleneck, crf, clamps = _parse_stack(_stack(synth.model_spec("hac", n_lstm=2)))
    assert conv_clamps == [None] * 3 and bottleneck is None and len(clamps) == 1
    clamp, lin = layers[1], layers[9]
    bad = [
        layers[:7] + [clamp] + layers[7:],                  # Clamp between Permute and the LSTMs
        layers[:8] + [clamp] + layers[8:],                  # Clamp between two LSTMs
        layers[:9] + [clamp] + layers[9:],                  # Clamp between the LSTMs and the Linear
        layers[:10] + [clamp] + layers[10:],                # Clamp between the Linear and the head
        layers[:2] + [clamp] + layers[2:],                  # two Clamps behind a convolution
        layers + [clamp],                                   # two Clamps behind the head
        layers[:6] + [lin] + layers[6:],                    # Linear in front of the Permute
        layers[:8] + [lin] + layers[8:],                    # Linear between two LSTMs
        layers[:10] + [lin] + layers[10:],                  # two Linears
        layers[:11],                                        # no head clamp is fine ... (checked below)
    ]
    for stack in bad[:-1]:
        with pytest.raises(UnsupportedModel, match="Clamp\\?"):
            _parse_stack(stack)
    assert _parse_stack(bad[-1])[5] == []


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

def _model(spec, seed=25, batchsize=32, chunksize=1998):
    from bonito_b200.crf.model import Model
    weights = synth.make_weights(spec, seed=seed)
    model = Model(synth.model_config(spec))
    model.load_state_dict(synth.state_dict_from_weights(spec, weights))
    model.use_koi(batchsize=batchsize, chunksize=chunksize, quantize=False)
    return model.half().eval().to("cuda"), weights


def _swish_clamp(v):
    """fp16 activation output of swish + Clamp(-0.5, 3.5) on fp16-rounded pre-activations (fp32 arithmetic)."""
    v = v.half().float()
    return torch.nn.functional.silu(v).half().float().clamp(-0.5, 3.5)


@pytest.mark.gpu
@pytest.mark.parametrize("stem_impl", ["tc", "fma"])
@pytest.mark.parametrize("c1", [16, 4])
def test_conv_stem_ex_swish_clamp(stem_impl, c1, monkeypatch):
    """b200_conv_stem_fwd_ex with B200_ACT_SWISH_CLAMP on both stem kernels against the oracle; the old entry point with the
    same weights and plain swish is unchanged."""
    from bonito_b200 import native
    if stem_impl == "fma":
        monkeypatch.setenv("B200_STEM_IMPL", "fma")
    elif c1 == 4:
        pytest.skip("the tensor-core stem kernel exists for the 16 -> 16 shape only")
    g = torch.Generator().manual_seed(c1)
    n, L, padl, Lp = 3, 1000, 9, 1020
    x = (synth.squiggle(n, L, seed=1)[:, 0] * 1.3).half()
    w1 = (torch.randn(c1, 1, 5, generator=g) * 2.5 / 5 ** 0.5).half()
    b1 = (torch.randn(c1, generator=g) * 0.1).half()
    w2 = (torch.randn(16, c1, 5, generator=g) * 2.5 / (5 * c1) ** 0.5).half()
    b2 = (torch.randn(16, generator=g) * 0.1).half()
    dev = [t.cuda().contiguous() for t in (x, w1, b1, w2, b2)]
    out = torch.full((n * Lp * 16,), float("nan"), dtype=torch.float16, device="cuda")
    native.conv_stem(dev[0], dev[1], dev[2], native.ACT_SWISH_CLAMP, dev[3], dev[4], native.ACT_SWISH_CLAMP, out, Lp, padl,
                     bounds=(-0.5, 3.5, -0.5, 3.5))
    got = out.view(n, Lp, 16).float().cpu()
    a1 = _swish_clamp(torch.nn.functional.conv1d(x.float()[:, None], w1.float(), b1.float(), padding=2))
    want = _swish_clamp(torch.nn.functional.conv1d(a1, w2.float(), b2.float(), padding=2)).permute(0, 2, 1)
    err = (got[:, padl:padl + L] - want).abs()
    assert err.max().item() <= TOL_FP16_MAX and err.mean().item() <= TOL_FP16_MEAN, (err.max().item(), err.mean().item())
    assert torch.all(got[:, :padl] == 0) and torch.all(got[:, padl + L:] == 0)
    assert (want == 3.5).float().mean().item() > 0.03 and got.max().item() == 3.5
    plain = torch.empty_like(out)
    native.conv_stem(dev[0], dev[1], dev[2], native.ACT_SWISH, dev[3], dev[4], native.ACT_SWISH, plain, Lp, padl)
    assert plain.float().max().item() > 3.5                         # the old entry point does not clamp


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["wgmma", "mma"])
def test_gemm_swish_clamp_epilogue(impl):
    from bonito_b200 import native
    g = torch.Generator().manual_seed(3)
    m, n, k = 1000, 1024, 304
    a = (torch.randn(m, k, generator=g)).half()
    b = (torch.randn(n, k, generator=g) * 2.5 / k ** 0.5).half()
    bias = (torch.randn(n, generator=g) * 0.1).half()
    c = torch.full((m, n), float("nan"), dtype=torch.float16, device="cuda")
    native.gemm(a.cuda(), k, b.cuda(), bias.cuda(), c, n, m, n, k, act=native.ACT_SWISH_CLAMP, lo=-0.5, hi=3.5,
                impl=native.GEMM_TCGEN05 if impl == "wgmma" else native.GEMM_MMA_SYNC)
    want = _swish_clamp(a.float() @ b.float().T + bias.float())
    err = (c.float().cpu() - want).abs()
    assert err.max().item() <= TOL_FP16_MAX and err.mean().item() <= TOL_FP16_MEAN
    assert (want == 3.5).float().mean().item() > 0.03 and c.max().item() == 3.5


@pytest.mark.gpu
@pytest.mark.parametrize("which,n,L", [("v40", 6, 1995), ("v40", 70, 995), ("v3", 6, 2000)])
def test_encoder_matches_oracle(which, n, L):
    """The v4.0 stack (per-layer features, bottleneck) and the v3 learned-blank head through the engine against the oracle
    with fp16 rounding points and the fp32 oracle; the kernel decoder and the oracle decoder agree on the engine's scores."""
    from bonito_b200.decode import beam_search
    spec = synth.v40_spec() if which == "v40" else synth.old_style_spec(blank_score=None)
    model, weights = _model(spec, seed=31, chunksize=L)
    x = synth.squiggle(n, L, seed=n).half()
    events = []
    with torch.inference_mode():
        scores, feats = model.native_plan("cuda").forward(x.cuda(), return_features=True, events=events)
        seqs, _, _ = beam_search(scores)
    names = {"conv_stem", "conv_gemm", "lstm_in_gemm", "lstm_rec", "crf_gemm"}
    assert {name for name, _, _ in events} == (names | {"bottleneck_gemm"} if which == "v40" else names)
    width = 4096 if which == "v40" else 5120
    budgets = ((True, TOL_FP16_MAX, TOL_FP16_MEAN), (False, TOL_FP32_MAX, TOL_FP32_MEAN))
    if which == "v3":       # old-style tanh x 5 head: the fp16 budgets of test_old_style_v3_1_shape_matches_oracle
        budgets = ((True, 2.5e-2, 1.5e-3), budgets[1])

    def rel(got, want):     # feature errors relative to max(1, |value|): the unclamped swish stem of v3 reaches ~30
        return ((got.float().cpu() - want).abs() / want.abs().clamp(min=1.0)).max().item()

    for fp16, tol_max, tol_mean in budgets:
        with torch.no_grad():
            ref, rfeats = X.lstm_crf_forward(weights, spec, x.float(), return_features=True, fp16=fp16)
        ref = _native_layout(ref, spec)
        errs = {"stem": rel(feats["stem"].permute(0, 2, 1), rfeats["conv1"]),
                "conv": rel(feats["conv"], rfeats["conv2"].permute(2, 0, 1))}
        if which == "v40":
            errs["linear"] = rel(feats["linear"], rfeats["linear"])
        err = (scores.float().cpu() - ref).abs()
        errs["scores_max"], errs["scores_mean"] = err.max().item(), err.mean().item()
        print(which, n, L, "oracle-fp16" if fp16 else "oracle-fp32", {k: f"{v:.2e}" for k, v in errs.items()})
        assert scores.shape == (n, ref.shape[1], width)
        assert max(errs.values()) <= tol_max, errs
        assert errs["scores_mean"] <= tol_mean, errs
    if which == "v40":
        assert float(feats["stem"].max()) == 3.5 and float(feats["conv"].max()) == 3.5
        assert float((feats["conv"] == 3.5).float().mean()) > 0.03
    _, o_seq, _, _ = _decode_oracle(scores.float().cpu().numpy(), spec)
    got = [r[r != 0].tobytes() for r in seqs.numpy()]
    assert got == [r[r != 0].tobytes() for r in o_seq] and min(len(s) for s in got) > 100


@pytest.mark.gpu
def test_v40_full_size():
    """The v4.0 basecaller batch at full size (96 x 9996 samples, T = 2000): determinism, sub-batch independence, and 4
    chunks against the fp16-rounding oracle within the fp16 budgets."""
    spec = synth.v40_spec()
    model, weights = _model(spec, batchsize=96, chunksize=9996)
    x = synth.squiggle(96, 9996, seed=7).half()
    with torch.inference_mode():
        s1 = model(x.cuda()).clone()
        s2 = model(x.cuda()).clone()
        small = model(x[40:73].cuda()).clone()
    assert s1.shape == (96, 2000, 4096)
    assert torch.equal(s1, s2) and torch.equal(small, s1[40:73])
    picks = [0, 41, 72, 95]
    with torch.no_grad():
        ref = _native_layout(X.lstm_crf_forward(weights, spec, x[picks].float(), fp16=True), spec)
    err = (s1[picks].float().cpu() - ref).abs()
    within = (err <= 1e-3 * ref.abs().clamp(min=1.0) + 1e-3).float().mean().item()
    print(f"v4.0 full size vs fp16-rounding oracle: max {err.max().item():.2e} mean {err.mean().item():.2e} within {within:.5f}")
    assert err.max().item() <= TOL_FP16_MAX and err.mean().item() <= TOL_FP16_MEAN


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["v40", "v3"])
def test_against_the_reference_fixture(golden_dir, which):
    """The native engine against the reference module tree's fp32 forward, with the criteria of
    test_sup_lstm_against_the_reference_fixture; Model.decode_batch decodes learned blanks without a fixed blank score.
    The chunks are 68 frames long, so a string may also differ by at most two edits (a repeat such as GAGA... shifted by
    one frame against the fp32 reference)."""
    from _helpers import edit_distance, identity
    from bonito_b200.crf.model import Model
    gold, spec, weights = _gold(golden_dir, which)
    model = Model(synth.model_config(spec, batchsize=8, chunksize=340, overlap=0))
    model.load_state_dict(synth.state_dict_from_weights(spec, weights))
    model.use_koi(batchsize=8, chunksize=340, quantize=False)
    model = model.half().eval().cuda()
    with torch.inference_mode():
        scores = model(torch.from_numpy(gold["x"].astype(np.float16)).cuda())
        strings = model.decode_batch(scores)
    assert scores.shape == (2, 68, 4096 if which == "v40" else 5120)
    err = (scores[..., ::int(gold["col_stride"])].float().cpu() - torch.from_numpy(gold["scores_ntc"])).abs()
    print(which, "vs reference fixture: max", err.max().item(), "mean", err.mean().item())
    assert err.max().item() <= 2e-2 and err.mean().item() <= 2e-3
    for got, want in zip(strings, json.loads(str(gold["strings"]))):
        assert identity(got, want) >= 0.99 or edit_distance(got, want) <= 2, (got, want)


def _random_lb(n, t, k, seed, blank=None):
    g = torch.Generator().manual_seed(seed)
    s = (torch.randn(n, t, 4 ** k, 5, generator=g) * 1.7).clamp(-5, 5)
    if blank is not None:
        s[..., 0] = blank
    return s.reshape(n, t, -1).half()


@pytest.mark.gpu
@pytest.mark.parametrize("state_len,n,t", [(3, 3, 1), (4, 2, 1), (5, 2, 1), (3, 4, 17), (4, 3, 33), (5, 2, 61),
                                           (3, 2, 2000), (4, 2, 2000), (5, 1, 2000)])
def test_learned_blank_decode_matches_oracle(state_len, n, t):
    from bonito_b200.engine import CrfDecoder
    scores = _random_lb(n, t, state_len, seed=state_len * 100 + t)
    moves, seq, qual = CrfDecoder()(scores.cuda(), state_len, qscale=1.05, qbias=0.2)
    o_moves, o_seq, o_qual, _ = X.decode_native_lb(scores.float().numpy(), state_len, 1.05, 0.2)
    assert np.array_equal(moves.cpu().numpy(), o_moves)
    assert np.array_equal(seq.cpu().numpy(), o_seq)
    dq = np.abs(qual.cpu().numpy().astype(int) - o_qual.astype(int))
    assert dq.max() <= 1 and (dq != 0).mean() < 0.01
    if t > 1:
        assert 0.2 < o_moves.mean() < 0.95                          # the case is not degenerate


@pytest.mark.gpu
@pytest.mark.parametrize("state_len,n,t", [(3, 5, 333), (4, 3, 2000), (5, 2, 2000), (5, 3, 7)])
def test_learned_blank_decode_of_a_constant_blank_is_the_fixed_blank_decode(state_len, n, t):
    """A blank column of constant 2.0 through the learned-blank kernel gives bit-identical moves, sequence and qstring to
    the fixed-blank kernel on the same move scores."""
    from bonito_b200.engine import CrfDecoder
    scores = _random_lb(n, t, state_len, seed=t + state_len, blank=2.0).cuda()
    moves_only = scores.view(n, t, -1, 5)[..., 1:].reshape(n, t, -1).contiguous()
    lb = CrfDecoder()(scores, state_len, qscale=1.05, qbias=0.2)
    fixed = CrfDecoder()(moves_only, state_len, blank_score=2.0, qscale=1.05, qbias=0.2)
    for a, b in zip(lb, fixed):
        assert torch.equal(a, b)
    assert lb[0].float().mean().item() > 0.2


@pytest.mark.gpu
def test_learned_blank_scores_refuse_the_beam_search(monkeypatch):
    from bonito_b200.decode import beam_search
    scores = _random_lb(2, 50, 3, seed=1).cuda()
    with pytest.raises(ValueError, match="fixed blank"):
        beam_search(scores, decoder="beam")
    monkeypatch.setenv("B200_DECODER", "beam")
    with pytest.raises(ValueError, match="fixed blank"):
        beam_search(scores)
    seq, _, _ = beam_search(scores[..., :256].contiguous())     # 4^4 columns: fixed-blank scores still take the beam search
    assert seq.shape == (2, 50)


@pytest.mark.gpu
def test_revcomp_of_learned_blank_scores():
    """`--revcomp` on v3: the result is the decode of the reference's reverse_complement of the full scores, and the
    blank_score argument (2.0 by default, as the reference passes it) does not enter."""
    from bonito_b200.crf.basecall import compute_scores
    from bonito_b200.engine import CrfDecoder
    spec = synth.old_style_spec(n_lstm=2, blank_score=None)
    model, _ = _model(spec, seed=9, chunksize=2000)
    x = synth.squiggle(4, 2000, seed=5)
    res = compute_scores(model, x, reverse=True)
    res7 = compute_scores(model, x, reverse=True, blank_score=7.0)
    with torch.inference_mode():
        scores = model(x.half().cuda())
        rc = model.seqdist.reverse_complement(scores.permute(1, 0, 2)).permute(1, 0, 2).contiguous()
        moves, seq, qual = CrfDecoder()(rc, spec["state_len"])
    assert torch.equal(res["moves"], moves.cpu()) and torch.equal(res["sequence"], seq.cpu())
    assert torch.equal(res["qstring"], qual.cpu())
    assert all(torch.equal(res[k], res7[k]) for k in res)
    fwd = compute_scores(model, x)
    assert not torch.equal(fwd["sequence"], res["sequence"])


@pytest.mark.gpu
@pytest.mark.parametrize("change", ["conv_clamp", "bottleneck", "learned_blank"])
@pytest.mark.parametrize("shape", ["hac", "fast"])
def test_narrow_widths_refuse_the_new_layers(change, shape):
    from bonito_b200.crf.model import Model
    from bonito_b200.engine import UnsupportedModel
    spec = synth.model_spec(shape, n_lstm=2)
    if change == "conv_clamp":
        spec["conv_clamp"] = (-0.5, 3.5)
        spec["convs"][2] = spec["convs"][2][:5] + ("swish",)
    elif change == "bottleneck":
        spec["bottleneck"] = 64
    else:
        spec["blank_score"] = None
    model = Model(synth.model_config(spec))
    model.load_state_dict(synth.state_dict_from_weights(spec, synth.make_weights(spec, seed=1)))
    model.use_koi(batchsize=8, chunksize=1998, quantize=False)
    model = model.half().eval().cuda()
    with pytest.raises(UnsupportedModel, match="wide LSTM path only"):
        model.native_plan("cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["v40", "v3"])
def test_cli_basecaller(tmp_path, which):
    """`python -m bonito_b200 basecaller` on v4.0 / v3 model directories prints the FASTQ basecall() produces."""
    import toml
    from bonito_b200.crf.basecall import basecall
    from bonito_b200.reader import Reader
    from bonito_b200.util import load_model
    spec = synth.v40_spec(n_lstm=3) if which == "v40" else synth.old_style_spec(n_lstm=3, blank_score=None)
    weights = synth.make_weights(spec, seed=4)
    mdir = tmp_path / "model"
    mdir.mkdir()
    with open(mdir / "config.toml", "w") as fh:
        toml.dump(synth.model_config(spec, batchsize=8, chunksize=2000, overlap=120), fh)
    torch.save(synth.state_dict_from_weights(spec, weights), mdir / "weights_1.tar")
    rdir = tmp_path / "reads"
    rdir.mkdir()
    for i, n in enumerate([5000, 1500, 7777]):
        sig = synth.squiggle(1, n, seed=20 + i)[0, 0].numpy()
        np.save(rdir / f"read{i}.npy", 93.7 + 23.5 * sig if which == "v40" else sig)
    out = subprocess.run([sys.executable, "-m", "bonito_b200", "basecaller", str(mdir), str(rdir), "--no-trim"], cwd=ROOT,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = out.stdout.strip().split("\n")
    records = {lines[i][1:]: (lines[i + 1], lines[i + 3]) for i in range(0, len(lines), 4)}
    assert sorted(records) == ["read0", "read1", "read2"]
    model = load_model(str(mdir), "cuda", use_koi=True)
    reads = Reader(str(rdir)).get_reads(str(rdir), do_trim=False, scaling_strategy=model.config.get("scaling"),
                                        norm_params=model.config.get("standardisation"))
    p = model.config["basecaller"]
    for read, res in basecall(model, reads, batchsize=p["batchsize"], chunksize=p["chunksize"], overlap=p["overlap"]):
        assert records[read.read_id] == (res["sequence"], res["qstring"]) and len(res["sequence"]) > 0
