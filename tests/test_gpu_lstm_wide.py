"""The wide LSTM-CRF models (hidden 768: dna_r9.4.1@v3.1, hidden 1024: dna_r10.4.1@v4.3) on the grid-wide recurrent kernel
(lstm_rec_wide.cu): the kernel, the encoder, the old-style config, the full v4.3 batch, the reference fixture and the CLI."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import crf_oracle as O
from oracle import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the budgets of test_gpu_pipeline.py
TOL_FP16_MAX, TOL_FP16_MEAN = 8.0e-3, 6.0e-4
TOL_FP32_MAX, TOL_FP32_MEAN = 6.0e-2, 3.0e-3


def _perms(H):
    unit = torch.arange(H)
    perm_ih = (torch.arange(4)[None, :] * H + unit[:, None]).reshape(-1)                        # [unit][gate]
    perm_hh = (torch.arange(H // 8)[:, None, None] * 8 + torch.arange(4)[None, :, None] * H
               + torch.arange(8)[None, None, :]).reshape(-1)                                    # [unit/8][gate][unit%8]
    return perm_ih, perm_hh


def _model(spec, seed=25, batchsize=32, chunksize=1998):
    from bonito_b200.crf.model import Model
    weights = synth.make_weights(spec, seed=seed)
    model = Model(synth.model_config(spec))
    model.load_state_dict(synth.state_dict_from_weights(spec, weights))
    model.use_koi(batchsize=batchsize, chunksize=chunksize, quantize=False)
    return model.half().eval().to("cuda"), weights


# ---------------------------------------------------------------------------------------------------------------------
# CPU: fixture, seeded weights, old-style config
# ---------------------------------------------------------------------------------------------------------------------

def _gold(golden_dir):
    from oracle.make_golden import weights_digest
    gold = np.load(os.path.join(golden_dir, "forward_sup_lstm.npz"))
    spec = synth.model_spec("sup_lstm")
    weights = synth.make_weights(spec, seed=int(gold["seed"]), qr_f64=True)
    if weights_digest(weights) != str(gold["digest"]):
        pytest.skip("seeded sup_lstm weights round differently on this CPU: fixture not comparable")
    return gold, spec, weights


def test_oracle_reproduces_the_sup_lstm_fixture(golden_dir):
    """The CPU oracle (fp32) reproduces the reference module tree's v4.3-shaped forward and its decode_batch strings."""
    gold, spec, weights = _gold(golden_dir)
    x = torch.from_numpy(gold["x"].astype(np.float32))
    with torch.no_grad():
        ref = O.lstm_crf_forward(weights, spec, x).permute(1, 0, 2)
    want = torch.from_numpy(gold["scores_ntc"])           # every col_stride-th score column
    cs = int(gold["col_stride"])
    assert ref.shape == (2, 67, 4096) and want.shape == (2, 67, 4096 // cs)
    assert torch.allclose(ref[..., ::cs], want, atol=5e-5, rtol=0), (ref[..., ::cs] - want).abs().max().item()
    _, seq, _, _ = O.decode_native(ref.numpy(), spec["state_len"], spec["blank_score"])
    assert [r[r != 0].tobytes().decode() for r in seq] == json.loads(str(gold["strings"]))


def test_seeded_sup_lstm_weights_are_not_degenerate(golden_dir):
    """The width-normalised gains give H = 1024 outputs that differ from chunk to chunk and rarely hit the +-5 clamp."""
    spec = synth.model_spec("sup_lstm", n_lstm=2)
    weights = synth.make_weights(spec, seed=25)
    x = synth.squiggle(4, 1200, seed=3).half().float()
    with torch.no_grad():
        s = O.lstm_crf_forward(weights, spec, x).permute(1, 0, 2)
    _, seq, _, _ = O.decode_native(s.numpy(), spec["state_len"], spec["blank_score"])
    strings = [r[r != 0].tobytes().decode() for r in seq]
    saturated = float((s.abs() >= 5.0).float().mean())
    print("sup_lstm seeded weights: bases per chunk", [len(t) for t in strings], f"clamped {saturated:.4f}")
    assert len(set(strings)) == len(strings) and min(len(t) for t in strings) > 40
    assert saturated < 0.02


def test_old_style_config_builds_the_v3_1_encoder():
    """An old-style `[encoder]` config (dna_r9.4.1@v3.1 keys) builds through rnn_encoder into the module tree the oracle
    describes: 1 -> 4 -> 16 stem, conv3 k19 stride 5 swish, 5 LSTMs of width 768, tanh x 5 head with bias."""
    from bonito_b200 import nn as bnn
    from bonito_b200.crf.model import Model
    spec = synth.old_style_spec(n_lstm=2)
    cfg = synth.old_style_config(spec)
    assert "type" not in cfg["encoder"] and cfg["encoder"]["features"] == 768 and cfg["encoder"]["stride"] == 5
    weights = synth.make_weights(spec, seed=5)
    model = Model(cfg)
    model.load_state_dict(synth.state_dict_from_weights(spec, weights))
    assert model.stride == 5
    lstms = [m for m in model.encoder.children() if isinstance(m, bnn.LSTM)]
    assert [bool(m.reverse) for m in lstms] == spec["reverse"]
    x = synth.squiggle(2, 400, seed=2)
    with torch.no_grad():
        got = model.encoder(x)
        want = O.lstm_crf_forward(weights, spec, x, expand_blanks=True)
    assert got.shape == want.shape and (got - want).abs().max().item() < 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_wide_kernel_is_exposed_for_768_and_1024_only():
    from bonito_b200 import native
    assert native.lstm_wide_ctas(768) == 96 and native.lstm_wide_ctas(1024) == 128
    assert native.lstm_wide_ctas(384) == 0 and native.lstm_wide_ctas(512) == 0
    assert native.lstm_cluster_size(768) == 0 and native.lstm_cluster_size(1024) == 0     # the generic kernel's query
    assert native.lstm_wide_resident(1024) >= 128 and native.lstm_wide_resident(768) >= 96


@pytest.mark.gpu
@pytest.mark.parametrize("hidden,n,t,reverse", [
    (768, 1, 1, False), (768, 5, 17, True), (768, 65, 40, False), (768, 200, 2, True), (768, 130, 17, False),
    (1024, 1, 40, True), (1024, 5, 2, False), (1024, 64, 17, True), (1024, 130, 40, False), (1024, 200, 17, True),
])
def test_wide_lstm_layer_matches_oracle(hidden, n, t, reverse):
    from bonito_b200 import native
    H, G = hidden, native.lstm_wide_ctas(hidden)
    g = torch.Generator().manual_seed(hidden + n + t)
    x = (torch.randn(t, n, H, generator=g) * 0.5).half()
    w_ih = (torch.randn(4 * H, H, generator=g) / H ** 0.5).half()
    w_hh = (torch.randn(4 * H, H, generator=g) / H ** 0.5).half()
    b = (torch.randn(4 * H, generator=g) * 0.3).half()
    perm_ih, perm_hh = _perms(H)
    wih, bias, whh = (v.cuda().contiguous() for v in (w_ih[perm_ih], b[perm_ih], w_hh[perm_hh]))

    def run(xs):
        xs = xs.cuda().contiguous()
        gx = torch.full((t, G, n, 32), float("nan"), dtype=torch.float16, device="cuda")
        native.gemm(xs, H, wih, bias, gx, 32, t * n, 4 * H, H, rows_inner=n, valid_inner=n, stride_inner=1,
                    stride_outer=G * n, cb_width=32, cb_rows=n)
        y = torch.full((t, n, H), float("nan"), dtype=torch.float16, device="cuda")
        ws = torch.empty(native.lstm_rec_wide_workspace_bytes(n, H), dtype=torch.uint8, device="cuda")
        native.lstm_rec_wide(gx, whh, y, t, n, H, reverse, workspace=ws)
        off = native.lstm_rec_wide_status_offset(n, H)
        torch.cuda.synchronize()
        assert int(ws[off:off + 4].view(torch.int32).item()) == 0
        return y.cpu()

    y = run(x)
    ref = O.lstm_layer(x.float(), w_ih.float(), w_hh.float(), b.float(), torch.zeros(4 * H), reverse)
    err = (y.float() - ref).abs().max().item()
    print(f"wide LSTM H={H} n={n} t={t} reverse={reverse}: max|err| {err:.2e}")
    assert err <= 5e-3, err
    assert torch.equal(run(x), y)                                  # two launches are bitwise identical
    flipped = run(x.flip(1))                                       # chunk order reversed: every chunk changes position
    assert torch.equal(flipped.flip(1), y)


def _features_errors(feats, rfeats, n_lstm):
    errs = {"stem": (feats["stem"].float().cpu().permute(0, 2, 1) - rfeats["conv1"]).abs().max().item(),
            "conv": (feats["conv"].float().cpu() - rfeats["conv2"].permute(2, 0, 1)).abs().max().item()}
    for i in range(n_lstm):
        errs[f"lstm{i}"] = (feats[f"lstm{i}"].float().cpu() - rfeats[f"lstm{i}"]).abs().max().item()
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize("n,L", [(6, 1998), (70, 996)])
def test_sup_lstm_encoder_matches_oracle(n, L):
    """The v4.3 shape (H = 1024, 5 LSTM layers, 4096 scores) through the engine, with per-layer features, against the oracle
    with fp16 rounding points and the fp32 oracle."""
    spec = synth.model_spec("sup_lstm")
    model, weights = _model(spec)
    x = synth.squiggle(n, L, seed=n).half()
    events = []
    with torch.inference_mode():
        scores, feats = model.native_plan("cuda").forward(x.cuda(), return_features=True, events=events)
    torch.cuda.synchronize()
    assert {name for name, _, _ in events} == {"conv_stem", "conv_gemm", "lstm_in_gemm", "lstm_rec", "crf_gemm"}
    for fp16, tol_max, tol_mean in ((True, TOL_FP16_MAX, TOL_FP16_MEAN), (False, TOL_FP32_MAX, TOL_FP32_MEAN)):
        with torch.no_grad():
            ref, rfeats = O.lstm_crf_forward(weights, spec, x.float(), return_features=True, fp16=fp16)
        errs = _features_errors(feats, rfeats, spec["n_lstm"])
        err = (scores.float().cpu() - ref.permute(1, 0, 2)).abs()
        errs["scores_max"], errs["scores_mean"] = err.max().item(), err.mean().item()
        print("sup_lstm", n, L, "oracle-fp16" if fp16 else "oracle-fp32", {k: f"{v:.2e}" for k, v in errs.items()})
        assert scores.shape == (n, ref.shape[0], 4096)
        assert errs["scores_max"] <= tol_max, errs
        assert errs["scores_mean"] <= tol_mean, errs


@pytest.mark.gpu
def test_old_style_v3_1_shape_matches_oracle():
    """dna_r9.4.1@v3.1 through its old-style config: H = 768, 4-channel stem, stride 5, tanh x 5 head with bias.  Budgets of
    test_old_style_crf_head_tanh_and_scale; the kernel decoder and the oracle decoder give the same bases on the same scores."""
    from bonito_b200.decode import beam_search
    spec = synth.old_style_spec()
    model, weights = _model(spec, seed=31, chunksize=2000)
    n, L = 6, 2000
    x = synth.squiggle(n, L, seed=n + 1).half()
    with torch.inference_mode():
        scores = model(x.cuda())
        seqs, _, _ = beam_search(scores)
    with torch.no_grad():
        ref = O.lstm_crf_forward(weights, spec, x.float(), fp16=True).permute(1, 0, 2)
    got = scores.float().cpu()
    err = (got - ref).abs()
    print(f"v3.1 shape: max |err| {err.max().item():.2e} mean {err.mean().item():.2e}")
    assert got.shape == (n, 400, 4096) and got.abs().max().item() <= 5.0 + 1e-6
    assert err.max().item() <= 2.5e-2 and err.mean().item() <= 1.5e-3, (err.max().item(), err.mean().item())
    _, o_seq, _, _ = O.decode_native(got.numpy(), spec["state_len"], spec["blank_score"])
    got_seqs = [r[r != 0].tobytes() for r in seqs.cpu().numpy()]
    assert got_seqs == [r[r != 0].tobytes() for r in o_seq]
    assert min(len(s) for s in got_seqs) > 100


@pytest.mark.gpu
def test_sup_lstm_full_size():
    """The v4.3 basecaller batch at full size (96 x 9996 samples, T = 1666): determinism, sub-batch independence, 8 chunks
    against the fp16-rounding oracle, and sequences against oracle forward + oracle decode by edit distance."""
    from _helpers import edit_distance
    from bonito_b200.decode import beam_search, to_str
    from oracle import build_ref
    spec = synth.model_spec("sup_lstm")
    model, weights = _model(spec, batchsize=96, chunksize=9996)
    x = synth.squiggle(96, 9996, seed=7).half()
    with torch.inference_mode():
        s1 = model(x.cuda()).clone()
        s2 = model(x.cuda()).clone()
        small = model(x[40:73].cuda()).clone()
        seq, _, _ = beam_search(s1, scale=1.05, offset=0.2)
    assert s1.shape == (96, 1666, 4096)
    assert torch.equal(s1, s2) and torch.equal(small, s1[40:73])
    picks = [0, 17, 40, 63, 64, 72, 90, 95]
    with torch.no_grad():
        ref = O.lstm_crf_forward(weights, spec, x[picks].float(), fp16=True).permute(1, 0, 2).contiguous()
    got = s1[picks].float().cpu()
    err = (got - ref).abs()
    within = (err <= 1e-3 * ref.abs().clamp(min=1.0) + 1e-3).float().mean().item()
    print(f"sup_lstm full size vs fp16-rounding oracle: max {err.max().item():.2e} mean {err.mean().item():.2e} "
          f"within 1e-3 rel: {within:.5f}")
    assert err.max().item() <= 8e-3 and err.mean().item() <= 6e-4 and within >= 0.999
    o_moves, o_seq, o_q = build_ref.decode(ref.numpy(), spec["state_len"], 2.0, 1.05, 0.2)
    total = dist = exact = 0
    for k, i in enumerate(picks):
        a, b = to_str(seq[i]), o_seq[k][o_seq[k] != 0].tobytes().decode()
        d = edit_distance(a, b)
        dist, total, exact = dist + d, total + len(b), exact + (d == 0)
        assert len(b) > 500 and d <= 0.03 * len(b), (i, d, len(b))
    print(f"sequences: {exact}/{len(picks)} chunks identical, edit distance {dist} over {total} bases")
    assert dist <= 1e-2 * total and exact >= len(picks) // 2, (dist, total, exact)


@pytest.mark.gpu
def test_sup_lstm_against_the_reference_fixture(golden_dir):
    """The native engine against the reference module tree's fp32 forward (tests/golden/forward_sup_lstm.npz), with the
    criteria of test_headline_shape_against_the_reference_fixture."""
    from _helpers import identity
    from bonito_b200.crf.model import Model
    from bonito_b200.decode import beam_search, to_str
    gold, spec, weights = _gold(golden_dir)
    model = Model(synth.model_config(spec, batchsize=8, chunksize=400, overlap=0))
    model.load_state_dict(synth.state_dict_from_weights(spec, weights))
    model.use_koi(batchsize=8, chunksize=400, quantize=False)
    model = model.half().eval().cuda()
    with torch.inference_mode():
        scores = model(torch.from_numpy(gold["x"].astype(np.float16)).cuda())
        seq, _, _ = beam_search(scores)
    assert scores.shape == (2, 67, 4096)
    err = (scores[..., ::int(gold["col_stride"])].float().cpu() - torch.from_numpy(gold["scores_ntc"])).abs()
    print("vs reference fixture: max", err.max().item(), "mean", err.mean().item())
    assert err.max().item() <= 2e-2 and err.mean().item() <= 2e-3
    for got, want in zip([to_str(r) for r in seq], json.loads(str(gold["strings"]))):
        assert identity(got, want) >= 0.99, (got, want)


def _write_v43_model_dir(path, spec, weights, **cfg_kwargs):
    """config.toml + weights_1.tar in the v4.3 layout, with BatchNorm after every convolution (non-trivial statistics, so
    that fuse_bn_ changes the weights)."""
    import toml
    from bonito_b200.crf.model import Model
    cfg = synth.model_config(spec, batchnorm=True, **cfg_kwargs)
    sd = synth.state_dict_from_weights(spec, weights)
    full = Model(cfg).state_dict()
    gen = torch.Generator().manual_seed(11)
    for k in full:
        if k in sd:
            full[k] = sd[k]
        elif k.endswith("bn.weight"):
            full[k] = 1.0 + 0.2 * torch.randn(full[k].shape, generator=gen)
        elif k.endswith("bn.bias"):
            full[k] = 0.1 * torch.randn(full[k].shape, generator=gen)
        elif k.endswith("running_mean"):
            full[k] = 0.2 * torch.randn(full[k].shape, generator=gen)
        elif k.endswith("running_var"):
            full[k] = 0.5 + torch.rand(full[k].shape, generator=gen)
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.toml"), "w") as fh:
        toml.dump(cfg, fh)
    torch.save(full, os.path.join(path, "weights_1.tar"))
    return str(path)


@pytest.mark.gpu
def test_cli_basecaller_sup_lstm_model_dir(tmp_path):
    """`python -m bonito_b200 basecaller` on a v4.3-layout model directory prints the FASTQ basecall() produces."""
    from bonito_b200.crf.basecall import basecall
    from bonito_b200.nn import fuse_bn_
    from bonito_b200.reader import Reader
    from bonito_b200.util import load_model
    spec = synth.model_spec("sup_lstm", n_lstm=3)
    weights = synth.make_weights(spec, seed=4)
    mdir = _write_v43_model_dir(tmp_path / "model", spec, weights, batchsize=8, chunksize=2000, overlap=120)
    rdir = tmp_path / "reads"
    rdir.mkdir()
    for i, n in enumerate([5000, 1500, 7777]):
        np.save(rdir / f"read{i}.npy", 93.7 + 23.5 * synth.squiggle(1, n, seed=20 + i)[0, 0].numpy())
    out = subprocess.run([sys.executable, "-m", "bonito_b200", "basecaller", mdir, str(rdir), "--no-trim"], cwd=ROOT,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = out.stdout.strip().split("\n")
    records = {lines[i][1:]: (lines[i + 1], lines[i + 3]) for i in range(0, len(lines), 4)}
    assert sorted(records) == ["read0", "read1", "read2"]
    model = load_model(mdir, "cuda", use_koi=True).apply(fuse_bn_)
    reads = Reader(str(rdir)).get_reads(str(rdir), do_trim=False, scaling_strategy=model.config["scaling"],
                                        norm_params=model.config["standardisation"])
    p = model.config["basecaller"]
    for read, res in basecall(model, reads, batchsize=p["batchsize"], chunksize=p["chunksize"], overlap=p["overlap"]):
        assert records[read.read_id] == (res["sequence"], res["qstring"]) and len(res["sequence"]) > 50


@pytest.mark.gpu
def test_cli_refuses_a_width_without_a_kernel(tmp_path):
    spec = synth.model_spec("hac", n_lstm=1)
    spec["hidden"] = 512
    spec["convs"][2] = (16, 512, 19, 6, 9, "tanh")
    weights = synth.make_weights(spec, seed=4)
    mdir = synth.write_model_dir(str(tmp_path / "model"), spec, weights, batchsize=8, chunksize=2000, overlap=120)
    rdir = tmp_path / "reads"
    rdir.mkdir()
    np.save(rdir / "read0.npy", 93.7 + 23.5 * synth.squiggle(1, 3000, seed=1)[0, 0].numpy())
    out = subprocess.run([sys.executable, "-m", "bonito_b200", "basecaller", mdir, str(rdir)], cwd=ROOT,
                         capture_output=True, text=True, timeout=300)
    assert out.returncode != 0 and "no native path for this model" in out.stderr, out.stderr[-1500:]
    assert "768, 1024" in out.stderr


@pytest.mark.gpu
def test_quantize_stays_refused_on_the_wide_widths():
    from bonito_b200.crf.model import Model
    from bonito_b200.engine import UnsupportedModel
    spec = synth.model_spec("sup_lstm", n_lstm=1)
    model = Model(synth.model_config(spec))
    model.load_state_dict(synth.state_dict_from_weights(spec, synth.make_weights(spec, seed=1)))
    model.use_koi(batchsize=8, chunksize=1998, quantize=True)
    model = model.half().eval().cuda()
    with pytest.raises(UnsupportedModel, match="--quantize"):
        model.native_plan("cuda")
