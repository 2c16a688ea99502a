"""
QuartzNet CTC models (dna_r9.4.1@v1, @v2): fixtures, oracle, greedy decode, layer-stack refusals (CPU) and the depthwise,
strided first-conv, relu-epilogue and CTC-head kernels, the full forward, basecall and the CLI (GPU).

Forward budgets: the noise floor is the spread between the oracle's reference-rounding mode (fp16 wherever the reference's
half model rounds) and its fp64 mode on the same input.  On the 2 x 1200 fixtures it is max 3.2e-2 / mean 5.0e-3 (v1) and
max 4.5e-2 / mean 6.2e-3 (v2) in log-prob units; the GPU must stay within twice the floor measured in the same test.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _oracle_ctc as oc  # noqa: E402
from bonito_b200 import synth  # noqa: E402
from bonito_b200.ctc.model import Model, greedy_collapse, greedy_step  # noqa: E402
from bonito_b200.engine import UnsupportedModel  # noqa: E402
from bonito_b200.engine_ctc import CtcPlan  # noqa: E402

SEEDS = {"v1": 51, "v2": 52}


def _model(version, state=None, max_repeat=None, **cfg):
    spec = synth.quartznet_spec(version, max_repeat=max_repeat)
    config = synth.quartznet_config(spec, **cfg)
    if state is None:
        state = synth.make_quartznet_weights(spec, seed=SEEDS[version])
    m = Model(config)
    m.load_state_dict(state)
    return m.eval(), config, state


def _fixture(golden_dir, version):
    return np.load(os.path.join(golden_dir, f"forward_ctc_{version}.npz"))


def _decode_str(labels, probs, qscale=1.0, qbias=0.0):
    s, q, mv = greedy_collapse(labels, probs, "NACGT", qscale, qbias)
    return s[s != 0].tobytes().decode(), q[q != 0].tobytes().decode(), mv


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("version", ["v1", "v2"])
def test_fixture_oracle_decode_and_activity(golden_dir, version):
    from oracle.make_golden import weights_digest
    fx = _fixture(golden_dir, version)
    _, config, state = _model(version)
    assert weights_digest(state) == str(fx["digest"]) and int(fx["seed"]) == SEEDS[version]
    x = torch.from_numpy(fx["x"].astype(np.float32))
    logp, blocks = oc.forward(state, config, x, return_blocks=True)
    assert float((logp - torch.from_numpy(fx["logp"]).double()).abs().max()) <= 5e-5
    ref = fx["logp"]
    strings = json.loads(str(fx["strings"]))
    assert [oc.greedy(row)[0] for row in ref] == strings
    assert [_decode_str(*greedy_step(row))[0] for row in ref] == strings
    rms = [float(b.pow(2).mean().sqrt()) for b in blocks]
    assert np.allclose(rms, fx["block_rms"], rtol=1e-4) and min(rms) > 0.2 and max(rms) < 3.0, rms
    for row, s in zip(ref, strings):
        labels, _ = greedy_step(row)
        assert (labels != 0).mean() >= 0.15
        assert set(s) == set("ACGT")
        assert len(s) >= 20
    # eps 1e-5 instead of the modules' 1e-3 visibly changes the output (channel 0 of every BatchNorm has var 0.01)
    assert float((oc.forward(state, config, x, eps=1e-5) - logp).abs().max()) > 1e-2


@pytest.mark.parametrize("version", ["v1", "v2"])
def test_reference_tree_matches_oracle_and_loads_into_model(tmp_path, version):
    from oracle import reference_shim
    if not reference_shim.available():
        pytest.skip("reference checkout not present")
    ref = oc.load_ctc()
    spec = synth.quartznet_spec(version, max_repeat=2)
    config = synth.quartznet_config(spec)
    state = synth.make_quartznet_weights(spec, seed=7)
    rm = ref.Model(config)
    rm.load_state_dict(state)
    rm.eval()
    x = synth.squiggle(2, 600, seed=3).half().float()
    with torch.no_grad():
        r = rm(x).permute(1, 0, 2).double()
    assert float((r - oc.forward(state, config, x)).abs().max()) <= 5e-5
    # a state_dict saved from the reference's module tree loads into our Model through load_model / match_names
    synth.write_quartznet_dir(str(tmp_path / "m"), spec, rm.state_dict())
    from bonito_b200.util import load_model
    ours = load_model(str(tmp_path / "m"), "cpu", half=False)
    assert isinstance(ours, Model) and ours.stride == 3 and ours.alphabet == ["N", "A", "C", "G", "T"]
    with torch.no_grad():
        o = ours(x).permute(1, 0, 2).double()
    assert float((o - r).abs().max()) <= 1e-5


def _logp(rows):
    """Log-probs whose argmax follows `rows` (labels), probability 0.8 on the label."""
    out = np.full((len(rows), 5), np.log(0.05), dtype=np.float32)
    out[np.arange(len(rows)), rows] = np.log(0.8)
    return out


def test_greedy_decode_hand_worked_cases():
    # all blank
    s, q, mv = _decode_str(*greedy_step(_logp([0, 0, 0])))
    assert (s, q, mv.tolist()) == ("", "", [0, 0, 0])
    # T = 1
    s, q, mv = _decode_str(*greedy_step(_logp([2])))
    assert (s, mv.tolist()) == ("C", [1]) and q == chr(int(np.rint(-10 * np.log10(0.2))) + 33)
    # A A _ A: the repeat collapses, the blank resets -> two A; the first A's quality averages frames 0 and 1
    labels = np.array([1, 1, 0, 1], dtype=np.uint8)
    probs = np.array([0.9, 0.5, 0.99, 0.6], dtype=np.float32)
    s, q, mv = _decode_str(labels, probs)
    assert s == "AA" and mv.tolist() == [1, 0, 0, 1]
    assert q == chr(int(np.rint(-10 * np.log10(1 - 0.7))) + 33) + chr(int(np.rint(-10 * np.log10(0.4))) + 33)
    assert oc.greedy(_logp([1, 1, 0, 1]))[0] == "AA"
    # equal fp16 log-probs: the highest index wins
    row = np.array([[np.log(0.1), np.log(0.4), np.log(0.1), np.log(0.4), np.log(0.0001)]], dtype=np.float16).astype(np.float32)
    assert greedy_step(row)[0].tolist() == [3] and oc.greedy(row)[0] == "G"
    # [qscore] scale / bias
    s, q, _ = _decode_str(np.array([4], dtype=np.uint8), np.array([0.9], dtype=np.float32), qscale=2.0, qbias=1.0)
    assert q == chr(int(np.rint(10 * 2.0 + 1.0)) + 33)
    # qualities are clipped to [33, 126]
    assert _decode_str(np.array([4], dtype=np.uint8), np.array([1.0], dtype=np.float32), qscale=10.0)[1] == chr(126)


def test_greedy_collapse_runs_on_the_stitched_read():
    """A run of one label across a chunk join emits one base (a per-chunk collapse would emit two); a short read is cut to
    floor(length / stride) frames."""
    from bonito_b200.crf.basecall import stitch_results
    chunksize, overlap, stride = 30, 12, 3        # 10 frames per chunk, 2 dropped at each side of a join
    length = 48                                   # two chunks: windows [0, 30) and [18, 48)
    a = np.zeros((2, 10), dtype=np.uint8)
    a[0, 6:8] = 2                                 # C at the end of what chunk 0 keeps (frames 0..7) ...
    a[1, 2:4] = 2                                 # ... continuing at the start of what chunk 1 keeps (frames 2..9)
    a[1, 6] = 4
    probs = np.full((2, 10), 0.5, dtype=np.float32)
    st = stitch_results({"labels": torch.from_numpy(a), "probs": torch.from_numpy(probs)}, length, chunksize, overlap, stride)
    assert st["labels"].shape[0] == length // stride
    assert _decode_str(st["labels"].numpy(), st["probs"].numpy())[0] == "CT"
    assert "".join(_decode_str(a[i], probs[i])[0] for i in range(2)) == "CCT"
    short = stitch_results({"labels": torch.from_numpy(a[:1])}, 20, chunksize, overlap, stride)
    assert short["labels"].shape[0] == 20 // 3


def test_stack_refusals_and_decode_options():
    m, config, _ = _model("v1", max_repeat=2)
    CtcPlan(m, "cpu")                                         # the configs' own shapes are accepted
    with pytest.raises(UnsupportedModel, match="int8"):
        CtcPlan(m, "cpu", quantize=True)

    def refused(edit, match):
        spec = synth.quartznet_spec("v1", max_repeat=2)
        cfg = synth.quartznet_config(spec)
        edit(cfg)
        with pytest.raises(UnsupportedModel, match=match):
            CtcPlan(Model(cfg).eval(), "cpu")
    refused(lambda c: c["block"][2].update(dilation=[2]), "dilated")
    refused(lambda c: c["block"][2].update(stride=[2]), "only the first block")
    refused(lambda c: c["block"][0].update(separable=True), "first block")
    refused(lambda c: c["block"][7].update(residual=True), "residual connection on a non-separable")
    refused(lambda c: c["block"][7].update(repeat=2), "repeat > 1")
    refused(lambda c: c["encoder"].update(activation="tanh"), "activation")
    refused(lambda c: c["block"][2].update(kernel=[35]), "depthwise convolution")
    refused(lambda c: c["block"][3].update(filters=640), "depthwise convolution")
    refused(lambda c: c["block"][7].update(kernel=[4]), "even kernel")
    with pytest.raises(NotImplementedError, match="beam search"):
        m.decode(torch.zeros(4, 5), beamsize=5)
    from bonito_b200.ctc.basecall import basecall
    with pytest.raises(ValueError, match="revcomp"):
        basecall(m, [], reverse=True)
    with pytest.raises(NotImplementedError, match="beam search"):
        basecall(m, [], beamsize=5)
    assert m.decode(torch.from_numpy(_logp([0, 1, 1, 2]))) == "AC"


def _stacked_dense_spec():
    """v2 at two repeats with two more dense blocks (384 -> 256 k3, 256 -> 384 k5) in front of C3 (384 -> 48 k15): three
    consecutive dense blocks that each read overlapping rows of a zero-haloed buffer."""
    spec = synth.quartznet_spec("v2", max_repeat=2)
    spec["blocks"][7:7] = [(256, 1, 3, 1, False, False), (384, 1, 5, 1, False, False)]
    return spec


def test_stacked_haloed_dense_blocks_get_their_own_buffers():
    spec = _stacked_dense_spec()
    m = Model(synth.quartznet_config(spec))
    m.load_state_dict(synth.make_quartznet_weights(spec, seed=9))
    plan = CtcPlan(m.eval(), "cpu")
    N, L = 2, 600
    T = plan.frames(L)
    bufs = plan._buffers(N, L)
    assert sorted(bufs["halo"]) == [7, 8, 9]
    spans = []
    for i, (cin, k) in {7: (384, 3), 8: (256, 5), 9: (384, 15)}.items():
        h = bufs["halo"][i]
        assert h.numel() == N * (T + 2 * (k // 2)) * cin + k * cin and not bool(h.any())
        spans.append((h.data_ptr(), h.data_ptr() + 2 * h.numel()))
        dst, ld, lp = plan._dest(bufs, i - 1, N, T)     # the block in front writes frame rows of block i's own buffer
        assert dst.data_ptr() == h.data_ptr() + 2 * (k // 2) * cin and (ld, lp) == (cin, T + 2 * (k // 2))
    spans.sort()
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))


def test_ctc_package_alias():
    from bonito_b200.util import load_symbol
    assert load_symbol({"model": {"package": "bonito.ctc"}}, "Model") is Model


# ------------------------------------------------------------------------------------------------ GPU
DW_SHAPES = sorted({(c, k) for c, k in [(256, 33), (256, 39), (256, 51), (512, 51), (512, 63), (512, 75), (512, 87),
                                        (344, 115), (424, 115), (424, 5), (464, 5), (464, 123), (456, 123), (456, 9),
                                        (440, 9), (440, 31), (280, 31), (280, 67)]})


def _ulps(got, ref16):
    """|got - ref| in units of the fp16 spacing at ref (both fp16 tensors)."""
    g, r = got.double().cpu(), ref16.double().cpu()
    sp = torch.from_numpy(np.spacing(np.abs(ref16.cpu().numpy())).astype(np.float64))
    return ((g - r).abs() / sp).max().item()


@pytest.mark.gpu
def test_depthwise_matches_conv1d_every_config_shape():
    from bonito_b200 import native
    dev = "cuda"
    gen = torch.Generator().manual_seed(0)
    for c, k in DW_SHAPES:
        for t in (1, k - 1, 1333):
            n = 3
            x = torch.randn(n, t, c, generator=gen).half()
            w = (torch.randn(c, 1, k, generator=gen) / np.sqrt(k)).half()
            # pitched: input columns [8, 8 + c) of rows of c + 16, output columns [16, 16 + c) of rows of c + 24
            xb = torch.zeros(n * t, c + 16, dtype=torch.float16)
            xb[:, 8:8 + c] = x.reshape(n * t, c)
            xb = xb.to(dev)
            yb = torch.full((n * t, c + 24), 7.0, dtype=torch.float16, device=dev)
            native.depthwise_conv(xb[:, 8:], c + 16, w.to(dev), yb[:, 16:], c + 24, n, t)
            torch.cuda.synchronize()
            conv = lambda a, b: torch.nn.functional.conv1d(a.permute(0, 2, 1), b, padding=k // 2, groups=c)  # noqa: E731
            ref = conv(x.double(), w.double()).permute(0, 2, 1).reshape(n * t, c)
            # within 1 fp16 ulp of the exact result, widened where cancellation makes the fp32 accumulation error (at most
            # k * 2^-24 * sum |w x|, the same for any fp32-accumulating conv) larger than that ulp
            bound = k * 2.0 ** -24 * conv(x.double().abs(), w.double().abs()).permute(0, 2, 1).reshape(n * t, c)
            tol = torch.from_numpy(np.spacing(np.abs(ref.half().numpy())).astype(np.float64)) + bound
            got = yb[:, 16:16 + c].cpu().double()
            bad = (got - ref).abs() > tol
            assert not bool(bad.any()), (c, k, t, float(((got - ref).abs() / tol).max()))
            assert torch.all(yb[:, :16].cpu() == 7.0) and torch.all(yb[:, 16 + c:].cpu() == 7.0)
            # first and last K frames of each chunk (zero padding, nothing from the neighbouring chunks) are among the rows
            # checked above; a leak would also show as an error far above the tolerance there
            edge = bad.reshape(n, t, c)
            assert not bool(edge[:, :k].any()) and not bool(edge[:, max(0, t - k):].any())
    with pytest.raises(native.NativeError, match="unsupported shape"):
        native.depthwise_conv(xb, c + 16, torch.zeros(c, 1, 7, dtype=torch.float16, device=dev), yb, c + 24, n, t)


@pytest.mark.gpu
def test_conv_first_ex_strided_relu_and_gemm_relu():
    from bonito_b200 import native
    dev = "cuda"
    gen = torch.Generator().manual_seed(1)
    n, L = 3, 1001
    x = synth.squiggle(n, L, seed=2)[:, 0].half()
    for c, k, act in ((256, 33, native.ACT_RELU), (344, 9, native.ACT_SWISH)):
        w = (torch.randn(c, 1, k, generator=gen) / np.sqrt(k)).half()
        b = (0.1 * torch.randn(c, generator=gen)).half()
        T = (L - 1) // 3 + 1
        ld, padl, lp = c + 8, 2, T + 5
        out = torch.full((n * lp, ld), 9.0, dtype=torch.float16, device=dev)
        native.conv_first_ex(x.to(dev), w.to(dev), b.to(dev), act, out[:, 8:], ld, lp, padl, stride=3)
        torch.cuda.synchronize()
        ref = torch.nn.functional.conv1d(x[:, None].double(), w.double(), b.double(), stride=3, padding=k // 2).half().double()
        ref = torch.clamp(ref, min=0) if act == native.ACT_RELU else ref * torch.sigmoid(ref)
        got = out.cpu().reshape(n, lp, ld)
        assert torch.all(got[:, :, :8] == 9.0)
        assert torch.all(got[:, :padl, 8:] == 0) and torch.all(got[:, padl + T:, 8:] == 0)
        assert _ulps(got[:, padl:padl + T, 8:].reshape(-1, c), ref.permute(0, 2, 1).reshape(-1, c).half()) <= 2.0
    # stride 1 at the transformer stem's shape: bit-identical to b200_conv_first_fwd (same accumulation order)
    w = (torch.randn(64, 1, 5, generator=gen) / 2).half().to(dev)
    b = (0.1 * torch.randn(64, generator=gen)).half().to(dev)
    a = torch.empty(n * (L + 4), 64, dtype=torch.float16, device=dev)
    e = torch.empty_like(a)
    native.conv_first(x.to(dev), w, b, native.ACT_SWISH, a, L + 4, 2)
    native.conv_first_ex(x.to(dev), w, b, native.ACT_SWISH, e, 64, L + 4, 2, stride=1)
    assert torch.equal(a, e)
    # relu in both GEMM kernels
    A = torch.randn(300, 256, generator=gen).half()
    B = (torch.randn(72, 256, generator=gen) / 16).half()
    bias = torch.randn(72, generator=gen).half()
    exact = A.double() @ B.double().T + bias.double()
    ref = torch.clamp(exact, min=0)
    # 1 fp16 ulp, plus the fp32 accumulation bound k * 2^-24 * sum |a b| where cancellation makes that larger
    tol = torch.from_numpy(np.spacing(np.abs(ref.half().numpy())).astype(np.float64)) + \
        256 * 2.0 ** -24 * (A.double().abs() @ B.double().abs().T + bias.double().abs())
    for impl in (native.GEMM_TCGEN05, native.GEMM_MMA_SYNC):
        C = torch.empty(300, 72, dtype=torch.float16, device=dev)
        native.gemm(A.to(dev), 256, B.to(dev), bias.to(dev), C, 72, 300, 72, 256, act=native.ACT_RELU, impl=impl)
        torch.cuda.synchronize()
        assert bool(((C.cpu().double() - ref).abs() <= tol).all()) and bool((C >= 0).all())
        assert bool((C.cpu()[exact < -1e-2] == 0).all())


@pytest.mark.gpu
def test_conv_first_outputs_unchanged_from_the_recorded_build(golden_dir):
    """b200_conv_first_fwd at its own shapes computes bit for bit what the build recorded in the fixture computed (commit
    f0e678c, before B200_ACT_RELU joined the shared epilogue activation): scripts/make_golden_conv_first.py."""
    from bonito_b200 import native
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import make_golden_conv_first as g
    fx = np.load(os.path.join(golden_dir, "conv_first_outputs.npz"))
    assert str(fx["commit"]) == "f0e678c"
    for i, case in enumerate(g.CASES):
        name, c, k, act, n, l, padl, padr = case
        x, w, b = (t.cuda() for t in g.inputs(c, k, n, l, seed=100 + i))
        lp = padl + l + padr
        out = torch.full((n * lp, c), 3.0, dtype=torch.float16, device="cuda")
        native.conv_first(x, w, b, act, out, lp, padl)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy().view(np.uint16), fx[name].view(np.uint16)), name


@pytest.mark.gpu
@pytest.mark.parametrize("F,M", [(48, 1001), (1024, 777)])
def test_ctc_head_logp_labels_probs(F, M):
    from bonito_b200 import native
    dev = "cuda"
    gen = torch.Generator().manual_seed(F)
    x = torch.randn(M, F, generator=gen).half()
    w = (torch.randn(5, F, generator=gen) * (2 / np.sqrt(F))).half()
    w[4] = w[2]                                   # classes 2 and 4 tie on every row: 4 must win where they lead
    b = (0.3 * torch.randn(5, generator=gen)).half()
    b[4] = b[2]
    labels = torch.empty(M, dtype=torch.uint8, device=dev)
    probs = torch.empty(M, dtype=torch.float32, device=dev)
    logp = torch.empty(M, 5, dtype=torch.float16, device=dev)
    native.ctc_head(x.to(dev), M, w.to(dev), b.to(dev), labels, probs, logp=logp)
    lab2 = torch.empty_like(labels)
    pr2 = torch.empty_like(probs)
    native.ctc_head(x.to(dev), M, w.to(dev), b.to(dev), lab2, pr2)
    torch.cuda.synchronize()
    lp = logp.float()
    exp_lab = 4 - torch.argmax(lp.flip(-1), dim=-1)
    assert torch.equal(labels.long(), exp_lab) and torch.equal(lab2, labels) and torch.equal(pr2, probs)
    assert torch.equal(probs, torch.exp(lp.gather(1, exp_lab[:, None])[:, 0]))
    assert int((labels == 2).sum()) == 0 and int((labels == 4).sum()) > 0
    logits = (x.double() @ w.double().T + b.double()).half().double()
    ref = torch.log_softmax(logits, dim=-1).half()
    assert _ulps(logp.cpu(), ref) <= 1.0


def _plan(version, **kw):
    m, config, state = _model(version, **kw)
    m.use_koi(batchsize=64, chunksize=3999, quantize=False)
    m = m.half().to("cuda")
    return m, config, state


@pytest.mark.gpu
@pytest.mark.parametrize("version", ["v1", "v2"])
def test_forward_fixture_and_full_batch_against_oracle(golden_dir, version):
    m, config, state = _plan(version)
    plan = m.native_plan()
    fx = _fixture(golden_dir, version)
    cases = [torch.from_numpy(fx["x"].astype(np.float32)), synth.squiggle(64, 3999, seed=9).half().float()]
    for x in cases:
        with torch.inference_mode():
            got = plan.forward(x.half().cuda()).double()
            labels, probs = plan.greedy(x.half().cuda())
            labels, probs = labels.cpu().numpy(), probs.cpu().numpy()
        sd = {k: v.cuda() for k, v in state.items()}
        ref = oc.forward(sd, config, x.cuda())
        rnd = oc.forward(sd, config, x.cuda(), rounding=True)
        floor_max, floor_mean = float((rnd - ref).abs().max()), float((rnd - ref).abs().mean())
        err = (got - ref).abs()
        assert float(err.max()) <= 2 * floor_max and float(err.mean()) <= 2 * floor_mean, \
            (float(err.max()), float(err.mean()), floor_max, floor_mean)
        # decode exactness on the GPU's own log-probs: host collapse of the GPU labels / probs == oracle greedy
        gl = got.float().cpu().numpy()
        for i in range(min(len(gl), 8)):
            s, q, mv = _decode_str(labels[i], probs[i])
            os_, oq, omv = oc.greedy(gl[i])
            assert (s, q) == (os_, oq) and np.array_equal(mv, omv)
    if version == "v1":       # the fixture's reference log-probs themselves
        with torch.inference_mode():
            got = plan.forward(torch.from_numpy(fx["x"]).cuda()).double().cpu()
        assert float((got - torch.from_numpy(fx["logp"]).double()).abs().max()) <= 2 * 3.2e-2


@pytest.mark.gpu
def test_stacked_haloed_dense_blocks_against_oracle():
    spec = _stacked_dense_spec()
    config = synth.quartznet_config(spec)
    state = synth.make_quartznet_weights(spec, seed=9)
    m = Model(config)
    m.load_state_dict(state)
    m.use_koi(batchsize=8, chunksize=3999, quantize=False)
    m = m.half().eval().to("cuda")
    x = synth.squiggle(8, 3999, seed=12).half().float()
    with torch.inference_mode():
        got = m(x.half().cuda()).double()
    sd = {k: v.cuda() for k, v in state.items()}
    ref = oc.forward(sd, config, x.cuda())
    rnd = oc.forward(sd, config, x.cuda(), rounding=True)
    err = (got - ref).abs()
    floor = (rnd - ref).abs()
    assert float(err.max()) <= 2 * float(floor.max()) and float(err.mean()) <= 2 * float(floor.mean()), \
        (float(err.max()), float(err.mean()), float(floor.max()), float(floor.mean()))


@pytest.mark.gpu
@pytest.mark.parametrize("version", ["v1", "v2"])
def test_basecall_matches_oracle_pipeline(version):
    from bonito_b200.crf.basecall import stitch_results
    from bonito_b200.ctc.basecall import basecall
    from bonito_b200.util import chunk
    m, _, _ = _plan(version)

    class R:
        def __init__(self, rid, sig):
            self.read_id, self.signal = rid, sig

    lengths = (9000, 2500, 12345)
    sig = synth.squiggle(len(lengths), max(lengths), seed=21)[:, 0].numpy()
    reads = [R(f"r{i}", sig[i, :n].copy()) for i, n in enumerate(lengths)]
    chunksize, overlap = 3999, 498
    out = list(basecall(m, iter(reads), chunksize=chunksize, overlap=overlap, batchsize=5))
    assert [r.read_id for r, _ in out] == ["r0", "r1", "r2"]
    plan = m.native_plan()
    for read, res in out:
        chunks = chunk(torch.from_numpy(read.signal), chunksize, overlap)
        with torch.inference_mode():
            logp = plan.forward(chunks.half().cuda()).float().cpu()
        st = stitch_results(logp, len(read.signal), chunksize, overlap, 3).numpy()
        s, q, mv = oc.greedy(st)
        assert res["sequence"] == s and res["qstring"] == q and np.array_equal(res["moves"], mv) and res["stride"] == 3
        if len(read.signal) < chunksize:
            assert len(res["moves"]) == len(read.signal) // 3
        assert len(s) > 50


@pytest.mark.gpu
def test_cli_fastq_sam_and_refusals(tmp_path):
    reads = tmp_path / "reads"
    reads.mkdir()
    sig = synth.squiggle(2, 9000, seed=4)[:, 0].numpy()
    for i in range(2):
        np.save(reads / f"read{i}.npy", (90 + 20 * sig[i]).astype(np.float32))
    env = dict(os.environ, PYTHONPATH=ROOT)
    for version in ("v1", "v2"):
        spec = synth.quartznet_spec(version)
        d = synth.write_quartznet_dir(str(tmp_path / version), spec, synth.make_quartznet_weights(spec, seed=SEEDS[version]))
        for suffix in ("fastq", "sam"):
            path = tmp_path / f"{version}.{suffix}"
            with open(path, "w") as fh:
                p = subprocess.run([sys.executable, "-m", "bonito_b200", "basecaller", d, str(reads)], cwd=ROOT, env=env,
                                   stdout=fh, stderr=subprocess.PIPE, text=True)
            assert p.returncode == 0, p.stderr
            text = open(path).read()
            if suffix == "fastq":
                recs = text.strip().split("\n")
                assert len(recs) == 8 and recs[0].startswith("@read") and len(recs[1]) > 100 and len(recs[1]) == len(recs[3])
            else:
                rows = [r for r in text.strip().split("\n") if not r.startswith("@")]
                assert len(rows) == 2 and all("\tmv:B:c,3," in r for r in rows)
        for flag, msg in (("--revcomp", "--revcomp is not supported for the QuartzNet CTC models"),
                          ("--quantize", "no native path for this model")):
            p = subprocess.run([sys.executable, "-m", "bonito_b200", "basecaller", d, str(reads), flag], cwd=ROOT, env=env,
                               capture_output=True, text=True)
            assert p.returncode != 0 and msg in p.stderr and "Traceback" not in p.stderr, p.stderr
