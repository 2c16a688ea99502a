"""GPU parity tests of the transformer (sup) path against the CPU oracle (oracle/transformer_oracle.py)."""
import numpy as np
import pytest
import torch

from oracle import crf_oracle as O
from oracle import synth
from oracle import transformer_oracle as TO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from bonito_b200 import native as nat
    nat.require()
    return nat


def _dev(t):
    return t.to("cuda", torch.float16).contiguous()


@pytest.mark.parametrize("n,t,window", [(2, 200, (127, 128)), (1, 833, (127, 128)), (3, 70, (127, 128)), (2, 130, (5, 9)),
                                        (1, 100, (-1, -1))])
def test_attention_matches_oracle(native, n, t, window):
    g = torch.Generator().manual_seed(t)
    nh, hd = 8, 64
    qkv = (torch.randn(n, t, 3, nh, hd, generator=g) * 1.5).half()
    cos, sin = TO.rotary_tables(t, hd, fp16=True)
    out = torch.full((n, t, nh * hd), float("nan"), dtype=torch.float16, device="cuda")
    native.attention(_dev(qkv), _dev(torch.cat([cos, sin], dim=1)), out, n, t, nh, hd, window[0], window[1])
    torch.cuda.synchronize()
    x = qkv.float()
    q = TO._r16(TO.apply_rotary(x[:, :, 0], cos, sin), True).permute(0, 2, 1, 3)
    k = TO._r16(TO.apply_rotary(x[:, :, 1], cos, sin), True).permute(0, 2, 1, 3)
    v = x[:, :, 2].permute(0, 2, 1, 3)
    att = (q @ k.transpose(-1, -2)) / hd ** 0.5
    w = (t, t) if window == (-1, -1) else window
    att = att.masked_fill(~TO.window_mask(t, w), float("-inf"))
    ref = (torch.softmax(att, dim=-1) @ v).permute(0, 2, 1, 3).reshape(n, t, nh * hd)
    err = (out.float().cpu() - ref).abs().max().item()
    assert err <= 6e-3, err   # P is rounded to fp16 before the second product (as in flash-attn)


@pytest.mark.parametrize("n,t,window", [(2, 1666, (127, 128)), (1, 300, (127, 128)), (2, 257, (0, 128)), (1, 400, (127, 0))])
def test_attention_wgmma_and_mma_kernels_match_oracle(native, monkeypatch, n, t, window):
    """The wgmma kernel (default) and the mma.sync kernel (B200_ATTN_IMPL=mma) on the sup window shapes: both against the
    oracle, and against each other to the rounding of the output."""
    g = torch.Generator().manual_seed(t + 7)
    nh, hd = 8, 64
    qkv = (torch.randn(n, t, 3, nh, hd, generator=g) * 1.5).half()
    cos, sin = TO.rotary_tables(t, hd, fp16=True)
    cs = _dev(torch.cat([cos, sin], dim=1))
    outs = {}
    for impl in ("wgmma", "mma"):
        if impl == "mma":
            monkeypatch.setenv("B200_ATTN_IMPL", "mma")
        else:
            monkeypatch.delenv("B200_ATTN_IMPL", raising=False)
        out = torch.full((n, t, nh * hd), float("nan"), dtype=torch.float16, device="cuda")
        native.attention(_dev(qkv), cs, out, n, t, nh, hd, window[0], window[1])   # a fresh copy: q, k are rotated in place
        torch.cuda.synchronize()
        outs[impl] = out.float().cpu()
    x = qkv.float()
    q = TO._r16(TO.apply_rotary(x[:, :, 0], cos, sin), True).permute(0, 2, 1, 3)
    k = TO._r16(TO.apply_rotary(x[:, :, 1], cos, sin), True).permute(0, 2, 1, 3)
    v = x[:, :, 2].permute(0, 2, 1, 3)
    att = (q @ k.transpose(-1, -2)) / hd ** 0.5
    att = att.masked_fill(~TO.window_mask(t, window), float("-inf"))
    ref = (torch.softmax(att, dim=-1) @ v).permute(0, 2, 1, 3).reshape(n, t, nh * hd)
    for impl, got in outs.items():
        assert not torch.isnan(got).any(), impl
        err = (got - ref).abs().max().item()
        assert err <= 6e-3, (impl, err)
    assert (outs["wgmma"] - outs["mma"]).abs().max().item() <= 4e-3


def test_rmsnorm_swiglu_conv_first(native):
    g = torch.Generator().manual_seed(1)
    m, d, f = 1000, 512, 2048
    a, x, w = (torch.randn(m, d, generator=g)).half(), (torch.randn(m, d, generator=g)).half(), (1 + 0.1 * torch.randn(d, generator=g)).half()
    alpha = float(torch.tensor(2.4494897).half())
    out = torch.empty(m, d, dtype=torch.float16, device="cuda")
    native.rmsnorm_residual(_dev(a), _dev(x), _dev(w), alpha, 1e-5, out, m, d)
    ref = TO.rms_norm(a.float(), (alpha * x.float()).half().float(), w.float()).half().float()
    assert (out.float().cpu() - ref).abs().max().item() <= 4e-3
    h = torch.randn(m, 2 * f, generator=g).half()
    o2 = torch.empty(m, f, dtype=torch.float16, device="cuda")
    native.swiglu(_dev(h), o2, m, f)
    y, gate = h.float().chunk(2, dim=-1)
    ref2 = (gate * y / (1 + torch.exp(-gate))).half().float()
    assert (o2.float().cpu() - ref2).abs().max().item() <= 4e-3
    n, L, c, k, lp, padl = 3, 500, 64, 5, 520, 2
    xs = synth.squiggle(n, L, seed=3).half()
    wc, bc = (torch.randn(c, 1, k, generator=g) * 0.5).half(), (torch.randn(c, generator=g) * 0.1).half()
    o3 = torch.full((n, lp, c), float("nan"), dtype=torch.float16, device="cuda")
    native.conv_first(_dev(xs[:, 0]), _dev(wc), _dev(bc), native.ACT_SWISH, o3, lp, padl)
    torch.cuda.synchronize()
    ref3 = O.convolution(xs.float(), wc.float(), bc.float(), 1, 2, "swish", True).permute(0, 2, 1)
    got = o3.float().cpu()
    assert torch.all(got[:, :padl] == 0) and torch.all(got[:, padl + L:] == 0)
    assert (got[:, padl:padl + L] - ref3).abs().max().item() <= 4e-3


def _sup_model(depth=2, seed=3):
    from bonito_b200.transformer import Model
    spec = synth.sup_spec(depth=depth)
    weights = synth.make_sup_weights(spec, seed=seed)
    model = Model(synth.sup_config(spec))
    model.load_state_dict(synth.sup_state_dict(spec, weights))
    model.use_koi(batchsize=8, chunksize=1200, quantize=False)
    return model.half().eval().to("cuda"), spec, weights


@pytest.mark.parametrize("depth,n,L", [(2, 3, 1200), (3, 2, 3996)])
def test_sup_forward_matches_oracle(depth, n, L):
    model, spec, weights = _sup_model(depth)
    x = synth.squiggle(n, L, seed=n).half()
    with torch.inference_mode():
        scores, feats = model.native_plan("cuda").forward(x.cuda(), return_features=True)
    torch.cuda.synchronize()
    # scores reach |x| ~ 10-12 here (x5 scale): one fp16 ulp is 7.8e-3; same-rounding oracle within ~8 ulp, pure fp32 oracle
    # within what fp16 storage of 5 convolutions + the layers costs any half-precision implementation
    for fp16, tol_max, tol_mean in ((True, 8e-2, 4e-3), (False, 2.0e-1, 8e-3)):
        with torch.no_grad():
            ref, rf = TO.transformer_forward(weights, spec, x.float(), fp16=fp16, return_features=True)
        errs = {"conv": (feats["conv"].float().cpu() - rf[f"conv{len(spec['convs']) - 1}"].permute(0, 2, 1)).abs().max().item()}
        for l in range(depth):
            errs[f"layer{l}"] = (feats[f"layer{l}"].float().cpu() - rf[f"layer{l}"]).abs().max().item()
        e = (scores.float().cpu() - ref).abs()
        errs["scores_max"], errs["scores_mean"] = e.max().item(), e.mean().item()
        print("sup", depth, n, L, "oracle-fp16" if fp16 else "oracle-fp32", {k: f"{v:.2e}" for k, v in errs.items()},
              "score std %.2f max %.1f" % (ref.std().item(), ref.abs().max().item()))
        assert scores.shape == ref.shape
        assert errs["scores_max"] <= tol_max and errs["scores_mean"] <= tol_mean, errs


def test_sup_model_call_and_decode():
    """model(x) through the use_koi path, then the k=5 decode of its own scores against the oracle decoder."""
    from bonito_b200.decode import beam_search
    model, spec, _ = _sup_model(2)
    x = synth.squiggle(3, 1200, seed=9).half().cuda()
    with torch.inference_mode():
        scores = model(x)
        seq, q, moves = beam_search(scores, scale=1.05, offset=1.3)
    assert scores.shape == (3, 200, 4096) and scores.dtype == torch.float16
    o_moves, o_seq, o_q, _ = O.decode_native(scores.float().cpu().numpy(), 5, 2.0, 1.05, 1.3)
    got = [r[r != 0].tobytes() for r in seq.numpy()]
    want = [r[r != 0].tobytes() for r in o_seq]
    assert got == want and min(len(w) for w in want) > 20


@pytest.mark.gpu
@pytest.mark.parametrize("m,k,f", [(1000, 512, 2048), (77, 384, 96), (4096, 512, 256), (2000, 384, 192), (256 * 35 + 60, 512, 1024)])
def test_gemm_with_fused_swiglu(native, m, k, f):
    """B200_ACT_SWIGLU: fc1 with rows interleaved in [32 y | 32 gate] groups == GatedMlp's fc1 -> chunk -> swiglu."""
    from bonito_b200.engine_tf import _interleave_swiglu
    g = torch.Generator().manual_seed(4)
    x = torch.randn(m, k, generator=g).half()
    w1 = (torch.randn(2 * f, k, generator=g) / k ** 0.5 * 2).half()
    out = torch.full((m, f), float("nan"), dtype=torch.float16, device="cuda")
    native.gemm(_dev(x), k, _dev(_interleave_swiglu(w1)), None, out, f, m, 2 * f, k, act=native.ACT_SWIGLU)
    h = (x.float() @ w1.float().t()).half().float()
    y, gate = h.chunk(2, dim=-1)
    ref = (gate * y / (1 + torch.exp(-gate))).half().float()
    err = (out.float().cpu() - ref).abs()
    # y / gate are rounded to fp16 before the product, so a 1-ulp difference in either (accumulation order) moves the
    # result by up to 2^-10 relative each, plus the final rounding
    assert bool(torch.all(err <= 4e-3 + 4e-3 * ref.abs())) and err.mean().item() <= 2e-4, (err.max().item(), err.mean().item())
    with pytest.raises(RuntimeError):
        native.gemm(_dev(x), k, _dev(w1), None, out, f, m, 2 * f, k, act=native.ACT_SWIGLU, impl=native.GEMM_MMA_SYNC)


def test_sup_width_against_the_reference_fixture(golden_dir):
    """d_model 512 / 8 heads / ff 2048 / k = 5, 6 layers: the native engine against scores produced by the reference's own
    bonito.transformer classes (fp32 CPU, tests/golden/forward_sup_wide.npz)."""
    import os
    from oracle.make_golden import weights_digest
    from bonito_b200.transformer import Model
    gold = np.load(os.path.join(golden_dir, "forward_sup_wide.npz"))
    spec = synth.sup_spec(depth=int(gold["depth"]))
    weights = synth.make_sup_weights(spec, seed=int(gold["seed"]))
    if weights_digest(weights) != str(gold["digest"]):
        pytest.skip("seeded sup weights differ on this machine: fixture not comparable")
    model = Model(synth.sup_config(spec))
    model.load_state_dict(synth.sup_state_dict(spec, weights))
    model.use_koi(batchsize=2, chunksize=600, quantize=False)
    model = model.half().eval().cuda()
    x = torch.from_numpy(gold["x"]).cuda()
    with torch.inference_mode():
        scores, feats = model.native_plan("cuda").forward(x, return_features=True)
    ref = torch.from_numpy(gold["scores_ntc"])
    err = (scores.float().cpu() - ref).abs()
    e5 = (feats["layer5"].float().cpu() - torch.from_numpy(gold["layer5"])).abs().max().item()
    print(f"sup width vs reference fixture: scores max {err.max().item():.2e} mean {err.mean().item():.2e}; layer5 max {e5:.2e}")
    # fp16 storage through 5 convolutions + 6 layers against the reference in fp32; scores reach |x| ~ 11: ulp 7.8e-3
    assert err.max().item() <= 1.0e-1 and err.mean().item() <= 8e-3, (err.max().item(), err.mean().item())


def test_sup_full_depth_matches_same_rounding_oracle():
    """Benchmark config 3 architecture at full depth (18 layers, d_model 512, 8 heads, k = 5) on two 3996-sample chunks vs
    the oracle with fp16 storage rounding.  Budget: scores carry the x5 output scale and reach |x| in [8, 16), where one
    fp16 ulp is 7.8e-3; 18 layers of two half-precision implementations with different accumulation orders stay within
    10 ulp at the worst element, half an ulp on average, and 99 % of all scores within 2 ulp."""
    model, spec, weights = _sup_model(18, seed=5)
    x = synth.squiggle(2, 3996, seed=21).half()
    with torch.inference_mode():
        scores = model(x.cuda())
    with torch.no_grad():
        ref = TO.transformer_forward(weights, spec, x.float(), fp16=True)
    err = (scores.float().cpu() - ref).abs()
    within2 = (err <= 1.6e-2).float().mean().item()
    print(f"sup 18 layers vs fp16-rounding oracle: max {err.max().item():.2e} mean {err.mean().item():.2e} "
          f"within 2 ulp {within2:.4f}; score std {ref.std().item():.2f} max {ref.abs().max().item():.1f}")
    assert scores.shape == ref.shape == (2, 666, 4096)
    assert err.max().item() <= 8e-2, err.max().item()
    assert err.mean().item() <= 4e-3, err.mean().item()
    assert within2 >= 0.99, within2
