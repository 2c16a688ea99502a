"""
QuartzNet CTC training on the GPU (bonito_b200/csrc/ctc_train.cu, bonito_b200.engine_ctc.CtcTrainPlan): each kernel
against float64 at its edges, whole-model gradients against the float64 functional oracle (tests/_oracle_ctc_train.py)
next to torch's own autocast gradients with the same dropout masks, determinism, non-finite gradients, the stale-plan
rule and a short overfit.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _oracle_ctc_train as O
from bonito_b200 import native, synth
from bonito_b200.ctc.model import Model
from bonito_b200.engine_ctc import DEPTHWISE_TAPS, CtcTrainPlan

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _h(shape, seed, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return (offset + scale * torch.randn(*shape, generator=g)).half()


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("m,cout,k", [(300, 1024, 512), (50001, 48, 256), (4000, 1024, 64)])
def test_wgrad_gemm_plain(m, cout, k):
    dz, x = _h((m, cout), 1), _h((m, k), 2)
    dw = torch.empty(cout, k, dtype=torch.float32, device=DEV)
    native.wgrad_gemm(dz.to(DEV), cout, x.to(DEV), k, m, cout, k, dw)
    ref = dz.double().t() @ x.double()
    assert _rel(dw, ref) < 1e-5, _rel(dw, ref)
    slices = native.load().b200_wgrad_gemm_workspace_bytes(m, cout, k)
    assert (slices == 0) == (m == 300)      # one slice at 300 rows, split-K otherwise


def test_wgrad_gemm_haloed_k15():
    N, T, K, cin, cout = 3, 101, 15, 384, 48
    p = K // 2
    rows = T + 2 * p
    xh = torch.zeros(N, rows, cin).half()
    xh[:, p:p + T] = _h((N, T, cin), 3)
    buf = torch.cat([xh.reshape(-1), torch.zeros(K * cin).half()]).to(DEV)
    dz = _h((N * T, cout), 4)
    dw = torch.empty(cout, K * cin, dtype=torch.float32, device=DEV)
    native.wgrad_gemm(dz.to(DEV), cout, buf, cin, N * rows, cout, K * cin, dw, rows_inner=rows, valid_inner=T, lpz=T)
    x = xh[:, p:p + T].permute(0, 2, 1).double()                       # [N, cin, T]
    z = torch.zeros(N, cout, T, dtype=torch.float64, requires_grad=True)
    w = torch.zeros(cout, cin, K, dtype=torch.float64, requires_grad=True)
    out = F.conv1d(x, w, padding=p)
    out.backward(dz.double().view(N, T, cout).permute(0, 2, 1))
    ref = w.grad.permute(0, 2, 1).reshape(cout, K * cin)
    assert _rel(dw, ref) < 1e-5


@pytest.mark.parametrize("k", DEPTHWISE_TAPS)
@pytest.mark.parametrize("c,n,t", [(256, 2, 200), (280, 3, 40), (512, 2, 3)])
def test_depthwise_wgrad(k, c, n, t):
    x, dy = _h((n * t, c), 5), _h((n * t, c), 6)
    dw = torch.empty(c, 1, k, dtype=torch.float32, device=DEV)
    native.depthwise_wgrad(dy.to(DEV), c, x.to(DEV), c, n, t, dw)
    w = torch.zeros(c, 1, k, dtype=torch.float64, requires_grad=True)
    F.conv1d(x.double().view(n, t, c).permute(0, 2, 1), w, padding=k // 2, groups=c).backward(
        dy.double().view(n, t, c).permute(0, 2, 1))
    assert _rel(dw, w.grad) < 1e-5


@pytest.mark.parametrize("c,k,stride", [(256, 33, 3), (344, 9, 3), (256, 33, 1), (48, 5, 1)])
def test_conv_first_wgrad(c, k, stride):
    n, l = 3, 1001
    t = (l - 1) // stride + 1
    x, dz = _h((n, l), 7), _h((n * t, c), 8)
    dw = torch.empty(c, 1, k, dtype=torch.float32, device=DEV)
    native.conv_first_wgrad(dz.to(DEV), c, x.to(DEV), stride, dw)
    w = torch.zeros(c, 1, k, dtype=torch.float64, requires_grad=True)
    F.conv1d(x.double()[:, None], w, stride=stride, padding=k // 2).backward(dz.double().view(n, t, c).permute(0, 2, 1))
    assert _rel(dw, w.grad) < 1e-5


def test_bn_stats_large_offset():
    """mean 200, std 0.3: sumsq - mean^2 in fp32 would lose ~3 % of the variance."""
    m, c = 70001, 264
    z = _h((m, c), 9, scale=0.3, offset=200.0)
    mean = torch.empty(c, dtype=torch.float32, device=DEV)
    invstd = torch.empty_like(mean)
    rm, rv = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
    native.bn_stats(z.to(DEV), c, m, c, 1e-3, 0.1, mean, invstd, rm, rv)
    zd = z.double()
    mu, var = zd.mean(0), zd.var(0, unbiased=False)
    assert _rel(mean, mu) < 1e-7
    assert (invstd.double().cpu() * torch.sqrt(var + 1e-3) - 1).abs().max() < 1e-5
    assert _rel(rm, 0.1 * mu) < 1e-6
    assert (rv.double().cpu() - (0.9 + 0.1 * zd.var(0, unbiased=True))).abs().max() < 1e-5


def _bn_case(residual, act, p, seed=11, n=3, t=300, c=264):
    m = n * t
    g = torch.Generator().manual_seed(seed)
    z = _h((m, c), seed)
    zr = _h((m, c), seed + 1) if residual else None
    gamma, beta = 0.5 + torch.rand(c, generator=g), 0.1 * torch.randn(c, generator=g)
    gr, br = 0.5 + torch.rand(c, generator=g), 0.1 * torch.randn(c, generator=g)
    dy = _h((m, c), seed + 2)
    dev = lambda v: v.to(DEV).contiguous()      # noqa: E731
    stats = []
    for zz in (z, zr) if residual else (z,):
        mean, inv = torch.empty(c, device=DEV), torch.empty(c, device=DEV)
        native.bn_stats(dev(zz), c, m, c, 1e-3, 0.1, mean, inv)
        stats += [mean, inv]
    mask = torch.empty(m, c // 8, dtype=torch.uint8, device=DEV)
    res = (dev(zr), c, stats[2], stats[3], dev(gr), dev(br)) if residual else None
    # the struct holds raw pointers: `tensors` keeps everything it points to alive
    tensors = dict(z=dev(z), gamma=dev(gamma), beta=dev(beta), dy=dev(dy), res=res, stats=stats)
    args = native.bn_act_struct(m, c, t, act, p, 1234, 5, tensors["z"], c, stats[0], stats[1], tensors["gamma"],
                                tensors["beta"], residual=res, mask=mask)
    return args, tensors, mask, (z, zr, gamma, beta, gr, br, dy), (m, c, t)


@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("act,p", [(native.ACT_RELU, 0.0), (native.ACT_SWISH, 0.05)])
def test_bn_act_fwd_bwd(residual, act, p):
    args, tens, mask, (z, zr, gamma, beta, gr, br, dy), (m, c, t) = _bn_case(residual, act, p)
    out = torch.empty(m, c, dtype=torch.float16, device=DEV)
    native.bn_act_fwd(args, out, c, t)
    dg, db, dz = torch.empty(c, device=DEV), torch.empty(c, device=DEV), torch.empty(m, c, dtype=torch.float16, device=DEV)
    kw = {}
    if residual:
        kw = dict(dgamma_r=torch.empty(c, device=DEV), dbeta_r=torch.empty(c, device=DEV),
                  dzr=torch.empty(m, c, dtype=torch.float16, device=DEV))
    native.bn_act_bwd(args, tens["dy"], c, dg, db, dz, c, t, **kw)
    keep = O.unpack_masks(mask, 1, m, c)[0].t() if p > 0 else torch.ones(m, c, dtype=torch.bool)
    if p > 0:
        frac = keep.double().mean().item()
        sd = np.sqrt(p * (1 - p) / keep.numel())
        assert abs(frac - (1 - p)) < 5 * sd, frac
    leaves = [v.double().requires_grad_(True) for v in (z, gamma, beta)]
    zz = leaves[0]
    y = F.batch_norm(zz, None, None, leaves[1], leaves[2], training=True, eps=1e-3)
    if residual:
        rl = [v.double().requires_grad_(True) for v in (zr, gr, br)]
        y = y + F.batch_norm(rl[0], None, None, rl[1], rl[2], training=True, eps=1e-3)
    a = F.relu(y) if act == native.ACT_RELU else F.silu(y)
    o = a * keep.cpu().double() / (1 - p)
    o.backward(dy.double())
    assert _rel(out, o) < 2e-3
    # the kernel's activation input is rounded to fp16 (as under autocast) and the oracle's is not: relu' flips for the
    # few elements within one fp16 step of 0, which moves dz by ~1 % at this size
    assert _rel(dz, leaves[0].grad) < 2e-2 and _rel(dg, leaves[1].grad) < 2e-2 and _rel(db, leaves[2].grad) < 2e-2
    if residual:
        assert _rel(kw["dzr"], rl[0].grad) < 2e-2 and _rel(kw["dgamma_r"], rl[1].grad) < 2e-2
        assert torch.equal(kw["dbeta_r"], db)


def test_bn_act_bwd_zero_where_dropped():
    """dy only at dropped elements: every gradient is exactly zero."""
    args, tens, mask, _, (m, c, t) = _bn_case(False, native.ACT_SWISH, 0.3)
    native.bn_act_fwd(args, torch.empty(m, c, dtype=torch.float16, device=DEV), c, t)
    keep = O.unpack_masks(mask, 1, m, c)[0].t().to(DEV)
    dy = torch.where(keep, torch.zeros((), dtype=torch.float16, device=DEV), tens["dy"]).contiguous()
    dg, db, dz = torch.empty(c, device=DEV), torch.empty(c, device=DEV), torch.empty(m, c, dtype=torch.float16, device=DEV)
    native.bn_act_bwd(args, dy, c, dg, db, dz, c, t)
    assert (dy != 0).any() and not dg.any() and not db.any() and not dz.any()


def test_head_fwd_bwd():
    m, f = 5003, 1024
    x, w, b = _h((m, f), 12), _h((5, f), 13, 0.05), _h((5,), 14, 0.1)
    g = torch.randn(m, 5, generator=torch.Generator().manual_seed(15))
    logp = torch.empty(m, 5, device=DEV)
    native.ctc_head_train_fwd(x.to(DEV), m, w.to(DEV), b.to(DEV), logp)
    dw, db, dx = torch.empty(5, f, device=DEV), torch.empty(5, device=DEV), torch.empty(m, f, dtype=torch.float16, device=DEV)
    native.ctc_head_bwd(x.to(DEV), m, w.to(DEV), logp, g.to(DEV), dw, db, dx)
    xl, wl, bl = (v.double().requires_grad_(True) for v in (x, w, b))
    logits = xl @ wl.t() + bl
    ref = F.log_softmax(logits + (logits.half().double() - logits).detach(), dim=-1)     # at the fp16 logits, as the kernel
    ref.backward(g.double())
    assert _rel(logp, ref) < 1e-3
    assert _rel(dw, wl.grad) < 1e-4 and _rel(db, bl.grad) < 1e-4 and _rel(dx, xl.grad) < 2e-3


def test_kernels_refuse_bad_arguments():
    z = torch.zeros(64, 12, dtype=torch.float16, device=DEV)
    with pytest.raises(native.NativeError, match="multiples of 8"):
        native.wgrad_gemm(z, 12, z, 12, 64, 12, 12, torch.empty(12, 12, device=DEV))
    with pytest.raises(native.NativeError, match="depthwise_wgrad"):
        native.depthwise_wgrad(z, 12, z, 12, 2, 32, torch.empty(12, 1, 5, device=DEV))


# ------------------------------------------------------------------------------------------------ whole model
def _model(name, max_repeat, dropout=0.0, seed=31):
    spec = synth.quartznet_spec(name, max_repeat=max_repeat)
    cfg = synth.quartznet_config(spec)
    for b in cfg["block"]:
        b["dropout"] = dropout
    m = Model(cfg)
    m.load_state_dict(synth.make_quartznet_weights(spec, seed=seed))
    return m


def _batch(N, L, stride, seed=41):
    x = synth.squiggle(N, L, seed=seed).half().float()
    T = (L - 1) // stride + 1
    g = torch.Generator().manual_seed(seed)
    lengths = torch.full((N,), T // 8, dtype=torch.int64)
    targets = torch.randint(1, 5, (N, T // 8), generator=g)
    return x, targets, lengths


def _masks(S):
    out = []
    for rec in S["blocks"]:
        for u in ([rec["bn"]] if "bn" in rec else [r["bn"] for r in rec["reps"]]):
            C = u["bn"].num_features
            out.append(None if u["mask"] is None else O.unpack_masks(u["mask"], S["N"], S["T"], C).cpu())
    return out


@pytest.mark.parametrize("name,dropout", [("v1", 0.0), ("v2", 0.05)])
def test_model_gradients_against_float64(name, dropout):
    model = _model(name, 2, dropout)
    x, targets, lengths = _batch(4, 2400, model.stride)
    ref_model = _model(name, 2, dropout)      # untouched running statistics for the oracles
    model = model.to(DEV).train()
    model.use_koi()
    plan = CtcTrainPlan(model)
    logp, S = plan.forward(x.to(DEV), seed=777)
    masks = _masks(S)
    if dropout:
        kept = torch.cat([m.reshape(-1) for m in masks])
        sd = np.sqrt(dropout * (1 - dropout) / kept.numel())
        assert abs(kept.double().mean().item() - (1 - dropout)) < 5 * sd
    lp = logp.detach().requires_grad_(True)
    loss = model.loss(lp.permute(1, 0, 2), targets, lengths)["total_loss"]
    loss.backward()
    grads = plan.backward(S, lp.grad)

    o_logp, P64, B64 = O.forward(ref_model, x, masks)
    o_loss = O.loss(o_logp, targets, lengths)
    o_loss.backward()
    t_logp, P16, _ = O.forward(ref_model, x, masks, dtype=torch.float32, device=DEV, autocast=True)
    O.loss(t_logp, targets, lengths).backward()

    assert abs(loss.item() - o_loss.item()) < 2e-3 * abs(o_loss.item()), (loss.item(), o_loss.item())
    names = {id(p): n for n, p in model.named_parameters()}
    floor = 2e-3
    worst = []
    for p, g in zip(plan.params, grads):
        n = names[id(p)]
        e_nat, e_torch = _rel(g, P64[n].grad), _rel(P16[n].grad, P64[n].grad)
        worst.append((e_nat / (2 * e_torch + floor), n, e_nat, e_torch))
        assert e_nat <= 2 * e_torch + floor, (n, e_nat, e_torch)
    print(name, "worst native/(2 torch + floor):", max(worst)[:4])
    for n, b in model.named_buffers():
        if n.endswith("running_mean") or n.endswith("running_var"):
            assert _rel(b, B64[n]) < 1e-3, n
        elif n.endswith("num_batches_tracked"):
            assert b.item() == B64[n].item()


def test_two_steps_bitwise_and_interleaved():
    model = _model("v2", 1, 0.05).to(DEV).train()
    model.use_koi()
    x, targets, lengths = _batch(3, 1800, model.stride)
    plan = CtcTrainPlan(model)
    g = torch.randn(3, (1800 - 1) // model.stride + 1, 5, generator=torch.Generator().manual_seed(3)).to(DEV)
    state0 = {n: b.clone() for n, b in model.named_buffers()}

    def step(seed):
        logp, S = plan.forward(x.to(DEV), seed)
        return logp.clone(), plan.backward(S, g)

    def restore():
        for n, b in model.named_buffers():
            b.copy_(state0[n])

    a = step(5)
    sa = {n: b.clone() for n, b in model.named_buffers()}
    restore()
    b = step(5)
    assert torch.equal(a[0], b[0]) and all(torch.equal(u, v) for u, v in zip(a[1], b[1]))
    assert all(torch.equal(sa[n], bb) for n, bb in model.named_buffers())
    # two forwards, then two backwards == (forward, backward) twice
    restore()
    s1, s2 = step(6), step(7)
    restore()
    l1, S1 = plan.forward(x.to(DEV), 6)
    l2, S2 = plan.forward(x.to(DEV), 7)
    g2, g1 = plan.backward(S2, g), plan.backward(S1, g)
    assert torch.equal(l1, s1[0]) and torch.equal(l2, s2[0])
    assert all(torch.equal(u, v) for u, v in zip(g1, s1[1])) and all(torch.equal(u, v) for u, v in zip(g2, s2[1]))


def test_inf_gradient_is_non_finite_and_scaler_skips():
    model = _model("v1", 1).to(DEV).train()
    model.use_koi()
    x, _, _ = _batch(2, 1500, model.stride)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=1024.0)
    before = [p.detach().clone() for p in model.parameters()]
    out = model(x.to(DEV))
    w = torch.ones_like(out)
    w[0, 3, 1] = float("inf")
    scaler.scale((out * w).sum()).backward()
    torch.cuda.synchronize()
    assert any(not torch.isfinite(p.grad).all() for p in model.parameters())
    scaler.step(opt)
    scaler.update()
    assert scaler.get_scale() < 1024.0
    assert all(torch.equal(a, p.detach()) for a, p in zip(before, model.parameters()))


def test_stale_plan_rebuilds_after_in_place_update():
    model = _model("v1", 1).to(DEV).eval()
    model.use_koi()
    x = synth.squiggle(2, 1500, seed=2).half().to(DEV)
    with torch.no_grad():
        y1 = model(x).float()
        model.decoder.layers[0].bias.add_(torch.tensor([1.0, 0, 0, 0, 0], device=DEV))
        y2 = model(x).float()
        fresh = Model(model.config)
        fresh.load_state_dict(model.state_dict())
        fresh = fresh.to(DEV).eval()
        fresh.use_koi()
        y3 = fresh(x).float()
    assert not torch.equal(y1, y2)
    assert torch.equal(y2, y3)


def test_training_forward_only_in_train_mode_with_grad():
    model = _model("v1", 1).to(DEV)
    model.use_koi()
    x = synth.squiggle(2, 1500, seed=2).half().to(DEV)
    assert model.train()(x).dtype == torch.float32
    with torch.no_grad():
        assert model(x).dtype == torch.float16
    assert model.eval()(x).dtype == torch.float16


def test_overfit_one_batch():
    torch.manual_seed(0)
    model = _model("v1", 1).to(DEV).train()
    model.use_koi()
    x, targets, lengths = _batch(8, 3000, model.stride, seed=9)
    x = x.to(DEV)
    opt = torch.optim.AdamW(model.parameters(), lr=2e-3)
    losses = []
    for _ in range(40):
        opt.zero_grad()
        loss = model.loss(model(x).permute(1, 0, 2), targets, lengths)["total_loss"]
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print(f"overfit: loss {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert losses[-1] < 0.7 * losses[0]


# ------------------------------------------------------------------------------------------------ end to end
def _run(*argv, timeout=900):
    import subprocess
    import sys
    root = __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__)))
    return subprocess.run([sys.executable, "-m", "bonito_b200", *argv], cwd=root, capture_output=True, text=True, timeout=timeout)


def test_train_pretrained_evaluate_basecall_resume(tmp_path):
    """A seeded v1 model directory; a chunk dataset of its own greedy calls; `train --pretrained` for one epoch; `evaluate`
    and `basecaller` on the result; `train -f` resumes from epoch 1."""
    from bonito_b200.cli.evaluate import call_batch
    spec = synth.quartznet_spec("v1", max_repeat=1)
    mdir = synth.write_quartznet_dir(str(tmp_path / "model"), spec, synth.make_quartznet_weights(spec, seed=11),
                                     batchsize=16, chunksize=2000, overlap=200)
    n, L = 40, 2000
    chunks = synth.squiggle(n, L, seed=5)[:, 0].numpy().astype(np.float32)
    model = Model(synth.quartznet_config(spec))
    model.load_state_dict(synth.make_quartznet_weights(spec, seed=11))
    model = model.to(DEV).eval()
    model.use_koi()
    with torch.inference_mode():
        seqs = call_batch(model, torch.from_numpy(chunks)[:, None].half().to(DEV))
    width = max(len(s) for s in seqs)
    lut = {c: i for i, c in enumerate("NACGT")}
    refs = np.zeros((n, width), dtype=np.uint8)
    for i, s in enumerate(seqs):
        refs[i, :len(s)] = [lut[c] for c in s]
    keep = np.array([len(s) > 0 for s in seqs])
    data = tmp_path / "data"
    data.mkdir()
    np.save(data / "chunks.npy", chunks[keep])
    np.save(data / "references.npy", refs[keep])
    np.save(data / "reference_lengths.npy", np.array([len(s) for s in seqs], dtype=np.uint16)[keep])

    wd = tmp_path / "run"
    p = _run("train", str(wd), "--pretrained", mdir, "--directory", str(data), "--epochs", "1", "--batch", "8",
             "--valid-chunks", "8", "--lr", "1e-4", "--num-workers", "0")
    assert p.returncode == 0, p.stderr[-3000:]
    for f in ("config.toml", "weights_1.tar", "losses_1.csv", "training.csv"):
        assert (wd / f).exists(), f
    lines = (wd / "losses_1.csv").read_text().splitlines()
    assert lines[0].split(",")[:5] == ["chunks", "time", "grad_norm", "lr", "scale"] and len(lines) == 1 + 4
    header = (wd / "training.csv").read_text().splitlines()[0]
    assert header == "time,duration,epoch,train_loss,validation_loss,validation_mean,validation_median"

    p = _run("evaluate", str(wd), "--directory", str(data), "--chunks", "8", "--weights", "1")
    assert p.returncode == 0, p.stderr[-3000:]
    reads = tmp_path / "reads"
    reads.mkdir()
    np.save(reads / "read0.npy", 93.7 + 23.5 * synth.squiggle(1, 9000, seed=70)[0, 0].numpy())
    p = _run("basecaller", str(wd), str(reads))
    assert p.returncode == 0 and p.stdout.startswith("@read0"), p.stderr[-3000:]

    p = _run("train", str(wd), "-f", "--pretrained", mdir, "--directory", str(data), "--epochs", "2", "--batch", "8",
             "--valid-chunks", "8", "--num-workers", "0")
    assert p.returncode == 0, p.stderr[-3000:]
    assert "picking up weights state from epoch 1" in p.stderr
    assert (wd / "weights_2.tar").exists() and not (wd / "losses_1.csv").read_text().count("\n") > 5
    assert len((wd / "training.csv").read_text().splitlines()) == 3
