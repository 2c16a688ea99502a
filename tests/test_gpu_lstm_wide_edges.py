"""
The grid-persistent wide LSTM recurrence (lstm_rec_wide.cu, H = 768 and 1024) at its tile, grid and launch edges.

gx [T][G][N][32] is built from natural-order gate pre-activations with the per-CTA column order [unit - 8g][gate] of the
kernel header; y [T][N][H] carries canary margins (_edges.py).  The kernel's cell math is the shared
`gate_activations` / `tanh_f` of the other LSTM kernels, so the bound is `_lstm_reference`'s (carried per element through
the recurrence: |W_hh| e_h from the h error, H 2^-23 sum|w h| for the fp32 wgmma accumulation, the gx add, sigma' <= 1/4
and tanh' <= 1 into c and h, 2^-19 per SFU evaluation; the fp16 output in [rn16(h - e), rn16(h + e)]).  After every
launch the workspace's control words are read back: the status word must be 0 and the barrier counter G (T - 1), one
arrival per CTA and exchanged step.
"""
import numpy as np
import pytest
import torch

from _edges import (CANARY16, _lstm_inputs, _lstm_reference, _perm_hh, bits16, canary16, check_between, check_guarded,
                    fp16_values_admitted, rn16)

FRONT, BACK = 64, 64                                       # canary margins of y (elements), 16-byte aligned


@pytest.fixture(scope="module")
def native():
    from bonito_b200 import native as nat
    nat.require()
    return nat


def _gx_wide(gx, G):
    """gx [T, n, 4, H] natural order -> [T][G][n][32], CTA g's columns [unit - 8g][gate]."""
    T, n, _, H = gx.shape
    return gx.view(T, n, 4, G, 8).permute(0, 3, 1, 4, 2).reshape(T, G, n, 32).contiguous()


def _control(native, ws, n, H):
    """(barrier counter, status word) of a workspace after a launch with n chunks."""
    off = native.lstm_rec_wide_status_offset(n, H)
    words = ws[off - 128:off + 4].view(torch.int32).cpu().numpy()
    return int(words[0]), int(words[-1])


def _launch(native, gx_k, whh_k, T, n, H, reverse, ws=None):
    """One guarded launch; returns (y bits [T, n, H] as int64, y values as float64, workspace)."""
    if ws is None:
        ws = torch.empty(native.lstm_rec_wide_workspace_bytes(n, H), dtype=torch.uint8, device="cuda")
    buf = canary16(FRONT + T * n * H + BACK)
    native.lstm_rec_wide(gx_k, whh_k, buf[FRONT:FRONT + T * n * H], T, n, H, reverse, workspace=ws)
    torch.cuda.synchronize()
    bits = bits16(buf)
    check_guarded(bits, FRONT + np.arange(T * n * H), CANARY16)
    y = buf[FRONT:FRONT + T * n * H].double().cpu().numpy().reshape(T, n, H)
    return bits[FRONT:FRONT + T * n * H].reshape(T, n, H), y, ws


# ------------------------------------------------------------------------------------------------ 1. interval test
def _cases():
    c = []
    for H in (768, 1024):
        c += [(H, 1, 37, False, "N=1-T=37"), (H, 63, 37, True, "N=63-T=37-reverse"), (H, 64, 3, False, "N=64-T=3-both-parities"),
              (H, 65, 2, True, "N=65-T=2-second-tile-one-chunk-reverse"), (H, 65, 1, False, "N=65-T=1-no-exchange"),
              (H, 129, 37, H == 768, "N=129-T=37-third-tile"),
              (H, 2560, 3, H == 1024, "N=2560-T=3-40-tiles-cell-state-limit"), (H, 2560, 1, False, "N=2560-T=1")]
    return [pytest.param(H, n, T, r, id=f"H={H}-{name}") for H, n, T, r, name in c]


@pytest.mark.gpu
@pytest.mark.parametrize("H,n,T,reverse", _cases())
def test_wide_lstm_in_interval_at_tile_and_grid_edges(native, H, n, T, reverse):
    """Partial, single-chunk and 40 tiles (the cell-state limit), T = 1 (no exchange), 2 and 3 (both exchange parities)
    and 37, both directions: y inside the carried interval, every element of y written and nothing around it, status 0,
    counter G (T - 1)."""
    G = native.lstm_wide_ctas(H)
    assert native.lstm_wide_max_chunks(H) == 2560
    gx, whh = _lstm_inputs(T, n, H, seed=H + n + T)
    _, y, ws = _launch(native, _gx_wide(gx, G).cuda(), whh[_perm_hh(H)].cuda(), T, n, H, reverse)
    assert _control(native, ws, n, H) == (G * (T - 1), 0)
    lo, hi = _lstm_reference(gx, whh, reverse)
    check_between(y, lo, hi, f"lstm_rec_wide H={H} n={n} T={T} reverse={reverse}")
    print(f"wide LSTM H={H} n={n} T={T}: widest interval {int(fp16_values_admitted(lo, hi).max())} fp16 values")


# ------------------------------------------------------------------------------------------------ 2. dirty workspace
@pytest.mark.gpu
@pytest.mark.parametrize("H", [768, 1024])
def test_wide_lstm_ignores_what_the_workspace_held(native, H):
    """A workspace filled with 0xFF and a zeroed one give bitwise equal outputs: the counter and the status word are reset
    on the stream, and no step reads exchange data it did not write.  Then two consecutive launches with different n and
    directions on one dirty workspace sized for the larger n equal the launches on fresh workspaces."""
    G = native.lstm_wide_ctas(H)
    runs = []
    for n, T, reverse in ((130, 5, False), (65, 4, True)):
        gx, whh = _lstm_inputs(T, n, H, seed=7 * n + T)
        args = (_gx_wide(gx, G).cuda(), whh[_perm_hh(H)].cuda(), T, n, H, reverse)
        size = native.lstm_rec_wide_workspace_bytes(n, H)
        want, _, _ = _launch(native, *args, ws=torch.zeros(size, dtype=torch.uint8, device="cuda"))
        got, _, ws = _launch(native, *args, ws=torch.full((size,), 0xFF, dtype=torch.uint8, device="cuda"))
        assert np.array_equal(got, want), f"n={n}: a dirty workspace changed the output"
        assert _control(native, ws, n, H) == (G * (T - 1), 0)
        runs.append((args, want))
    shared = torch.full((native.lstm_rec_wide_workspace_bytes(130, H),), 0xFF, dtype=torch.uint8, device="cuda")
    for args, want in runs:
        got, _, _ = _launch(native, *args, ws=shared)
        T, n = args[2], args[3]
        assert np.array_equal(got, want), f"n={n} after another launch on the same workspace"
        assert _control(native, shared, n, H) == (G * (T - 1), 0)


# ------------------------------------------------------------------------------------------------ 3. refusals
def _operands(native, T, n, H):
    G = max(native.lstm_wide_ctas(H), 1)
    gx = torch.zeros(T * G * n * 32 + 8, dtype=torch.float16, device="cuda")
    whh = torch.zeros(4 * H * H + 8, dtype=torch.float16, device="cuda")
    y = torch.zeros(T * n * H + 8, dtype=torch.float16, device="cuda")
    ws = torch.zeros(max(native.lstm_rec_wide_workspace_bytes(n, H), 256) + 16, dtype=torch.uint8, device="cuda")
    return gx, whh, y, ws


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["n=2561", "gx", "y", "workspace", "hidden=512"])
def test_wide_lstm_refusals(native, what):
    """Each refusal raises NativeError with its message before any launch: one chunk over the 40-tile cell-state limit,
    an operand that is not 16-byte aligned (a view one element in), a hidden size without a wide kernel.  The operands
    are sized for the call, so nothing outside them could be touched either way."""
    H, T, n = (512 if what == "hidden=512" else 1024), 1, (2561 if what == "n=2561" else 64)
    gx, whh, y, ws = _operands(native, T, n, H)
    gx_a, y_a, ws_a = gx[:-8], y[:-8], ws[:-16]
    if what == "gx":
        gx_a = gx[1:-7]
    elif what == "y":
        y_a = y[1:-7]
    elif what == "workspace":
        ws_a = ws[1:-15]
    msg = {"n=2561": "at most 2560 chunks per launch \\(got 2561\\)", "hidden=512": "hidden size 512 is not supported"}
    with pytest.raises(native.NativeError, match=msg.get(what, "operands must be 16-byte aligned")):
        native.lstm_rec_wide(gx_a, whh[:4 * H * H], y_a, T, n, H, False, workspace=ws_a)
    torch.cuda.synchronize()
    assert not y.any().item(), "a refused call wrote y"


@pytest.mark.gpu
@pytest.mark.parametrize("T,n", [pytest.param(0, 5, id="T=0"), pytest.param(5, 0, id="n=0")])
def test_wide_lstm_empty_calls_write_nothing(native, T, n):
    H = 1024
    gx, whh, _, ws = _operands(native, 5, 5, H)
    buf = canary16(FRONT + 5 * 5 * H + BACK)
    native.lstm_rec_wide(gx[:-8], whh[:4 * H * H], buf[FRONT:FRONT + 5 * 5 * H], T, n, H, True, workspace=ws[:-16])
    torch.cuda.synchronize()
    assert (bits16(buf) == CANARY16).all()


# ------------------------------------------------------------------------------------------------ 4. engine sub-batching
@pytest.mark.gpu
def test_engine_splits_batches_over_the_chunk_limit(native):
    """A batch of 2563 chunks runs as sub-batches of 2560 and 3 (engine.forward_wide).  Chunks are computed
    independently, so rows 2555 .. 2562, across the boundary, equal bitwise a forward of those 8 chunks alone;
    return_features is refused for such a batch."""
    from bonito_b200.crf.model import Model
    from oracle import synth
    spec = synth.model_spec("sup_lstm", n_lstm=1)
    model = Model(synth.model_config(spec))
    model.load_state_dict(synth.state_dict_from_weights(spec, synth.make_weights(spec, seed=9)))
    model.use_koi(batchsize=64, chunksize=300, quantize=False)
    model = model.half().eval().cuda()
    plan = model.native_plan("cuda")
    x = synth.squiggle(2563, 300, seed=4).half().cuda()
    with torch.inference_mode():
        full = plan.forward(x).clone()
        part = plan.forward(x[2555:2563].contiguous()).clone()
        with pytest.raises(ValueError, match="at most 2560 chunks"):
            plan.forward(x, return_features=True)
    torch.cuda.synchronize()
    assert full.shape[0] == 2563 and torch.isfinite(full.float()).all()
    assert torch.equal(full[2555:2563], part)


# ------------------------------------------------------------------------------------------------ 5. discriminative power
def _lstm_point(gx, whh, reverse, swap_if=False, delay=False):
    """fp16 outputs of a float64 recurrence with the kernels' rounding points, optionally wrong: i and f gates swapped, or
    the recurrent input h_{t-2} instead of h_{t-1}."""
    gx64, w = gx.double().numpy(), whh.double().numpy()
    T, n, _, H = gx64.shape
    h16, h_prev, c = np.zeros((n, H)), np.zeros((n, H)), np.zeros((n, H))
    out = np.empty((T, n, H))
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        G = gx64[t].reshape(n, 4 * H) + (h_prev if delay else h16) @ w.T
        gi, gf, gg, go = (G[:, q * H:(q + 1) * H] for q in range(4))
        if swap_if:
            gi, gf = gf, gi
        sig = lambda z: 0.5 * (1.0 + np.tanh(0.5 * z))
        c = sig(gf) * c + sig(gi) * np.tanh(gg)
        h_prev, h16 = h16, rn16(sig(go) * np.tanh(c))
        out[t] = h16
    return out


def test_wide_lstm_check_rejects_wrong_references():
    """The interval check admits the exact emulation and rejects the direction flipped, the i and f gates swapped, and
    h_{t-1} delayed by one step."""
    H, n, T = 768, 4, 6
    gx, whh = _lstm_inputs(T, n, H, seed=3)
    for reverse in (False, True):
        lo, hi = _lstm_reference(gx, whh, reverse)
        check_between(_lstm_point(gx, whh, reverse), lo, hi, "exact emulation")
        for wrong in (dict(reverse=not reverse), dict(reverse=reverse, swap_if=True), dict(reverse=reverse, delay=True)):
            with pytest.raises(AssertionError):
                check_between(_lstm_point(gx, whh, **wrong), lo, hi, f"wrong reference {wrong}")
