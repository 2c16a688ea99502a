"""The width-384 LSTM layer with its input projection fused into the tile-layout recurrence (b200_lstm_fused_tile_fwd):
bitwise against the unfused path it replaces (input GEMM into gate pre-activations + b200_lstm_rec_tile_fwd) and against
the float64 LSTM reference."""
import pytest
import torch

from oracle import crf_oracle as O

pytestmark = pytest.mark.gpu

H = 384


@pytest.fixture(scope="module")
def native():
    from bonito_b200 import native as nat
    nat.require()
    return nat


def _dev(t):
    return t.to("cuda", torch.float16).contiguous()


@pytest.mark.parametrize("n,t,reverse", [(5, 1, False), (5, 2, True), (64, 2, False), (64, 1, True), (65, 300, True),
                                         (130, 300, False), (130, 17, True), (512, 40, False), (512, 3, True)])
def test_fused_tile_layer_matches_unfused_and_reference(native, n, t, reverse):
    """Partial, single and multiple 64-chunk tiles, T = 1 .. 300, both directions; the output starts as NaN so that rows of
    chunks beyond the batch are checked to stay unwritten, and the input rows of those chunks hold values that must not
    reach any valid chunk."""
    tb, cs = native.lstm_tile_chunks(H), native.lstm_tile_cluster(H)
    cw = 4 * H // cs
    nt = -(-n // tb)
    g = torch.Generator().manual_seed(7000 + n + t)
    x = (torch.randn(t, n, H, generator=g) * 0.5).half()
    w_ih = (torch.randn(4 * H, H, generator=g) / H ** 0.5).half()
    w_hh = (torch.randn(4 * H, H, generator=g) / H ** 0.5).half()
    b = (torch.randn(4 * H, generator=g) * 0.3).half()
    unit = torch.arange(H)
    perm_ih = (torch.arange(4)[None, :] * H + unit[:, None]).reshape(-1)
    perm_hh = (torch.arange(H // 8)[:, None, None] * 8 + torch.arange(4)[None, :, None] * H
               + torch.arange(8)[None, None, :]).reshape(-1)
    xt = (torch.randn(nt, t, tb, H, generator=g) * 4).half()                # rows of chunks >= n: stray values
    for i in range(nt):
        nb = min(tb, n - i * tb)
        xt[i, :, :nb] = x[:, i * tb:i * tb + nb]
    xt = xt.cuda()
    wih, bias, whh = _dev(w_ih[perm_ih]), _dev(b[perm_ih]), _dev(w_hh[perm_hh])

    y = torch.full((nt, t, tb, H), float("nan"), dtype=torch.float16, device="cuda")
    native.lstm_fused_tile(xt, wih, bias, whh, y, t, n, H, reverse)
    gx = torch.zeros(nt, t, cs, tb, cw, dtype=torch.float16, device="cuda")
    native.gemm(xt, H, wih, bias, gx, cw, nt * t * tb, 4 * H, H, rows_inner=tb, valid_inner=tb, stride_inner=1,
                stride_outer=cs * tb, cb_width=cw, cb_rows=tb)
    y_ref = torch.full((nt, t, tb, H), float("nan"), dtype=torch.float16, device="cuda")
    native.lstm_rec_tile(gx, whh, y_ref, t, n, H, reverse)
    torch.cuda.synchronize()

    got = y.cpu().permute(1, 0, 2, 3).reshape(t, nt * tb, H)
    assert torch.isnan(got[:, n:]).all()          # rows of chunks beyond the batch are not written
    assert torch.equal(got[:, :n], y_ref.cpu().permute(1, 0, 2, 3).reshape(t, nt * tb, H)[:, :n])
    ref = O.lstm_layer(x.double(), w_ih.double(), w_hh.double(), b.double(), torch.zeros(4 * H, dtype=torch.float64), reverse)
    err = (got[:, :n].double() - ref).abs().max().item()
    assert err <= 5e-3, err


def test_fused_tile_layer_accepts_zero_steps(native):
    """T = 0 is a no-op, like the unfused recurrent kernel."""
    y = torch.full((1, 1, 64, H), float("nan"), dtype=torch.float16, device="cuda")
    x = torch.zeros(1, 1, 64, H, dtype=torch.float16, device="cuda")
    w = torch.zeros(4 * H, H, dtype=torch.float16, device="cuda")
    bias = torch.zeros(4 * H, dtype=torch.float16, device="cuda")
    native.lstm_fused_tile(x, w, bias, w, y, 0, 5, H, False)
    torch.cuda.synchronize()
    assert torch.isnan(y.cpu()).all()
