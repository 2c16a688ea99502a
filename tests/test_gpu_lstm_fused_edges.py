"""The fused width-384 LSTM layer (b200_lstm_fused_tile_fwd) at batch sizes that end inside a 64-chunk tile at and around
its midpoint (32 chunks), with odd and even T so that both exchange staging parities end the layer at those tile edges.
Same checks as test_gpu_lstm_fused.py: bitwise against the unfused path, within 5e-3 of the float64 LSTM, and rows of
chunks beyond the batch left NaN."""
import pytest

import test_gpu_lstm_fused as base

pytestmark = pytest.mark.gpu

native = base.native


@pytest.mark.parametrize("n,t,reverse", [(40, 7, False), (40, 6, True), (32, 3, False), (96, 5, True), (96, 1, False),
                                         (100, 33, False), (100, 64, True), (100, 2, False)])
def test_fused_tile_layer_mid_tile_edges(native, n, t, reverse):
    """n = 40 and 32: one tile, valid up to past or exactly at its midpoint; n = 96: a second tile of exactly 32 chunks;
    n = 100: a second tile of 36 chunks."""
    base.test_fused_tile_layer_matches_unfused_and_reference(native, n, t, reverse)
