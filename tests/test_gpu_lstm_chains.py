"""
The hac LSTM stack in chains of tiles (b200_lstm_crf_lstm_fwd, which b200_lstm_crf_fwd and the per-kernel path run) against
one launch of the fused kernel per layer over the whole batch, byte for byte.  Batch sizes give one tile, tile counts that
do not divide into the chains (3, 5) and a partial last tile; the stack also runs with no chain streams (one chain), and
layer by layer (`first`, `count`).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def plan():
    from bonito_b200.crf.model import Model
    from oracle import synth
    spec = synth.model_spec("hac")
    model = Model(synth.model_config(spec))
    model.load_state_dict(synth.state_dict_from_weights(spec, synth.make_weights(spec, seed=5)))
    model.use_koi(batchsize=64, chunksize=600, quantize=False)
    model = model.half().eval().to("cuda")
    return model.native_plan(torch.device("cuda"))


@pytest.mark.parametrize("n", [40, 190, 300])
@pytest.mark.parametrize("mode", ["chains", "one_chain", "per_layer"])
def test_chained_stack_matches_one_launch_per_layer(plan, n, mode):
    from bonito_b200 import native
    L = 600
    b = plan._buffers("tile", n, L, slot=0)
    T, nt, H = b["T"], b["nt"], plan.hidden
    g = torch.Generator().manual_seed(n)
    x = torch.zeros(nt, T, 64, H, dtype=torch.float16)     # rows of chunks beyond the batch stay zero, as in the engine
    flat = torch.rand(n, T, H, generator=g) * 2 - 1
    for k in range(n):
        x[k // 64, :, k % 64] = flat[k].half()
    x = x.cuda()

    ref_a, ref_b = x.clone(), torch.zeros_like(x)
    ws = torch.empty(nt, native.lstm_rec_tile_workspace_bytes(64), dtype=torch.uint8, device="cuda")
    for layer in plan.lstm:
        native.lstm_fused_tile(ref_a, layer["wih"], layer["bias"], layer["whh"], ref_b, T, n, H, layer["reverse"], workspace=ws)
        ref_a, ref_b = ref_b, ref_a

    b["ya"].copy_(x)
    b["yb"].zero_()
    p = plan._plan_struct(b, n, L)
    saved = list(p.chain_streams)
    if mode == "one_chain":
        for i in range(len(saved)):
            p.chain_streams[i] = None
    try:
        if mode == "per_layer":
            for i in range(len(plan.lstm)):
                native.lstm_crf_lstm_fwd(p, i, 1)
        else:
            native.lstm_crf_lstm_fwd(p, 0, len(plan.lstm))
        torch.cuda.synchronize()
    finally:
        for i, s in enumerate(saved):
            p.chain_streams[i] = s
    out = b["yb"] if len(plan.lstm) % 2 else b["ya"]
    assert torch.equal(out.view(torch.int16), ref_a.view(torch.int16))
