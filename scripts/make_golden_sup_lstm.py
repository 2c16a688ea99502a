"""
Generate tests/golden/forward_sup_lstm.npz: the LSTM sup shape (dna_r10.4.1@v4.3: H = 1024, 5 LSTM layers, state_len 5, 4096
scores per frame) through the REFERENCE's own module tree, fp32 on the CPU, as oracle/make_golden.py's forward_hac does for
the hac shape.  Needs the reference checkout that oracle/reference_shim.py imports; the committed fixture is only replayed.

    python scripts/make_golden_sup_lstm.py

Contents: the fp16-representable input [2, 1, 400], every 8th score column of the scores without the blank column
([N, T, 512] of [N, T, 4096], fp32: the full table would make the fixture ten times larger; the decode strings pin the rest),
the decode_batch strings of the full scores, the weight seed and the digest of the seeded weights
(`make_weights(..., qr_f64=True)`: the orthogonal init factorised in float64, so that the fp16 weights are the same on every
CPU; the tests regenerate them and compare the digest).
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import reference_shim, synth  # noqa: E402
from oracle.make_golden import weights_digest  # noqa: E402

SEED = 33
COL_STRIDE = 8     # stored score columns: 0, 8, 16, ...


def main():
    ref = reference_shim.load()
    spec = synth.model_spec("sup_lstm")
    model = ref.crf_model.Model(synth.model_config(spec, batchnorm=False))
    weights = synth.make_weights(spec, seed=SEED, qr_f64=True)
    model.load_state_dict(synth.state_dict_from_weights(spec, weights))
    model.eval()
    x = synth.squiggle(2, 400, seed=14).half().float()      # fp16-representable input: identical for every implementation
    with torch.inference_mode():
        scores = model.encoder(x)                            # [T, N, C + blanks]
        strings = model.decode_batch(scores)
    t, n, _ = scores.shape
    s5 = scores.reshape(t, n, -1, 5)
    assert torch.all(s5[..., 0] == 2.0)
    ntc = s5[..., 1:].reshape(t, n, -1).permute(1, 0, 2).contiguous()
    out = {"x": x.numpy().astype(np.float16), "scores_ntc": ntc[..., ::COL_STRIDE].contiguous().numpy(),
           "col_stride": np.array(COL_STRIDE), "strings": np.array(json.dumps(strings)),
           "digest": np.array(weights_digest(weights)), "seed": np.array(SEED), "stride": np.array(model.stride)}
    path = os.path.join(ROOT, "tests", "golden", "forward_sup_lstm.npz")
    np.savez_compressed(path, **out)
    sat = float((ntc.abs() >= 5.0).float().mean())
    print("forward_sup_lstm.npz scores", tuple(ntc.shape), "strings", [len(s) for s in strings], "max|s| %.2f" % float(ntc.abs().max()),
          "clamped %.4f" % sat, "bytes", os.path.getsize(path))


if __name__ == "__main__":
    main()
