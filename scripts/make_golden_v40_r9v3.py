"""
Generate tests/golden/forward_sup_lstm_v40.npz (dna_r10.4.1@v4.0: H = 1024, Clamp(-0.5, 3.5) behind each convolution, conv3
stride 5 swish, Linear 1024 -> 256 in front of the head, 4096 scores per frame plus the fixed blank) and
tests/golden/forward_r9_v3.npz (dna_r9.4.1@v3: the old-style H = 768 stack whose head learns its blank scores, 5120 scores per
frame in the layout [state][stay, m0..m3]) through the REFERENCE's own module tree, fp32 on the CPU, as
scripts/make_golden_sup_lstm.py does for v4.3.  Needs the reference checkout that oracle/reference_shim.py imports; the
committed fixtures are only replayed.  The shim's `posteriors` (koi.ctc, a closed binary) is the oracle's restatement, so the
decode strings are the reference's decode_batch on top of that restatement.

    python scripts/make_golden_v40_r9v3.py

Contents of each: the fp16-representable input [2, 1, 340], every col_stride-th score column, fp32 (v4.0: of the 4096 scores
without the blank column, stride 8; v3: of all 5120 columns, stride 11, so that every fifth stored column is a learned blank
column), the decode_batch strings of the full scores, the weight seed and the digest of the seeded weights
(`make_weights(..., qr_f64=True)`; the tests regenerate them and compare the digest).
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

FIXTURES = {
    # file: (spec, seed, column stride)
    "forward_sup_lstm_v40.npz": (synth.v40_spec(), 41, 8),
    "forward_r9_v3.npz": (synth.old_style_spec(blank_score=None), 43, 11),
}


def make(ref, name, spec, seed, col_stride):
    model = ref.crf_model.Model(synth.model_config(spec, batchnorm=False))
    weights = synth.make_weights(spec, seed=seed, qr_f64=True)
    model.load_state_dict(synth.state_dict_from_weights(spec, weights))
    model.eval()
    x = synth.squiggle(2, 340, seed=15).half().float()      # fp16-representable input: identical for every implementation
    with torch.inference_mode():
        scores = model.encoder(x)                            # [T, N, 5 * 4^k]: fixed blanks expanded, or learned blanks
        strings = model.decode_batch(scores)
    t, n, _ = scores.shape
    if spec["blank_score"] is not None:
        s5 = scores.reshape(t, n, -1, 5)
        assert torch.all(s5[..., 0] == spec["blank_score"])
        ntc = s5[..., 1:].reshape(t, n, -1).permute(1, 0, 2).contiguous()
    else:
        ntc = scores.permute(1, 0, 2).contiguous()
    out = {"x": x.numpy().astype(np.float16), "scores_ntc": ntc[..., ::col_stride].contiguous().numpy(),
           "col_stride": np.array(col_stride), "strings": np.array(json.dumps(strings)),
           "digest": np.array(weights_digest(weights)), "seed": np.array(seed), "stride": np.array(model.stride)}
    path = os.path.join(ROOT, "tests", "golden", name)
    np.savez_compressed(path, **out)
    print(name, "scores", tuple(ntc.shape), "strings", [len(s) for s in strings], "max|s| %.2f" % float(ntc.abs().max()),
          "bytes", os.path.getsize(path))


def main():
    ref = reference_shim.load()
    for name, (spec, seed, col_stride) in FIXTURES.items():
        make(ref, name, spec, seed, col_stride)


if __name__ == "__main__":
    main()
