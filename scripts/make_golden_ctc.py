"""
Generate tests/golden/forward_ctc_v1.npz and forward_ctc_v2.npz (the QuartzNet CTC models dna_r9.4.1@v1 and @v2) through the
REFERENCE's own module tree (bonito/ctc/model.py `Model(config)`), fp32 on the CPU, with the seeded weights of
`synth.make_quartznet_weights`.  Needs the reference checkout that oracle/reference_shim.py imports; the committed fixtures
are only replayed.  The reference's decoders (fast_ctc_decode) are not used: the strings are the oracle's greedy decode.

    python scripts/make_golden_ctc.py

Contents: the fp16-representable input [2, 1, 1200], the log-probs of all 5 classes [2, 400, 5] (fp32, batch-first),
the oracle greedy strings and quality strings, the RMS of each block's output (oracle, fp64), the weight seed and the digest of the seeded weights.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import synth  # noqa: E402
from oracle.make_golden import weights_digest  # noqa: E402
import _oracle_ctc  # noqa: E402

FIXTURES = {"forward_ctc_v1.npz": ("v1", 51), "forward_ctc_v2.npz": ("v2", 52)}


def main():
    ref = _oracle_ctc.load_ctc()
    for name, (version, seed) in FIXTURES.items():
        spec = synth.quartznet_spec(version)
        config = synth.quartznet_config(spec)
        state = synth.make_quartznet_weights(spec, seed=seed)
        model = ref.Model(config)
        model.load_state_dict(state)
        model.eval()
        x = synth.squiggle(2, 1200, seed=15).half().float()
        with torch.inference_mode():
            logp = model(x).permute(1, 0, 2).contiguous()            # [T, N, 5] -> [N, T, 5]
        decoded = [_oracle_ctc.greedy(row.numpy()) for row in logp]
        _, blocks = _oracle_ctc.forward(state, config, x, return_blocks=True)
        block_rms = np.array([float(b.pow(2).mean().sqrt()) for b in blocks])
        out = {"x": x.numpy().astype(np.float16), "logp": logp.numpy(), "strings": np.array(json.dumps([d[0] for d in decoded])),
               "qstrings": np.array(json.dumps([d[1] for d in decoded])), "digest": np.array(weights_digest(state)),
               "block_rms": block_rms, "seed": np.array(seed), "stride": np.array(model.stride)}
        path = os.path.join(ROOT, "tests", "golden", name)
        np.savez_compressed(path, **out)
        print(name, "logp", tuple(logp.shape), "bases", [len(d[0]) for d in decoded], "block rms", np.round(block_rms, 2), "bytes", os.path.getsize(path))


if __name__ == "__main__":
    main()
