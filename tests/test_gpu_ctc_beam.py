"""
The CTC prefix beam search kernel (bonito_b200/csrc/ctc_beam.cu) against its CPU oracle (tests/_oracle_ctc_beam.py), and
the layers above it: `bonito_b200.ctc.model.beam_search`, `Model.decode`, `basecall(..., beamsize=W)` and the
`B200_CTC_BEAMSIZE` switch of the `basecaller` CLI.

Planted / peaked log-probs must match the oracle byte for byte.  On flat random log-probs (softmax of N(0, 1) logits) the
fp32 sums of the kernel and the float64 sums of the oracle can rank two nearly equal candidates differently; measured on
one NVIDIA H100 80GB HBM3, 192 of 192 such reads were identical, and the test requires 90 % and that every differing
call is as probable as the oracle's to within 1e-3 in log-probability.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _oracle_ctc as oc  # noqa: E402
import _oracle_ctc_beam as ob  # noqa: E402
from bonito_b200 import native, synth  # noqa: E402
from bonito_b200.ctc.model import Model, beam_search  # noqa: E402

pytestmark = pytest.mark.gpu
CANARY8 = 0xA5
LABEL = {"A": 1, "C": 2, "G": 3, "T": 4}


def _planted(rows, hi, rng=None):
    """fp16 log-probs whose argmax follows `rows`: `hi` on the label, the rest shared (unequally when `rng` is given)."""
    rows = np.asarray(rows)
    T = len(rows)
    rest = np.full((T, 5), (1 - hi) / 4)
    if rng is not None:
        w = rng.uniform(0.2, 1.0, size=(T, 5))
        w[np.arange(T), rows] = 0
        rest = (1 - hi) * w / w.sum(-1, keepdims=True)
    rest[np.arange(T), rows] = hi
    return np.log(rest).astype(np.float16)


def _rows(T, seed):
    """Labels with repeats, blanks between and inside runs, and runs of every length up to the whole read."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < T:
        out += [int(rng.integers(0, 5))] * int(rng.integers(1, 5))
    return out[:T]


def _flat(T, seed):
    rng = np.random.default_rng(seed)
    logits = rng.normal(size=(T, 5))
    return (logits - np.log(np.exp(logits).sum(-1, keepdims=True))).astype(np.float16)


def _strings(out, lo, hi):
    seq, qual, moves = (out[i, lo:hi] for i in range(3))
    return seq[seq != 0].tobytes().decode(), qual[qual != 0].tobytes().decode(), moves


def _run(reads, width, threshold=1e-3, qscale=1.0, qbias=0.0):
    """The kernel on a list of [T, 5] fp16 arrays packed in order -> [(sequence, qstring, moves)] per read."""
    offsets = np.concatenate([[0], np.cumsum([len(r) for r in reads])]).astype(np.int64)
    logp = torch.from_numpy(np.concatenate(reads).reshape(-1, 5)).cuda()
    out = beam_search(logp, offsets, width, threshold, qscale, qbias).cpu().numpy()
    return [_strings(out, lo, hi) for lo, hi in zip(offsets, offsets[1:])]


def _same(got, want):
    return got[0] == want[0] and got[1] == want[1] and np.array_equal(got[2], want[2])


@pytest.mark.parametrize("width", [1, 2, 5, 32])
def test_kernel_matches_oracle_on_planted_reads(width):
    rng = np.random.default_rng(width)
    empty = np.zeros((0, 5), dtype=np.float16)
    # unequal shares for the other classes wherever the read is long or flat enough for two different prefixes to come
    # out equal in exact arithmetic (fp32 and float64 would round such a tie differently)
    reads = [_planted(_rows(T, 10 * T + width), hi, rng if T > 40 or hi < 0.9 else None)
             for T, hi in [(1, 0.9), (2, 0.6), (31, 0.9), (32, 0.7), (33, 0.998), (4000, 0.9), (257, 0.55)]]
    reads += [_planted([3] * 40, 0.9), _planted([0] * 33, 0.9), _planted([1, 1, 0, 1], 0.8)]
    for order in (reads[:5] + [empty] + reads[5:], [empty] + reads[::-1], reads[::2] + [empty]):
        got = _run(order, width, qscale=1.25, qbias=-0.5)
        for i, (lp, g) in enumerate(zip(order, got)):
            want = ob.beam_search(lp, width, qscale=1.25, qbias=-0.5)
            assert _same(g, want), (width, i, len(lp), g[0][:60], want[0][:60])
            assert int(g[2].sum()) == len(g[0]) == len(g[1])
    for lp in (empty, reads[0], reads[5]):                         # the only read of a launch
        assert _same(_run([lp], width)[0], ob.beam_search(lp, width))
    assert _run([_planted([3] * 40, 0.99)], width)[0][0] == "G"             # at 0.9, "GAG" over 40 frames outweighs "G"
    assert _run([_planted([1, 1, 0, 1], 0.8)], width)[0][0] == "AA"


def test_cut_ties_and_the_case_where_the_beam_beats_greedy():
    with np.errstate(divide="ignore"):
        beats = np.log(np.array([[0.40, 0.35, 0.25, 0.0, 0.0]] * 2)).astype(np.float16)
        tie4 = np.log(np.array([[0.0, 0.25, 0.25, 0.25, 0.25]])).astype(np.float16)
        tie2 = np.log(np.array([[0.5, 0.5, 0.0, 0.0, 0.0]])).astype(np.float16)
        cut = np.log(np.array([[0.05, 0.90, 0.05, 0.0, 0.0], [0.0008, 0.0002, 0.999, 0.0, 0.0]])).astype(np.float16)
    flat = np.log(np.full((3, 5), 0.2)).astype(np.float16)
    mixed = np.concatenate([_planted([3], 0.8), flat, _planted([3], 0.8)])
    got = _run([beats, tie4, tie2, cut], 5)
    assert got[0][0] == "A" and got[0][2].tolist() == [1, 0] and oc.greedy(beats.astype(np.float32))[0] == ""
    assert [g[0] for g in got[1:]] == ["A", "", "AC"]
    for reads, threshold in (([beats, tie4, tie2, cut], 1e-3), ([cut, cut[:1]], 0.1), ([flat, mixed], 0.5), ([mixed, beats], 0.0)):
        for lp, g in zip(reads, _run(reads, 5, threshold=threshold)):
            assert _same(g, ob.beam_search(lp, 5, threshold=threshold)), threshold
    assert _run([flat, mixed], 5, threshold=0.5)[1][0] == "G"


def test_flat_random_reads_agree_with_the_oracle_up_to_near_ties():
    reads = [_flat(150 + 7 * (i % 9), 1000 + i) for i in range(192)]
    same = 0
    for width in (5, 32):
        for lp, g in zip(reads[width % 2::2], _run(reads[width % 2::2], width)):
            want = ob.beam_search(lp, width)
            if _same(g, want):
                same += 1
                continue
            a = ob.ctc_log_prob(lp, [LABEL[c] for c in g[0]])
            b = ob.ctc_log_prob(lp, [LABEL[c] for c in want[0]])
            assert abs(a - b) <= 1e-3, (width, a, b)
            assert int(g[2].sum()) == len(g[0]) == len(g[1])
    print(f"flat random reads identical to the oracle: {same} of {len(reads)}")
    assert same >= 0.9 * len(reads)


def _quartznet(version="v1", **cfg):
    spec = synth.quartznet_spec(version)
    m = Model(synth.quartznet_config(spec, **cfg))
    m.load_state_dict(synth.make_quartznet_weights(spec, seed={"v1": 51, "v2": 52}[version]))
    m.use_koi(batchsize=64, chunksize=3999, quantize=False)
    return m.eval().half().to("cuda")


def test_every_width_on_a_quartznet_output_and_model_decode():
    m = _quartznet("v1", qscore=(1.5, 0.25))
    x = synth.squiggle(2, 3999, seed=9).half().cuda()
    with torch.inference_mode():
        logp = m.native_plan().forward(x)
    host = logp.cpu().numpy()
    for width in range(1, 33):
        got = _run([host[0], host[1]], width)
        for g in got:
            assert int(g[2].sum()) == len(g[0]) == len(g[1]) and set(g[0]) <= set("ACGT")
        if width in (2, 5, 32):
            assert _same(got[1], ob.beam_search(host[1], width)), width
    assert len(got[0][0]) > 50
    # Model.decode on a CUDA tensor: one read through the same kernel, with the model's [qscore] calibration
    want = ob.beam_search(host[0], 5, qscale=1.5, qbias=0.25)
    assert m.decode(logp[0], beamsize=5) == want[0]
    assert m.decode(logp[0], beamsize=5, qscores=True) == want[0] + want[1]
    seq, path = m.decode(logp[0].float(), beamsize=5, return_path=True)
    assert seq == want[0] and np.array_equal(path, np.flatnonzero(want[2]))
    assert m.decode(logp[0], beamsize=5, threshold=0.05) == ob.beam_search(host[0], 5, threshold=0.05)[0]
    assert m.decode(logp[0]) == oc.greedy(host[0].astype(np.float32))[0]          # beamsize=1 is still the greedy decode
    with pytest.raises(NotImplementedError, match="no CPU path"):
        m.decode(logp[0].cpu(), beamsize=5)


def test_long_read_keeps_its_range_and_runs_are_reproducible():
    unit = [1, 1, 0, 2, 0, 0, 3, 3, 3, 4, 0, 1, 0, 1, 0]
    rows = unit * (300_000 // len(unit))
    lp = _planted(rows, 0.9, np.random.default_rng(3))
    short = _planted(_rows(500, 8), 0.8)
    a = beam_search(torch.from_numpy(np.concatenate([short, lp])).cuda(), [0, 500, 300_500], 5)
    b = beam_search(torch.from_numpy(np.concatenate([short, lp])).cuda(), [0, 500, 300_500], 5)
    assert torch.equal(a, b)
    seq, qual, moves = _strings(a.cpu().numpy(), 500, 300_500)
    assert seq == "ACGTAA" * (300_000 // len(unit))
    assert len(qual) == len(seq) == int(moves.sum()) and set(qual) <= {chr(c) for c in range(34, 74)}
    assert _same(_strings(a.cpu().numpy(), 0, 500), ob.beam_search(short, 5))


def test_qualities_are_the_greedy_ones_on_the_greedy_path():
    rows = _rows(3000, 4)
    lp = _planted(rows, 0.999, np.random.default_rng(5))           # every other class is below the 1e-3 cut
    seq, qual, moves = _run([lp], 5, qscale=1.1, qbias=0.3)[0]
    gs, gq, gmv = oc.greedy(lp.astype(np.float32), qscale=np.float32(1.1), qbias=np.float32(0.3))
    assert seq == gs and np.array_equal(moves, gmv) and qual == gq and len(seq) > 500


def test_output_and_workspace_bounds_and_the_workspace_check():
    """Canary bytes around the three outputs and the workspace stay intact, frames outside the reads are not written, and
    a workspace one node short is refused by the status of the call before anything is launched."""
    reads = [_planted(_rows(T, T), 0.7) for T in (65, 1, 300)]
    gap, front = 7, 64
    frames = gap + sum(len(r) for r in reads) + 2 * gap
    logp = torch.zeros(frames, 5, dtype=torch.float16)
    off, pos = [], gap
    for r in reads:                                                 # reads out of order in the buffer, gaps between them
        off.append(pos)
        logp[pos:pos + len(r)] = torch.from_numpy(r)
        pos += len(r) + gap // 2
    off, ln = np.array(off[::-1], dtype=np.int64), np.array([len(r) for r in reads[::-1]], dtype=np.int32)
    need = native.ctc_beam_workspace_bytes(3, int(ln.sum()), 32)
    bufs = [torch.full((front + frames + front,), CANARY8, dtype=torch.uint8, device="cuda") for _ in range(3)]
    ws = torch.full((front + need + front,), CANARY8, dtype=torch.uint8, device="cuda")
    # 256-byte aligned views: torch allocations are 512-byte aligned and `front` is a multiple of 64
    views = [b[front:front + frames] for b in bufs]
    native.ctc_beam_search(logp.cuda(), off, ln, 32, 1e-3, 1.0, 0.0, ws[front:front + need], *views)
    torch.cuda.synchronize()
    inside = np.zeros(frames, dtype=bool)
    for o, n in zip(off, ln):
        inside[o:o + n] = True
    for b in bufs:
        host = b.cpu().numpy()
        assert (host[:front] == CANARY8).all() and (host[front + frames:] == CANARY8).all()
        assert (host[front:front + frames][~inside] == CANARY8).all()
    assert (bufs[2].cpu().numpy()[front:front + frames][inside] <= 1).all()
    wsh = ws.cpu().numpy()
    assert (wsh[:front] == CANARY8).all() and (wsh[front + need:] == CANARY8).all()
    out = np.stack([b.cpu().numpy()[front:front + frames] for b in bufs])
    for r, o in zip(reads[::-1], off):
        assert _same(_strings(out, o, o + len(r)), ob.beam_search(r, 32))
    # one node (8 bytes) short
    for b in bufs:
        b.fill_(CANARY8)
    with pytest.raises(native.NativeError, match="workspace has"):
        native.ctc_beam_search(logp.cuda(), off, ln, 32, 1e-3, 1.0, 0.0, ws[front:front + need - 8], *views)
    torch.cuda.synchronize()
    assert all(bool((b == CANARY8).all()) for b in bufs)
    # argument checks of the wrapper
    with pytest.raises(native.NativeError, match="outside the"):
        native.ctc_beam_search(logp.cuda(), off + frames, ln, 5, 1e-3, 1.0, 0.0, ws, *views)
    with pytest.raises(native.NativeError, match="beam_width"):
        native.ctc_beam_search(logp.cuda(), off, ln, 33, 1e-3, 1.0, 0.0, ws, *views)
    with pytest.raises(native.NativeError, match="sequence"):
        native.ctc_beam_search(logp.cuda(), off, ln, 5, 1e-3, 1.0, 0.0, ws, views[0][1:], views[1], views[2])
    with pytest.raises(native.NativeError, match="threshold"):
        native.ctc_beam_search(logp.cuda(), off, ln, 5, 1.5, 1.0, 0.0, ws, *views)


class _Read:
    def __init__(self, rid, sig):
        self.read_id, self.signal = rid, sig


@pytest.mark.parametrize("version", ["v1", "v2"])
def test_basecall_with_the_beam_search_matches_the_oracle_pipeline(version):
    from bonito_b200.crf.basecall import stitch_results
    from bonito_b200.ctc.basecall import basecall
    from bonito_b200.util import chunk
    m = _quartznet(version)
    lengths = (9000, 2500, 12345)
    sig = synth.squiggle(len(lengths), max(lengths), seed=21)[:, 0].numpy()
    reads = [_Read(f"r{i}", sig[i, :n].copy()) for i, n in enumerate(lengths)]
    chunksize, overlap = 3999, 498
    out = list(basecall(m, iter(reads), beamsize=5, chunksize=chunksize, overlap=overlap, batchsize=5))
    assert [r.read_id for r, _ in out] == ["r0", "r1", "r2"]
    plan = m.native_plan()
    for read, res in out:
        with torch.inference_mode():
            logp = plan.forward(chunk(torch.from_numpy(read.signal), chunksize, overlap).half().cuda()).cpu()
        st = stitch_results(logp, len(read.signal), chunksize, overlap, 3).numpy()
        s, q, mv = ob.beam_search(st, 5)
        assert res["sequence"] == s and res["qstring"] == q and np.array_equal(res["moves"], mv) and res["stride"] == 3
        assert len(res["moves"]) == len(read.signal) // 3 and len(s) > 50
    # the calls do not depend on how the reads are grouped or batched
    for kw in (dict(group_reads=1), dict(group_frames=4000), dict(batchsize=2), dict(group_reads=2, batchsize=64)):
        again = list(basecall(m, iter(reads), beamsize=5, chunksize=chunksize, overlap=overlap, **{"batchsize": 5, **kw}))
        assert [r.read_id for r, _ in again] == ["r0", "r1", "r2"]
        for (_, a), (_, b) in zip(out, again):
            assert a["sequence"] == b["sequence"] and a["qstring"] == b["qstring"] and np.array_equal(a["moves"], b["moves"])
    greedy = list(basecall(m, iter(reads), chunksize=chunksize, overlap=overlap, batchsize=5))
    assert all(len(g["sequence"]) > 50 for _, g in greedy)


def test_cli_beamsize_switch(tmp_path):
    reads = tmp_path / "reads"
    reads.mkdir()
    sig = synth.squiggle(2, 9000, seed=4)[:, 0].numpy()
    for i in range(2):
        np.save(reads / f"read{i}.npy", (90 + 20 * sig[i]).astype(np.float32))
    spec = synth.quartznet_spec("v2")
    d = synth.write_quartznet_dir(str(tmp_path / "v2"), spec, synth.make_quartznet_weights(spec, seed=52))
    cmd = [sys.executable, "-m", "bonito_b200", "basecaller", d, str(reads)]
    env = dict(os.environ, PYTHONPATH=ROOT)
    env.pop("B200_CTC_BEAMSIZE", None)
    texts = {}
    for width, suffix in ((None, "fastq"), ("1", "fastq"), ("5", "fastq"), ("5", "sam")):
        path = tmp_path / f"w{width}.{suffix}"
        with open(path, "w") as fh:
            p = subprocess.run(cmd, cwd=ROOT, env=env if width is None else dict(env, B200_CTC_BEAMSIZE=width), stdout=fh,
                               stderr=subprocess.PIPE, text=True)
        assert p.returncode == 0, p.stderr
        texts[width, suffix] = open(path).read()
    assert texts[None, "fastq"] == texts["1", "fastq"]              # unset is the greedy decode, as before
    recs = texts["5", "fastq"].strip().split("\n")
    assert len(recs) == 8 and all(len(recs[i + 1]) > 100 and len(recs[i + 1]) == len(recs[i + 3]) for i in (0, 4))
    assert texts["5", "fastq"] != texts["1", "fastq"]
    rows = [r for r in texts["5", "sam"].strip().split("\n") if not r.startswith("@")]
    assert len(rows) == 2 and all("\tmv:B:c,3," in r for r in rows)
    for bad in ("99", "0", "five"):
        p = subprocess.run(cmd, cwd=ROOT, env=dict(env, B200_CTC_BEAMSIZE=bad), capture_output=True, text=True)
        assert p.returncode != 0 and "B200_CTC_BEAMSIZE must be an integer in 1..32" in p.stderr, p.stderr
        assert "Traceback" not in p.stderr
