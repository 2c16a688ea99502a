"""`evaluate`: the CPU alignment oracle, chunk-dataset loading, the summary, and on the GPU b200_sw_align against the oracle
and the whole subcommand on synthetic models and datasets."""
import io
import os
import random
import subprocess
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

import _oracle_align as O
from bonito_b200 import synth
from bonito_b200.align import AlignResult

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ oracle, by hand
@pytest.mark.parametrize("q,r,want", [
    ("ACGTACGT", "ACGTACGT", (40, 7, 7, "8=")),                          # identity
    ("ACGTTCGTAC", "ACGTACGTAC", (41, 9, 9, "4=1X5=")),                  # one substitution
    ("ACGTACTGTACGT", "ACGTACGTACGT", (52, 12, 11, "6=1I6=")),           # one insertion inside
    ("ACGTACGTACGT", "ACGTACTGTACGT", (52, 11, 12, "6=1D6=")),           # one deletion inside
    ("GACGTACGT", "ACGTACGT", (40, 8, 7, "8=")),                         # an extra query base at the start is clipped
    ("ACGTACGTT", "ACGTACGT", (40, 7, 7, "8=")),                         # ... and at the end
    ("ACGTACGT", "ACGTACGTT", (40, 7, 7, "8=")),                         # an extra reference base at the end is clipped
    ("ACGTACGT", "TACGTACGT", (40, 7, 8, "8=")),                         # ... and at the start
    ("ACGTAAAACGT", "ACGTAAAAACGT", (47, 10, 11, "4=1D7=")),             # homopolymer: the gap goes first in the run
    ("AAAA", "CCCC", (0, -1, -1, "")),                                   # no common letter
    ("", "ACGT", (0, -1, -1, "")),                                       # empty sides
    ("ACGT", "", (0, -1, -1, "")),
    ("ACGT", "ACGTTTTTACGT", (20, 3, 3, "4=")),                          # end-cell tie: the smaller end_ref
    ("AAGG", "GGAA", (10, 1, 3, "2=")),                                  # end-cell tie: the smaller end_query first
])
def test_oracle_hand_worked_cases(q, r, want):
    res = O.align(q, r)
    assert (res["score"], res["end_query"], res["end_ref"], res["cigar"]) == want


def test_oracle_counts_and_align_result_fields():
    res = O.align("ACGTACTGTACGT", "ACGTACGTACGT")
    assert (res["n_eq"], res["n_x"], res["n_ins"], res["n_del"]) == (12, 0, 1, 0)
    f = O.align_result_fields(ref="TTACGTACGTACGT", seq="GACGTACGTACG")
    assert (f.num_correct, f.align_seq_start, f.align_seq_end, f.align_ref_start, f.align_ref_end) == (11, 1, 11, 2, 12)
    assert f.accuracy == 1.0 and (f.ref_len, f.seq_len) == (14, 12)
    assert O.align_result_fields(ref="ACGT", seq="") == AlignResult()
    zero = O.align_result_fields(ref="CCCC", seq="AAA")
    assert zero == AlignResult(accuracy=0.0, ref_len=4, seq_len=3)


# ------------------------------------------------------------------------------------------------ host checks
def test_align_batch_refuses_bad_input_before_any_launch():
    from bonito_b200.align import align_batch
    with pytest.raises(ValueError, match="other than A, C, G, T"):
        align_batch(["ACGT", "ACNT"], ["ACGT", "ACGT"], device="cpu")
    with pytest.raises(ValueError, match="other than A, C, G, T"):
        align_batch(["ACGT"], ["acgt"], device="cpu")
    with pytest.raises(ValueError, match="at most 65535"):
        align_batch(["A" * 65536], ["ACGT"], device="cpu")
    with pytest.raises(ValueError, match="references for"):
        align_batch(["ACGT"], [], device="cpu")


def _write_chunks(directory, n, length=40, seed=0, ref_len=12):
    rng = np.random.default_rng(seed)
    os.makedirs(directory, exist_ok=True)
    chunks = rng.standard_normal((n, length)).astype(np.float32)
    lengths = rng.integers(1, ref_len + 1, size=n)
    refs = np.zeros((n, ref_len), dtype=np.uint8)
    for i, k in enumerate(lengths):
        refs[i, :k] = rng.integers(1, 5, size=k)
    chunks[:, 0] = np.arange(n)                 # chunk i is recognisable by its first sample
    np.save(os.path.join(directory, "chunks.npy"), chunks)
    np.save(os.path.join(directory, "references.npy"), refs)
    np.save(os.path.join(directory, "reference_lengths.npy"), lengths.astype(np.uint16))
    return chunks, refs, lengths


def test_load_numpy_split_validation_and_indices(tmp_path):
    from bonito_b200.data import ChunkDataSet, load_numpy, load_numpy_datasets
    _write_chunks(tmp_path / "a", 20)
    train, valid = load_numpy(15, tmp_path / "a", valid_chunks=4)          # split: the last 4 of the first 15
    assert train["shuffle"] and not valid["shuffle"]
    assert [int(x) for x in train["dataset"].chunks[:, 0, 0]] == list(range(11))
    assert [int(x) for x in valid["dataset"].chunks[:, 0, 0]] == [11, 12, 13, 14]
    train, valid = load_numpy(3, tmp_path / "a", valid_chunks=5)            # more valid chunks than loaded: split at 0
    assert [int(x) for x in valid["dataset"].chunks[:, 0, 0]] == [0, 1, 2]
    assert len(train["dataset"]) == 0 and not train["shuffle"]              # an empty split gives a loader all the same
    from torch.utils.data import DataLoader
    assert list(DataLoader(**train)) == []
    train, valid = load_numpy(None, tmp_path / "a")                         # no count: 97 % / 3 %
    assert len(train["dataset"]) == 19 and len(valid["dataset"]) == 1
    _write_chunks(tmp_path / "a" / "validation", 6, seed=1)
    train, valid = load_numpy(15, tmp_path / "a", valid_chunks=4)           # validation/ takes precedence
    assert len(train["dataset"]) == 15 and [int(x) for x in valid["dataset"].chunks[:, 0, 0]] == [0, 1, 2, 3]
    np.save(tmp_path / "a" / "indices.npy", np.array([7, 99, 3, 25, 5, 1], dtype=np.int64))
    chunks, targets, lengths = load_numpy_datasets(limit=3, directory=tmp_path / "a")
    assert [int(x) for x in chunks[:, 0]] == [7, 3, 5]                      # indices past the end dropped, then limited
    item = ChunkDataSet(chunks, targets, lengths)[1]
    assert item[0].shape == (1, 40) and item[0].dtype == np.float32 and item[1].dtype == np.int64
    assert item[2].dtype == np.int64


def test_load_data_script_and_errors(tmp_path):
    from bonito_b200.data import ComputeSettings, DataSettings, ModelSetup, load_data
    (tmp_path / "s").mkdir()
    (tmp_path / "s" / "dataset.py").write_text(
        "import numpy as np\n"
        "from bonito_b200.data import ChunkDataSet\n"
        "class Loader:\n"
        "    def __init__(self, **kw):\n"
        "        self.kw = kw\n"
        "    def _set(self, n):\n"
        "        s = self.kw['standardisation']\n"
        "        c = np.full((n, 30), s['mean'], dtype=np.float32)\n"
        "        return ChunkDataSet(c, np.ones((n, 4), dtype=np.int64), np.full(n, 4))\n"
        "    def train_loader_kwargs(self, **kw):\n"
        "        return {'dataset': self._set(kw['chunks']), 'shuffle': True}\n"
        "    def valid_loader_kwargs(self, **kw):\n"
        "        return {'dataset': self._set(kw['valid_chunks']), 'shuffle': False, 'batch_size': 2}\n")
    setup = ModelSetup(3, 1, {"mean": 7.5, "stdev": 2.0})
    train, valid = load_data(DataSettings(tmp_path / "s", 5, 3, None), setup, ComputeSettings(4, 0, 9, pin_memory=False))
    assert len(train.dataset) == 5 and len(valid.dataset) == 3 and valid.batch_size == 2 and train.batch_size == 4
    x, y, n = next(iter(valid))
    assert x.shape == (2, 1, 30) and float(x[0, 0, 0]) == 7.5
    with pytest.raises(IOError, match="Failed to load input data"):
        load_data(DataSettings(tmp_path / "nothing", 5, 3, None), setup, ComputeSettings(4, 0, 9))


def test_evaluate_help_and_flag_surface():
    out = subprocess.run([sys.executable, "-m", "bonito_b200", "evaluate", "-h"], cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.startswith("usage: bonito_b200 evaluate")
    from bonito_b200.cli.evaluate import argparser
    flags = {a for act in argparser()._actions for a in act.option_strings}
    assert flags == {"--output_dir", "--directory", "--dataset", "--device", "--seed", "--weights", "--chunks", "--batchsize",
                     "--standardise"}                                      # bonito/cli/evaluate.py:140-156
    args = argparser().parse_args(["model"])
    assert (args.dataset, args.device, args.seed, args.weights, args.chunks, args.batchsize, args.standardise) == \
        ("valid", "cuda", 9, 0, 512, 256, False)


def test_summary_block_and_table():
    from bonito_b200.cli.evaluate import summary, summary_table
    rows = [AlignResult(0.9, 9, 1, 0, 0, 12, 10, 1, 10, 0, 9),
            AlignResult(),                                                 # an empty call
            AlignResult(0.5, 0, 1, 1, 0, 6, 4, 2, 3, 1, 2)]                # n_eq 0: sub / ins rate inf
    text = summary(rows)
    lines = text.split("\n")
    assert lines[0] == "" and lines[-1] == "" and len(lines) == 13
    assert lines[1] == "* num_chunks      3"
    assert lines[2] == f"* accuracy        {(0.9 + 0 + 0.5) / 3:.2%}"
    assert lines[3] == "* sub-rate        inf%"            # 1/9, NaN (0/0, skipped), inf
    assert lines[4] == "* ins-rate        inf%"
    assert lines[5] == "* del-rate        0.00%"           # 0/9, NaN, 0/0 = NaN: the mean of what is left
    assert lines[6] == "* seq_len         4.7"
    assert lines[8] == f"* seq_rclip       {((10 - 9 - 1) + (0 - 0 - 1) + (4 - 2 - 1)) / 3:.1f}"
    assert lines[11] == f"* ref_rclip       {((12 - 10 - 1) + (0 - 0 - 1) + (6 - 3 - 1)) / 3:.1f}"
    nan = summary([AlignResult(0.0, 0, 0, 0, 0, 5, 5, 0, 0, 0, 0)])
    assert "* sub-rate        nan%" in nan and "* accuracy        0.00%" in nan
    table = summary_table(rows).split("\n")
    assert table[0] == "\taccuracy\tnum_correct\tnum_mismatches\tnum_insertions\tnum_deletions\tref_len\tseq_len\t" \
                       "align_ref_start\talign_ref_end\talign_seq_start\talign_seq_end"
    assert table[1] == "0\t0.9\t9\t1\t0\t0\t12\t10\t1\t10\t0\t9"
    assert table[2] == "1\t0.0\t0\t0\t0\t0\t0\t0\t0\t0\t0\t0"          # pandas makes the mixed column float64
    assert table[4] == ""


# ------------------------------------------------------------------------------------------------ GPU: the kernel
def _mutate(rng, s, sub, ins, dele):
    out = []
    for c in s:
        x = rng.random()
        if x < sub:
            out.append(rng.choice([b for b in "ACGT" if b != c]))
        elif x < sub + ins:
            out.append(c)
            out.append(rng.choice("ACGT"))
        elif x < sub + ins + dele:
            continue
        else:
            out.append(c)
    return "".join(out)


def _rand(rng, n):
    return "".join(rng.choice("ACGT") for _ in range(n))


def _repeats(rng, n):
    parts = []
    while sum(map(len, parts)) < n:
        parts.append(rng.choice("ACGT") * rng.randint(2, 9) if rng.random() < 0.5 else
                     _rand(rng, rng.randint(2, 4)) * rng.randint(2, 6))
    return "".join(parts)[:n]


PROFILES = ["identical", "edits_5_2_3", "edits_25", "unrelated", "repeats", "query_in_ref", "ref_in_query"]


def _pair(rng, profile, n):
    """(ref, query) with a reference of n bases."""
    if profile == "repeats":
        r = _repeats(rng, n)
        return r, _mutate(rng, r, 0.05, 0.02, 0.03)
    r = _rand(rng, n)
    if profile == "identical":
        return r, r
    if profile == "edits_5_2_3":
        return r, _mutate(rng, r, 0.05, 0.02, 0.03)
    if profile == "edits_25":
        return r, _mutate(rng, r, 0.12, 0.06, 0.07)
    if profile == "unrelated":
        return r, _rand(rng, n)
    if profile == "query_in_ref":
        a = n // 4
        return r, _mutate(rng, r[a:n - a], 0.03, 0.01, 0.01)
    return r, _rand(rng, n // 3 + 1) + _mutate(rng, r, 0.03, 0.01, 0.01) + _rand(rng, n // 3 + 1)


def _kernel_pairs():
    rng = random.Random(2024)
    pairs = [("", ""), ("ACGT", ""), ("", "ACGT"), ("A", "A"), ("A", "C")]
    for n in (1, 2, 31, 32, 33, 255, 256, 257, 1000):
        for profile in PROFILES:
            pairs.append(_pair(rng, profile, n))
    for profile in ("edits_5_2_3", "repeats", "ref_in_query"):
        pairs.append(_pair(rng, profile, 4097))
    long = _rand(rng, 20000)
    pairs.append((long, _mutate(rng, long[9000:9600], 0.05, 0.02, 0.03)))       # a 600-base query inside 20000
    pairs.append((long[4000:4600], _mutate(rng, long, 0.05, 0.02, 0.03)))       # a 600-base reference inside ~20000
    return pairs


@pytest.mark.gpu
def test_kernel_matches_oracle_and_is_independent_of_the_batch():
    from bonito_b200.align import sw_align_batch
    pairs = _kernel_pairs()
    refs, seqs = [r for r, _ in pairs], [q for _, q in pairs]
    got = sw_align_batch(refs, seqs)
    assert got.shape == (len(pairs), 7)
    bad = []
    for k, (r, q) in enumerate(pairs):
        want = O.as_row(O.align(q, r))
        if got[k].tolist() != want:
            bad.append((k, len(q), len(r), got[k].tolist(), want))
    assert not bad, bad[:5]
    # every pair alone gives what it gave in the batch
    for k, (r, q) in enumerate(pairs):
        assert sw_align_batch([r], [q])[0].tolist() == got[k].tolist(), k
    # and a reordered batch gives the same rows
    order = list(range(len(pairs)))[::-1]
    again = sw_align_batch([refs[i] for i in order], [seqs[i] for i in order])
    assert np.array_equal(again[::-1], got)
    assert sw_align_batch([], []).shape == (0, 7)


@pytest.mark.gpu
def test_kernel_refuses_long_and_non_acgt_input():
    from bonito_b200 import native
    from bonito_b200.align import align_batch
    with pytest.raises(ValueError):
        align_batch(["A" * 65536], ["A" * 10])
    with pytest.raises(ValueError):
        align_batch(["ACGT"], ["ACGU"])
    # the entry point itself refuses a length over 65535
    n = 70000
    buf = torch.full((n,), ord("A"), dtype=torch.uint8, device="cuda")
    off = torch.zeros(1, dtype=torch.int64)
    ws = torch.empty(native.sw_align_workspace_bytes(1, n), dtype=torch.uint8, device="cuda")
    out = torch.empty(1, 7, dtype=torch.int32, device="cuda")
    with pytest.raises(native.NativeError, match="65535"):
        native.sw_align(buf, off, torch.tensor([n], dtype=torch.int32), buf, off, torch.tensor([10], dtype=torch.int32), ws, out)


# ------------------------------------------------------------------------------------------------ GPU: evaluate
def _hac_dir(tmp_path):
    spec = synth.model_spec("hac")
    return synth.write_model_dir(str(tmp_path / "hac"), spec, synth.make_weights(spec, seed=3)), 1998


def _ctc_dir(tmp_path):
    spec = synth.quartznet_spec("v1")
    return synth.write_quartznet_dir(str(tmp_path / "ctc"), spec, synth.make_quartznet_weights(spec, seed=11)), 2001


def _sup_dir(tmp_path):
    import toml
    spec = synth.sup_spec(depth=2)
    d = tmp_path / "sup"
    d.mkdir()
    with open(d / "config.toml", "w") as fh:
        toml.dump(synth.sup_config(spec), fh)
    torch.save(synth.sup_state_dict(spec, synth.make_sup_weights(spec, seed=3)), d / "weights_1.tar")
    return str(d), 1200


def _dataset(directory, chunks, refs):
    os.makedirs(directory, exist_ok=True)
    width = max(1, max(len(r) for r in refs))
    labels = np.zeros((len(refs), width), dtype=np.uint8)
    for i, r in enumerate(refs):
        labels[i, :len(r)] = ["NACGT".index(c) for c in r]
    np.save(os.path.join(directory, "chunks.npy"), chunks)
    np.save(os.path.join(directory, "references.npy"), labels)
    np.save(os.path.join(directory, "reference_lengths.npy"), np.array([len(r) for r in refs], dtype=np.uint16))


def _read_fasta(path):
    lines = open(path).read().split("\n")
    return [lines[i + 1] for i in range(0, len(lines) - 1, 2)]


def _run(model_dir, data_dir, out_dir, n, batchsize):
    from bonito_b200.cli.evaluate import argparser, main
    args = argparser().parse_args([model_dir, "--directory", str(data_dir), "--chunks", str(n), "--batchsize",
                                   str(batchsize), "--weights", "1", "--output_dir", str(out_dir)])
    buf = io.StringIO()
    with redirect_stdout(buf):
        main(args)
    return buf.getvalue()


@pytest.mark.gpu
@pytest.mark.parametrize("make", [_hac_dir, _ctc_dir, _sup_dir], ids=["hac_lstm_crf", "quartznet_v1", "sup_transformer"])
def test_evaluate_end_to_end(tmp_path, make):
    model_dir, length = make(tmp_path)
    n, batchsize = 24, 16                       # a short last batch too
    chunks = synth.squiggle(n, length, seed=5)[:, 0].numpy()
    # pass 1: learn the model's own calls
    _dataset(tmp_path / "d0", chunks, ["ACGT"] * n)
    _run(model_dir, tmp_path / "d0", tmp_path / "o0", n, batchsize)
    calls = _read_fasta(tmp_path / "o0" / "seqs.fasta")
    assert len(calls) == n and min(len(c) for c in calls) >= 10, [len(c) for c in calls]
    # pass 2: references equal to the calls -> every chunk is 100 % accurate
    _dataset(tmp_path / "d1", chunks, calls)
    text = _run(model_dir, tmp_path / "d1", tmp_path / "o1", n, batchsize)
    assert "* num_chunks      24\n* accuracy        100.00%\n* sub-rate        0.00%" in text
    rows = open(tmp_path / "o1" / "summ.txt").read().rstrip("\n").split("\n")[1:]
    assert len(rows) == n and all(float(r.split("\t")[1]) == 1.0 for r in rows)
    # pass 3: seeded edits in the references -> summ.txt is the oracle's alignment of the written fasta files
    rng = random.Random(7)
    edited = [_mutate(rng, c, 0.05, 0.02, 0.03) or "A" for c in calls]
    _dataset(tmp_path / "d2", chunks, edited)
    text = _run(model_dir, tmp_path / "d2", tmp_path / "o2", n, batchsize)
    seqs, refs = _read_fasta(tmp_path / "o2" / "seqs.fasta"), _read_fasta(tmp_path / "o2" / "refs.fasta")
    assert seqs == calls and refs == edited
    table = [r.split("\t") for r in open(tmp_path / "o2" / "summ.txt").read().rstrip("\n").split("\n")]
    assert table[0][0] == "" and len(table) == n + 1
    for k, (seq, ref) in enumerate(zip(seqs, refs)):
        want = O.align_result_fields(ref=ref, seq=seq)
        row = table[k + 1]
        assert int(row[0]) == k
        assert abs(float(row[1]) - want.accuracy) <= 1e-12
        assert [int(v) for v in row[2:]] == [getattr(want, f) for f in table[0][2:]], (k, row)
    assert "* accuracy        100.00%" not in text


@pytest.mark.gpu
def test_evaluate_cli_prints_the_summary_and_writes_outputs(tmp_path):
    model_dir, length = _hac_dir(tmp_path)
    chunks = synth.squiggle(32, length, seed=8)[:, 0].numpy()
    _dataset(tmp_path / "d", chunks, ["ACGTACGTTGCA" * 3] * 32)
    env = dict(os.environ, PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable, "-m", "bonito_b200", "evaluate", model_dir, "--directory", str(tmp_path / "d"),
                        "--chunks", "32", "--weights", "1", "--output_dir", str(tmp_path / "out")], cwd=ROOT, env=env,
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    keys = [line.split()[1] for line in p.stdout.split("\n") if line.startswith("* ") and not line.startswith("* *")]
    assert keys[-11:] == ["num_chunks", "accuracy", "sub-rate", "ins-rate", "del-rate", "seq_len", "seq_lclip", "seq_rclip",
                          "ref_len", "ref_lclip", "ref_rclip"]
    assert sorted(os.listdir(tmp_path / "out")) == ["refs.fasta", "seqs.fasta", "summ.txt"]
    # a model that cannot be loaded: one line on stderr, no traceback
    p = subprocess.run([sys.executable, "-m", "bonito_b200", "evaluate", str(tmp_path / "missing"), "--directory",
                        str(tmp_path / "d")], cwd=ROOT, env=env, capture_output=True, text=True)
    assert p.returncode != 0 and "Traceback" not in p.stderr and p.stderr.count("\n") == 1, p.stderr
