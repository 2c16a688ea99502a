"""
Writes the POD5 fixtures under tests/golden/ (needs the system libzstd.so.1; the GPU tests that use them do not):

  pod5_vbz.pod5, pod5_raw.pod5   the same eight synthetic reads, VBZ-compressed (signal rows of 8000 samples, so most reads
                                 span two rows) and uncompressed, written by tests/_pod5_writer.py;
  pod5_expected.npz              their read ids and int16 signals;
  zstd_corpus.npz                zstd streams from libzstd with the length and SHA-256 of what libzstd decompresses
                                 them to (the outputs themselves are not stored, to keep the fixture small): levels -5,
                                 1, 3, 9 and 19, with and without checksum and content size, small target block sizes, a
                                 1 KiB window, multi-block streams up to 1 MiB, random bytes (Raw blocks), constant runs
                                 (RLE), text, svb16 rows of synthetic squiggles, two frames with a skippable frame between
                                 them, and an empty frame.

    python scripts/make_golden_pod5.py
"""
import hashlib
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _pod5_writer as W  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def words(n, seed):
    rng = np.random.default_rng(seed)
    vocab = ["the", "read", "signal", "pore", "base", "of", "and", "a", "current", "strand", "motor", "protein", "flow",
             "cell", "channel", "sample", "model", "call", "quality", "score", "in", "to", "is", "was", "nanopore"]
    out = bytearray()
    while len(out) < n:
        out += (" ".join(rng.choice(vocab, 12)) + ".\n").encode()
    return bytes(out[:n])


def repeats(n, seed):
    """n bytes of one 16 kB text repeated with 64 bytes changed in each copy: long matches over many blocks."""
    rng = np.random.default_rng(seed)
    base = np.frombuffer(words(16000, seed), np.uint8)
    out = np.concatenate([base] * (n // len(base) + 1))[:n].copy()
    for at in range(0, n, len(base)):
        pos = at + rng.integers(0, len(base), 64)
        out[pos[pos < n]] = rng.integers(32, 127, int((pos < n).sum()))
    return out.tobytes()


def squiggle_svb(n, seed):
    return W.svb16_encode(W.synthetic_reads(1, seed=seed, min_len=n, max_len=n + 1)[0]["signal"])


def corpus():
    rng = np.random.default_rng(11)
    sources = {"text": words(20000, 1), "random": rng.bytes(4000), "constant": b"\x5a" * 70000,
               "svb16": squiggle_svb(8000, 2), "svb16_big": squiggle_svb(120000, 3), "text_big": repeats(1 << 20, 4),
               "tiny": b"ACGT", "empty": b""}
    entries = []  # (label, stream, source name)
    for name in ("text", "random", "constant", "svb16"):
        for level in (-5, 1, 3, 9, 19):
            for checksum, size in ((False, True), (True, False)):
                entries.append((f"{name}/L{level}/ck{int(checksum)}/cs{int(size)}",
                                W.zstd_compress(sources[name], level, checksum, size), name))
    for name in ("text", "svb16"):
        for block in (1340, 4096):
            entries.append((f"{name}/L3/block{block}", W.zstd_compress(sources[name], 3, True, True, target_block=block), name))
        entries.append((f"{name}/L19/window10", W.zstd_compress(sources[name], 19, True, True, window_log=10), name))
    entries.append(("svb16_big/L1", W.zstd_compress(sources["svb16_big"], 1, True, True), "svb16_big"))
    for level in (1, 9):
        entries.append((f"text_big/L{level}", W.zstd_compress(sources["text_big"], level, True, True), "text_big"))
    for name in ("tiny", "empty"):
        entries.append((f"{name}/L3", W.zstd_compress(sources[name], 3, True, True), name))
    a, b = W.zstd_compress(sources["text"], 3, True, True), W.zstd_compress(sources["svb16"], 1, False, False)
    skip = struct.pack("<II", 0x184D2A5E, 7) + b"skipped"
    sources["text+svb16"] = sources["text"] + sources["svb16"]
    entries.append(("two frames with a skippable frame", a + skip + b, "text+svb16"))
    for label, blob, name in entries:  # libzstd agrees
        assert W.zstd_decompress(blob, len(sources[name])) == sources[name], label
    blobs = [e[1] for e in entries]
    return dict(labels=np.array([e[0] for e in entries]), streams=np.frombuffer(b"".join(blobs), np.uint8),
                stream_offsets=np.cumsum([0] + [len(x) for x in blobs]).astype(np.int64),
                out_lengths=np.array([len(sources[e[2]]) for e in entries], np.int64),
                sha256=np.array([list(hashlib.sha256(sources[e[2]]).digest()) for e in entries], np.uint8))


def main():
    os.makedirs(GOLDEN, exist_ok=True)
    reads = W.synthetic_reads(8, seed=5, min_len=4000, max_len=16000)
    W.write_pod5(os.path.join(GOLDEN, "pod5_vbz.pod5"), reads, vbz=True, row_samples=8000, level=1)
    W.write_pod5(os.path.join(GOLDEN, "pod5_raw.pod5"), reads, vbz=False, row_samples=8000)
    np.savez_compressed(os.path.join(GOLDEN, "pod5_expected.npz"), read_ids=np.array([str(r["read_id"]) for r in reads]),
                        signals=np.concatenate([r["signal"] for r in reads]),
                        offsets=np.cumsum([0] + [len(r["signal"]) for r in reads]).astype(np.int64))
    np.savez_compressed(os.path.join(GOLDEN, "zstd_corpus.npz"), **corpus())


if __name__ == "__main__":
    main()
