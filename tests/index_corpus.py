"""Inputs for bm2_index's tests: small FASTA / FASTQ files whose .pac / .ann / .amb must equal `bwa-mem2 index`'s, and seeded genomes."""
from __future__ import annotations
import gzip
import numpy as np

IUPAC = b"RYKMSWBDHV"


def _wrap(seq: bytes, width: int, eol: bytes = b"\n") -> bytes:
    return b"".join(seq[i:i + width] + eol for i in range(0, len(seq), width)) if seq else b""


def _random_seq(rng, n: int, amb_rate: float = 0.0, lower_rate: float = 0.0) -> bytes:
    s = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].copy()
    if amb_rate:
        m = rng.random(n) < amb_rate
        s[m] = np.frombuffer(b"N" + IUPAC, np.uint8)[rng.integers(0, 11, int(m.sum()))]
    if lower_rate:
        m = rng.random(n) < lower_rate
        s[m] = s[m] | 0x20
    return s.tobytes()


def corpus() -> dict[str, bytes]:
    """name -> file bytes (names ending in .gz are gzip)."""
    rng = np.random.default_rng(7)
    c: dict[str, bytes] = {}
    seq = _random_seq(rng, 900)
    runs = seq[:100] + b"N" * 37 + seq[100:300] + b"NNNNnnnn" + seq[300:400] + b"NAN" + seq[400:500] + IUPAC + seq[500:600] + b"RRYY" + seq[600:]
    c["n_runs_iupac.fa"] = b">chr1 a comment here\n" + _wrap(runs, 60) + b">chr2\n" + _wrap(_random_seq(rng, 333, 0.05), 70)
    c["case.fa"] = b">lc\n" + _wrap(b"acgtNNnnacgtnNnNaaccGGTTnnNNrRyY" * 5, 50) + b">mixed\tx y\n" + _wrap(_random_seq(rng, 400, 0.1, 0.3), 61)
    c["n_only.fa"] = b">allN\n" + b"N" * 50 + b"\n>acgt\nACGTACGTA\n>alln2\nnnnnNNNN\n"
    c["edges.fa"] = (b">s1\nNNNACGTACGTNNN\n>s2\nNNNNGATTACANN\n>s3\nNACGTN\n>s4\nN\n>s5\nACGTTGCA\n>s6\nNNNN\n>s7\nNNACG\n")
    c["empty_records.fa"] = (b">empty1 has a comment\n>x/1 pair-like name\nACGTACGTAC\n>empty2\n\n>r/2\nGGGCCCAAT\n>last\n"
                             + b"ACGTN" * 7 + b"\n>trailing_empty\n")
    c["crlf.fa"] = b">c1 crlf comment\r\n" + _wrap(_random_seq(rng, 300, 0.05), 60, b"\r\n") + b">c2\r\nACGTNNNNAC\r\nGT\r\n"
    c["junk.fa"] = b"some junk line\nmore junk >not-a-header? no\n>j1\nACGTACGTTTGA\n>j2 c\nAACCGGTTNN\n"
    c["reads.fq"] = b"@q1 cm\nACGTNACGT\n+\nIIIIIIIII\n@q2\nGGGNNNCCC\n+q2\n#########\n@q3/1\nAC\n+\nII\n"
    c["mixed_fa_fq.fa"] = b">a\nACGTRYACGT\n@b\nACGNNA\n+\nIIIIII\n>c\nTTTT\n"
    for k in range(4):                                   # l_pac % 4 == 0, 1, 2, 3
        c[f"lpac_mod{k}.fa"] = b">m\n" + _wrap(_random_seq(rng, 96 + k, 0.03), 60) + b">n\nACGT\n"
    big = b"".join(b">ctg%d desc %d\n" % (i, i) + _wrap(_random_seq(rng, int(rng.integers(1, 3000)), 0.01, 0.1), 60) for i in range(12))
    c["multi_contig.fa"] = big
    c["plain_gz.fa.gz"] = gzip.compress(c["n_runs_iupac.fa"])
    c["multi_member.fa.gz"] = gzip.compress(c["case.fa"]) + gzip.compress(c["edges.fa"]) + gzip.compress(b">tail\nACGTNNAC\n")
    return c


def synthetic_fasta(n_bp: int, seed: int, n_contigs: int = 8, width: int = 60) -> bytes:
    """A random genome of n_bp bases in n_contigs contigs with planted N runs (1-5000 bases) and scattered IUPAC codes, wrapped at width."""
    rng = np.random.default_rng(seed)
    g = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n_bp)].copy()
    for _ in range(max(1, n_bp // 200000)):
        p = int(rng.integers(0, n_bp)); L = int(rng.integers(1, 5000))
        g[p:p + L] = ord("N")
    m = rng.random(n_bp) < 1e-4
    g[m] = np.frombuffer(IUPAC, np.uint8)[rng.integers(0, len(IUPAC), int(m.sum()))]
    cuts = np.sort(rng.choice(np.arange(1, n_bp), n_contigs - 1, replace=False))
    out = []
    for i, (a, b) in enumerate(zip(np.r_[0, cuts], np.r_[cuts, n_bp])):
        out.append(b">chr%d synthetic\n" % (i + 1) + fasta_lines(g[a:b], width))
    return b"".join(out)


def fasta_lines(seq: np.ndarray, width: int) -> bytes:
    """Bytes of seq (uint8) wrapped at width, built without a Python loop over lines."""
    n = len(seq)
    if n == 0:
        return b""
    full = n // width
    body = np.empty(full * (width + 1), np.uint8)
    v = body.reshape(full, width + 1) if full else body.reshape(0, width + 1)
    v[:, :width] = seq[:full * width].reshape(full, width)
    v[:, width] = 10
    tail = seq[full * width:]
    return body.tobytes() + (tail.tobytes() + b"\n" if len(tail) else b"")


def low_entropy_fasta(n_bp: int, seed: int) -> bytes:
    """A genome that forces many doubling rounds: long identical copies of a block, (AT)n and poly-A runs, and two identical contigs."""
    rng = np.random.default_rng(seed)
    unit = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 50000)]
    parts = []
    left = n_bp // 2
    while left > 0:
        k = int(rng.integers(0, 4))
        L = int(min(left, rng.integers(1000, 200000)))
        if k == 0:
            s = np.resize(unit, L)                       # copies of one 50 kbp block
        elif k == 1:
            s = np.resize(np.frombuffer(b"AT", np.uint8), L)
        elif k == 2:
            s = np.full(L, ord("A"), np.uint8)
        else:
            s = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, L)]
        parts.append(s); left -= L
    half = np.concatenate(parts)[:n_bp // 2]
    return b">dup1\n" + fasta_lines(half, 60) + b">dup2 same as dup1\n" + fasta_lines(half, 60) + b">tail\n" + fasta_lines(np.resize(np.frombuffer(b"AC", np.uint8), 777), 60)
