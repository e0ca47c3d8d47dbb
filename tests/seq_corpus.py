"""Inputs in every shape kseq reads (FASTA, wrapped FASTQ, mixed, CRLF, lone '\\r' lines, blank lines, junk, empty sequences, ...) for
tests/test_seq_input_cpu.py and tests/test_zz_seq_input_gpu.py, and the parser of the record dumps of tests/host_emul/bseq_dump.cpp and
seq_emul.cpp."""
import numpy as np

IUPAC = b"ACGTACGTACGTacgtNnRYKMSWBDHVrykmswbdhv"


def _seq(rng, n, alphabet=b"ACGT"):
    return bytes(np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)])


def _qual(rng, n):
    return bytes(rng.integers(33, 75, n).astype(np.uint8))           # '!'..'J': includes '>' (62) and '@' (64)


def _wrap(s, width, eol=b"\n"):
    if width is None or not s:
        return s + eol
    widths = width if isinstance(width, list) else [width]
    out, i, k = [], 0, 0
    while i < len(s):
        w = widths[k % len(widths)]; k += 1
        out.append(s[i:i + w] + eol); i += w
    return b"".join(out)


def fasta(recs, width=None, eol=b"\n"):
    return b"".join(b">" + h + eol + _wrap(s, width, eol) for h, s, _ in recs)


def fastq(recs, width=None, eol=b"\n"):
    return b"".join(b"@" + h + eol + _wrap(s, width, eol) + b"+" + eol + _wrap(q, width, eol) for h, s, q in recs)


def records(rng, n, lo=1, hi=300, alphabet=b"ACGT", names=b"r", comments=True):
    out = []
    for i in range(n):
        L = int(rng.integers(lo, hi))
        h = names + b"%d" % i
        if comments and i % 3 == 1:
            h += b" c%d\tBX:Z:%d" % (i, i)
        elif comments and i % 3 == 2:
            h += b"\tcomment %d" % i
        out.append((h, _seq(rng, L, alphabet), _qual(rng, L)))
    return out


def _quals_start_with(rng, recs, width, chars=b"@>"):
    """qualities whose wrapped lines start with '@' or '>' (a quality line that looks like a header)"""
    out = []
    for k, (h, s, q) in enumerate(recs):
        q = bytearray(q)
        for i in range(0, len(q), width):
            q[i] = chars[(i // width + k) % len(chars)]
        out.append((h, s, bytes(q)))
    return out


# hand-written records for the corner cases of kseq's line and '\r' rules (each a valid record for kseq)
CORNERS = (
    b"@lone_cr\n\r\n+\n\r\n"                               # a sequence that is a lone '\r' keeps it (length 1)
    b"@crcr\nA\r\r\n+\nI\r\r\n"                            # "A\r\r" -> "A\r"
    b"@crcr_empty\nACG\n+\nI\r\r\n\nII\n"                  # qualities "I\r\r" -> "I\r", an empty line strips that '\r' too: "I" + "II"
    b"@mid_cr\nAC\r\nGT\n\r\n+\nII\nII\n"                  # a lone '\r' line inside a sequence is dropped
    b">fa_cr\r\nACGT\r\n\r\nAC\r\n"                        # FASTA with CRLF and a lone-'\r' line
    b"@blank\n\nACGT\n\nAC\n+\nIIIIII\n"                   # blank sequence lines are skipped
    b"@empty\n+\n\n"                                        # empty sequence: one (empty) quality line
    b">empty_fa\n"
    b">empty_fa2 with comment\n"
    b"@vt\x0bname c\nACGT\n+\nIIII\n"                      # '\v' ends the name
    b"@ff\x0cname\nACGT\n+\nIIII\n"                        # '\f' ends the name
    b"@cr_name\rtail\nACGT\n+\nIIII\n"                     # '\r' ends the name mid-line; the rest is the comment
    b"@sp_cr \r\nACGT\n+\nIIII\n"                          # comment "\r" (one byte: kept)
    b"@slash/1\nACGT\n+\nIIII\n@slash/2 x\nACGT\n+\nIIII\n@s/x\nA\n+\nI\n@/1\nA\n+\nI\n"
    b"@tab\tcomment\twith tabs\nACGT\n+\nIIII\n"
    b"@plus_rest\nACGT\n+plus line text\nIIII\n"
    b"@wrapq\nACGTACGT\n+\n@III\n>III\n"                    # quality lines that start with '@' and '>'
    b"junk line\nmore junk @mid\nACGT\n+\nIIII\n"           # junk between records: the header is the '@' inside the line
    b">fa_then_fq\nACGT\nAC\n@fq_after\nAC\n+\nII\n"
)


def corpus(seed=1):
    """name -> (bytes of file 1, bytes of file 2 or None)"""
    rng = np.random.default_rng(seed)
    c = {}
    r = records(rng, 300, 1, 400)
    c["fa_single"] = (fasta(r), None)
    c["fa_60"] = (fasta(r, 60), None)
    c["fa_80"] = (fasta(r, 80), None)
    c["fa_ragged"] = (fasta(r, [61, 17, 80, 1, 33]), None)
    c["fq_4line"] = (fastq(r), None)
    c["fq_wrapped_at"] = (fastq(_quals_start_with(rng, r, 60), 60), None)
    c["fq_wrapped_crlf"] = (fastq(_quals_start_with(rng, r, 50, b">@"), 50, b"\r\n"), None)
    mixed = []
    for k in range(0, 300, 30):
        part = r[k:k + 30]
        mixed.append([fasta(part), fastq(part, 70), fasta(part, 60, b"\r\n"), fastq(part), fastq(part, None, b"\r\n")][(k // 30) % 5])
    c["mixed"] = (b"".join(mixed), None)
    iu = records(rng, 120, 0, 200, IUPAC)
    c["iupac_lower_empty"] = (fasta(iu, 60) + fastq(iu, 45), None)
    c["corners"] = (CORNERS, None)
    c["junk_first_blank_end"] = (b"some junk\nno header here\n\n" + fastq(r[:50]) + b"\n\n", None)
    c["junk_mid_line"] = (b"xx" + b"".join(b"junk %d " % i + fastq([t]) for i, t in enumerate(r[:60])), None)
    c["no_final_newline"] = (fasta(r[:40], 60)[:-1], None)
    c["no_final_newline_fq"] = (fastq(r[:40])[:-1], None)
    c["header_at_eof"] = (fastq(r[:40]) + b"@", None)
    c["fa_header_at_eof"] = (fasta(r[:40], 60) + b">", None)
    # paired: the same records as /1 and /2
    p1 = [(h.split(b" ")[0].split(b"\t")[0] + b"/1" + h[len(h.split(b" ")[0].split(b"\t")[0]):], s, q) for h, s, q in r[:200]]
    p2 = [(h.split(b" ")[0].split(b"\t")[0] + b"/2", s[::-1], q[::-1]) for h, s, q in r[:200]]
    c["pe_fa_60"] = (fasta(p1, 60), fasta(p2, 60))
    c["pe_mixed"] = (fastq(p1, 60), fasta(p2, 80, b"\r\n"))
    inter = []
    for a, b in zip(p1, p2):
        inter += [a, b]
    c["interleaved_fa"] = (fasta(inter, 60), None)
    return c


MALFORMED = {
    "short_quality": (b"@a\nACGT\n+\nIIII\n@b\nACGT\n+\nII\n", 1),
    "long_quality": (b">x\nAC\n@a\nACGT\n+\nIIIIII\n", 1),
    "plus_at_eof": (b"@a\nACGT\n+\nIIII\n@b\nACGT\n+", 1),
    "empty_seq_with_quality": (b"@a\n+\nII\n", 0),
}


def parse_dump(out: bytes):
    """records of a dump: list of chunks, each a list of (name, comment or None, seq, qual or None); plus the "E" / "S" lines"""
    chunks, extra, i = [], {}, 0
    while i < len(out):
        j = out.index(b"\n", i)
        tag, rest = out[i:i + 1], out[i + 2:j]
        if tag in (b"C", b"R"):
            n = int(rest); i = j + 1; recs = []
            for _ in range(n):
                f = []
                for _k in range(4):
                    c = out.index(b":", i); ln = int(out[i:c])
                    f.append(None if ln < 0 else out[c + 1:c + 1 + ln]); i = c + 1 + max(ln, 0)
                assert out[i:i + 1] == b"\n"; i += 1
                recs.append(tuple(f))
            chunks.append(recs)
        else:
            extra[tag.decode()] = [int(x) for x in rest.split()]
            i = j + 1
    return chunks, extra


def nt4(seq: bytes) -> bytes:
    """nst_nt4_table as bm2_fastq_encode / bm2_seq_encode encode a base: A C G T (either case) 0-3, '-' 5, anything else 4"""
    a = np.frombuffer(seq, np.uint8)
    u = a & 0xDF
    out = np.full(len(a), 4, np.uint8)
    for k, ch in enumerate(b"ACGT"):
        out[u == ch] = k
    out[a == ord("-")] = 5
    return out.tobytes()


def digest(recs) -> str:
    """SHA-256 of records (name, comment or None, sequence as nt4 codes, qualities or None): what the encoders must reproduce"""
    import hashlib
    h = hashlib.sha256()
    for rec in recs:
        for f in rec:
            h.update(b"-1:" if f is None else b"%d:" % len(f) + f)
        h.update(b"\n")
    return h.hexdigest()


def encoded(recs):
    """records of a dump with the sequence as nt4 codes"""
    return [(n, c, nt4(s), q) for n, c, s, q in recs]
