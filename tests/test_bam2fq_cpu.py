"""bm2_bam2fq on the CPU: the host emulation (tests/host_emul/bam2fq_emul.cpp, which runs bwa-mem2_b200/csrc/bam2fq.h unchanged) writes the
streams that the rule restated in Python (tests/bam2fq_util.py) gives, interleaved and split, plain and BGZF, on crafted records for each
branch of the rule and on random records, at every window size down to one record; the complement table is htslib's; read errors exit 1
and leave no file; the option errors exit 1 before anything is read."""
import gzip, os, subprocess
import numpy as np
import pytest
import bam2fq_util as bf
import bam_util as bu
import markdup_bam_util as mb

WINDOWS = (1, 200, 4096, 256 << 20)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return bf.build_emul(tmp_path_factory)


def _q(n, base=30):
    return [(base + 7 * i) % 42 for i in range(n)]


def crafted():
    r = bf.rec
    recs = []
    recs.append(r("iupac", 0x10, bf.LETTERS, _q(16)))                                 # 0x10 with every code: other
    recs.append(r("iupac_fwd", 0, bf.LETTERS, _q(16)))
    recs.append(r("fa1", 0x41, "ACGTN", None))                                         # QUAL '*': FASTA, a pair of them
    recs.append(r("x" * 254, 0x41 | 0x10, "ACGTTGCA" * 9, _q(72)))                     # the longest QNAME, mate far below
    recs.append(r("both", 0x1 | 0x40 | 0x80, "ACG", _q(3)))                            # both end bits: other
    recs.append(r("neither", 0x1, "GGA", [93, 0, 40]))                                 # neither, with 0x1: other; 93 is allowed
    recs.append(r("sec", 0x141, "AAAA", _q(4)))                                        # 0x100 and 0x800: skipped
    recs.append(r("sup", 0x881, "CCCC", _q(4)))
    recs.append(r("qcdup", 0x1 | 0x80 | 0x200 | 0x400, "TTTT", _q(4)))                 # QC-fail and duplicate READ2: kept, mate below
    recs.append(r("fa1", 0x81 | 0x10, "ACGTNR", None))
    recs.append(r("lonely", 0x41, "ACGT", _q(4)))                                      # a mate that never comes
    recs.append(r("sec2", 0x100, "", None))                                            # a skipped record without bases is fine
    for k in range(30):                                                                # filler, so that the far mates lie windows apart
        recs.append(r("f%d" % (k // 2), 0x81 if k % 2 else 0x41, "ACGT" * (k + 1), _q(4 * k + 4)))
    recs.append(r("qcdup", 0x41 | 0x200, "GATT", _q(4)))
    recs.append(r("x" * 254, 0x81, "TTTT", _q(4)))
    recs.append(r("lonely2", 0x81 | 0x10, "ACGTAC", _q(6)))
    return recs


def random_records(rng, n):
    r = bf.rec
    recs, open_ = [], []
    for i in range(n):
        u = rng.random()
        seq = "".join(rng.choice(list("ACGTN"), int(rng.integers(1, 160))))
        q = None if rng.random() < 0.05 else [int(x) for x in rng.integers(0, 42, len(seq))]
        rev = 0x10 if rng.random() < 0.5 else 0
        if u < 0.1:
            recs.append(r("o%d" % i, rev | (0xC1 if rng.random() < 0.5 else 0), seq, q))
        elif u < 0.15:
            recs.append(r("s%d" % i, rev | 0x41 | (0x100 if rng.random() < 0.5 else 0x800), seq, q))
        elif open_ and rng.random() < 0.5:
            name, fl = open_.pop(int(rng.integers(0, len(open_))))
            recs.append(r(name, rev | (0x81 if fl & 0x40 else 0x41), seq, q))
        else:
            name = "p%d" % i
            fl = 0x41 if rng.random() < 0.5 else 0x81
            open_.append((name, fl))
            recs.append(r(name, rev | fl, seq, q))
    return recs


def _write(d, recs, stem="in"):
    h, refs = mb.header(so="unsorted")
    p = str(d / (stem + ".bam"))
    mb.write_bam(p, h, refs, recs, 97)
    return p


def _check_all(emul, d, recs, tag, windows=WINDOWS):
    p = _write(d, recs, tag)
    for split in (False, True):
        for opt in ([True, True], [False, False], [True, False]):
            if not split and opt != [True, True]:
                continue
            want, wst = bf.convert(recs, split=split, other=opt[0], single=opt[1])
            for gz in (False, True):
                ext = ".fq.gz" if gz else ".fq"
                names = ["main"] if not split else ["1", "2", "0", "s"]
                base = None
                for w in windows:
                    paths = [str(d / ("%s_%s_%d%s" % (tag, n, w, ext))) if (n in want) else "" for n in names]
                    rc, msg, st = bf.emul_run(emul, p, paths, split=split, window=w, threads=1 + w % 3)
                    assert rc == 0, msg
                    for n, path in zip(names, paths):
                        if not path:
                            continue
                        raw = open(path, "rb").read()
                        got = gzip.decompress(raw) if gz else raw
                        assert got == want[n], (tag, split, opt, gz, w, n)
                        if gz:
                            sizes = [len(x) for _, x in bu.members(raw)]
                            assert raw.endswith(bu.EOF_BLOCK) and all(s == 65280 for s in sizes[:-2]), sizes[-3:]
                        if base is not None:
                            assert raw == base[n]
                    for k in ("records", "kept", "pairs", "others", "singletons", "others_dropped", "singletons_dropped"):
                        assert st[k] == wst[k], k
                    if w == 1:
                        bounds = list(range(len(recs) + 1))
                        assert st["pending_max"] == bf.window_pending_max(recs, bounds)
                    if (st["others_dropped"] or st["singletons_dropped"]):
                        assert "were not written" in msg
                    base = base or {n: open(path, "rb").read() for n, path in zip(names, paths) if path}
                    assert not [f for f in os.listdir(d) if f.endswith(".tmp")]


def test_complement_is_htslib_seq_comp_table(emul):
    recs = [bf.rec("c%d" % c, 0x10, bf.LETTERS[c], [30]) for c in range(16)]
    for c, r in enumerate(recs):
        assert bf.text(r, False).split(b"\n")[1] == bf.LETTERS[bf.SEQ_COMP_TABLE[c]].encode()
        assert bf.emul_text(emul, recs, [c], [], False) == bf.text(r, False)
    assert bf.SEQ_COMP_TABLE == [int("{:04b}".format(c)[::-1], 2) for c in range(16)]


def test_crafted_records_equal_python(emul, tmp_path):
    recs = crafted()
    out, st = bf.convert(recs)
    text = out["main"]
    assert b"@iupac\n" + bf.LETTERS[::-1].encode().translate(bytes.maketrans(b"ACMGRSVTWYHKDBN", b"TGKCYSBAWRDMHVN")) + b"\n" in text
    assert b">fa1/1\nACGTN\n>fa1/2\nYNACGT\n" in text and b"@neither\nGGA\n+\n~!I\n" in text
    assert b"sec" not in text and b"sup" not in text and st["pairs"] == 3 + 15 and st["singletons"] == 2
    assert text.endswith(b"@lonely/1\nACGT\n+\n" + bytes(x + 33 for x in _q(4)) + b"\n" + b"@lonely2/2\nGTACGT\n+\n" + bytes(x + 33 for x in _q(6)[::-1]) + b"\n")
    got, err = bf.emul_records(emul, recs, True)
    assert err == -1 and [int(x) for x in got["kind"]] == [bf.kind(bf.fields(r)[1]) for r in recs]
    assert [int(x) for x in got["text_len"]] == [len(bf.text(r, True)) if bf.kind(bf.fields(r)[1]) else 0 for r in recs]
    _check_all(emul, tmp_path, recs, "c")


def test_random_records_equal_python(emul, tmp_path):
    rng = np.random.default_rng(301)
    recs = random_records(rng, 2500)
    out, st = bf.convert(recs)
    assert len(out["main"]) > 3 * 65280 and st["singletons"] > 10 and st["others"] > 100
    _check_all(emul, tmp_path, recs, "r", windows=(1, 5000, 256 << 20))


def _errors():
    r = bf.rec
    ok = [r("a", 0x41, "ACGT", _q(4)), r("a", 0x81, "ACGT", _q(4))]
    yield "two READ1", ok[:1] + [r("b", 0, "A", [3])] * 3 + [r("a", 0x41, "AC", _q(2))], "read a: two READ1", ""
    yield "two READ2", [r("z", 0x81, "A", [3]), r("z", 0x81 | 0x10, "A", [3])], "read z: two READ2", ""
    yield "empty", ok + [r("e", 0, "", None)], "read e (record ", "of the window) has no bases (l_seq 0)"
    yield "quality", ok + [r("q", 0x41, "AC", [30, 94])], "read q (record ", "of the window) has a quality above 93"


@pytest.mark.parametrize("case", [c[0] for c in _errors()])
def test_errors_exit_1_and_leave_no_file(emul, tmp_path, case):
    _, recs, t1, t2 = next(c for c in _errors() if c[0] == case)
    p = _write(tmp_path, recs)
    with pytest.raises(bf.Bam2fqError):
        bf.convert(recs)
    for w in (1, 256 << 20):
        for paths, split in (([str(tmp_path / "o.fq.gz")], False), ([str(tmp_path / "1.fq"), str(tmp_path / "2.fq"), str(tmp_path / "0.fq"), ""], True)):
            rc, msg, _ = bf.emul_run(emul, p, paths, split=split, window=w)
            assert rc == 1 and t1 in msg and t2 in msg, msg
            assert sorted(os.listdir(tmp_path)) == ["in.bam"]


def test_option_errors(tmp_path):
    if not os.path.exists(bf.TOOL):
        pytest.skip("bm2_bam2fq not built")
    missing = str(tmp_path / "no_such.bam")                                            # never opened: the options fail first
    o1, o2 = str(tmp_path / "1.fq"), str(tmp_path / "2.fq")
    for argv, text in [(["-1", o1, missing], "-1 and -2 must be given together"), (["-2", o2, missing], "-1 and -2 must be given together"),
                       (["-s", o1, missing], "-s needs split output"), (["-0", o1, "-o", o2, missing], "-0 needs split output"),
                       (["-1", o1, "-2", o2, "-o", str(tmp_path / "i.fq"), missing], "-o cannot be given with -1 and -2"),
                       (["-n", "-N", missing], "-n and -N cannot both be given"), (["--window", "0", missing], "--window"),
                       (["-t", "0", missing], "-t takes"), ([], "no input"), (["-x", missing], "unknown option"), (["a.bam", "b.bam"], "more than one input")]:
        r = subprocess.run([bf.TOOL] + argv, capture_output=True, timeout=60)
        assert r.returncode == 1 and text in r.stderr.decode(), (argv, r.stderr)
    assert os.listdir(tmp_path) == []
