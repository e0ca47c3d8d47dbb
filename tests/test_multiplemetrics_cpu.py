"""bm2_multiplemetrics without a GPU: the host emulation (tests/host_emul/multiplemetrics_emul.cpp: mm.cu's check and count kernels over
mm_device.cuh's rule, mm_metrics.h's reference reader, formulas and text) writes byte for byte the two files that Picard's per-record loops
restated in Python (tests/multiplemetrics_util.py) give, on crafted records for each branch of the rule, on 2 000 random pairs in any order
cut into windows of every size down to one record, and over files; every read, reference and header error is named; the tool rejects
every bad option."""
import os, subprocess
import numpy as np
import pytest
import multiplemetrics_util as mu

M, I, D, N, S, H, EQ, X = 0, 1, 2, 3, 4, 5, 7, 8
REF = mu.Ref([("c1", 3000), ("c2", 2000), ("c3", 500)], holes=[(100, 20, "N"), (300, 10, "n"), (400, 5, "R"), (3100, 8, "."), (3200, 4, "Y")])
P1, P2 = 0x1 | 0x40, 0x1 | 0x80
AD = mu.ADAPTERS[3][:16]                     # PAIRED_END 3'


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return mu.build_emul(tmp_path_factory)


def pair(name, pos1, pos2, tlen, s1=0, s2=0x10, rid=0, mrid=None, extra=0, len1=50, len2=50, mapq=60):
    """A mapped pair: the first read at pos1 and the second at pos2 (strands s1, s2), TLEN as given on the first read (negated on the second)."""
    mrid = rid if mrid is None else mrid
    f1 = P1 | extra | s1 | (0x20 if s2 else 0)
    f2 = P2 | extra | s2 | (0x20 if s1 else 0)
    return [mu.rec(name, f1, rid, pos1, [(len1, M)], mapq=mapq, mrid=mrid, mpos=pos2, tlen=tlen),
            mu.rec(name, f2, mrid, pos2, [(len2, M)], mapq=mapq, mrid=rid, mpos=pos1, tlen=-tlen)]


def crafted():
    """Records for each branch of the rule, in no particular order."""
    r = []
    r += pair("fr", 500, 700, 250, extra=0x2) + pair("fr2", 600, 800, 251, extra=0x2) + pair("dup", 500, 700, 250, extra=0x2 | 0x400)
    r += [mu.rec("sec", 0x100 | P1, 0, 500, [(50, M)]), mu.rec("supp", 0x800 | P1, 0, 520, [(50, M)], tags=mu.tag_z("SA", "c1,1,+,5M,60,0;"))]
    r += pair("qcfail", 900, 1000, 150, extra=0x200)
    r += [mu.rec("noise", 0, 0, 1000, [(30, M)], tags=mu.tag_i("XN", 1)), mu.rec("noise_c", 0, 0, 1000, [(30, M)], tags=mu.tag_i("XN", 1, "C")),
          mu.rec("noise2", 0, 0, 1000, [(30, M)], tags=mu.tag_i("XN", 2)), mu.rec("noise_z", 0, 0, 1000, [(30, M)], tags=mu.tag_z("XN", "1")),
          mu.rec("noise_qc", 0x200, 0, 1000, [(30, M)], tags=mu.tag_i("XN", 1))]
    # adapters: exact, 1 and 2 mismatches, N, reverse complement, shorter than 16, non-PF, mapped
    un = lambda name, seq, flag=0x4: mu.rec(name, flag, -1, -1, [], seq=seq)
    r += [un("ad0", AD + "ACGT"), un("ad1", "T" + AD[1:] + "AC"), un("ad2", "TT" + AD[2:] + "AC"), un("adN", "NN" + AD[2:]),
          un("adN1", "NT" + AD[2:]), un("adrc", mu.revcomp(AD) + "G"), un("adshort", AD[:15]), un("adqc", AD, 0x4 | 0x200),
          un("adrev", AD + "A", 0x4 | 0x10), mu.rec("admapped", 0, 0, 1100, [(16, M)], seq=AD)]
    # mismatches at an N hole, an n hole, an IUPAC hole, with read N, and exact matches
    r += [mu.rec("holeN", 0, 0, 95, [(30, M)], seq="A" * 10 + "N" * 10 + "C" * 10), mu.rec("holen", 0, 0, 295, [(20, M)]),
          mu.rec("holeR", 0, 0, 398, [(10, M)], seq="AARRRRRAAA"), mu.rec("c2Y", 0, 1, 198, [(10, M)], seq="ACYYYYACGT"),
          mu.rec("exact", 0, 0, 1500, [(40, EQ)], seq=mu.ref_seq(REF, 0, 1500, 40)), mu.rec("exactX", 0, 1, 50, [(40, X)], seq=mu.ref_seq(REF, 1, 50, 40)),
          mu.rec("readN", 0x10, 0, 1600, [(20, M)], seq=mu.ref_seq(REF, 0, 1600, 10) + "NNNNN" + mu.ref_seq(REF, 0, 1615, 5))]
    # QUAL '*', qualities at the threshold, low MAPQ
    r += [mu.rec("noqual", 0, 0, 1700, [(30, M)], None), mu.rec("atq", 0, 0, 1750, [(20, M)], [19, 20] * 10),
          mu.rec("mapq19", 0, 0, 1800, [(30, M)], mapq=19), mu.rec("mapq20", 0, 0, 1800, [(30, M)], mapq=20)]
    # clips and indels on each strand
    r += [mu.rec("sc_f", 0, 0, 1900, [(5, S), (40, M), (7, S)]), mu.rec("sc_r", 0x10, 0, 1900, [(5, S), (40, M), (7, S)]),
          mu.rec("hc_f", 0, 0, 1950, [(3, H), (5, S), (40, M), (6, S), (4, H)]), mu.rec("hc_r", 0x10, 0, 1950, [(3, H), (5, S), (40, M), (4, H)]),
          mu.rec("indel", 0, 0, 2000, [(20, M), (2, I), (20, M), (3, D), (10, M), (30, N), (5, M)])]
    # chimeras: other contig, |TLEN| 100000 against 100001, RF, tandem, SA on a single-end read; a mate unmapped; improper pairs
    r += pair("chim_contig", 2100, 50, 0, mrid=1) + pair("tl100000", 2200, 2300, 100000) + pair("tl100001", 2200, 2300, 100001)
    r += pair("rf", 2300, 2400, 150, s1=0x10, s2=0) + pair("rf2", 2310, 2400, 140, s1=0x10, s2=0) + pair("tandem", 2400, 2500, 150, s1=0x10, s2=0x10)
    r += [mu.rec("sa", 0, 0, 2600, [(30, M)], tags=mu.tag_z("SA", "c2,5,+,30M,60,0;")), mu.rec("nosa", 0, 0, 2600, [(30, M)]),
          mu.rec("mate_unmapped", P1 | 0x8, 0, 2700, [(30, M)], tags=mu.tag_z("SA", "c2,5,+,30M,60,0;")),
          mu.rec("mate_unmapped", P2 | 0x4, 0, 2700, [], seq="A" * 30)]
    # inserts above 2^20, a median that ends in .5, a second read without TLEN
    r += pair("big", 100, 300, (1 << 20) + 3) + pair("big2", 100, 300, 1 << 20) + pair("big3", 100, 300, (1 << 20) - 1)
    r += pair("m100", 200, 300, 100) + pair("m101", 200, 300, 101) + pair("t0", 200, 300, 0)
    # no-calls: cycle 3 of unpaired reads in 4 of 5 forward reads, reversed for a reverse read
    r += [mu.rec("nc%d" % k, 0, 1, 1000 + k, [(8, M)], seq="ACGNACGT" if k < 3 else "ACGTACGT") for k in range(5)]
    r += [mu.rec("nc_rev", 0x10, 1, 1100, [(8, M)], seq="ACGTNCGT")]
    return r


def _cmp(emul, recs, sizes_list=([10 ** 9], [1], [2, 3], [7])):
    want = mu.files(recs, REF, "a b")
    for sizes in sizes_list:
        got = mu.emul_run(emul, REF, mu.windows(recs, sizes), "a b")
        assert got[4] is None, got[4]
        assert (got[0], got[1]) == want, sizes
    return want


def _rows(text):
    lines = text.split("\n")
    cols = lines[4].split("\t")
    out = []
    for l in lines[5:]:
        if not l:
            break
        out.append(dict(zip(cols, l.split("\t"))))
    return out


def test_crafted_equals_python(emul):
    recs = crafted()
    summ, ins = _cmp(emul, recs)
    rows = {r["CATEGORY"]: r for r in _rows(summ)}
    assert list(rows) == ["FIRST_OF_PAIR", "SECOND_OF_PAIR", "PAIR", "UNPAIRED"]
    u = rows["UNPAIRED"]
    assert int(u["PF_NOISE_READS"]) == 2 and u["SAMPLE"] == u["READ_GROUP"] == ""
    assert float(u["PCT_ADAPTER"]) > 0 and float(u["PCT_CHIMERAS"]) > 0 and float(u["PCT_SOFTCLIP"]) > 0 and float(u["PCT_HARDCLIP"]) > 0
    assert float(rows["PAIR"]["PCT_CHIMERAS"]) > 0 and int(rows["PAIR"]["TOTAL_READS"]) == int(rows["FIRST_OF_PAIR"]["TOTAL_READS"]) + \
        int(rows["SECOND_OF_PAIR"]["TOTAL_READS"])
    ir = _rows(ins)
    assert [r["PAIR_ORIENTATION"] for r in ir] == ["FR", "RF", "TANDEM"]
    assert "\n## HISTOGRAM\tjava.lang.Integer\ninsert_size\tAll_Reads.fr_count\tAll_Reads.rf_count\tAll_Reads.tandem_count\n" in ins


def test_each_rule():
    """The Python rule itself, branch by branch."""
    def one(recs):
        cats, ins, err = mu.metrics(recs, REF)
        assert err is None
        return cats, ins
    un = lambda seq: mu.rec("u", 0x4, -1, -1, [], seq=seq)
    assert [one([un(s)])[0]["UNPAIRED"]["adapter"] for s in (AD, "T" + AD[1:], "TT" + AD[2:], "NN" + AD[2:], "NT" + AD[2:], AD[:15],
                                                             mu.revcomp(AD))] == [1, 1, 0, 1, 1, 0, 1]
    seq = "A" * 10 + "N" * 10 + "C" * 10                                        # loci 100..119 are an N hole: read N matches there
    c = one([mu.rec("h", 0, 0, 95, [(30, M)], seq=seq)])[0]["UNPAIRED"]
    assert c["mism"] == sum(seq[k] != REF.letter(95 + k) for k in range(30)) and REF.letter(100) == "N"
    assert one([mu.rec("h", 0, 0, 95, [(30, M)], seq="A" * 30)])[0]["UNPAIRED"]["mism"] >= 20
    c = one([mu.rec("r", 0, 0, 400, [(5, M)], seq="RRRRA")])[0]["UNPAIRED"]
    assert c["mism"] == 1 and c["nocall"] == {}
    c = one([mu.rec("q", 0, 0, 1700, [(30, M)], None)])[0]["UNPAIRED"]
    assert c["hq_bases"] == 30 and c["q20"] == 0
    c = one([mu.rec("s", 0x10, 0, 1950, [(3, H), (5, S), (40, M), (4, H)]), mu.rec("s", 0, 0, 1950, [(40, M), (6, S), (4, H)])])[0]["UNPAIRED"]
    assert (c["sc3_sum"], c["sc3_reads"], c["hard"], c["soft"]) == (11, 2, 11, 11)
    for p, chim in ((pair("a", 2200, 2300, 100000), 0), (pair("a", 2200, 2300, 100001), 2), (pair("a", 2300, 2400, 150, s1=0x10, s2=0), 2),
                    (pair("a", 2400, 2500, 150, s1=0x10, s2=0x10), 2), (pair("a", 2100, 50, 0, mrid=1), 2)):
        assert one(p)[0]["FIRST_OF_PAIR"]["chim"] + one(p)[0]["SECOND_OF_PAIR"]["chim"] == chim
    fr = [x for k in range(19) for x in pair("f%d" % k, 100, 300, 250)]
    rf = pair("r", 300, 400, 150, s1=0x10, s2=0)
    assert mu.insert_text(one(fr + rf)[1], "").count("\tRF\t") == 1                          # 1 of 20: 5 %
    assert mu.insert_text(one(fr + pair("f", 100, 300, 250) + rf)[1], "").count("\tRF\t") == 0  # 1 of 21
    assert _rows(mu.insert_text(one(pair("a", 1, 2, 100) + pair("b", 1, 2, 101))[1], ""))[0]["MEDIAN_INSERT_SIZE"] == "100.5"


def test_bad_cycle_at_80_percent(emul):
    # cycle 3 holds an N in 4 of 5 reads (the reverse read's stored base 4 is its cycle 3), then in 3 of 5
    for n_bad, want in ((4, "1"), (3, "0")):
        recs = [mu.rec("nc%d" % k, 0, 1, 1000 + k, [(8, M)], seq="ACGNACGT" if k < n_bad - 1 else "ACGTACGT") for k in range(4)]
        recs += [mu.rec("nc_rev", 0x10, 1, 1100, [(8, M)], seq="ACGTNCGT")]
        summ, _ = _cmp(emul, recs, ([10 ** 9], [1]))
        assert _rows(summ)[0]["BAD_CYCLES"] == want


@pytest.mark.parametrize("which", ["single", "pairs", "empty"])
def test_shapes(emul, which):
    recs = crafted()
    if which == "single":
        recs = [r for r in recs if not mu.bu.fields(r)["flag"] & 1]
    elif which == "pairs":
        recs = [r for r in recs if mu.bu.fields(r)["flag"] & 1]
    else:
        recs = []
    summ, ins = _cmp(emul, recs, ([10 ** 9], [3]) if recs else ([1],))
    cats = [r["CATEGORY"] for r in _rows(summ)]
    assert cats == {"single": ["UNPAIRED"], "pairs": ["FIRST_OF_PAIR", "SECOND_OF_PAIR", "PAIR"], "empty": ["UNPAIRED"]}[which]
    assert ("## HISTOGRAM" in ins) == (which == "pairs") and _rows(ins) == ([] if which != "pairs" else _rows(ins))


def test_random_pairs_every_window(emul):
    rng = np.random.default_rng(101)
    recs = mu.random_records(REF, rng, 2000)
    want = mu.files(recs, REF, "x")
    rows = {r["CATEGORY"]: r for r in _rows(want[0])}
    assert len(rows) == 4 and all(float(rows[c]["PF_MISMATCH_RATE"]) > 0 for c in rows)
    assert len(_rows(want[1])) >= 2
    for sizes in ([len(recs)], [1], [2], [17], [1000], [3, 1, 250]):
        got = mu.emul_run(emul, REF, mu.windows(recs, sizes), "x")
        assert got[4] is None and (got[0], got[1]) == want, sizes


def test_read_errors(emul):
    ok = mu.rec("ok", 0, 0, 100, [(10, M)])
    cases = [(mu.rec("lseq0", 0, 0, 200, [(10, D)], [], seq=""), "read lseq0 (record 1) has l_seq 0 or above 1048576"),
             (mu.rec("lseq0u", 0x4, -1, -1, [], [], seq=""), "read lseq0u (record 1) has l_seq 0"),
             (mu.rec("past", 0, 0, 2995, [(10, M)]), "read past (record 1) does not lie inside a contig"),
             (mu.rec("badrid", 0, 3, 5, [(10, M)]), "read badrid (record 1) does not lie inside a contig"),
             (mu.rec("badcig", 0, 0, 200, [(10, M), (2, I)], seq="A" * 10), "read badcig (record 1) has a CIGAR that does not match")]
    for bad, msg in cases:
        recs = [ok, bad, ok]
        assert mu.metrics(recs, REF)[2][0] == 1
        got = mu.emul_run(emul, REF, [recs])
        assert got[4] is not None and msg in got[4], (msg, got[4])
    long = mu.rec("long", 0x4, -1, -1, [], 30, seq="A" * ((1 << 20) + 1))
    assert "read long (record 0) has l_seq 0 or above 1048576" in mu.emul_run(emul, REF, [[long]])[4]
    # records that are not counted, or not aligned, are not checked against the reference
    for r in (mu.rec("s", 0x100, 0, 2995, [(10, M)]), mu.rec("q", 0x200, 0, 2995, [(10, M)]), mu.rec("u", 0x4, 0, 2995, [(10, M)]),
              mu.rec("lseq0s", 0x800, 0, 200, [(10, D)], [], seq="")):
        assert mu.metrics([r], REF)[2] is None and mu.emul_run(emul, REF, [[r]])[4] is None


def test_tool_emulation_over_files(emul, tmp_path):
    rng = np.random.default_rng(102)
    pre = str(tmp_path / "ref.fa")
    REF.write(pre)
    back = mu.Ref.read(pre)
    assert back.holes == REF.holes and np.array_equal(back.codes, REF.codes)
    recs = mu.random_records(REF, rng, 600)
    (tmp_path / "in.bam").write_bytes(mu.bam_bytes(REF, recs))
    want = mu.files(recs, REF, "x")
    for window in (1, 4096, 1 << 30):
        a, b, st = mu.emul_tool(emul, pre, str(tmp_path / "in.bam"), window=window, args="x")
        assert (a, b) == want and st["records"] == len(recs)
    bad = {"names.bam": (mu.bam_bytes(REF, recs, refs=[("c1", 3000), ("cX", 2000), ("c3", 500)]), "reference 1 is cX of length 2000 in the header"),
           "count.bam": (mu.bam_bytes(REF, recs, refs=[("c1", 3000), ("c2", 2000)]), "the header has 2 references, the index 3 contigs")}
    for name, (data, msg) in bad.items():
        (tmp_path / name).write_bytes(data)
        with pytest.raises(ValueError) as e:
            mu.emul_tool(emul, pre, str(tmp_path / name))
        assert msg in str(e.value), (name, str(e.value))
    # the reference files
    pac = open(pre + ".pac", "rb").read()
    for cut, msg in ((pac[:-1], "ref.fa.pac: its size does not fit the 5500 bases"), (pac + b"\0", "its size does not fit"),
                     (pac[:-1] + b"\3", "its size does not fit"), (None, "cannot open " + pre + ".pac")):
        if cut is None:
            os.unlink(pre + ".pac")
        else:
            open(pre + ".pac", "wb").write(cut)
        with pytest.raises(ValueError, match=msg):
            mu.emul_tool(emul, pre, str(tmp_path / "in.bam"))
    REF.write(pre)
    amb = open(pre + ".amb").read().split("\n")
    open(pre + ".amb", "w").write("\n".join([amb[0], amb[2], amb[1]] + amb[3:]))
    with pytest.raises(ValueError, match="the holes are not sorted"):
        mu.emul_tool(emul, pre, str(tmp_path / "in.bam"))
    with pytest.raises(ValueError, match="cannot open .*nothere.ann"):
        mu.emul_tool(emul, str(tmp_path / "nothere"), str(tmp_path / "in.bam"))


def _run(args):
    return subprocess.run([mu.TOOL] + args, capture_output=True, timeout=120)


@pytest.mark.skipif(not os.path.exists(mu.TOOL), reason="bm2_multiplemetrics not built")
def test_option_errors(tmp_path):
    pre = str(tmp_path / "ref.fa")
    REF.write(pre)
    (tmp_path / "u.bam").write_bytes(mu.bam_bytes(REF, [], refs=[("c1", 3000)]))
    bam, o = str(tmp_path / "u.bam"), str(tmp_path / "o")
    for args, msg in (([], "no index prefix"), ([pre], "no input BAM"), ([pre, bam], "no output prefix (-o)"), (["-o", o, pre, bam, "x"], "more than one input"),
                      (["-t", "0", "-o", o, pre, bam], "-t takes a whole number from 1 to 1024"), (["--window", "12Q", "-o", o, pre, bam], "--window takes a size"),
                      (["--window", "0", "-o", o, pre, bam], "--window takes a size"), (["--bogus", pre, bam], "unknown option --bogus"),
                      (["-o"], "-o takes a value"), (["-o", o, str(tmp_path / "none"), bam], "cannot open"),
                      (["-o", o, pre, str(tmp_path / "none.bam")], "cannot open"),
                      (["-o", o, pre, bam], "the header has 1 references, the index 3 contigs")):
        r = _run(args)
        assert r.returncode == 1 and msg in r.stderr.decode(), (args, r.stderr)
    assert sorted(os.listdir(tmp_path)) == ["ref.fa.amb", "ref.fa.ann", "ref.fa.pac", "u.bam"]
