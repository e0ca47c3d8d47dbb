"""bm2_sort without a GPU: bam_qname_cmp (bwa-mem2_b200/csrc/bam_sort_device.cuh, compiled for the host) equals the literal Python port of
samtools' strnum_cmp on crafted and random names, and the comparison is antisymmetric, transitive and equal only on identical names; the sink
of bam_sort.h driven by the host emulation (tests/host_emul/bamsort_emul.cpp) writes Python's order of the records in both orders, at run
sizes from one record up, with many runs and merge windows, with the same bytes at every run size and no temporary file left; equal names
come out by flag & 0xc0 and then input order; the shared @HD rewrite keeps bm2_mem's output; and the option errors exit 1 and leave no file."""
import itertools, json, os, subprocess
import numpy as np
import pytest
import bam_util as bu
import bam_sort_util as bs
import bamsort_util as su
import markdup_bam_util as mb

MEM = os.path.join(su.ROOT, "bwa-mem2_b200", "bm2_mem")
IDX = os.path.join(su.ROOT, "tests", "golden", "c0_index", "ref.fa")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return su.build_emul(tmp_path_factory)


CRAFTED = [
    b"a", b"b", b"A", b"a1", b"aa", b"a:", b"1", b"9", b"10", b"a9", b"a10", b"a09", b"a009", b"a0010",         # digits against letters
    b"r007", b"r7", b"r0007x", b"r7x", b"r07y", b"x0", b"x00", b"x000", b"x0a", b"x00a", b"0", b"00", b"000",      # leading zeros, all-zero runs
    b"n" + b"9" * 25, b"n" + b"1" + b"0" * 24, b"n" + b"9" * 24, b"n" + b"0" * 3 + b"9" * 25, b"n" + b"9" * 25 + b"a",   # runs of more than 20 digits
    b"n12345678901234567890123", b"n12345678901234567890124", b"n012345678901234567890123",
    b"read", b"read1", b"read12", b"read12/1", b"read12/2", b"rea",                                           # prefixes
    bytes([0x80]), bytes([0xff]), b"a" + bytes([0xc3, 0xa9]), b"a" + bytes([0x7f]), b"a" + bytes([0x80]) + b"1",  # bytes >= 0x80
    b"x" * 254, b"x" * 253 + b"y", b"x" * 253, b"7" * 254, b"7" * 253 + b"8", b"0" * 254,                    # 254-byte names
    b"A00123:45:HXXX:1:1101:1234:5678", b"A00123:45:HXXX:1:1101:1234:05678", b"A00123:45:HXXX:1:1101:12340:5678",  # Illumina style
    b"A00123:45:HXXX:1:1101:999:5678", b"A00123:45:HXXX:1:2101:1234:5678", b"A00123:45:HXXX:2:1101:1234:5678",
    b"A00123:45:HXXY:1:1101:1234:5678", b"A0123:45:HXXX:1:1101:1234:5678",
]


def illumina_name(rng):
    inst = "A%05d" % rng.integers(0, 200) if rng.random() < 0.7 else "A%d" % rng.integers(0, 200)
    return ("%s:%d:H%s:%d:%d:%d:%d" % (inst, rng.integers(0, 60), "".join(rng.choice(list("XYZ0"), 3)), rng.integers(1, 5),
                                       int(rng.choice([1101, 1102, 2101, 2210])), rng.integers(0, 40000), rng.integers(0, 40000))).encode()


def small_name(rng):
    return bytes(rng.choice(list(b"a0:1"), int(rng.integers(0, 9))).tolist())


def _check_equal(emul, names, pairs):
    got = su.emul_cmp(emul, names, pairs)
    want = [su.sign(su.strnum_cmp(names[i], names[j])) for i, j in pairs]
    assert got == want


def test_crafted_names_equal_python(emul):
    n = len(CRAFTED)
    _check_equal(emul, CRAFTED, [(i, j) for i in range(n) for j in range(n)])
    c = lambda a, b: su.sign(su.strnum_cmp(a, b))
    assert c(b"a9", b"a10") < 0 and c(b"a09", b"a9") < 0 and c(b"r7", b"r007") > 0 and c(b"x00", b"x0") < 0
    assert c(b"n" + b"9" * 24, b"n" + b"1" + b"0" * 24) < 0 and c(b"n" + b"0" * 3 + b"9" * 25, b"n" + b"9" * 25) < 0
    assert c(b"read1", b"read12") < 0 and c(b"rea", b"read") < 0 and c(b"a", b"A") > 0 and c(bytes([0xff]), b"z") > 0
    assert c(b"A00123:45:HXXX:1:1101:999:5678", b"A00123:45:HXXX:1:1101:1234:5678") < 0


@pytest.mark.parametrize("grammar", ["illumina", "small"])
def test_random_names_equal_python(emul, grammar):
    rng = np.random.default_rng(11 if grammar == "illumina" else 12)
    make = illumina_name if grammar == "illumina" else small_name
    names = [make(rng) for _ in range(3000)]
    names += [n[:int(rng.integers(0, len(n) + 1))] for n in names[:300]]           # prefixes of each other
    pairs = [tuple(int(x) for x in rng.integers(0, len(names), 2)) for _ in range(40000)] + [(i, i) for i in range(len(names))]
    _check_equal(emul, names, pairs)


def test_order_is_total(emul):
    """Antisymmetric, transitive and equal only on identical names, on random triples and on every pair of names up to 4 letters of a0:1."""
    rng = np.random.default_rng(13)
    small = [bytes(t) for n in range(5) for t in itertools.product(b"a0:1", repeat=n)]
    names = small + [illumina_name(rng) for _ in range(400)] + CRAFTED
    cache = {}

    def c(i, j):
        if (i, j) not in cache:
            cache[(i, j)] = su.sign(su.strnum_cmp(names[i], names[j]))
        return cache[(i, j)]
    for i in range(len(small)):
        for j in range(len(small)):
            assert c(i, j) == -c(j, i) and (c(i, j) == 0) == (names[i] == names[j])
    for _ in range(150000):
        i, j, k = (int(x) for x in rng.integers(0, len(names), 3))
        if c(i, j) <= 0 and c(j, k) <= 0:
            assert c(i, k) <= 0 and (c(i, k) < 0 or (c(i, j) == 0 and c(j, k) == 0)), (names[i], names[j], names[k])
        assert c(i, j) == -c(j, i) and (c(i, j) == 0) == (names[i] == names[j])
    pairs = list(cache)[:60000]
    assert su.emul_cmp(emul, names, pairs) == [cache[p] for p in pairs]              # the C function has what was checked


def records(rng, n, contigs=3):
    out = []
    for i in range(n):
        name = illumina_name(rng) if rng.random() < 0.5 else small_name(rng) + b"r%d" % rng.integers(0, 50)
        if rng.random() < 0.3 and out:
            name = su.name_of(out[int(rng.integers(0, len(out)))])                  # equal names
        rid = int(rng.integers(-1, contigs))
        flag = int(rng.choice([0x41, 0x81, 0x1, 0xc1, 0, 0x10 | 0x41, 0x100 | 0x81])) | (4 if rid < 0 else 0)
        out.append(bs.make_rec(rid, int(rng.integers(0, 90000)) if rid >= 0 else -1, flag, cigar=((int(rng.integers(20, 151)), 0),), name=name))
    return out


def _sorted_file(emul, tmp, data, budget, by_name, chunk=20000):
    d = tmp / ("b%d_%d" % (budget, by_name)); d.mkdir()
    out = str(d / "out.bam")
    st = su.emul_file(emul, data, budget, str(d / "out.bam.tmp."), out, by_name=by_name, n_ref=3, chunk=chunk)
    assert os.listdir(d) == ["out.bam"]                                              # no temporary file survives
    return open(out, "rb").read(), st


@pytest.mark.parametrize("by_name", [True, False])
def test_emulated_tool_equals_python_at_every_run_size(emul, tmp_path, by_name):
    rng = np.random.default_rng(21 + by_name)
    recs = records(rng, 3000)
    data = b"".join(recs)
    want = su.expected_records(recs, by_name)
    base, windows = None, 0
    for budget in (1 << 40, 200_000, 100_000, 1):
        if budget == 1:                                                              # one record per run: a temporary file each
            sub = recs[:200]
            got, st = _sorted_file(emul, tmp_path, b"".join(sub), 1, by_name)
            assert [r for _, r in bu.records(bu.inflate(got))] == su.expected_records(sub, by_name)
            assert st["runs"] == 200 and st["windows"] >= 1
            continue
        got, st = _sorted_file(emul, tmp_path, data, budget, by_name)
        assert [r for _, r in bu.records(bu.inflate(got))] == want, budget
        if budget > len(data):
            assert st["runs"] == 0 and st["spill_bytes"] == 0
        else:
            assert st["runs"] >= 3
            windows = max(windows, st["windows"])
        base = base or got
        assert got == base, budget
    assert windows >= 2
    one = [recs[5]]
    got, _ = _sorted_file(emul, tmp_path, one[0], 2, by_name)
    assert [r for _, r in bu.records(bu.inflate(got))] == one


def test_equal_names_come_out_by_flag_then_input_order(emul, tmp_path):
    recs = []
    for k, f in enumerate([0xc1, 0x81, 0x41, 0x1, 0x81 | 0x10, 0x41 | 0x100, 0x1 | 0x800, 0xc1 | 0x10, 0x41 | 0x10, 0]):
        r = mb.rec(k % 3, 100 * k, f, "q7")
        recs.append(r)
    recs += [mb.rec(0, 5, 0x41, "q07"), mb.rec(0, 5, 0x41, "q6"), mb.rec(0, 5, 0x81, "q7x")]
    want = su.name_order(recs)
    flags = [su.flag_of(r) for r in want]
    names = [su.name_of(r) for r in want]
    assert names == [b"q6", b"q07"] + [b"q7"] * 10 + [b"q7x"]                        # q07 < q7: the side that consumed fewer bytes is greater
    assert flags[2:12] == [0x1, 0x1 | 0x800, 0, 0x41, 0x41 | 0x100, 0x41 | 0x10, 0x81, 0x81 | 0x10, 0xc1, 0xc1 | 0x10]
    for budget in (1 << 40, 1):
        got, _ = _sorted_file(emul, tmp_path, b"".join(recs), budget, True, chunk=0)
        assert [r for _, r in bu.records(bu.inflate(got))] == want


def test_merge_windows_carry_the_stream_cut(emul):
    """Slices of the name-sorted stream passed one after another with the carry equal the whole stream compressed at once."""
    rng = np.random.default_rng(31)
    srt = su.name_order(records(rng, 2500))
    blob = b"".join(srt)
    whole = su.emul_once(emul, blob, [a for a, _ in bu.records(blob)])
    z, carry, k = b"", b"", 0
    for size in (1, 7, 500, 40, 1000, 2000):
        part = b"".join(srt[k:k + size])
        k += size
        o = su.emul_once(emul, part, [a for a, _ in bu.records(part)], carry, last=k >= len(srt))
        z += o["z"]; carry = o["carry"]
    assert carry == b"" and z == whole["z"]


def test_header_rewrite_and_pg_rule():
    h = "@SQ\tSN:c0\tLN:10\n@HD\tVN:1.4\tSO:unsorted\tGO:query\tSO:x\n@PG\tID:bm2_sort\tPN:a\n@PG\tID:bm2_sort.1\tPN:b\n@CO\tz\n"
    out = su.out_header(h + "\0\0", True, ["bm2_sort", "-n", "in.bam"])
    assert out.split("\n") == ["@HD\tVN:1.4\tSO:queryname\tGO:query", "@SQ\tSN:c0\tLN:10", "@PG\tID:bm2_sort\tPN:a", "@PG\tID:bm2_sort.1\tPN:b",
                               "@CO\tz", "@PG\tID:bm2_sort.2\tPN:bm2_sort\tPP:bm2_sort.1\tVN:b200-r2\tCL:bm2_sort -n in.bam", ""]
    assert su.out_header("", False, ["s"]) == "@HD\tVN:1.6\tSO:coordinate\n@PG\tID:bm2_sort\tPN:bm2_sort\tVN:b200-r2\tCL:s\n"
    assert su.header_with_sort_order("@CO\ta\n@HD", "coordinate") == "@HD\tSO:coordinate\n@CO\ta\n"


@pytest.mark.skipif(not os.path.exists(MEM), reason="bm2_mem not built")
def test_bm2_mem_header_is_unchanged():
    """bm2_mem --sort's @HD rewrite now comes from the shared header: the same text as the Python restatement."""
    for extra in ([], ["-H", "@CO\tfirst", "-H", "@HD\tVN:1.4\tSO:unsorted\tGO:query"]):
        plain = json.loads(subprocess.run([MEM, "--dump-opt"] + extra + [IDX, "a.fq"], capture_output=True, text=True, timeout=60).stdout)["header"]
        srt = json.loads(subprocess.run([MEM, "--dump-opt", "--sort"] + extra + [IDX, "a.fq"], capture_output=True, text=True, timeout=60).stdout)["header"]
        assert srt == su.header_with_sort_order(plain, "coordinate")


def test_option_errors(tmp_path):
    if not os.path.exists(su.TOOL):
        pytest.skip("bm2_sort not built")
    missing = str(tmp_path / "no_such.bam")                                          # never opened: the options fail first
    o = str(tmp_path / "o.bam")
    for argv, text in [(["-n", "--write-index", "-o", o, missing], "--write-index needs coordinate order"),
                       (["--write-index", missing], "--write-index needs -o"),
                       (["--sort-mem", "0", missing], "--sort-mem"), (["--sort-mem", "12X", missing], "--sort-mem"),
                       (["--sort-mem", "-5", missing], "--sort-mem"), (["--sort-mem"], "--sort-mem takes a value"),
                       (["--window", "0", missing], "--window"), (["--window", "K", missing], "--window"),
                       (["-t", "0", missing], "-t takes"), ([], "no input"), (["-x", missing], "unknown option"),
                       (["-o", o, "a.bam", "b.bam"], "more than one input"), (["-o", o, missing], "cannot open")]:
        r = subprocess.run([su.TOOL] + argv, capture_output=True, timeout=60)
        assert r.returncode == 1 and text in r.stderr.decode(), (argv, r.stderr)
    assert os.listdir(tmp_path) == []
