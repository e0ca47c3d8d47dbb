"""Writes tests/golden/option_regs.json: for every option set of tests/test_option_surface_cpu.py (and the ALT-contig case), the
digest (oracle_lib.dump_digest) of the regs the UNMODIFIED reference computes on the C0 reads (oracle/_ref/<isa>/ref_driver, regs
dumped by its link-time hooks).  Needs oracle/_ref:  python tests/golden/make_option_golden.py"""
import json, os, shutil, subprocess, sys, tempfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cigar_util as cu  # noqa: E402
import oracle_lib as ol  # noqa: E402
import refdump  # noqa: E402
from test_option_surface_cpu import CASES  # noqa: E402


def main():
    gdir = os.path.join(ROOT, "tests", "golden")
    exe = cu.refbin()
    assert exe, "oracle/_ref is not built"
    reads = np.load(os.path.join(gdir, "c0_reads.npz"))["reads"]
    work = tempfile.mkdtemp(prefix="bm2_optgold_")
    fq = []
    for k, name in ((0, "r1.fq"), (1, "r2.fq")):
        fq.append(os.path.join(work, name))
        with open(fq[-1], "w") as f:
            for i, r in enumerate(reads[k::2]):
                f.write(f"@p{i}\n{''.join('ACGTN'[c] for c in r)}\n+\n{'I' * len(r)}\n")
    alt = os.path.join(work, "altidx")
    shutil.copytree(os.path.join(gdir, "c0_index"), alt)
    with open(os.path.join(alt, "ref.fa.alt"), "w") as f:
        f.write("chr3\t0\tchr1\t1\t60\t100M\t*\t0\t0\t*\t*\nchr4\t0\tchr1\t1\t60\t100M\t*\t0\t0\t*\t*\n")
    out = {}
    for name, args, prefix in [(n, a, os.path.join(gdir, "c0_index", "ref.fa")) for n, a in CASES] + [("alt", [], os.path.join(alt, "ref.fa"))]:
        env = dict(os.environ, BM2_DUMP_PREFIX=os.path.join(work, name))
        subprocess.check_call([exe, "mem", "-t", "1", "-K", "100000000"] + args + [prefix] + fq,
                              stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, env=env)
        out[name] = ol.dump_digest(*refdump.read_regs(os.path.join(work, name + ".regs.bin")))
    with open(os.path.join(gdir, "option_regs.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    shutil.rmtree(work)


if __name__ == "__main__":
    main()
