"""Seeded inputs for BAM tests and scripts/bam_rate.py: Illumina-like quality strings (a constant quality would make any compressor look
good) and synthetic uncompressed BAM records of 151 bp pairs."""
import struct
import numpy as np


def illumina_quals(n, length, rng):
    """n quality strings (Phred+33 bytes, uint8[n, length]) from a position-dependent Markov walk: high at the start, drifting down towards
    the 3' end with growing spread, occasional dips, and a tail of '#' (Q2) on some reads."""
    q = np.empty((n, length), np.int16)
    cur = rng.integers(30, 39, n)
    for i in range(length):
        drift = -1 if rng.random() < 0.02 + 0.25 * i / length else 0
        step = rng.choice([-2, -1, 0, 0, 0, 0, 1, 2], n) + drift
        dip = rng.random(n) < 0.01
        cur = np.clip(np.where(dip, cur - rng.integers(8, 20, n), cur + step), 2, 41)
        cur = np.where(rng.random(n) < 0.05, np.clip(cur + 6, 2, 41), cur)        # recover after a dip
        q[:, i] = cur
    tail = rng.random(n) < 0.08
    cut = rng.integers(length // 2, length, n)
    for r in np.nonzero(tail)[0]:
        q[r, cut[r]:] = 2
    return (q + 33).astype(np.uint8)


def bam_records(n_reads=3000, seed=7, length=151):
    """-> (uncompressed BAM records, record starts): pairs on two contigs, with NM / MD / MC / AS / XS / RG tags like bm2_mem writes."""
    rng = np.random.default_rng(seed)
    quals = illumina_quals(n_reads, length, rng) - 33
    out, starts = bytearray(), []
    pos = 1000
    for r in range(n_reads):
        starts.append(len(out))
        name = b"A00123:45:HXXXXDSXX:%d:%d:%d:%d" % (1 + r % 4, 1101 + (r // 4000) % 50, 1000 + (r * 37) % 30000, 1000 + (r * 91) % 30000)
        pos += int(rng.integers(0, 200)) if r % 2 == 0 else 0
        seq = rng.integers(0, 4, length)
        packed = bytes(((np.array([1, 2, 4, 8])[seq[0::2]] << 4) | np.concatenate([np.array([1, 2, 4, 8])[seq[1::2]], [0]])[:len(seq[0::2])]).astype(np.uint8))
        cigar = struct.pack("<I", length << 4)
        mate = pos + int(rng.integers(100, 400))
        tags = b"NMC" + bytes([int(rng.integers(0, 4))]) + b"MDZ%d\0" % length + b"MCZ151M\0" + b"ASC" + bytes([int(rng.integers(120, 152))])
        tags += b"XSC" + bytes([int(rng.integers(0, 40))]) + b"RGZgrp1\0"
        body = struct.pack("<iiBBHHHiiii", r % 2, pos, len(name) + 1, 60, 4681 + (pos >> 14), 1, 99 if r % 2 == 0 else 147, length, r % 2, mate,
                           mate - pos + length)
        body += name + b"\0" + cigar + packed + bytes(quals[r]) + tags
        out += struct.pack("<i", len(body)) + body
    return bytes(out), starts
