"""ctypes binding of libbm2b200.so (include/bm2_b200.h).  Fails loudly when the library or a CUDA
device is missing: there is no CPU fallback."""
from __future__ import annotations
import ctypes as C, os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbm2b200.so")

PAIR_DT = np.dtype([("idr", "<i4"), ("idq", "<i4"), ("id", "<i4"), ("len1", "<i4"), ("len2", "<i4"), ("h0", "<i4"),
                    ("seqid", "<i4"), ("regid", "<i4"), ("score", "<i4"), ("tle", "<i4"), ("gtle", "<i4"),
                    ("qle", "<i4"), ("gscore", "<i4"), ("max_off", "<i4")])
SMEM_DT = np.dtype([("rid", "<u4"), ("m", "<u4"), ("n", "<u4"), ("_pad", "<u4"), ("k", "<i8"), ("l", "<i8"), ("s", "<i8")])
SEED_DT = np.dtype([("rbeg", "<i8"), ("qbeg", "<i4"), ("len", "<i4"), ("score", "<i4"), ("chain", "<i4")])
CHAIN_DT = np.dtype([("pos", "<i8"), ("seqid", "<i4"), ("rid", "<i4"), ("n_seeds", "<i4"), ("seed_off", "<i4"),
                     ("w", "<i4"), ("kept", "<i4"), ("first", "<i4"), ("is_alt", "<i4"), ("frac_rep", "<f4"), ("_pad", "<i4")])
REG_DT = np.dtype([("rb", "<i8"), ("re", "<i8"), ("qb", "<i4"), ("qe", "<i4"), ("rid", "<i4"), ("_p0", "<i4"), ("c", "<u8"),
                   ("score", "<i4"), ("truesc", "<i4"), ("sub", "<i4"), ("alt_sc", "<i4"), ("csub", "<i4"), ("sub_n", "<i4"),
                   ("w", "<i4"), ("seedcov", "<i4"), ("secondary", "<i4"), ("secondary_all", "<i4"), ("seedlen0", "<i4"),
                   ("n_comp_is_alt", "<i4"), ("frac_rep", "<f4"), ("_p1", "<i4"), ("hash", "<u8"), ("flg", "<i4"), ("_p2", "<i4")])


class MemOpt(C.Structure):
    _fields_ = [("a", C.c_int), ("b", C.c_int), ("o_del", C.c_int), ("e_del", C.c_int), ("o_ins", C.c_int), ("e_ins", C.c_int),
                ("pen_unpaired", C.c_int), ("pen_clip5", C.c_int), ("pen_clip3", C.c_int), ("w", C.c_int), ("zdrop", C.c_int),
                ("max_mem_intv", C.c_uint64), ("T", C.c_int), ("flag", C.c_int), ("min_seed_len", C.c_int),
                ("min_chain_weight", C.c_int), ("max_chain_extend", C.c_int), ("split_factor", C.c_float),
                ("split_width", C.c_int), ("max_occ", C.c_int), ("max_chain_gap", C.c_int), ("n_threads", C.c_int),
                ("chunk_size", C.c_int64), ("mask_level", C.c_float), ("drop_ratio", C.c_float), ("XA_drop_ratio", C.c_float),
                ("mask_level_redun", C.c_float), ("mapQ_coef_len", C.c_float), ("mapQ_coef_fac", C.c_int), ("max_ins", C.c_int),
                ("max_matesw", C.c_int), ("max_XA_hits", C.c_int), ("max_XA_hits_alt", C.c_int), ("mat", C.c_int8 * 25)]


class IndexDesc(C.Structure):
    _fields_ = [("reference_seq_len", C.c_int64), ("count", C.c_int64 * 5), ("sentinel_index", C.c_int64),
                ("cp_occ", C.c_void_p), ("sa_ms_byte", C.c_void_p), ("sa_ls_word", C.c_void_p), ("ref_string", C.c_void_p),
                ("l_pac", C.c_int64), ("n_seqs", C.c_int32), ("ann_offset", C.c_void_p), ("ann_len", C.c_void_p),
                ("ann_is_alt", C.c_void_p)]


# seam 3 (bm2_gen_cigar): request / record layouts of include/bm2_b200.h
CIGAR_REQ_DT = np.dtype([("rb", "<i8"), ("re", "<i8"), ("read", "<i4"), ("qb", "<i4"), ("qe", "<i4"), ("w", "<i4")])
CIGAR_REC_DT = np.dtype([("score", "<i4"), ("n_cigar", "<i4"), ("nm", "<i4"), ("n_md", "<i4"), ("cigar_off", "<i8"), ("md_off", "<i8")])


# seam 4, first piece (bm2_pestat): mem_pestat_t of the four orientations FF, FR, RF, RR
PESTAT_DT = np.dtype([("low", "<i4"), ("high", "<i4"), ("failed", "<i4"), ("_pad", "<i4"), ("avg", "<f8"), ("std", "<f8")])


# seam 4 (bm2_sam_pe): one record per SAM line, XA entries; layouts of include/bm2_b200.h
SAM_REC_DT = np.dtype([("read", "<i4"), ("flag", "<i4"), ("rid", "<i4"), ("rnext", "<i4"), ("mapq", "<i4"), ("nm", "<i4"), ("score", "<i4"), ("sub", "<i4"),
                       ("alt_sc", "<i4"), ("reg", "<i4"), ("n_cigar", "<i4"), ("n_md", "<i4"), ("is_alt", "<i4"), ("n_mc", "<i4"),
                       ("pos", "<i8"), ("pnext", "<i8"), ("tlen", "<i8"), ("cigar_off", "<i8"), ("md_off", "<i8")])
SAM_XA_DT = np.dtype([("read", "<i4"), ("reg", "<i4"), ("rid", "<i4"), ("is_rev", "<i4"), ("nm", "<i4"), ("n_cigar", "<i4"), ("pos", "<i8"), ("cigar_off", "<i8")])


# finer seam under seam 4 (bm2_ksw_align2): request / result layouts of include/bm2_b200.h
KSW_REQ_DT = np.dtype([("qoff", "<i8"), ("toff", "<i8"), ("qlen", "<i4"), ("tlen", "<i4"), ("xtra", "<i4"), ("_pad", "<i4")])
KSW_RES_DT = np.dtype([("score", "<i4"), ("te", "<i4"), ("qe", "<i4"), ("score2", "<i4"), ("te2", "<i4"), ("tb", "<i4"), ("qb", "<i4"), ("_pad", "<i4")])


class SamResult(C.Structure):
    _fields_ = [("n_recs", C.c_int64), ("recs", C.c_void_p), ("n_xa", C.c_int64), ("xa", C.c_void_p), ("n_ops", C.c_int64), ("cigar", C.c_void_p),
                ("n_md", C.c_int64), ("md", C.c_void_p)]


class CigarResult(C.Structure):
    _fields_ = [("n", C.c_int64), ("recs", C.c_void_p), ("n_ops", C.c_int64), ("cigar", C.c_void_p), ("n_md", C.c_int64), ("md", C.c_void_p)]


class SamTextIn(C.Structure):
    _fields_ = [("res", C.c_void_p), ("reads", C.c_void_p), ("names", C.c_void_p), ("quals", C.c_void_p), ("contig_names", C.c_void_p),
                ("name_buf", C.c_char_p * 2), ("name_beg", C.c_void_p), ("name_len", C.c_void_p)]


class FastqBatch(C.Structure):
    _fields_ = [("n_reads", C.c_int32), ("d_codes", C.c_void_p), ("d_offsets", C.c_void_p), ("codes", C.c_void_p), ("offsets", C.c_void_p),
                ("quals", C.c_void_p), ("name_beg", C.c_void_p), ("name_len", C.c_void_p)]


class FastqSplit(C.Structure):
    _fields_ = [("set", FastqBatch * 2), ("comment_beg", C.c_void_p * 2), ("comment_len", C.c_void_p * 2), ("read_index", C.c_void_p * 2)]


class SamTextExtra(C.Structure):
    _fields_ = [("rg_id", C.c_char_p), ("comment_beg", C.c_void_p), ("comment_len", C.c_void_p), ("contig_anno", C.c_void_p), ("ref_hdr", C.c_int32),
                ("qual_present", C.c_void_p)]


def _host(p, n, dt):
    dt = np.dtype(dt)
    return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(max(n, 1) * dt.itemsize,))[:n * dt.itemsize].view(dt).copy()


def sam_format(recs, xa, cigar, md, codes, offsets, contig_names, read_names=None, quals=None, n_threads=1, name_spans=None,
               rg_id=None, comments=None, contig_anno=None, ref_hdr=False, qual_present=None) -> bytes:
    """bm2_sam_format: the SAM text of a batch from the records of bm2_sam_pe / bm2_sam_se (one line per record, QNAME to the last tag).
    read_names: list of names, or name_spans = (buf1, buf2 or None, name_beg int64[], name_len int32[]) as bm2_fastq_encode returns them.
    With rg_id (-R), comments = (comment_beg int64[], comment_len int32[]) into the buffers of name_spans (-C) or contig_anno (list of str)
    with ref_hdr (-V), or qual_present (uint8[] per read, 0: QUAL '*', as bm2_seq_encode returns it): bm2_sam_format_ex."""
    recs = np.ascontiguousarray(recs, SAM_REC_DT); xa = np.ascontiguousarray(xa, SAM_XA_DT)
    cigar = np.ascontiguousarray(cigar, np.uint32); md = np.ascontiguousarray(md, np.uint8)
    codes = np.ascontiguousarray(codes, np.uint8); offsets = np.ascontiguousarray(offsets, np.int64)
    res = SamResult(len(recs), recs.ctypes.data, len(xa), xa.ctypes.data, len(cigar), cigar.ctypes.data, len(md), md.ctypes.data)
    rb = ReadBatch(len(offsets) - 1, codes.ctypes.data, offsets.ctypes.data)
    cn = (C.c_char_p * len(contig_names))(*[s.encode() for s in contig_names])
    rn = (C.c_char_p * len(read_names))(*[s.encode() if isinstance(s, str) else bytes(s) for s in read_names]) if read_names is not None else None
    q = np.ascontiguousarray(np.frombuffer(quals, np.uint8) if isinstance(quals, (bytes, bytearray)) else quals, np.uint8) if quals is not None else None
    tin = SamTextIn(C.cast(C.byref(res), C.c_void_p), C.cast(C.byref(rb), C.c_void_p), C.cast(rn, C.c_void_p) if rn is not None else None,
                    q.ctypes.data if q is not None else None, C.cast(cn, C.c_void_p))
    if name_spans is not None:
        b1, b2, nbeg, nlen = name_spans
        nbeg = np.ascontiguousarray(nbeg, np.int64); nlen = np.ascontiguousarray(nlen, np.int32)
        tin.name_buf[0] = b1; tin.name_buf[1] = b2
        tin.name_beg = nbeg.ctypes.data; tin.name_len = nlen.ctypes.data
    text = C.c_void_p(); n = C.c_int64()
    if rg_id is None and comments is None and contig_anno is None and not ref_hdr and qual_present is None:
        f = lib().bm2_sam_format
        f.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        rc = f(C.byref(tin), int(n_threads), C.byref(text), C.byref(n))
    else:
        x = SamTextExtra(rg_id.encode() if isinstance(rg_id, str) else rg_id, None, None, None, int(bool(ref_hdr)))
        if comments is not None:
            cb = np.ascontiguousarray(comments[0], np.int64); cl = np.ascontiguousarray(comments[1], np.int32)
            x.comment_beg = cb.ctypes.data; x.comment_len = cl.ctypes.data
        if contig_anno is not None:
            ca = (C.c_char_p * len(contig_anno))(*[s.encode() if isinstance(s, str) else bytes(s) for s in contig_anno])
            x.contig_anno = C.cast(ca, C.c_void_p)
        if qual_present is not None:
            qp = np.ascontiguousarray(qual_present, np.uint8)
            x.qual_present = qp.ctypes.data
        f = lib().bm2_sam_format_ex
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        rc = f(C.byref(tin), C.byref(x), int(n_threads), C.byref(text), C.byref(n))
    if rc:
        raise Bm2Error(f"bm2_sam_format failed ({rc})")
    out = C.string_at(text, n.value)
    lib().bm2_free.argtypes = [C.c_void_p]
    lib().bm2_free(text)
    return out


def bam_format(recs, xa, cigar, md, codes, offsets, contig_names, read_names=None, quals=None, n_threads=1, name_spans=None,
               rg_id=None, comments=None, contig_anno=None, ref_hdr=False, qual_present=None):
    """bm2_bam_format_ex: the records of sam_format(...) (same arguments) as uncompressed BAM records -> (bytes, read_off int64[n_reads + 1]:
    where each read's records start).  A long QNAME or a comment that is not SAM tags raises Bm2Error naming the read."""
    recs = np.ascontiguousarray(recs, SAM_REC_DT); xa = np.ascontiguousarray(xa, SAM_XA_DT)
    cigar = np.ascontiguousarray(cigar, np.uint32); md = np.ascontiguousarray(md, np.uint8)
    codes = np.ascontiguousarray(codes, np.uint8); offsets = np.ascontiguousarray(offsets, np.int64)
    res = SamResult(len(recs), recs.ctypes.data, len(xa), xa.ctypes.data, len(cigar), cigar.ctypes.data, len(md), md.ctypes.data)
    rb = ReadBatch(len(offsets) - 1, codes.ctypes.data, offsets.ctypes.data)
    cn = (C.c_char_p * len(contig_names))(*[s.encode() for s in contig_names])
    rn = (C.c_char_p * len(read_names))(*[s.encode() if isinstance(s, str) else bytes(s) for s in read_names]) if read_names is not None else None
    q = np.ascontiguousarray(np.frombuffer(quals, np.uint8) if isinstance(quals, (bytes, bytearray)) else quals, np.uint8) if quals is not None else None
    tin = SamTextIn(C.cast(C.byref(res), C.c_void_p), C.cast(C.byref(rb), C.c_void_p), C.cast(rn, C.c_void_p) if rn is not None else None,
                    q.ctypes.data if q is not None else None, C.cast(cn, C.c_void_p))
    keep = []
    if name_spans is not None:
        b1, b2, nbeg, nlen = name_spans
        nbeg = np.ascontiguousarray(nbeg, np.int64); nlen = np.ascontiguousarray(nlen, np.int32); keep += [nbeg, nlen]
        tin.name_buf[0] = b1; tin.name_buf[1] = b2
        tin.name_beg = nbeg.ctypes.data; tin.name_len = nlen.ctypes.data
    x = SamTextExtra(rg_id.encode() if isinstance(rg_id, str) else rg_id, None, None, None, int(bool(ref_hdr)))
    if comments is not None:
        cb = np.ascontiguousarray(comments[0], np.int64); cl = np.ascontiguousarray(comments[1], np.int32); keep += [cb, cl]
        x.comment_beg = cb.ctypes.data; x.comment_len = cl.ctypes.data
    if contig_anno is not None:
        ca = (C.c_char_p * len(contig_anno))(*[s.encode() if isinstance(s, str) else bytes(s) for s in contig_anno]); keep.append(ca)
        x.contig_anno = C.cast(ca, C.c_void_p)
    if qual_present is not None:
        qp = np.ascontiguousarray(qual_present, np.uint8); keep.append(qp)
        x.qual_present = qp.ctypes.data
    buf = C.c_void_p(); n = C.c_int64(); ro = C.c_void_p()
    f = lib().bm2_bam_format_ex
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    rc = f(C.byref(tin), C.byref(x), int(n_threads), C.byref(buf), C.byref(n), C.byref(ro))
    if rc:
        raise Bm2Error(f"bm2_bam_format failed ({rc}): " + (lib().bm2_last_error(None) or b"").decode(errors="replace"))
    out = C.string_at(buf, n.value)
    off = _host(ro, rb.n_reads + 1, np.int64)
    lib().bm2_free.argtypes = [C.c_void_p]
    lib().bm2_free(buf); lib().bm2_free(ro)
    return out, off


class ReadBatch(C.Structure):
    _fields_ = [("n_reads", C.c_int32), ("codes", C.c_void_p), ("offsets", C.c_void_p)]


class SmemResult(C.Structure):
    _fields_ = [("n", C.c_int64), ("smems", C.c_void_p), ("read_off", C.c_void_p)]


class ChainResult(C.Structure):
    _fields_ = [("n_chains", C.c_int64), ("n_seeds", C.c_int64), ("chains", C.c_void_p), ("seeds", C.c_void_p),
                ("read_off", C.c_void_p)]


class RegResult(C.Structure):
    _fields_ = [("n", C.c_int64), ("regs", C.c_void_p), ("read_off", C.c_void_p)]


# bm2_bam_sort_compress: per record in output order (include/bm2_b200.h)
SORT_REC_DT = np.dtype([("rid", "<i4"), ("pos", "<i4"), ("end", "<i4"), ("bin", "<u2"), ("flag", "<u2"), ("block", "<i8"), ("offset", "<i4"), ("_pad", "<i4")])


# bm2_dup_signatures / bm2_dup_resolve: one entry of a duplicate space (include/bm2_b200.h); kind 0 pair, 1 fragment, 2 pair end
DUP_ENTRY_DT = np.dtype([("k1", "<u8"), ("k2", "<u8"), ("tid", "<i8"), ("score", "<i4"), ("kind", "<i4")])
# bm2_dup_signatures_ex / bm2_dup_resolve_ex: a located pair entry; loc bit 0 has a location, bit 1 the orientation class (reverse)
DUP_LOC_ENTRY_DT = np.dtype([("k1", "<u8"), ("k2", "<u8"), ("tid", "<i8"), ("score", "<i4"), ("kind", "<i4"), ("tile", "<i4"), ("x", "<i4"),
                             ("y", "<i4"), ("loc", "<i4")])


# bm2_bqsr_tables: the recalibration counts (include/bm2_b200.h)
class BqsrTables(C.Structure):
    _fields_ = [("qual_obs", C.c_void_p), ("qual_err", C.c_void_p), ("ctx_obs", C.c_void_p), ("ctx_err", C.c_void_p), ("cyc_obs", C.c_void_p),
                ("cyc_err", C.c_void_p), ("reads", C.c_int64), ("bases", C.c_int64), ("ms", C.c_double), ("err_kind", C.c_int32),
                ("err_index", C.c_int64), ("err_name", C.c_char_p), ("read_group", C.c_char_p)]


BQSR_NQ, BQSR_NCTX, BQSR_NCYC = 94, 16, 1001


# bm2_bqsr_apply_set / bm2_last_bqsr_apply_stats (include/bm2_b200.h)
class BqsrApplyTables(C.Structure):
    _fields_ = [("n_rg", C.c_int32), ("P", C.c_void_p), ("ctx", C.c_void_p), ("cyc", C.c_void_p), ("n_ids", C.c_int32), ("ids", C.c_void_p),
                ("id_table", C.c_void_p)]


class BqsrApplyStats(C.Structure):
    _fields_ = [("apply_ms", C.c_double), ("bgzf_ms", C.c_double), ("bases_changed", C.c_int64), ("recal_records", C.c_int64),
                ("kept_records", C.c_int64), ("err_kind", C.c_int32), ("err_index", C.c_int64), ("err_name", C.c_char_p)]


# bm2_recal_set (include/bm2_b200.h)
class RecalSet(C.Structure):
    _fields_ = [("n_contigs", C.c_int32), ("contig_off", C.c_void_p), ("contig_len", C.c_void_p), ("l_pac", C.c_int64), ("pac", C.c_void_p),
                ("holes", C.c_void_p), ("n_holes", C.c_int64), ("covered", C.c_void_p), ("junction", C.c_void_p), ("n_ids", C.c_int32),
                ("ids", C.c_void_p), ("id_cov", C.c_void_p), ("n_cov", C.c_int32)]


# bm2_wgs_set / bm2_wgs_finish (include/bm2_b200.h)
class WgsParams(C.Structure):
    _fields_ = [("min_mapq", C.c_int32), ("min_baseq", C.c_int32), ("coverage_cap", C.c_int32), ("count_unpaired", C.c_int32)]


class WgsResult(C.Structure):
    _fields_ = [("hist", C.c_void_p), ("cap", C.c_int32), ("exc", C.c_int64 * 6), ("records", C.c_int64), ("counted_records", C.c_int64),
                ("carried_max", C.c_int64), ("add_ms", C.c_double), ("finish_ms", C.c_double)]


# bm2_mm_finish (include/bm2_b200.h)
class MmResult(C.Structure):
    _fields_ = [("counts", C.c_int64 * 63), ("max_len", C.c_int32), ("len_hist", C.c_void_p), ("mism_hist", C.c_void_p), ("nocall", C.c_void_p),
                ("max_insert", C.c_int32), ("insert_hist", C.c_void_p), ("insert_big", C.c_void_p), ("n_big", C.c_int64), ("records", C.c_int64),
                ("add_ms", C.c_double), ("finish_ms", C.c_double)]


# bm2_mm_gc_finish (include/bm2_b200.h)
class MmGcResult(C.Structure):
    _fields_ = [("windows", C.c_int64 * 101), ("reads", C.c_int64 * 101), ("bases", C.c_int64 * 101), ("errors", C.c_int64 * 101),
                ("total_clusters", C.c_int64), ("aligned_reads", C.c_int64), ("scan_ms", C.c_double), ("add_ms", C.c_double)]


class SortOut(C.Structure):
    _fields_ = [("z", C.c_void_p), ("z_len", C.c_int64), ("member_size", C.c_void_p), ("n_members", C.c_int64), ("carry", C.c_void_p),
                ("carry_len", C.c_int64), ("recs", C.c_void_p), ("n_recs", C.c_int64)]


EXPORTS = ["bm2_create_sibling", "bm2_fastq_encode", "bm2_seq_encode", "bm2_fastq_comments", "bm2_fastq_smart_pair", "bm2_sam_format", "bm2_sam_format_ex", "bm2_free", "bm2_create_resident", "bm2_gather_probe", "bm2_set_sam_staged", "bm2_last_sam_stats", "bm2_gather64_gbs", "bm2_set_sub_batches", "bm2_seed_chain_extend_resident", "bm2_last_counters", "bm2_set_stream", "bm2_int_pipe_gops", "bm2_abi_version", "bm2_opt_init", "bm2_index_load", "bm2_index_free", "bm2_create", "bm2_destroy",
           "bm2_last_error", "bm2_extend_pairs", "bm2_extend_pairs_device", "bm2_collect_smems", "bm2_seed_chain",
           "bm2_seed_chain_extend", "bm2_last_stage_ms", "bm2_gen_cigar", "bm2_pestat", "bm2_sam_pe", "bm2_sam_se", "bm2_ksw_align2",
           "bm2_fasta_pack", "bm2_index_build", "bm2_bam_format_ex", "bm2_bgzf_compress", "bm2_last_bgzf_stats",
           "bm2_bam_sort_compress", "bm2_last_sort_stats", "bm2_bam_sort_memory", "bm2_bam_sort_memory_ex", "bm2_bam_sort_compress_ex",
           "bm2_dup_signatures", "bm2_dup_resolve", "bm2_last_dup_stats", "bm2_dup_set", "bm2_dup_signatures_ex", "bm2_dup_resolve_ex",
           "bm2_bqsr_sites", "bm2_bqsr_count", "bm2_bqsr_tables", "bm2_bqsr_apply_set", "bm2_bqsr_apply", "bm2_last_bqsr_apply_stats",
           "bm2_bqsr_apply_memory", "bm2_wgs_set", "bm2_wgs_memory", "bm2_wgs_add", "bm2_wgs_finish",
           "bm2_mm_set", "bm2_mm_memory", "bm2_mm_add", "bm2_mm_finish", "bm2_mm_gc_set", "bm2_mm_gc_memory", "bm2_mm_gc_finish", "bm2_markdup_set", "bm2_markdup_records", "bm2_markdup_pair", "bm2_markdup_counts",
           "bm2_markdup_mark", "bm2_last_markdup_stats", "bm2_markdup_memory", "bm2_recal_memory", "bm2_recal_set", "bm2_recal_add", "bm2_recal_tables",
           "bm2_bam2fq_records", "bm2_bam2fq_format", "bm2_last_bam2fq_stats", "bm2_bam2fq_memory",
           "bm2_bam_qname_sort_compress", "bm2_bam_qname_sort_memory"]

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with __graft_entry__.build() (no CPU fallback exists)")
        _lib = C.CDLL(LIB_PATH)
        _lib.bm2_last_error.restype = C.c_char_p
        _lib.bm2_last_error.argtypes = [C.c_void_p]
        _lib.bm2_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_void_p, C.c_void_p]
        _lib.bm2_destroy.argtypes = [C.c_void_p]
        _lib.bm2_index_load.argtypes = [C.c_char_p, C.POINTER(C.POINTER(IndexDesc))]
        _lib.bm2_index_free.argtypes = [C.POINTER(IndexDesc)]
        _lib.bm2_extend_pairs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
        _lib.bm2_extend_pairs_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                                 C.c_int32, C.c_void_p]
        for f in ("bm2_collect_smems", "bm2_seed_chain", "bm2_seed_chain_extend"):
            if hasattr(_lib, f):
                getattr(_lib, f).argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def default_opt() -> MemOpt:
    o = MemOpt()
    lib().bm2_opt_init(C.byref(o))
    return o


class Bm2Error(RuntimeError):
    pass


def pestat(opt, l_pac, regs, read_off):
    """bm2_pestat: insert-size statistics of a chunk (reads 2i, 2i+1 are mates) from the regs of bm2_seed_chain_extend -> PESTAT_DT[4]."""
    regs = np.ascontiguousarray(regs, REG_DT); read_off = np.ascontiguousarray(read_off, np.int64)
    out = np.zeros(4, PESTAT_DT)
    f = lib().bm2_pestat
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    rc = f(C.addressof(opt), int(l_pac), len(read_off) - 1, regs.ctypes.data, read_off.ctypes.data, out.ctypes.data)
    if rc:
        raise Bm2Error(f"bm2_pestat failed ({rc})")
    return out


class FastaPackStats(C.Structure):
    _fields_ = [("l_pac", C.c_int64), ("n_seqs", C.c_int64), ("n_holes", C.c_int64), ("seconds", C.c_double)]


class IndexBuildStats(C.Structure):
    _fields_ = [("n", C.c_int64), ("peak_device_bytes", C.c_int64), ("rounds", C.c_int32), ("groups", C.c_int32), ("windows", C.c_int32),
                ("pieces", C.c_int64), ("unresolved", C.c_int64), ("unresolved_on_host", C.c_int32),
                ("load_s", C.c_double), ("pass1_s", C.c_double), ("refine_s", C.c_double), ("emit_s", C.c_double), ("total_s", C.c_double)]


def _stats_dict(st) -> dict:
    return {name: getattr(st, name) for name, _ in st._fields_}


def fasta_pack(path: str, prefix: str) -> dict:
    """bm2_fasta_pack (host only): <prefix>.pac / .ann / .amb of a FASTA or FASTQ file, plain or gzip, as `bwa-mem2 index` writes them."""
    st = FastaPackStats()
    f = lib().bm2_fasta_pack
    f.restype = C.c_int
    f.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p]
    if f(path.encode(), prefix.encode(), C.byref(st)):
        raise Bm2Error(lib().bm2_last_error(None).decode())
    return _stats_dict(st)


def index_build(prefix: str, device: int = 0, work_bytes: int = 0) -> dict:
    """bm2_index_build: <prefix>.0123 and <prefix>.bwt.2bit.64 from <prefix>.pac on the GPU.  work_bytes sizes the working buffers
    (0: from the free device memory); returns the build's stats (peak device bytes, rounds, groups, pieces, windows, stage times)."""
    st = IndexBuildStats()
    f = lib().bm2_index_build
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_char_p, C.c_int64, C.c_void_p]
    if f(int(device), prefix.encode(), int(work_bytes), C.byref(st)):
        raise Bm2Error(lib().bm2_last_error(None).decode())
    return _stats_dict(st)


class Index:
    """Host-resident index loaded by the native loader (bm2_index_load)."""

    def __init__(self, prefix: str):
        self._p = C.POINTER(IndexDesc)()
        rc = lib().bm2_index_load(prefix.encode(), C.byref(self._p))
        if rc:
            lib().bm2_index_io_error.restype = C.c_char_p
            raise Bm2Error(f"bm2_index_load({prefix}): {lib().bm2_index_io_error().decode()}")
        self.desc = self._p.contents

    def close(self):
        if self._p:
            lib().bm2_index_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Context:
    """bm2_ctx wrapper; mirrors the reference seams (see include/bm2_b200.h)."""

    def __init__(self, device: int = 0, index=None, opt: MemOpt | None = None, resident: bool = False):
        """index: an Index (host arrays, uploaded by bm2_create) or an IndexDesc; resident=True: the four big arrays of the
        descriptor are device pointers already in `device`'s memory (bm2_create_resident; the caller keeps them alive)."""
        self._ctx = C.c_void_p()
        self.opt = opt if opt is not None else default_opt()
        self._index = index
        idx_ptr = None
        if index is not None:
            idx_ptr = C.cast(C.byref(index.desc if isinstance(index, Index) else index), C.c_void_p)
        f = lib().bm2_create_resident if resident else lib().bm2_create
        rc = f(C.byref(self._ctx), device, idx_ptr, C.cast(C.byref(self.opt), C.c_void_p))
        if rc:
            raise Bm2Error(("bm2_create_resident: " if resident else "bm2_create: ") + lib().bm2_last_error(None).decode())

    def close(self):
        if self._ctx:
            lib().bm2_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc:
            raise Bm2Error(f"{what}: " + lib().bm2_last_error(self._ctx).decode())

    # seam 1 (BandedPairWiseSW::getScores16 & co.)
    def extend_pairs(self, pairs: np.ndarray, ref: np.ndarray, qer: np.ndarray, w: int, end_bonus: int):
        assert pairs.dtype == PAIR_DT and pairs.flags.c_contiguous
        ref = np.ascontiguousarray(ref, np.uint8); qer = np.ascontiguousarray(qer, np.uint8)
        self._check(lib().bm2_extend_pairs(self._ctx, pairs.ctypes.data, ref.ctypes.data, qer.ctypes.data,
                                           len(pairs), w, end_bonus), "bm2_extend_pairs")
        return pairs

    def extend_pairs_device(self, d_pairs_ptr, d_ref_ptr, d_qer_ptr, n, w, end_bonus, d_cells_ptr=None):
        self._check(lib().bm2_extend_pairs_device(self._ctx, d_pairs_ptr, d_ref_ptr, d_qer_ptr, n, w, end_bonus,
                                                  d_cells_ptr), "bm2_extend_pairs_device")

    # seam 2
    @staticmethod
    def _batch(codes: np.ndarray, offsets: np.ndarray):
        codes = np.ascontiguousarray(codes, np.uint8); offsets = np.ascontiguousarray(offsets, np.int64)
        rb = ReadBatch(len(offsets) - 1, codes.ctypes.data, offsets.ctypes.data)
        return rb, (codes, offsets)

    def collect_smems(self, codes, offsets):
        rb, keep = self._batch(codes, offsets)
        res = SmemResult()
        self._check(lib().bm2_collect_smems(self._ctx, C.byref(rb), C.byref(res)), "bm2_collect_smems")
        n = res.n
        sm = np.ctypeslib.as_array(C.cast(res.smems, C.POINTER(C.c_uint8)), shape=(n * SMEM_DT.itemsize,)).view(SMEM_DT).copy() if n else np.zeros(0, SMEM_DT)
        off = np.ctypeslib.as_array(C.cast(res.read_off, C.POINTER(C.c_int64)), shape=(rb.n_reads + 1,)).copy()
        return sm, off

    def seed_chain(self, codes, offsets):
        rb, keep = self._batch(codes, offsets)
        res = ChainResult()
        self._check(lib().bm2_seed_chain(self._ctx, C.byref(rb), C.byref(res)), "bm2_seed_chain")
        nc, ns = res.n_chains, res.n_seeds
        ch = np.ctypeslib.as_array(C.cast(res.chains, C.POINTER(C.c_uint8)), shape=(nc * CHAIN_DT.itemsize,)).view(CHAIN_DT).copy() if nc else np.zeros(0, CHAIN_DT)
        sd = np.ctypeslib.as_array(C.cast(res.seeds, C.POINTER(C.c_uint8)), shape=(ns * SEED_DT.itemsize,)).view(SEED_DT).copy() if ns else np.zeros(0, SEED_DT)
        off = np.ctypeslib.as_array(C.cast(res.read_off, C.POINTER(C.c_int64)), shape=(rb.n_reads + 1,)).copy()
        return ch, sd, off

    def seed_chain_extend(self, codes, offsets, copy=True):
        rb, keep = self._batch(codes, offsets)
        res = RegResult()
        self._check(lib().bm2_seed_chain_extend(self._ctx, C.byref(rb), C.byref(res)), "bm2_seed_chain_extend")
        n = res.n
        regs = np.ctypeslib.as_array(C.cast(res.regs, C.POINTER(C.c_uint8)), shape=(n * REG_DT.itemsize,)).view(REG_DT) if n else np.zeros(0, REG_DT)
        off = np.ctypeslib.as_array(C.cast(res.read_off, C.POINTER(C.c_int64)), shape=(rb.n_reads + 1,))
        return (regs.copy(), off.copy()) if copy else (regs, off)

    def gen_cigar(self, codes, offsets, reqs):
        """bm2_gen_cigar: reqs is a CIGAR_REQ_DT array -> (recs CIGAR_REC_DT, cigar uint32[], md bytes)."""
        rb, keep = self._batch(codes, offsets)
        reqs = np.ascontiguousarray(reqs, CIGAR_REQ_DT)
        res = CigarResult()
        lib().bm2_gen_cigar.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        self._check(lib().bm2_gen_cigar(self._ctx, C.byref(rb), reqs.ctypes.data_as(C.c_void_p), len(reqs), C.byref(res)), "bm2_gen_cigar")
        def arr(p, n, dt):
            dt = np.dtype(dt)
            return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n * dt.itemsize,)).view(dt).copy() if n else np.zeros(0, dt)
        return arr(res.recs, res.n, CIGAR_REC_DT), arr(res.cigar, res.n_ops, "<u4"), arr(res.md, res.n_md, "u1")

    def ksw_align2(self, reqs):
        """bm2_ksw_align2: reqs = [(query codes, window codes, xtra), ...] -> int32[n, 7] (score, te, qe, score2, te2, tb, qb)."""
        seqs = np.concatenate([np.concatenate([np.asarray(q, np.uint8), np.asarray(t, np.uint8)]) for q, t, _ in reqs]) if reqs else np.zeros(0, np.uint8)
        rq = np.zeros(len(reqs), KSW_REQ_DT); pos = 0
        for i, (q, t, x) in enumerate(reqs):
            rq[i] = (pos, pos + len(q), len(q), len(t), x, 0); pos += len(q) + len(t)
        out = np.zeros(len(reqs), KSW_RES_DT)
        f = lib().bm2_ksw_align2
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
        self._check(f(self._ctx, seqs.ctypes.data_as(C.c_void_p), len(seqs), rq.ctypes.data_as(C.c_void_p), len(rq), out.ctypes.data_as(C.c_void_p)), "bm2_ksw_align2")
        return np.stack([out[k] for k in ("score", "te", "qe", "score2", "te2", "tb", "qb")], axis=1).astype(np.int32) if len(out) else np.zeros((0, 7), np.int32)

    def sam_se(self, codes, offsets, regs, read_off, id_base=0):
        """bm2_sam_se: the SAM stage of a batch of single-end reads -> (recs SAM_REC_DT, xa SAM_XA_DT, cigar uint32[], md bytes)."""
        rb, keep = self._batch(codes, offsets)
        regs = np.ascontiguousarray(regs, REG_DT); read_off = np.ascontiguousarray(read_off, np.int64)
        res = SamResult()
        f = lib().bm2_sam_se
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        self._check(f(self._ctx, C.byref(rb), regs.ctypes.data_as(C.c_void_p), read_off.ctypes.data_as(C.c_void_p), int(id_base), C.byref(res)), "bm2_sam_se")
        def arr(p, n, dt):
            dt = np.dtype(dt)
            return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n * dt.itemsize,)).view(dt).copy() if n else np.zeros(0, dt)
        return arr(res.recs, res.n_recs, SAM_REC_DT), arr(res.xa, res.n_xa, SAM_XA_DT), arr(res.cigar, res.n_ops, "<u4"), arr(res.md, res.n_md, "u1")

    def sam_pe(self, codes, offsets, regs, read_off, pes, id_base=0):
        """bm2_sam_pe: the SAM stage of a batch of pairs -> (recs SAM_REC_DT, xa SAM_XA_DT, cigar uint32[], md bytes)."""
        rb, keep = self._batch(codes, offsets)
        regs = np.ascontiguousarray(regs, REG_DT); read_off = np.ascontiguousarray(read_off, np.int64); pes = np.ascontiguousarray(pes, PESTAT_DT)
        res = SamResult()
        f = lib().bm2_sam_pe
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        self._check(f(self._ctx, C.byref(rb), regs.ctypes.data_as(C.c_void_p), read_off.ctypes.data_as(C.c_void_p), pes.ctypes.data_as(C.c_void_p),
                      int(id_base), C.byref(res)), "bm2_sam_pe")
        def arr(p, n, dt):
            dt = np.dtype(dt)
            return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n * dt.itemsize,)).view(dt).copy() if n else np.zeros(0, dt)
        return arr(res.recs, res.n_recs, SAM_REC_DT), arr(res.xa, res.n_xa, SAM_XA_DT), arr(res.cigar, res.n_ops, "<u4"), arr(res.md, res.n_md, "u1")

    def fastq_encode(self, buf1: bytes, buf2: bytes | None = None, want_names: bool = True):
        """bm2_fastq_encode: raw FASTQ bytes of a chunk (two files for pairs) -> dict(n_reads, codes, offsets, quals, names, d_codes, d_offsets);
        the device pointers stay valid until the context's next call."""
        b = FastqBatch()
        f = lib().bm2_fastq_encode
        f.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_void_p]
        self._check(f(self._ctx, buf1, len(buf1), buf2, len(buf2) if buf2 is not None else 0, C.byref(b)), "bm2_fastq_encode")
        return self._fq_batch(b, buf1, buf2, want_names)

    def _fq_batch(self, b, buf1, buf2, want_names):
        n = b.n_reads
        self._fq_n = n
        offs = np.ctypeslib.as_array(C.cast(b.offsets, C.POINTER(C.c_int64)), shape=(n + 1,)).copy()
        tot = int(offs[-1])
        codes = np.ctypeslib.as_array(C.cast(b.codes, C.POINTER(C.c_uint8)), shape=(max(tot, 1),))[:tot].copy()
        quals = np.ctypeslib.as_array(C.cast(b.quals, C.POINTER(C.c_uint8)), shape=(max(tot, 1),))[:tot].copy()
        nb = np.ctypeslib.as_array(C.cast(b.name_beg, C.POINTER(C.c_int64)), shape=(max(n, 1),))[:n].copy()
        nl = np.ctypeslib.as_array(C.cast(b.name_len, C.POINTER(C.c_int32)), shape=(max(n, 1),))[:n].copy()
        bufs = (buf1, buf2 if buf2 is not None else buf1)
        stride = 2 if buf2 is not None else 1
        names = [bufs[r % stride][nb[r]:nb[r] + nl[r]] for r in range(n)] if want_names else None
        return dict(n_reads=n, codes=codes, offsets=offs, quals=quals, names=names, d_codes=b.d_codes, d_offsets=b.d_offsets,
                    name_spans=(buf1, buf2, nb, nl))

    def seq_encode(self, buf1: bytes, buf2: bytes | None = None, want_names: bool = True):
        """bm2_seq_encode: raw bytes of whole FASTA / FASTQ records of a chunk (two files for pairs), any shape kseq reads -> the dict of
        fastq_encode plus qual_present (uint8 per read, 0: no qualities; their bytes in quals are then unset)."""
        b = FastqBatch(); qp = C.c_void_p()
        f = lib().bm2_seq_encode
        f.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, buf1, len(buf1), buf2, len(buf2) if buf2 is not None else 0, C.byref(b), C.byref(qp)), "bm2_seq_encode")
        out = self._fq_batch(b, buf1, buf2, want_names)
        out["qual_present"] = _host(qp, out["n_reads"], np.uint8)
        return out

    def fastq_comments(self):
        """bm2_fastq_comments: (comment_beg int64[], comment_len int32[]) of the reads of the last fastq_encode, into their buffers."""
        beg = C.c_void_p(); ln = C.c_void_p()
        f = lib().bm2_fastq_comments
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, C.byref(beg), C.byref(ln)), "bm2_fastq_comments")
        n = self._fq_n
        return _host(beg, n, np.int64), _host(ln, n, np.int32)

    def fastq_smart_pair(self):
        """bm2_fastq_smart_pair: the last single-end fastq_encode batch split as bseq_classify does -> two dicts (single-end reads, pairs) with
        n_reads, codes, offsets, quals, name_beg, name_len, comment_beg, comment_len, read_index, d_codes, d_offsets."""
        sp = FastqSplit()
        f = lib().bm2_fastq_smart_pair
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, C.byref(sp)), "bm2_fastq_smart_pair")
        out = []
        for s in range(2):
            b = sp.set[s]; n = b.n_reads
            offs = _host(b.offsets, n + 1, np.int64); tot = int(offs[-1])
            out.append(dict(n_reads=n, offsets=offs, codes=_host(b.codes, tot, np.uint8), quals=_host(b.quals, tot, np.uint8),
                            name_beg=_host(b.name_beg, n, np.int64), name_len=_host(b.name_len, n, np.int32),
                            comment_beg=_host(sp.comment_beg[s], n, np.int64), comment_len=_host(sp.comment_len[s], n, np.int32),
                            read_index=_host(sp.read_index[s], n, np.int32), d_codes=b.d_codes, d_offsets=b.d_offsets))
        return out

    def bgzf_compress(self, data: bytes, cut=None):
        """bm2_bgzf_compress: BGZF members of data (bytes) on this context's GPU, blocks cut at the record starts cut (int64[], ascending; None:
        one record) by htslib's rule -> (members bytes, device ms, member count).  No EOF block."""
        cut = np.ascontiguousarray(cut if cut is not None else np.zeros(0), np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        out = C.c_void_p(); n = C.c_int64()
        f = lib().bm2_bgzf_compress
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, buf.ctypes.data, len(data), cut.ctypes.data, len(cut), C.byref(out), C.byref(n)), "bm2_bgzf_compress")
        ms = C.c_double(); m = C.c_int64()
        lib().bm2_last_bgzf_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib().bm2_last_bgzf_stats(self._ctx, C.byref(ms), C.byref(m))
        return (C.string_at(out, n.value) if n.value else b""), ms.value, m.value

    def bam_sort_compress(self, data: bytes, starts, carry: bytes = b"", last: bool = True):
        """bm2_bam_sort_compress: the records of data (uncompressed BAM) starting at starts, stably sorted by the coordinate key and compressed
        after carry -> dict(z: whole members, member_size, carry: the unfinished block's bytes, recs: SORT_REC_DT in output order,
        ms: device ms of keys, sort, gather, BGZF)."""
        starts = np.ascontiguousarray(starts, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        cb = np.frombuffer(carry, np.uint8) if len(carry) else np.zeros(1, np.uint8)
        o = SortOut()
        f = lib().bm2_bam_sort_compress
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
        self._check(f(self._ctx, buf.ctypes.data, len(data), starts.ctypes.data, len(starts), cb.ctypes.data, len(carry), int(last), C.byref(o)),
                    "bm2_bam_sort_compress")
        ms = (C.c_double * 4)()
        lib().bm2_last_sort_stats.argtypes = [C.c_void_p, C.c_void_p]
        lib().bm2_last_sort_stats(self._ctx, ms)
        recs = np.ctypeslib.as_array(C.cast(o.recs, C.POINTER(C.c_uint8)), shape=(o.n_recs * SORT_REC_DT.itemsize,)).view(SORT_REC_DT).copy() \
            if o.n_recs else np.zeros(0, SORT_REC_DT)
        sizes = _host(o.member_size, o.n_members, np.int32) if o.n_members else np.zeros(0, np.int32)
        return dict(z=C.string_at(o.z, o.z_len) if o.z_len else b"", member_size=sizes, carry=C.string_at(o.carry, o.carry_len) if o.carry_len else b"",
                    recs=recs, ms=dict(keys=ms[0], sort=ms[1], gather=ms[2], bgzf=ms[3]))

    def bam_qname_sort_compress(self, data: bytes, starts, carry: bytes = b"", last: bool = True):
        """bm2_bam_qname_sort_compress: bam_sort_compress in read-name order (samtools sort -n: the names by samtools' strnum_cmp, then
        flag & 0xc0, then input order) -> bam_sort_compress's dict (ms: device ms of keys, merge sort, gather, BGZF)."""
        starts = np.ascontiguousarray(starts, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        cb = np.frombuffer(carry, np.uint8) if len(carry) else np.zeros(1, np.uint8)
        o = SortOut()
        f = lib().bm2_bam_qname_sort_compress
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
        self._check(f(self._ctx, buf.ctypes.data, len(data), starts.ctypes.data, len(starts), cb.ctypes.data, len(carry), int(last), C.byref(o)),
                    "bm2_bam_qname_sort_compress")
        ms = (C.c_double * 4)()
        lib().bm2_last_sort_stats.argtypes = [C.c_void_p, C.c_void_p]
        lib().bm2_last_sort_stats(self._ctx, ms)
        recs = np.ctypeslib.as_array(C.cast(o.recs, C.POINTER(C.c_uint8)), shape=(o.n_recs * SORT_REC_DT.itemsize,)).view(SORT_REC_DT).copy() \
            if o.n_recs else np.zeros(0, SORT_REC_DT)
        sizes = _host(o.member_size, o.n_members, np.int32) if o.n_members else np.zeros(0, np.int32)
        return dict(z=C.string_at(o.z, o.z_len) if o.z_len else b"", member_size=sizes, carry=C.string_at(o.carry, o.carry_len) if o.carry_len else b"",
                    recs=recs, ms=dict(keys=ms[0], sort=ms[1], gather=ms[2], bgzf=ms[3]))

    def bam_qname_sort_memory(self, run_bytes: int):
        """bm2_bam_qname_sort_memory -> (bytes needed, bytes free)."""
        need, free = C.c_int64(), C.c_int64()
        f = lib().bm2_bam_qname_sort_memory
        f.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, int(run_bytes), C.byref(need), C.byref(free)), "bm2_bam_qname_sort_memory")
        return need.value, free.value

    def bam_sort_compress_ex(self, data: bytes, starts, tids, carry: bytes = b"", last: bool = True):
        """bm2_bam_sort_compress_ex: bam_sort_compress with each record's template id (int64[]) carried through the sort; records of the
        templates set by dup_set get 0x400 unless unmapped -> bam_sort_compress's dict plus tids (int64[], output order)."""
        starts = np.ascontiguousarray(starts, np.int64); tids = np.ascontiguousarray(tids, np.int64)
        assert len(tids) == len(starts)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        cb = np.frombuffer(carry, np.uint8) if len(carry) else np.zeros(1, np.uint8)
        tb = tids if len(tids) else np.zeros(1, np.int64)
        o = SortOut(); to = C.c_void_p()
        f = lib().bm2_bam_sort_compress_ex
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, buf.ctypes.data, len(data), starts.ctypes.data, len(starts), tb.ctypes.data, cb.ctypes.data, len(carry), int(last),
                      C.byref(o), C.byref(to)), "bm2_bam_sort_compress_ex")
        ms = (C.c_double * 4)()
        lib().bm2_last_sort_stats.argtypes = [C.c_void_p, C.c_void_p]
        lib().bm2_last_sort_stats(self._ctx, ms)
        recs = np.ctypeslib.as_array(C.cast(o.recs, C.POINTER(C.c_uint8)), shape=(o.n_recs * SORT_REC_DT.itemsize,)).view(SORT_REC_DT).copy() \
            if o.n_recs else np.zeros(0, SORT_REC_DT)
        sizes = _host(o.member_size, o.n_members, np.int32) if o.n_members else np.zeros(0, np.int32)
        return dict(z=C.string_at(o.z, o.z_len) if o.z_len else b"", member_size=sizes, carry=C.string_at(o.carry, o.carry_len) if o.carry_len else b"",
                    recs=recs, tids=_host(to.value, o.n_recs, np.int64) if o.n_recs else np.zeros(0, np.int64),
                    ms=dict(keys=ms[0], sort=ms[1], gather=ms[2], bgzf=ms[3]))

    def dup_signatures(self, data: bytes, starts, tmpl_first, tmpl_id):
        """bm2_dup_signatures: the entries of the templates [tmpl_first[t], tmpl_first[t+1]) of the records of data (uncompressed BAM) starting
        at starts, with ids tmpl_id -> (pair entries, fragment-space entries, device ms), DUP_ENTRY_DT in template order."""
        starts = np.ascontiguousarray(starts, np.int64); tf = np.ascontiguousarray(tmpl_first, np.int64); ti = np.ascontiguousarray(tmpl_id, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        sb = starts if len(starts) else np.zeros(1, np.int64)
        tib = ti if len(ti) else np.zeros(1, np.int64)
        p, f_ = C.c_void_p(), C.c_void_p(); n_p, n_f = C.c_int64(), C.c_int64()
        f = lib().bm2_dup_signatures
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64] + [C.c_void_p] * 4
        self._check(f(self._ctx, buf.ctypes.data, len(data), sb.ctypes.data, len(starts), tf.ctypes.data, tib.ctypes.data, len(ti),
                      C.byref(p), C.byref(n_p), C.byref(f_), C.byref(n_f)), "bm2_dup_signatures")
        ms = C.c_double()
        lib().bm2_last_dup_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib().bm2_last_dup_stats(self._ctx, C.byref(ms), None)
        return (_host(p.value, n_p.value, DUP_ENTRY_DT) if n_p.value else np.zeros(0, DUP_ENTRY_DT),
                _host(f_.value, n_f.value, DUP_ENTRY_DT) if n_f.value else np.zeros(0, DUP_ENTRY_DT), ms.value)

    def dup_resolve(self, entries, resolve: bool = True):
        """bm2_dup_resolve: entries (DUP_ENTRY_DT) of one space sorted by (k1, k2, score descending, tid) -> (the sorted entries, device ms)
        when not resolve, else (the duplicates' template ids in sorted order, device ms)."""
        e = np.ascontiguousarray(entries, DUP_ENTRY_DT)
        eb = e if len(e) else np.zeros(1, DUP_ENTRY_DT)
        srt, d = C.c_void_p(), C.c_void_p(); nd = C.c_int64()
        f = lib().bm2_dup_resolve
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, eb.ctypes.data, len(e), int(resolve), None if resolve else C.byref(srt), C.byref(d) if resolve else None,
                      C.byref(nd) if resolve else None), "bm2_dup_resolve")
        ms = C.c_double()
        lib().bm2_last_dup_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib().bm2_last_dup_stats(self._ctx, None, C.byref(ms))
        if resolve:
            return (_host(d.value, nd.value, np.int64) if nd.value else np.zeros(0, np.int64)), ms.value
        return (_host(srt.value, len(e), DUP_ENTRY_DT) if len(e) else np.zeros(0, DUP_ENTRY_DT)), ms.value

    def dup_signatures_ex(self, data: bytes, starts, tmpl_first, tmpl_id):
        """bm2_dup_signatures_ex: dup_signatures with the pair entries located -> (pair entries DUP_LOC_ENTRY_DT, fragment-space entries
        DUP_ENTRY_DT, (secondary or supplementary records, unmapped primaries), device ms)."""
        starts = np.ascontiguousarray(starts, np.int64); tf = np.ascontiguousarray(tmpl_first, np.int64); ti = np.ascontiguousarray(tmpl_id, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        sb = starts if len(starts) else np.zeros(1, np.int64)
        tib = ti if len(ti) else np.zeros(1, np.int64)
        p, f_ = C.c_void_p(), C.c_void_p(); n_p, n_f = C.c_int64(), C.c_int64()
        counts = np.zeros(2, np.int64)
        f = lib().bm2_dup_signatures_ex
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64] + [C.c_void_p] * 5
        self._check(f(self._ctx, buf.ctypes.data, len(data), sb.ctypes.data, len(starts), tf.ctypes.data, tib.ctypes.data, len(ti),
                      C.byref(p), C.byref(n_p), C.byref(f_), C.byref(n_f), counts.ctypes.data), "bm2_dup_signatures_ex")
        ms = C.c_double()
        lib().bm2_last_dup_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib().bm2_last_dup_stats(self._ctx, C.byref(ms), None)
        return (_host(p.value, n_p.value, DUP_LOC_ENTRY_DT) if n_p.value else np.zeros(0, DUP_LOC_ENTRY_DT),
                _host(f_.value, n_f.value, DUP_ENTRY_DT) if n_f.value else np.zeros(0, DUP_ENTRY_DT), (int(counts[0]), int(counts[1])), ms.value)

    def dup_resolve_ex(self, entries, distance: int = 100, resolve: bool = True):
        """bm2_dup_resolve_ex: located entries (DUP_LOC_ENTRY_DT) of one space -> (the sorted located entries, device ms) when not resolve,
        else (the duplicates' template ids in sorted order, the optical count at pixel distance `distance`, device ms)."""
        e = np.ascontiguousarray(entries, DUP_LOC_ENTRY_DT)
        eb = e if len(e) else np.zeros(1, DUP_LOC_ENTRY_DT)
        srt, d = C.c_void_p(), C.c_void_p(); nd, nopt = C.c_int64(), C.c_int64()
        f = lib().bm2_dup_resolve_ex
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, eb.ctypes.data, len(e), int(resolve), int(distance), None if resolve else C.byref(srt), C.byref(d) if resolve else None,
                      C.byref(nd) if resolve else None, C.byref(nopt) if resolve else None), "bm2_dup_resolve_ex")
        ms = C.c_double()
        lib().bm2_last_dup_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib().bm2_last_dup_stats(self._ctx, None, C.byref(ms))
        if resolve:
            return (_host(d.value, nd.value, np.int64) if nd.value else np.zeros(0, np.int64)), nopt.value, ms.value
        return (_host(srt.value, len(e), DUP_LOC_ENTRY_DT) if len(e) else np.zeros(0, DUP_LOC_ENTRY_DT)), ms.value

    def dup_set(self, dup_tids, n_bits: int):
        """bm2_dup_set: the bitset of n_bits bits with the templates dup_tids set, kept on this context for bam_sort_compress_ex."""
        bits = np.zeros(max((n_bits + 63) // 64, 1), np.uint64)
        for t in np.asarray(dup_tids, np.int64):
            bits[t >> 6] |= np.uint64(1) << np.uint64(t & 63)
        f = lib().bm2_dup_set
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        self._check(f(self._ctx, bits.ctypes.data, int(n_bits)), "bm2_dup_set")

    def bqsr_sites(self, covered, junction, n_bits: int, holes, read_group: str):
        """bm2_bqsr_sites: the known-site bitsets (uint64 words, n_bits = the index's l_pac), the .amb holes ([beg, end) pairs) and the read
        group to this context (which must hold an index); zeroes the counts and arms counting."""
        cov = np.ascontiguousarray(covered, np.uint64); jun = np.ascontiguousarray(junction, np.uint64)
        h = np.ascontiguousarray(holes, np.int64).reshape(-1)
        hb = h if len(h) else np.zeros(2, np.int64)
        f = lib().bm2_bqsr_sites
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_char_p]
        self._check(f(self._ctx, cov.ctypes.data, jun.ctypes.data, int(n_bits), hb.ctypes.data, len(h) // 2, read_group.encode()), "bm2_bqsr_sites")

    def bqsr_count(self, data: bytes, starts):
        """bm2_bqsr_count: counts the records of data (uncompressed BAM) starting at starts."""
        starts = np.ascontiguousarray(starts, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        sb = starts if len(starts) else np.zeros(1, np.int64)
        f = lib().bm2_bqsr_count
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        self._check(f(self._ctx, buf.ctypes.data, len(data), sb.ctypes.data, len(starts)), "bm2_bqsr_count")

    def bqsr_tables(self):
        """bm2_bqsr_tables -> dict(qual_obs/qual_err [94], ctx_obs/ctx_err [94, 16], cyc_obs/cyc_err [94, 1001] (cycle + 500), reads, bases,
        ms, err_kind, err_index, err_name, read_group)."""
        t = BqsrTables()
        f = lib().bm2_bqsr_tables
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, C.byref(t)), "bm2_bqsr_tables")
        out = dict(reads=t.reads, bases=t.bases, ms=t.ms, err_kind=t.err_kind, err_index=t.err_index,
                   err_name=(t.err_name or b"").decode(), read_group=(t.read_group or b"").decode())
        for k, shape in (("qual", (BQSR_NQ,)), ("ctx", (BQSR_NQ, BQSR_NCTX)), ("cyc", (BQSR_NQ, BQSR_NCYC))):
            for s in ("obs", "err"):
                out[k + "_" + s] = _host(getattr(t, k + "_" + s), int(np.prod(shape)), np.int64).reshape(shape)
        return out

    def recal_memory(self, l_pac: int, window_bytes: int, n_cov: int):
        """bm2_recal_memory -> (bytes needed, bytes free)."""
        need, free = C.c_int64(), C.c_int64()
        f = lib().bm2_recal_memory
        f.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, int(l_pac), int(window_bytes), int(n_cov), C.byref(need), C.byref(free)), "bm2_recal_memory")
        return need.value, free.value

    def recal_set(self, contig_off, contig_len, l_pac: int, pac, holes, covered, junction, ids, id_cov, n_cov: int):
        """bm2_recal_set: the contigs, the packed reference ((l_pac + 3) // 4 bytes), the .amb holes ([beg, end) pairs), the known-site bitsets
        (uint64 words), the @RG IDs with each one's covariate, and the covariate count; zeroes the counts."""
        self._recal_keep = [np.ascontiguousarray(contig_off, np.int64), np.ascontiguousarray(contig_len, np.int32), np.ascontiguousarray(pac, np.uint8),
                            np.ascontiguousarray(holes, np.int64).reshape(-1), np.ascontiguousarray(covered, np.uint64),
                            np.ascontiguousarray(junction, np.uint64), np.ascontiguousarray(list(id_cov) + [0], np.int32)]
        off, ln, pb, h, cov, jun, ic = self._recal_keep
        names = (C.c_char_p * max(len(ids), 1))(*[i.encode() for i in ids])
        self._recal_keep.append(names)
        s = RecalSet(len(off), off.ctypes.data, ln.ctypes.data, int(l_pac), pb.ctypes.data, h.ctypes.data if len(h) else None, len(h) // 2,
                     cov.ctypes.data, jun.ctypes.data, len(ids), C.cast(names, C.c_void_p) if ids else None, ic.ctypes.data, int(n_cov))
        f = lib().bm2_recal_set
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, C.byref(s)), "bm2_recal_set")

    def recal_add(self, data: bytes, starts):
        """bm2_recal_add: one window of records (uncompressed BAM at starts, any order).  A read error raises Bm2Error naming the read (the
        tables still report it)."""
        starts = np.ascontiguousarray(starts, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        sb = starts if len(starts) else np.zeros(1, np.int64)
        f = lib().bm2_recal_add
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        self._check(f(self._ctx, buf.ctypes.data, len(data), sb.ctypes.data, len(starts)), "bm2_recal_add")

    def recal_tables(self, cov: int):
        """bm2_recal_tables -> bqsr_tables's dict for covariate cov (read_group empty)."""
        t = BqsrTables()
        f = lib().bm2_recal_tables
        f.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        self._check(f(self._ctx, int(cov), C.byref(t)), "bm2_recal_tables")
        out = dict(reads=t.reads, bases=t.bases, ms=t.ms, err_kind=t.err_kind, err_index=t.err_index, err_name=(t.err_name or b"").decode())
        for k, shape in (("qual", (BQSR_NQ,)), ("ctx", (BQSR_NQ, BQSR_NCTX)), ("cyc", (BQSR_NQ, BQSR_NCYC))):
            for s in ("obs", "err"):
                out[k + "_" + s] = _host(getattr(t, k + "_" + s), int(np.prod(shape)), np.int64).reshape(shape)
        return out

    def bqsr_apply_set(self, P, ctx, cyc, ids, id_table):
        """bm2_bqsr_apply_set: the dense tables (float64 [n_rg, 94], [n_rg, 94, 16], [n_rg, 94, 1001]) and the header's @RG IDs with each
        one's table index (-1: none)."""
        self._apply_keep = [np.ascontiguousarray(P, np.float64).reshape(-1), np.ascontiguousarray(ctx, np.float64).reshape(-1),
                            np.ascontiguousarray(cyc, np.float64).reshape(-1), np.ascontiguousarray(id_table, np.int32)]
        p, c, y, tb = self._apply_keep
        names = (C.c_char_p * max(len(ids), 1))(*[i.encode() for i in ids])
        t = BqsrApplyTables(len(p) // BQSR_NQ, p.ctypes.data if len(p) else None, c.ctypes.data if len(c) else None, y.ctypes.data if len(y) else None,
                            len(ids), C.cast(names, C.c_void_p) if ids else None, tb.ctypes.data if len(tb) else None)
        f = lib().bm2_bqsr_apply_set
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, C.byref(t)), "bm2_bqsr_apply_set")

    def bqsr_apply(self, data: bytes, starts, carry: bytes = b"", last: bool = True):
        """bm2_bqsr_apply: the contiguous records of data recalibrated and compressed after carry -> bam_sort_compress's dict (z, member_size,
        carry, recs in input order)."""
        starts = np.ascontiguousarray(starts, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        sb = starts if len(starts) else np.zeros(1, np.int64)
        cb = np.frombuffer(carry, np.uint8) if len(carry) else np.zeros(1, np.uint8)
        o = SortOut()
        f = lib().bm2_bqsr_apply
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
        self._check(f(self._ctx, buf.ctypes.data, len(data), sb.ctypes.data, len(starts), cb.ctypes.data, len(carry), int(last), C.byref(o)),
                    "bm2_bqsr_apply")
        recs = np.ctypeslib.as_array(C.cast(o.recs, C.POINTER(C.c_uint8)), shape=(o.n_recs * SORT_REC_DT.itemsize,)).view(SORT_REC_DT).copy() \
            if o.n_recs else np.zeros(0, SORT_REC_DT)
        sizes = _host(o.member_size, o.n_members, np.int32) if o.n_members else np.zeros(0, np.int32)
        return dict(z=C.string_at(o.z, o.z_len) if o.z_len else b"", member_size=sizes, carry=C.string_at(o.carry, o.carry_len) if o.carry_len else b"",
                    recs=recs)

    def bqsr_apply_stats(self):
        """bm2_last_bqsr_apply_stats -> dict(apply_ms, bgzf_ms, bases_changed, recal_records, kept_records, err_kind, err_index, err_name)."""
        s = BqsrApplyStats()
        f = lib().bm2_last_bqsr_apply_stats
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, C.byref(s)), "bm2_last_bqsr_apply_stats")
        out = {k: getattr(s, k) for k, _ in s._fields_}
        out["err_name"] = (s.err_name or b"").decode()
        return out

    def wgs_set(self, contig_off, contig_len, l_pac: int, nocall, min_mapq=20, min_baseq=20, coverage_cap=250, count_unpaired=False):
        """bm2_wgs_set: one coverage counter per reference base, the no-call ranges ([beg, end) pairs) and Picard's parameters."""
        off = np.ascontiguousarray(contig_off, np.int64); ln = np.ascontiguousarray(contig_len, np.int32)
        h = np.ascontiguousarray(nocall, np.int64).reshape(-1)
        hb = h if len(h) else np.zeros(2, np.int64)
        p = WgsParams(int(min_mapq), int(min_baseq), int(coverage_cap), int(bool(count_unpaired)))
        f = lib().bm2_wgs_set
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
        self._check(f(self._ctx, off.ctypes.data if len(off) else None, ln.ctypes.data if len(ln) else None, len(off), int(l_pac), hb.ctypes.data,
                      len(h) // 2, C.byref(p)), "bm2_wgs_set")

    def wgs_memory(self, l_pac: int, window_bytes: int):
        """bm2_wgs_memory -> (bytes needed, bytes free)."""
        need, free = C.c_int64(), C.c_int64()
        f = lib().bm2_wgs_memory
        f.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, int(l_pac), int(window_bytes), C.byref(need), C.byref(free)), "bm2_wgs_memory")
        return need.value, free.value

    def wgs_add(self, data: bytes, starts):
        """bm2_wgs_add: one window of records (uncompressed BAM at starts, in file order).  A read error raises Bm2Error naming the read."""
        starts = np.ascontiguousarray(starts, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        sb = starts if len(starts) else np.zeros(1, np.int64)
        f = lib().bm2_wgs_add
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        self._check(f(self._ctx, buf.ctypes.data, len(data), sb.ctypes.data, len(starts)), "bm2_wgs_add")

    def wgs_finish(self):
        """bm2_wgs_finish -> dict(hist [cap + 1], exc [6]: MAPQ, DUPE, UNPAIRED, BASEQ, OVERLAP, CAPPED, records, counted_records, carried_max,
        add_ms, finish_ms)."""
        r = WgsResult()
        f = lib().bm2_wgs_finish
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, C.byref(r)), "bm2_wgs_finish")
        return dict(hist=_host(r.hist, r.cap + 1, np.int64), exc=[int(x) for x in r.exc], records=r.records, counted_records=r.counted_records,
                    carried_max=r.carried_max, add_ms=r.add_ms, finish_ms=r.finish_ms)

    def mm_set(self, contig_off, contig_len, l_pac: int, pac, holes, hole_char: bytes):
        """bm2_mm_set: the contigs, the packed reference ((l_pac + 3) // 4 bytes) and the .amb holes ([beg, end) pairs, one letter each)."""
        off = np.ascontiguousarray(contig_off, np.int64); ln = np.ascontiguousarray(contig_len, np.int32)
        pb = np.ascontiguousarray(pac, np.uint8)
        h = np.ascontiguousarray(holes, np.int64).reshape(-1)
        hb = h if len(h) else np.zeros(2, np.int64)
        f = lib().bm2_mm_set
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int64]
        self._check(f(self._ctx, off.ctypes.data if len(off) else None, ln.ctypes.data if len(ln) else None, len(off), int(l_pac), pb.ctypes.data,
                      hb.ctypes.data, bytes(hole_char), len(h) // 2), "bm2_mm_set")

    def mm_memory(self, l_pac: int, window_bytes: int):
        """bm2_mm_memory -> (bytes needed, bytes free)."""
        need, free = C.c_int64(), C.c_int64()
        f = lib().bm2_mm_memory
        f.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, int(l_pac), int(window_bytes), C.byref(need), C.byref(free)), "bm2_mm_memory")
        return need.value, free.value

    def markdup_set(self, ids, libs, n_lib: int, unknown_lib: int):
        """bm2_markdup_set: the merged header's @RG IDs, each one's library index, the library count and the unknown library's index."""
        self._mdb_keep = np.ascontiguousarray(list(libs) + [0], np.int32)
        names = (C.c_char_p * max(len(ids), 1))(*[i.encode() for i in ids])
        f = lib().bm2_markdup_set
        f.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
        self._check(f(self._ctx, len(ids), C.cast(names, C.c_void_p), self._mdb_keep.ctypes.data, int(n_lib), int(unknown_lib)), "bm2_markdup_set")

    def markdup_records(self, data: bytes, starts):
        """bm2_markdup_records: one window of records (uncompressed BAM at starts, contiguous) -> structured array of bm2_markdup_rec
        (end, hash, score, kind, rg, lib, tile, x, y, loc)."""
        starts = np.ascontiguousarray(starts, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        sb = starts if len(starts) else np.zeros(1, np.int64)
        out = C.c_void_p()
        f = lib().bm2_markdup_records
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
        self._check(f(self._ctx, buf.ctypes.data, len(data), sb.ctypes.data, len(starts), C.byref(out)), "bm2_markdup_records")
        dt = np.dtype([("end", "<u8"), ("hash", "<u8"), ("score", "<i4"), ("kind", "<i4"), ("rg", "<i4"), ("lib", "<i4"), ("tile", "<i4"), ("x", "<i4"), ("y", "<i4"),
                       ("loc", "<i4")])
        if not len(starts):
            return np.zeros(0, dt)
        return np.frombuffer((C.c_uint8 * (len(starts) * dt.itemsize)).from_address(out.value), dt).copy()

    def markdup_pair(self, halves, names: bytes):
        """bm2_markdup_pair: halves (structured: hash u8, rg i4, name_len i4, name_off i8) and their names -> each one's partner or -1."""
        h = np.ascontiguousarray(halves)
        buf = np.frombuffer(names + b"\0", np.uint8)
        out = C.c_void_p()
        f = lib().bm2_markdup_pair
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
        self._check(f(self._ctx, h.ctypes.data if len(h) else None, len(h), buf.ctypes.data, len(names), C.byref(out)), "bm2_markdup_pair")
        if not len(h):
            return []
        return np.frombuffer((C.c_int32 * len(h)).from_address(out.value), np.int32).tolist()

    def markdup_counts(self, n_lib: int):
        """bm2_markdup_counts -> int64 [n_lib, 2]: secondary or supplementary records, unmapped primaries."""
        c = np.zeros(2 * n_lib, np.int64)
        f = lib().bm2_markdup_counts
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, c.ctypes.data), "bm2_markdup_counts")
        return c.reshape(-1, 2)

    def markdup_stats(self):
        """bm2_last_markdup_stats -> (records_ms, pair_ms, mark_ms, bgzf_ms)."""
        v = (C.c_double * 4)()
        f = lib().bm2_last_markdup_stats
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, v), "bm2_last_markdup_stats")
        return tuple(v)

    def bam2fq_records(self, data: bytes, starts, suffixes: bool):
        """bm2_bam2fq_records: one window of records (uncompressed BAM at starts, contiguous) -> structured array of bm2_bam2fq_rec
        (hash, text_len, kind).  The window stays on the device for bam2fq_format.  A read error raises Bm2Error naming the read."""
        starts = np.ascontiguousarray(starts, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        sb = starts if len(starts) else np.zeros(1, np.int64)
        out = C.c_void_p()
        f = lib().bm2_bam2fq_records
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]
        self._check(f(self._ctx, buf.ctypes.data, len(data), sb.ctypes.data, len(starts), int(bool(suffixes)), C.byref(out)), "bm2_bam2fq_records")
        dt = np.dtype([("hash", "<u8"), ("text_len", "<i8"), ("kind", "<i4"), ("pad", "<i4")])
        if not len(starts):
            return np.zeros(0, dt)
        return np.frombuffer((C.c_uint8 * (len(starts) * dt.itemsize)).from_address(out.value), dt).copy()

    def bam2fq_format(self, order, extra_recs, suffixes: bool, carry: bytes = b"", compress: bool = False, last: bool = True):
        """bm2_bam2fq_format: order lists record i of the last bam2fq_records window as i and record k of extra_recs (a list of record
        bytes) as ~k -> (data, tail, text_len): the text, or with compress the BGZF members and the unfinished block."""
        lst = np.ascontiguousarray(list(order) + [0], np.int64)
        xb = b"".join(extra_recs)
        xbuf = np.frombuffer(xb + b"\0", np.uint8)
        xs = np.ascontiguousarray(np.cumsum([0] + [len(r) for r in extra_recs])[:-1].tolist() + [0], np.int64)
        cb = np.frombuffer(carry + b"\0", np.uint8)

        class Out(C.Structure):
            _fields_ = [("data", C.c_void_p), ("len", C.c_int64), ("tail", C.c_void_p), ("tail_len", C.c_int64), ("text_len", C.c_int64)]
        o = Out()
        f = lib().bm2_bam2fq_format
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_int32,
                      C.c_int32, C.c_void_p]
        self._check(f(self._ctx, lst.ctypes.data, len(lst) - 1, xbuf.ctypes.data, len(xb), xs.ctypes.data, len(extra_recs), int(bool(suffixes)),
                      cb.ctypes.data, len(carry), int(bool(compress)), int(bool(last)), C.byref(o)), "bm2_bam2fq_format")
        data = C.string_at(o.data, o.len) if o.len else b""
        tail = C.string_at(o.tail, o.tail_len) if o.tail_len else b""
        return data, tail, int(o.text_len)

    def bam2fq_stats(self):
        """bm2_last_bam2fq_stats -> (record_ms, format_ms, bgzf_ms)."""
        v = (C.c_double * 3)()
        f = lib().bm2_last_bam2fq_stats
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, v), "bm2_last_bam2fq_stats")
        return tuple(v)

    def mm_add(self, data: bytes, starts):
        """bm2_mm_add: one window of records (uncompressed BAM at starts, any order).  A read error raises Bm2Error naming the read."""
        starts = np.ascontiguousarray(starts, np.int64)
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        sb = starts if len(starts) else np.zeros(1, np.int64)
        f = lib().bm2_mm_add
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        self._check(f(self._ctx, buf.ctypes.data, len(data), sb.ctypes.data, len(starts)), "bm2_mm_add")

    def mm_finish(self):
        """bm2_mm_finish -> dict(counts [3, 21], len_hist / mism_hist / nocall [3, max_len + 1], insert_hist [3, max_insert + 1], insert_big
        (orientation << 32 | size, sorted), records, add_ms, finish_ms)."""
        r = MmResult()
        f = lib().bm2_mm_finish
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, C.byref(r)), "bm2_mm_finish")
        L, I = r.max_len + 1, r.max_insert + 1
        return dict(counts=np.array(r.counts, np.int64).reshape(3, 21), len_hist=_host(r.len_hist, 3 * L, np.int64).reshape(3, L),
                    mism_hist=_host(r.mism_hist, 3 * L, np.int64).reshape(3, L), nocall=_host(r.nocall, 3 * L, np.int64).reshape(3, L),
                    insert_hist=_host(r.insert_hist, 3 * I, np.int64).reshape(3, I),
                    insert_big=_host(r.insert_big, r.n_big, np.uint64) if r.n_big else np.zeros(0, np.uint64), records=r.records,
                    add_ms=r.add_ms, finish_ms=r.finish_ms)

    def mm_gc_set(self):
        """bm2_mm_gc_set: after mm_set, bins the reference's windows by GC and counts GC bias in the mm_add calls that follow."""
        f = lib().bm2_mm_gc_set
        f.argtypes = [C.c_void_p]
        self._check(f(self._ctx), "bm2_mm_gc_set")

    def mm_gc_memory(self, window_bytes: int):
        """bm2_mm_gc_memory -> the device bytes GC bias adds to mm_memory's figure."""
        need = C.c_int64()
        f = lib().bm2_mm_gc_memory
        f.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
        self._check(f(self._ctx, int(window_bytes), C.byref(need)), "bm2_mm_gc_memory")
        return need.value

    def mm_gc_finish(self):
        """bm2_mm_gc_finish -> dict(windows, reads, bases, errors [101] each, total_clusters, aligned_reads, scan_ms, add_ms)."""
        r = MmGcResult()
        f = lib().bm2_mm_gc_finish
        f.argtypes = [C.c_void_p, C.c_void_p]
        self._check(f(self._ctx, C.byref(r)), "bm2_mm_gc_finish")
        return dict(windows=np.array(r.windows, np.int64), reads=np.array(r.reads, np.int64), bases=np.array(r.bases, np.int64),
                    errors=np.array(r.errors, np.int64), total_clusters=r.total_clusters, aligned_reads=r.aligned_reads, scan_ms=r.scan_ms,
                    add_ms=r.add_ms)

    def set_sam_staged(self, on: int):
        """bm2_set_sam_staged: 1 / 2 = the rescue's local alignments as a batch (one window per warp / per thread) before the per-pair kernel, 0 = inside it."""
        lib().bm2_set_sam_staged.argtypes = [C.c_void_p, C.c_int]
        self._check(lib().bm2_set_sam_staged(self._ctx, int(on)), "bm2_set_sam_staged")

    def last_sam_stats(self):
        """bm2_last_sam_stats -> dict: device ms of the last bm2_sam_pe / bm2_sam_se call (jobs, ksw, pairs, gather) and the rescue counters."""
        ms = (C.c_double * 4)(); cnt = (C.c_ulonglong * 6)()
        lib().bm2_last_sam_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        self._check(lib().bm2_last_sam_stats(self._ctx, ms, cnt, 4, 6), "bm2_last_sam_stats")
        return {"ms": {"jobs": ms[0], "ksw": ms[1], "pairs": ms[2], "gather_and_copies": ms[3]}, "staged": int(cnt[0]), "jobs": int(cnt[1]),
                "looked_up": int(cnt[2]), "in_place": int(cnt[3]), "window_moved": int(cnt[4]), "waves": int(cnt[5])}

    def set_stream(self, cuda_stream_handle):
        lib().bm2_set_stream.argtypes = [C.c_void_p, C.c_void_p]
        self._check(lib().bm2_set_stream(self._ctx, cuda_stream_handle), "bm2_set_stream")

    def gather64_gbs(self, span_bytes: int = 0) -> float:
        v = C.c_double()
        lib().bm2_gather64_gbs.argtypes = [C.c_void_p, C.c_ulonglong, C.POINTER(C.c_double)]
        self._check(lib().bm2_gather64_gbs(self._ctx, int(span_bytes), C.byref(v)), "bm2_gather64_gbs")
        return v.value

    def gather_probe(self, span_bytes: int = 0, mlp: int = 4, shape: int = 0) -> float:
        """bm2_gather_probe: GB/s of random requests over the Occ table (shape 0: 64 B as 4 x 16 B, 1: 32 B as two 16-B loads of one sector, 2: 64 B as two such sectors)."""
        v = C.c_double()
        lib().bm2_gather_probe.argtypes = [C.c_void_p, C.c_ulonglong, C.c_int, C.c_int, C.POINTER(C.c_double)]
        self._check(lib().bm2_gather_probe(self._ctx, int(span_bytes), int(mlp), int(shape), C.byref(v)), "bm2_gather_probe")
        return v.value

    def set_sub_batches(self, k: int, min_reads: int = 16384):
        """Seam 2 runs a batch as k sub-batches in flight (bm2_set_sub_batches); k = 1 turns the split off."""
        lib().bm2_set_sub_batches.argtypes = [C.c_void_p, C.c_int, C.c_int]
        self._check(lib().bm2_set_sub_batches(self._ctx, int(k), int(min_reads)), "bm2_set_sub_batches")

    def int_pipe_gops(self) -> float:
        v = C.c_double()
        lib().bm2_int_pipe_gops.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        self._check(lib().bm2_int_pipe_gops(self._ctx, C.byref(v)), "bm2_int_pipe_gops")
        return v.value

    def seed_chain_extend_resident(self, codes, offsets, d_codes_ptr, d_offsets_ptr, copy_out=False, return_arrays=False):
        rb, keep = self._batch(codes, offsets)
        res = RegResult()
        lib().bm2_seed_chain_extend_resident.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        self._check(lib().bm2_seed_chain_extend_resident(self._ctx, C.byref(rb), d_codes_ptr, d_offsets_ptr, int(copy_out), C.byref(res)),
                    "bm2_seed_chain_extend_resident")
        if not return_arrays:
            return res.n
        n = res.n
        regs = np.ctypeslib.as_array(C.cast(res.regs, C.POINTER(C.c_uint8)), shape=(n * REG_DT.itemsize,)).view(REG_DT).copy() if n else np.zeros(0, REG_DT)
        off = np.ctypeslib.as_array(C.cast(res.read_off, C.POINTER(C.c_int64)), shape=(rb.n_reads + 1,)).copy()
        return regs, off

    def counters(self):
        v = (C.c_ulonglong * 7)()
        lib().bm2_last_counters.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        lib().bm2_last_counters(self._ctx, v, 7)
        return dict(n_ext=v[0], n_lf=v[1], cells=v[2], retry_left=v[3], retry_right=v[4], jobs_skipped=v[5], reads_done_wave1=v[6])

    def stage_ms(self):
        names = C.POINTER(C.c_char_p)(); ms = C.POINTER(C.c_float)(); n = C.c_int()
        lib().bm2_last_stage_ms(self._ctx, C.byref(names), C.byref(ms), C.byref(n))
        return {names[i].decode(): ms[i] for i in range(n.value)}
