/* bm2_b200.h — C ABI of libbm2b200.so: the H100-native seed-and-extend hot path of bwa-mem2.
 *
 * Plain C, pointers and sizes only.  Every entry point names the reference interface it replaces
 * (file:line under bwa-mem2 @ 97978f95).  The reference has no FFI; the seam is the C++ function
 * boundary below `mem_process_seqs` (src/bwamem.cpp:1338): `kt_for(worker_bwt)` + `kt_for(worker_aln)`
 * (src/bwamem.cpp:1359,1363), and the finer seams `BandedPairWiseSW::getScores16/getScores8/
 * scalarBandedSWAWrapper` (src/bandedSWA.h:130-297) and `FMI_search::getSMEMs*`/
 * `get_sa_entries_prefetch` (src/FMI_search.h:106-165).  INTEGRATION.md shows the reference-side
 * binding.  All functions return 0 on success, non-zero on error (`bm2_last_error`); there is no
 * CPU fallback: without a usable CUDA device every compute entry fails.
 */
#ifndef BM2_B200_H
#define BM2_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define BM2_ABI_VERSION 1

typedef struct bm2_ctx bm2_ctx;

/* Field-for-field mirror of `mem_opt_t` (src/bwamem.h:76-108) so a `const mem_opt_t*` can be
 * passed as `const bm2_mem_opt_t*`; defaults: src/bwamem.cpp:107-143. */
typedef struct bm2_mem_opt_t {
    int a, b;
    int o_del, e_del;
    int o_ins, e_ins;
    int pen_unpaired;
    int pen_clip5, pen_clip3;
    int w;
    int zdrop;
    uint64_t max_mem_intv;
    int T;
    int flag;
    int min_seed_len;
    int min_chain_weight;
    int max_chain_extend;
    float split_factor;
    int split_width;
    int max_occ;
    int max_chain_gap;
    int n_threads;
    int64_t chunk_size;
    float mask_level;
    float drop_ratio;
    float XA_drop_ratio;
    float mask_level_redun;
    float mapQ_coef_len;
    int mapQ_coef_fac;
    int max_ins;
    int max_matesw;
    int max_XA_hits, max_XA_hits_alt;
    int8_t mat[25];
} bm2_mem_opt_t;

/* `mem_opt_init()` defaults (src/bwamem.cpp:107-143) incl. `bwa_fill_scmat` (src/bwa.cpp:248). */
void bm2_opt_init(bm2_mem_opt_t *opt);

/* One checkpoint of the 2bit.64 Occ table: `CP_OCC` (src/FMI_search.h:54-58). */
typedef struct bm2_cp_occ {
    int64_t  cp_count[4];
    uint64_t one_hot_bwt_str[4];
} bm2_cp_occ;

/* Host view of the index the hot path reads (src/FMI_search.h:167-177, src/bntseq.h:53-61,
 * `ref_string` src/fastmap.cpp:860-881).  All pointers are HOST memory owned by the caller;
 * `bm2_create` copies them to HBM. */
typedef struct bm2_index_desc {
    int64_t reference_seq_len;      /* N = 2*l_pac + 1 (BWT length incl. sentinel)              */
    int64_t count[5];               /* as held in memory after load: (#symbols < b) + 1         */
    int64_t sentinel_index;
    const bm2_cp_occ *cp_occ;       /* (N >> 6) + 1 entries                                     */
    const int8_t   *sa_ms_byte;     /* (N >> 3) + 1 entries: bits 32..39 of sampled SA          */
    const uint32_t *sa_ls_word;     /* (N >> 3) + 1 entries: bits 0..31                         */
    const uint8_t  *ref_string;     /* 2*l_pac codes 0..3: forward then reverse complement      */
    int64_t l_pac;
    int32_t n_seqs;                 /* contigs (bntseq_t::n_seqs)                               */
    const int64_t *ann_offset;      /* n_seqs (bntann1_t::offset)                               */
    const int32_t *ann_len;         /* n_seqs (bntann1_t::len)                                  */
    const int32_t *ann_is_alt;      /* n_seqs, may be NULL (bntann1_t::is_alt)                  */
} bm2_index_desc;

/* Native loader of `<prefix>.bwt.2bit.64`, `.0123`, `.ann` (+ `.alt`): replaces
 * FMI_search::load_index (src/FMI_search.cpp:384-494), bwa_idx_load_ele (read_index_ele.cpp:60)
 * and the ref_string read (fastmap.cpp:860-881).  The returned descriptor owns its host memory. */
int  bm2_index_load(const char *prefix, bm2_index_desc **out);
void bm2_index_free(bm2_index_desc *idx);

/* Create a device context on CUDA device `device`: uploads the index to HBM and fixes the
 * parameters.  `idx` may be NULL for a BSW-only context (bm2_extend_pairs). */
int  bm2_create(bm2_ctx **out, int device, const bm2_index_desc *idx, const bm2_mem_opt_t *opt);
/* The same for an index that is ALREADY in the memory of `device` (multi-GPU start-up, SURVEY 8e: one rank reads the index files, the
 * others receive the four big arrays by one NCCL broadcast over NVLink instead of 8 x 16 GB of disk + PCIe traffic): `cp_occ`,
 * `sa_ms_byte`, `sa_ls_word` and `ref_string` of `dev_idx` are DEVICE pointers (file layout, sizes as in bm2_index_desc), the small
 * `ann_*` arrays HOST pointers.  The context does not own the four arrays: the caller keeps them alive until bm2_destroy and must not
 * read `cp_occ` afterwards - it is permuted in place into the device layout (fm_device.cuh) unless BM2_OCC_LAYOUT=0. */
int  bm2_create_resident(bm2_ctx **out, int device, const bm2_index_desc *dev_idx, const bm2_mem_opt_t *opt);
/* A second context on the same device that uses `ctx`'s index in place (no second copy in HBM), with its own streams and buffers and a copy of
 * `ctx`'s parameters: one context per host worker thread, the way the reference runs two chunks at a time in kt_pipeline (src/fastmap.cpp:
 * 952-1003, src/kthread.cpp:122-176) - a context serves one call at a time, two contexts serve two.  `ctx` must outlive the sibling. */
int  bm2_create_sibling(bm2_ctx **out, bm2_ctx *ctx);
void bm2_destroy(bm2_ctx *ctx);
const char *bm2_last_error(const bm2_ctx *ctx);   /* ctx may be NULL: last create error */
/* Launch on a caller-owned CUDA stream (cudaStream_t as void*), e.g. the caller's framework stream,
 * so that the caller's events bracket the kernels.  NULL restores the context's own stream. */
int  bm2_set_stream(bm2_ctx *ctx, void *cuda_stream);
/* Seam 2 runs a batch as `k` sub-batches in flight (own CUDA streams and scratch, shared index): the SMEM stage is
 * bound by memory latency and the extension stage by the integer pipe, so sub-batches at different stages fill
 * each other's stalls (more reads/s at k = 4 than unsplit).  A batch is only split when every sub-batch gets
 * at least `min_reads` reads; cuts are multiples of 512 reads so that results do not depend on k (the reference's
 * kt_for works in 512-read blocks, src/kthread.cpp:41-115).  Defaults: k = 4, min_reads = 16384; k = 1 turns it off.
 * The mem_collect_smem / mem_kernel1_core stage entries (bm2_collect_smems, bm2_seed_chain) always run unsplit. */
int  bm2_set_sub_batches(bm2_ctx *ctx, int k, int min_reads);
/* Measured integer-pipe throughput of this device (G lane-ops/s of dependent 32-bit add/max
 * chains over all SMs): the denominator of the BSW cell-update roofline (SURVEY.md 8d). */
int  bm2_int_pipe_gops(bm2_ctx *ctx, double *gops_s32);
/* Measured throughput (GB/s) of independent random 64-byte reads over the first `span_bytes` (0 = all) of this context's
 * Occ checkpoint table: what the memory system delivers for the SMEM stage's access shape (two random 64-B checkpoints
 * per interval extension) when no dependent address chain limits it.  Reported next to the HBM copy peak in bench.py. */
int  bm2_gather64_gbs(bm2_ctx *ctx, unsigned long long span_bytes, double *gbs);
/* The same probe with a selectable request shape and memory-level parallelism: shape 0 = 64 B as four 16-B loads of one thread,
 * 1 = 32 B as two 16-B loads of one sector (the half-checkpoint of the device Occ layout), 2 = 64 B as two such sectors, 3 = 32 B by cp.async.bulk
 * into shared memory behind an mbarrier (the TMA path; at most 4 in flight per thread), 4 = shape 3 and shape 1 together (mlp of each); `mlp` (1, 2, 4, 8)
 * independent requests in flight per thread.  GB/s of requested bytes.  Decides whether the SMEM stage is bound by DRAM, by the
 * load/store unit's request rate or by latency (DESIGN.md section 4). */
int  bm2_gather_probe(bm2_ctx *ctx, unsigned long long span_bytes, int mlp, int shape, double *gbs);
int  bm2_abi_version(void);

/* ---- seam 1: batched banded-SW seed extension -------------------------------------------------
 * Layout-compatible with `SeqPair` (src/bandedSWA.h:90-99). */
typedef struct bm2_seqpair {
    int32_t idr, idq, id;
    int32_t len1, len2;
    int32_t h0;
    int32_t seqid, regid;
    int32_t score, tle, gtle, qle;
    int32_t gscore, max_off;
} bm2_seqpair;

/* Replaces BandedPairWiseSW::getScores16 / getScores8 / scalarBandedSWAWrapper
 * (src/bandedSWA.cpp:2664, :1970, :242; AVX2 twins :1117, :412): for pair i, target = seq_buf_ref + idr (len1 codes 0..4),
 * query = seq_buf_qer + idq (len2), start score h0, band w; writes score/tle/gtle/qle/gscore/
 * max_off in place.  `end_bonus` is the constructor's end_bonus (pen_clip5 for left, pen_clip3 for
 * right extensions, src/bwamem.cpp:2456-2462).  Host buffers; copies are done inside. */
int bm2_extend_pairs(bm2_ctx *ctx, bm2_seqpair *pairs, const uint8_t *seq_buf_ref,
                     const uint8_t *seq_buf_qer, int32_t n_pairs, int32_t w, int32_t end_bonus);

/* Device-resident variant used by the throughput bench: same contract, all pointers are DEVICE
 * memory, the launch goes to the context's stream, no host sync.  `cells_out` (device, may be
 * NULL) accumulates the banded DP cells actually computed (sum over rows of end-beg). */
int bm2_extend_pairs_device(bm2_ctx *ctx, bm2_seqpair *d_pairs, const uint8_t *d_ref,
                            const uint8_t *d_qer, int32_t n_pairs, int32_t w, int32_t end_bonus,
                            unsigned long long *d_cells_out);

/* ---- seam 2: the whole hot path over a chunk of reads -----------------------------------------
 * Output record: layout-compatible with `mem_alnreg_t` (src/bwamem.h:137-160); the pointer slot
 * `c` is always NULL on output. */
typedef struct bm2_alnreg_t {
    int64_t rb, re;
    int32_t qb, qe;
    int32_t rid;
    int32_t pad0_;                  /* the compiler's padding of mem_alnreg_t, named so that it is written (0) */
    void   *c;
    int32_t score, truesc, sub, alt_sc, csub, sub_n, w, seedcov, secondary, secondary_all, seedlen0;
    int32_t n_comp_is_alt;          /* bit-field word: n_comp:30, is_alt:2                      */
    float   frac_rep;
    int32_t pad1_;
    uint64_t hash;
    int32_t flg;
    int32_t pad2_;
} bm2_alnreg_t;

/* SMEM record: `SMEM` (src/FMI_search.h:75-83). */
typedef struct bm2_smem {
    uint32_t rid;
    uint32_t m, n;
    int64_t  k, l, s;
} bm2_smem;

/* Seed / chain records (src/bwamem.h:113-135) as flat arrays. */
typedef struct bm2_seed {
    int64_t rbeg;
    int32_t qbeg, len, score;
    int32_t chain;                  /* index into the chunk's chain array                       */
} bm2_seed;

typedef struct bm2_chain {
    int64_t pos;
    int32_t seqid, rid;
    int32_t n_seeds, seed_off;      /* seeds [seed_off, seed_off+n_seeds) of the chunk's seeds   */
    int32_t w, kept, first, is_alt;
    float   frac_rep;
    int32_t _pad;
} bm2_chain;

/* A chunk of reads: concatenated base codes (0..3 = ACGT, 4 = other; exactly what
 * src/bwamem.cpp:992-1000 leaves in bseq1_t::seq) and n_reads+1 offsets. */
typedef struct bm2_read_batch {
    int32_t n_reads;
    const uint8_t *codes;
    const int64_t *offsets;
} bm2_read_batch;

/* Result arrays are owned by the context (pinned host memory) and stay valid until the next call
 * on the same context. */
typedef struct bm2_smem_result  { int64_t n; const bm2_smem *smems; const int64_t *read_off; } bm2_smem_result;
typedef struct bm2_chain_result { int64_t n_chains, n_seeds; const bm2_chain *chains; const bm2_seed *seeds;
                                  const int64_t *read_off; /* n_reads+1 offsets into chains */ } bm2_chain_result;
typedef struct bm2_reg_result   { int64_t n; const bm2_alnreg_t *regs; const int64_t *read_off; } bm2_reg_result;

/* Replaces mem_collect_smem (src/bwamem.cpp:626-804): three SMEM passes + ordering. */
int bm2_collect_smems(bm2_ctx *ctx, const bm2_read_batch *reads, bm2_smem_result *out);
/* Replaces mem_kernel1_core (src/bwamem.cpp:976-1091): SMEMs + SA lookup + chaining + filters. */
int bm2_seed_chain(bm2_ctx *ctx, const bm2_read_batch *reads, bm2_chain_result *out);
/* Replaces kt_for(worker_bwt) + kt_for(worker_aln) (src/bwamem.cpp:1359-1363): regs per read as
 * left by mem_kernel2_core (src/bwamem.cpp:1093-1172). */
int bm2_seed_chain_extend(bm2_ctx *ctx, const bm2_read_batch *reads, bm2_reg_result *out);

/* Device-resident variant for throughput measurement: `reads` still carries the HOST offsets (sizes
 * are needed on the host) but codes/offsets are taken from DEVICE memory (`d_codes`, `d_offsets`,
 * already uploaded by the caller), and the final regs stay on the device unless `copy_out` != 0
 * (out->regs is then NULL; out->n and out->read_off are valid). */
int bm2_seed_chain_extend_resident(bm2_ctx *ctx, const bm2_read_batch *reads, const uint8_t *d_codes,
                                   const int64_t *d_offsets, int copy_out, bm2_reg_result *out);

/* Per-stage device times (ms, CUDA events) of the last seam-2 call; names in `names`. */
int bm2_last_stage_ms(const bm2_ctx *ctx, const char *const **names, const float **ms, int *n);
/* Work counters of the last seam-2 call: v[0] interval extensions (128 algorithmic bytes each),
 * v[1] LF steps of the SA walk (64 B each), v[2] banded DP cells, v[3]/v[4] left/right jobs re-run
 * with the doubled band.  n >= 5.  With n >= 7 also v[5] extension jobs not run (their seeds proved
 * purged by the post-filter before extension) and v[6] reads whose seeds were all decided after the
 * first extension wave (both 0 with BM2_EXT_LAZY=0). */
int bm2_last_counters(const bm2_ctx *ctx, unsigned long long *v, int n);

/* ---------------------------------------------------------------------------------------------
 * Seam 3 (first widening step, SURVEY 8f item 2): CIGAR, NM and MD of alignments whose end points are
 * known.  Replaces bwa_gen_cigar2 (src/bwa.cpp:260-347) with its banded global alignment + backtrack
 * ksw_global2 (src/ksw.cpp:558-668), called per output alignment by mem_reg2aln (src/bwamem.cpp:1757-1768):
 *     cigar = bwa_gen_cigar2(opt->mat, o_del, e_del, o_ins, e_ins, w2, bns->l_pac, pac, qe - qb, &query[qb], rb, re,
 *                            &score, &n_cigar, &NM);
 * One request = one such call; the query is reads[read][qb, qe), the scoring comes from the context's mem_opt_t.
 * --------------------------------------------------------------------------------------------- */
typedef struct bm2_cigar_req {
    int64_t rb, re;            /* reference interval in the [0, 2*l_pac) coordinate (mem_alnreg_t / mem_aln_t) */
    int32_t read;              /* index of the read in the batch                                               */
    int32_t qb, qe;            /* query interval of the read                                                   */
    int32_t w;                 /* band limit (the w_ argument)                                                 */
} bm2_cigar_req;
typedef struct bm2_cigar_rec {
    int32_t score;             /* INT32_MIN when the reference returns without setting *score (rejected)      */
    int32_t n_cigar;           /* operations: len << 4 | op (0 M, 1 I, 2 D), as the reference's uint32_t cigar */
    int32_t nm;                /* NM (-1 when rejected)                                                        */
    int32_t n_md;              /* bytes of the MD string incl. its NUL (the block appended after the cigar)    */
    int64_t cigar_off, md_off; /* offsets into bm2_cigar_result::cigar / ::md                                  */
} bm2_cigar_rec;
typedef struct bm2_cigar_result {
    int64_t n; const bm2_cigar_rec *recs;
    int64_t n_ops; const uint32_t *cigar;
    int64_t n_md; const char *md;
} bm2_cigar_result;
/* Needs a context created with an index.  Result arrays are owned by the context (valid until its next call). */
int bm2_gen_cigar(bm2_ctx *ctx, const bm2_read_batch *reads, const bm2_cigar_req *reqs, int64_t n, bm2_cigar_result *out);

/* ---- seam 4, first piece: insert-size statistics -------------------------------------------------------------------------
 * Replaces mem_pestat (reference src/bwamem_pair.cpp:81-148), called once per chunk between the alignment regions (seam 2) and
 * the SAM stage (src/bwamem.cpp:1368-1378).  Host code, as in the reference: one pass over the best region of every read; no
 * context, no device.  regs / read_off: the output of bm2_seed_chain_extend for a chunk whose reads 2i, 2i+1 are mates.
 * pes[d], d = FF, FR, RF, RR: mem_pestat_t (src/bwamem.h:162-166).  Returns 0; 1 on bad arguments; 2 where the reference
 * asserts (no insert size inside the outlier bounds). */
typedef struct bm2_pestat_t {
    int32_t low, high;         /* proper-pair bounds of the insert size                      */
    int32_t failed;            /* too few pairs of this orientation                          */
    int32_t _pad;
    double avg, std;
} bm2_pestat_t;
int bm2_pestat(const bm2_mem_opt_t *opt, int64_t l_pac, int32_t n_reads, const bm2_alnreg_t *regs, const int64_t *read_off, bm2_pestat_t pes[4]);

/* ---- finer seam under seam 4: a batch of the local alignments of mate rescue -----------------------------------------------
 * Replaces ksw_align2 (reference src/ksw.cpp:324-381: ksw_u8 / ksw_i16 forward, then the reversed prefixes for the start) as
 * mem_matesw calls it (src/bwamem_pair.cpp:186-193).  seqs: codes 0-4; a request names its query and its reference window by
 * offsets into seqs; xtra as the reference's (KSW_XBYTE 0x10000, KSW_XSTOP 0x20000, KSW_XSUBO 0x40000, KSW_XSTART 0x80000 |
 * threshold).  Scoring from the context's mem_opt_t.  out: n results, caller's memory.  Queries up to 497 bases. */
typedef struct bm2_ksw_req { int64_t qoff, toff; int32_t qlen, tlen; int32_t xtra, _pad; } bm2_ksw_req;
typedef struct bm2_ksw_res { int32_t score, te, qe, score2, te2, tb, qb, _pad; } bm2_ksw_res;       /* kswr_t (src/ksw.h:45-50) */
int bm2_ksw_align2(bm2_ctx *ctx, const uint8_t *seqs, int64_t n_seq_bytes, const bm2_ksw_req *reqs, int64_t n, bm2_ksw_res *out);

/* ---- seam 4: the SAM stage of a chunk of read pairs ----------------------------------------------------------------------
 * Replaces, for all pairs of a chunk at once, what worker_sam does per pair through mem_sam_pe (reference
 * src/bwamem_pair.cpp:349-552, MATE_SORT == 0): mate rescue (mem_matesw :150-283 over ksw_align2, src/ksw.cpp:324-381),
 * mem_mark_primary_se (src/bwamem.cpp:1420-1468), -5 reordering, mem_pair (:285-346), the MAPQ logic, mem_reg2aln with its
 * CIGAR / NM / MD (src/bwamem.cpp:1732-1805), the record selection of mem_reg2sam (:1521-1577), the columns of mem_aln2sam
 * (:1592-1730) and the entries of the XA tags (mem_gen_alt, src/bwamem_extra.cpp:130-183).  What is left to the caller is text:
 * QNAME, SEQ / QUAL (trimmed by the hard clips of the record's CIGAR), the tag syntax, SA and MC (columns of the read's other
 * records / the mate's record), -C / -R / -V constants.
 * regs / read_off: the output of bm2_seed_chain_extend for the same batch (reads 2i, 2i+1 are mates); pes: bm2_pestat or the
 * -I values.  One bm2_sam_rec per SAM line, in output order (pair by pair, read 0 then read 1).
 * A record is a true secondary (SEQ / QUAL '*', no SA / pa tags) iff (flag & 0x100) && sub < 0; a -M supplementary has 0x100 and sub >= 0.
 * tests/sam_text.py formats the reference's text from these records byte for byte (SEQ / QUAL with hard clips, NM MD MC AS XS SA pa XA). */
typedef struct bm2_sam_rec {
    int32_t read;              /* read of the batch the line belongs to                                        */
    int32_t flag;              /* FLAG as printed                                                              */
    int32_t rid, rnext;        /* contig ids of RNAME / RNEXT, -1: '*'                                         */
    int32_t mapq, nm;          /* nm valid iff n_cigar > 0                                                     */
    int32_t score, sub;        /* AS (printed if >= 0), XS (printed if >= 0)                                   */
    int32_t alt_sc;            /* > 0 and not a 0x100 record: pa:f: = score / alt_sc                           */
    int32_t reg;               /* its XA tag = the bm2_sam_xa entries of this read with the same reg; -1: none */
    int32_t n_cigar, n_md;     /* printed operations (len << 4 | index into "MIDSH"); MD bytes incl. the NUL   */
    int32_t is_alt;            /* the hit lies on an ALT contig                                                */
    int32_t n_mc;              /* MC tag: the n_mc operations after the record's own (cigar_off + n_cigar)     */
    int64_t pos, pnext, tlen;  /* as printed (1-based; 0 where the column is 0)                                */
    int64_t cigar_off, md_off; /* into bm2_sam_result::cigar / ::md                                            */
} bm2_sam_rec;
typedef struct bm2_sam_xa {    /* one entry of an XA tag: name(rid),[+-]pos,CIGAR,nm;                          */
    int32_t read, reg;
    int32_t rid, is_rev, nm, n_cigar;      /* operations: len << 4 | index into "MIDSHN"                       */
    int64_t pos;               /* 0-based: printed as pos + 1                                                  */
    int64_t cigar_off;
} bm2_sam_xa;
typedef struct bm2_sam_result {
    int64_t n_recs; const bm2_sam_rec *recs;
    int64_t n_xa; const bm2_sam_xa *xa;        /* in the order the reference appends them                      */
    int64_t n_ops; const uint32_t *cigar;
    int64_t n_md; const char *md;
} bm2_sam_result;
/* Needs a context created with an index; uses the context's mem_opt_t (flag bits -a -M -P -S -Y -5 -q included).
 * Result arrays are owned by the context (valid until its next call).  id_base: number of pairs before this batch in the
 * run (the reference's `id`, which seeds the tie-breaking hashes). */
int bm2_sam_pe(bm2_ctx *ctx, const bm2_read_batch *reads, const bm2_alnreg_t *regs, const int64_t *read_off, const bm2_pestat_t pes[4],
               int64_t id_base, bm2_sam_result *out);
/* The single-end branch of worker_sam (src/bwamem.cpp:1320-1334: mem_mark_primary_se, -5, mem_reg2sam without a mate) for a batch of reads;
 * same records (no RNEXT / PNEXT / TLEN).  id_base: number of reads before this batch in the run. */
int bm2_sam_se(bm2_ctx *ctx, const bm2_read_batch *reads, const bm2_alnreg_t *regs, const int64_t *read_off, int64_t id_base, bm2_sam_result *out);
/* ---- seam 0 (SURVEY 8f item 3, host I/O on the fast side): FASTQ bytes -> read batch ----------------------------------------------
 * Replaces the parsing of bseq_read_orig (src/bwa.cpp:170-216 over kseq.h; name up to the first blank, trim_readno :62-66) and the base
 * encoding at the head of mem_kernel1_core (src/bwamem.cpp:992-1000, nst_nt4_table).  buf1 / buf2: the raw bytes of a chunk of the two
 * FASTQ files (buf2 NULL: single-end); the result interleaves them (reads 2i / 2i+1 from buf1 / buf2).  Parsing and encoding run on the
 * GPU; the batch is left on the device for bm2_seed_chain_extend_resident and copied to pinned host memory for the SAM stage.
 * Four-line records only; a chunk must stay below 2 GiB per buffer.  Arrays are owned by the context (valid until its next call). */
typedef struct bm2_fastq_batch {
    int32_t n_reads;
    const uint8_t *d_codes; const int64_t *d_offsets;     /* DEVICE: codes 0-4 ('-' = 5 as nst_nt4_table), n_reads + 1 offsets */
    const uint8_t *codes;   const int64_t *offsets;       /* HOST copies                                                      */
    const char *quals;                                    /* HOST: qualities laid out like codes                              */
    const int64_t *name_beg; const int32_t *name_len;     /* HOST: QNAME of read r = its buffer [name_beg[r], + name_len[r])  */
} bm2_fastq_batch;
int  bm2_fastq_encode(bm2_ctx *ctx, const char *buf1, int64_t n1, const char *buf2, int64_t n2, bm2_fastq_batch *out);
/* FASTQ comments of the reads of the context's last bm2_fastq_encode call, as kseq reads them (src/kseq.h:196): the rest of the header line after
 * the blank that ends the name, one trailing '\r' dropped from a comment longer than one byte.  Comment of read r = its buffer [beg[r], + len[r]);
 * len[r] == 0: none.  HOST arrays owned by the context (valid until its next bm2_fastq_* call).  This is what `bwa-mem2 mem -C` appends. */
int  bm2_fastq_comments(bm2_ctx *ctx, const int64_t **beg, const int32_t **len);
/* Smart pairing (`bwa-mem2 mem -p`, src/fastmap.cpp:249-296): splits the context's last single-end bm2_fastq_encode batch on the GPU as bseq_classify
 * (src/bwa.cpp:226-242) does - read i pairs with read i-1 when their names (after trim_readno) are equal and read i-1 is not already paired with
 * read i-2; every other read is single-end.  set[0]: the single-end reads, set[1]: the pairs (reads 2i, 2i+1 are mates), both in file order and
 * laid out as a bm2_fastq_batch is, with device and host arrays; names and comments are spans of the encoded buffer.  read_index[s][j]: the read of the
 * encoded batch that read j of set s is.  Arrays are owned by the context (valid until its next bm2_fastq_* call). */
typedef struct bm2_fastq_split {
    bm2_fastq_batch set[2];
    const int64_t *comment_beg[2]; const int32_t *comment_len[2];
    const int32_t *read_index[2];
} bm2_fastq_split;
int  bm2_fastq_smart_pair(bm2_ctx *ctx, bm2_fastq_split *out);
/* Every input kseq reads (kseq_read, src/kseq.h:185-227, as bseq_read_orig calls it, src/bwa.cpp:170-216): FASTA and FASTQ, wrapped or not and
 * mixed in one file, blank lines, junk before and between records, CRLF line ends - parsed on the GPU by the grammar of csrc/seq_grammar.cuh,
 * with kseq's '\r' rule and trim_readno.  The contract is that of bm2_fastq_encode: whole records of a chunk in (buf2 NULL: single-end), the same
 * batch out, and bm2_fastq_comments / bm2_fastq_smart_pair work on it.  *qual_present (HOST, n_reads, owned by the context): 0 where kseq leaves
 * the read without qualities (a FASTA record, or an empty quality string) and SAM prints '*'; the read's bytes in out->quals are then unset.
 * A malformed record (a '+' line without a line end, or qualities of another length than the sequence: kseq_read returns -2) is an error naming
 * the record; the reference instead stops reading there without a message.  A chunk must stay below 2 GiB per buffer. */
int  bm2_seq_encode(bm2_ctx *ctx, const char *buf1, int64_t n1, const char *buf2, int64_t n2, bm2_fastq_batch *out, const uint8_t **qual_present);

/* ---- seam 5 (SURVEY 8f item 3, host I/O on the fast side): SAM text of a chunk --------------------------------------------------------
 * The formatting half of mem_aln2sam (src/bwamem.cpp:1592-1730): QNAME, the tab-separated columns, SEQ / QUAL trimmed by the record's
 * hard clips and reverse-complemented on the reverse strand, tags NM MD MC AS XS SA pa XA in the reference's order, one line per
 * bm2_sam_rec, byte for byte what `bwa-mem2 mem` prints for the record (without the constant -C / -R / -V additions).  Host code on
 * n_threads threads (read ranges).  *text is malloc'd (release with bm2_free), NUL-terminated, *len bytes. */
typedef struct bm2_sam_text_in {
    const bm2_sam_result *res;          /* records of bm2_sam_pe / bm2_sam_se for this batch                       */
    const bm2_read_batch *reads;        /* the batch (codes 0-4, offsets): SEQ                                     */
    const char *const *names;           /* QNAME per read (mates carry the same name); NULL: "r<index>"            */
    const char *quals;                  /* qualities laid out like reads->codes (same offsets); NULL: '*'          */
    const char *const *contig_names;    /* RNAME by contig id (bntann1_t::name)                                    */
    /* names == NULL: QNAME of read r = name_buf[paired ? r & 1 : 0][name_beg[r], + name_len[r]) - the spans bm2_fastq_encode returns
     * (name_buf[1] NULL: single-end); all NULL: "r<index>" */
    const char *name_buf[2];
    const int64_t *name_beg; const int32_t *name_len;
} bm2_sam_text_in;
int  bm2_sam_format(const bm2_sam_text_in *in, int n_threads, char **text, int64_t *len);
/* The -R / -C / -V additions of mem_aln2sam (src/bwamem.cpp:1693, :1720-1728): RG:Z:<rg_id> after XS, the read's FASTQ comment after XA (a tab,
 * then the comment as it is), and XR:Z:<contig annotation> last on mapped records when ref_hdr is set and the annotation is not empty (its tabs
 * printed as spaces).  Comment of read r = the same buffer as its QNAME (bm2_sam_text_in::name_buf) [comment_beg[r], + comment_len[r]). */
typedef struct bm2_sam_text_extra {
    const char *rg_id;                            /* NULL or "": no RG tag                                                   */
    const int64_t *comment_beg;                   /* NULL: no comments; comment_len[r] == 0: none for read r                 */
    const int32_t *comment_len;
    const char *const *contig_anno;               /* annotation by contig id (bntann1_t::anno, "" for none); NULL: none    */
    int32_t ref_hdr;                              /* -V                                                                      */
    const uint8_t *qual_present;                  /* NULL: every read has qualities; qual_present[r] == 0: QUAL '*'         */
} bm2_sam_text_extra;
/* bm2_sam_format with the additions; x == NULL is bm2_sam_format. */
int  bm2_sam_format_ex(const bm2_sam_text_in *in, const bm2_sam_text_extra *x, int n_threads, char **text, int64_t *len);
/* The binary twin of bm2_sam_format_ex: the same records, fields and tags in the same order, as uncompressed BAM records (SAMv1 §4.2), each
 * what `samtools view -b` makes of the SAM line: SEQ in 4-bit codes, QUAL minus 33 (0xFF x l_seq without qualities; l_seq 0 on a true
 * secondary), 0-based pos / next_pos (-1 where the column is 0), bin = reg2bin of the CIGAR's reference span (4680 unplaced), integer tags in
 * the smallest type that holds them (c / s / i when negative, else C / S / I), pa as the float of its %.3f text, MD MC SA XA RG XR as Z.  More
 * than 65535 CIGAR operations: the placeholder <l_seq>S<ref_len>N and the operations in a CG:B,I tag after the others.  With a comment (-C) the
 * comment must be tab-separated TG:T:VALUE fields (types A c C s S i I f Z H B), stored typed as sam_parse1 stores them.
 * *bam: malloc'd (bm2_free), *len bytes; *read_off: malloc'd (bm2_free), n_reads + 1 offsets, where each read's records start.
 * Errors: a QNAME longer than 254 bytes, or a comment that does not parse, returns 4 with a message naming the read (bm2_last_error(NULL)). */
int  bm2_bam_format_ex(const bm2_sam_text_in *in, const bm2_sam_text_extra *x, int n_threads, char **bam, int64_t *len, int64_t **read_off);
void bm2_free(void *p);

/* ---- BGZF compression on the GPU (SAMv1 §4.1) -------------------------------------------------------------------------------------
 * in: n uncompressed bytes (HOST); cut: the n_cut ascending offsets where records start (bytes before cut[0] are a record of their own; NULL
 * with n_cut == 0: one record).  Blocks are cut as htslib's writer cuts them: at most 65280 bytes, a record that would overflow a non-empty
 * block starts the next one, a record larger than a block spans blocks.  Each block becomes one BGZF member of at most 65536 bytes: gzip header
 * with the BC subfield, raw DEFLATE (one dynamic Huffman block, or a stored block when that is not smaller), CRC32, ISIZE - compressed on the
 * context's device and stream, one block per CTA; the bytes depend on each block's input alone.  No EOF block is added.  *out: HOST, owned by the
 * context, valid until its next bm2_bgzf_compress call; *out_len bytes (0 for n == 0). */
int  bm2_bgzf_compress(bm2_ctx *ctx, const uint8_t *in, int64_t n, const int64_t *cut, int64_t n_cut, const uint8_t **out, int64_t *out_len);
/* The last bm2_bgzf_compress call: device time of its kernels (CUDA events, ms) and its member count. */
int  bm2_last_bgzf_stats(const bm2_ctx *ctx, double *device_ms, int64_t *members);

/* ---- Coordinate sort of BAM records on the GPU, compressed as they leave (bm2_mem --sort) -----------------------------------------------
 * One buffer of records (a sorted run, or a merge window) is stably sorted by samtools' coordinate key
 *   ((uint32) refID << 32) | ((uint32) (pos + 1) << 1) | (flag & 16 ? 1 : 0)
 * (refID -1 last, ties in input order) and compressed by bm2_bgzf_compress's kernels straight from device memory.  The stream is
 * carry + the sorted records, cut by htslib's rule over all of it: called window after window with each call's carry passed to the next, the
 * BGZF bytes are those of the whole sorted stream compressed at once.
 * recs: n bytes (HOST); starts: the n_recs record offsets, ascending, each record within n.  carry: carry_len (< 65280) bytes of the previous
 * call's unfinished block (HOST, may be the previous *out's carry).  last != 0: the final block is compressed too and the carry is empty.
 * Out (owned by the context, valid until its next call):
 *   z / z_len                  whole BGZF members, no EOF block; member_size[k]: the size of member k, n_members of them
 *   carry / carry_len          the unfinished last block's uncompressed bytes (0 when last or when the stream ends on a full block)
 *   recs[n_recs]               per record in output order: refID, pos, end (bam_endpos), bin = reg2bin(pos, end) (4680 for refID -1), flag,
 *                              block (0 = the member that starts with the carry; n_members = the new carry's block) and offset in it */
typedef struct { int32_t rid, pos, end; uint16_t bin, flag; int64_t block; int32_t offset, _pad; } bm2_sort_rec;
typedef struct {
    const uint8_t *z; int64_t z_len;
    const int32_t *member_size; int64_t n_members;
    const uint8_t *carry; int64_t carry_len;
    const bm2_sort_rec *recs; int64_t n_recs;
} bm2_sort_out;
int  bm2_bam_sort_compress(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const uint8_t *carry,
                           int64_t carry_len, int last, bm2_sort_out *out);
/* The last bm2_bam_sort_compress call: device ms (CUDA events) of its stages: ms[0] keys, ms[1] radix sort, ms[2] scan + gather, ms[3] BGZF. */
int  bm2_last_sort_stats(const bm2_ctx *ctx, double ms[4]);
/* Device bytes one bm2_bam_sort_compress call on run_bytes of records of about 300 bytes needs, and the bytes free on ctx's device now. */
int  bm2_bam_sort_memory(const bm2_ctx *ctx, int64_t run_bytes, int64_t *needed, int64_t *free_bytes);
/* The same with with_tids != 0: plus the template ids bm2_bam_sort_compress_ex carries (8 bytes per record in, 8 sorted). */
int  bm2_bam_sort_memory_ex(const bm2_ctx *ctx, int64_t run_bytes, int with_tids, int64_t *needed, int64_t *free_bytes);
/* bm2_bam_sort_compress in read-name order (bm2_sort -n), the natural order of `samtools sort -n`: the QNAMEs compared by samtools'
 * strnum_cmp (digit runs by value, never parsed: csrc/bam_sort_device.cuh), then flag & 0xc0 ascending, then input order.  Same arguments,
 * outputs and bm2_last_sort_stats stages (ms[1]: the merge sort).  Each record's QNAME must end with its NUL inside the record. */
int  bm2_bam_qname_sort_compress(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const uint8_t *carry,
                                 int64_t carry_len, int last, bm2_sort_out *out);
/* Device bytes one bm2_bam_qname_sort_compress call on run_bytes of records of about 300 bytes needs (bm2_bam_sort_memory's, plus cub's
 * merge-sort temporary storage), and the bytes free on ctx's device now. */
int  bm2_bam_qname_sort_memory(const bm2_ctx *ctx, int64_t run_bytes, int64_t *needed, int64_t *free_bytes);

/* ---- Duplicate marking (bm2_mem --markdup) ------------------------------------------------------------------------------------------------
 * The rule (csrc/markdup_device.cuh) follows Picard MarkDuplicates's defaults, SUM_OF_BASE_QUALITIES; optical duplicates are marked like any
 * other duplicate, and counted only for the metrics (bm2_dup_resolve_ex, below); equality with
 * Picard or samtools is not claimed.  A template is a read, or both reads of a pair; its id (tid) is the 0-based input-order index of its
 * first read.  Its primaries (no 0x100 / 0x800) give its entries:
 *   end    (refID, unclipped 5' coordinate, reverse) packed as refID << 34 | (coord + 2^32) << 1 | reverse (refID < 2^30, |coord| < 2^32):
 *          forward pos - leading S/H, reverse bam_endpos - 1 + trailing S/H; a CIGAR in CG:B,I is read from there
 *   score  of a read: min(sum of its qualities >= 15, 16383), 0 for QUAL '*'
 *   pair entry (kind 0)       both primaries of a pair mapped: k1 = min(endA, endB), k2 = max, score the sum of both
 *   pair-end entries (kind 2) of such a pair, one per end, in the fragment space: k1 = the end, k2 = 0, score that read's
 *   fragment entry (kind 1)   one mapped primary (single-end, or its mate unmapped): k1 = its end, k2 = 0, score its read's
 * Groups are the entries of one space with the same (k1, k2), ordered by score descending then tid.  Pair space: all but the first are
 * duplicates.  Fragment space: with a pair-end entry in the group every fragment entry is a duplicate, else all fragment entries but the first
 * are.  Pair-end entries are never duplicates. */
typedef struct { uint64_t k1, k2; int64_t tid; int32_t score, kind; } bm2_dup_entry;
/* Signatures of one chunk, one warp per template, on ctx's stream.  recs: n bytes of BAM records (HOST); starts: the n_recs record offsets;
 * tmpl_first: n_tmpl + 1 record indices, template t owning records [tmpl_first[t], tmpl_first[t+1]); tmpl_id: each template's id.
 * Out (HOST, owned by the context, valid until its next bm2_dup_signatures call): the pair entries and the fragment-space entries, both in
 * template order (a pair's two pair-end entries in the order of its primaries). */
int  bm2_dup_signatures(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tmpl_first,
                        const int64_t *tmpl_id, int64_t n_tmpl, const bm2_dup_entry **pairs, int64_t *n_pairs, const bm2_dup_entry **frags,
                        int64_t *n_frags);
/* Entries of one space (HOST, n of them) sorted by (k1, k2, score descending, tid) with a stable radix sort over the bits they use.
 * resolve == 0: *sorted gets them in that order (for a spilled run).  resolve != 0: every group is taken as whole, and *dups gets the ids of
 * the duplicate templates in sorted order, *n_dups of them.  Out: HOST, owned by the context, valid until its next bm2_dup_resolve call. */
int  bm2_dup_resolve(bm2_ctx *ctx, const bm2_dup_entry *entries, int64_t n, int resolve, const bm2_dup_entry **sorted, const int64_t **dups,
                     int64_t *n_dups);
/* Device ms (CUDA events) of the context's last bm2_dup_signatures and last bm2_dup_resolve call. */
int  bm2_last_dup_stats(const bm2_ctx *ctx, double *signatures_ms, double *resolve_ms);
/* The duplicate templates: bit t of bits (n_bits of them, 1 per input read; word w holds bits 64w..64w+63) set for a duplicate template t.
 * Copied to ctx's device and kept until the next call (n_bits == 0 clears it).  A bitset larger than the device's free memory is an error
 * that gives both numbers. */
int  bm2_dup_set(bm2_ctx *ctx, const uint64_t *bits, int64_t n_bits);
/* bm2_bam_sort_compress, with one template id per record (tids, NULL: none) carried through the sort: *tids_out (HOST, owned by the context,
 * valid until its next call; may be NULL) gets them in output order.  When a bitset was given to bm2_dup_set, a record whose template's bit is
 * set and that lacks 0x4 gets 0x400 in its flag (the uint16 at byte 18 of the record counted from block_size) and in its bm2_sort_rec.flag;
 * no other byte changes.  Without tids, or with no bitset, the bytes are bm2_bam_sort_compress's. */
int  bm2_bam_sort_compress_ex(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tids,
                              const uint8_t *carry, int64_t carry_len, int last, bm2_sort_out *out, const int64_t **tids_out);

/* ---- Duplication metrics and optical duplicates (bm2_mem --markdup-metrics) ------------------------------------------------------------
 * The rule (csrc/markdup_device.cuh) follows Picard MarkDuplicates's defaults; byte equality with Picard is not claimed.
 *   location  of a template: its first record's QNAME split on ':'.  Exactly 5 or 7 fields: tile, x, y are the last three, each parsed as
 *             Picard's rapidParseInt (an optional '-', then the digits up to the first non-digit, as a wrapping 32-bit int; no digit: no
 *             location).  Any other field count: no location.  The lane is not part of it.
 *   class     of a pair template: the strand (0x10) of its primary with 0x40 (of its first primary when neither has 0x40)
 *   optical   in a pair group of 2 .. 300000 members, two members are linked when both have a location, the same class and tile, and
 *             |x1 - x2| <= d and |y1 - y2| <= d (in 64 bits); the group's optical count is the sum over the connected components of
 *             size - 1, a member without a location being a component of its own.  Larger groups and fragment groups have none.
 * loc: bit 0 set when the template has a location, bit 1 its class (1: reverse), bits 2 and up a read-group index (0 from bm2_mem; bm2_markdup
 * sets it, and members of different read groups are never linked); tile, x, y are 0 without a location. */
typedef struct { bm2_dup_entry e; int32_t tile, x, y, loc; } bm2_dup_loc_entry;
/* bm2_dup_signatures, with the pair entries located.  counts[0] gets the chunk's records with 0x100 or 0x800, counts[1] its primary records
 * with 0x4.  The entries are bm2_dup_signatures's (pairs[i].e), in the same order. */
int  bm2_dup_signatures_ex(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tmpl_first,
                           const int64_t *tmpl_id, int64_t n_tmpl, const bm2_dup_loc_entry **pairs, int64_t *n_pairs, const bm2_dup_entry **frags,
                           int64_t *n_frags, int64_t counts[2]);
/* bm2_dup_resolve over located entries: the same order (*sorted: the located entries in it, when resolve == 0) and the same *dups.  With
 * resolve != 0, *n_optical (may be NULL) gets the optical count summed over the pair groups at pixel distance `distance` (0 .. 2^31-1). */
int  bm2_dup_resolve_ex(bm2_ctx *ctx, const bm2_dup_loc_entry *entries, int64_t n, int resolve, int64_t distance, const bm2_dup_loc_entry **sorted,
                        const int64_t **dups, int64_t *n_dups, int64_t *n_optical);

/* ---- Base quality recalibration tables (bm2_mem --recal-file) ---------------------------------------------------------------------------
 * The rule (csrc/bqsr_device.cuh) restates GATK 4 BaseRecalibrator at its defaults, substitution table only; byte equality with GATK is not
 * claimed.  Counted: records without 0x4 / 0x100 / 0x800 / 0x400 / 0x200, MAPQ not 0 or 255, after adaptor clipping and soft clips are
 * removed, with at least one base left.  A base is skipped when it is N, its quality is below 6, or it is a known-site base; an aligned base
 * is an error when it differs from the reference (N inside an .amb hole).  Keys: quality, context (two letters in sequencing order, the
 * low-quality tails written as N) and cycle (+-1..500, negative for the second of a pair). */
typedef struct bm2_bqsr_tables_t {
    const int64_t *qual_obs, *qual_err;   /* [94]: quality (the sum of the cycle table over the cycles)                        */
    const int64_t *ctx_obs, *ctx_err;     /* [94 * 16]: quality * 16 + context, context 4 * first + second letter, ACGT = 0..3   */
    const int64_t *cyc_obs, *cyc_err;     /* [94 * 1001]: quality * 1001 + cycle + 500                                          */
    int64_t reads, bases;                 /* records and bases counted                                                          */
    double ms;                            /* device time of the counting kernels (CUDA events)                                  */
    int32_t err_kind;                     /* the first read error: 0 none, 1 no qualities, 2 over 500 cycles after clipping,   */
    int64_t err_index;                    /*   3 a quality above 93 (bm2_recal_tables also: 4 no RG tag, 5 an RG tag that is no  */
                                          /*   ID); its record's index over all records seen since the sites                    */
    const char *err_name;                 /*   and its read name                                                                */
    const char *read_group;               /* the read group covariate given to bm2_bqsr_sites                                   */
} bm2_bqsr_tables_t;
/* The known sites over the context's index: covered and junction (n_bits == l_pac bits each over the forward strand's concatenated
 * contigs; word w holds bits 64w..64w+63) - covered bit p: a VCF record covers p; junction bit p: one record covers both p and p + 1 -, the
 * .amb holes as n_holes sorted [beg, end) pairs, and the read group covariate.  Zeroes the counts and arms counting: from then on
 * bm2_bam_sort_compress_ex also counts the records it sorts, after the gather (with their duplicate flags) and before BGZF; a record that is
 * a read error then makes that call fail with an error naming the read.  Bitsets larger than the free device memory are an error that gives
 * both numbers. */
int  bm2_bqsr_sites(bm2_ctx *ctx, const uint64_t *covered, const uint64_t *junction, int64_t n_bits, const int64_t *holes, int64_t n_holes,
                    const char *rg);
/* Counts the records of recs (uncompressed BAM records at starts) into the context's tables (after bm2_bqsr_sites).  A read error is not
 * counted and is reported by bm2_bqsr_tables. */
int  bm2_bqsr_count(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs);
/* The counts since bm2_bqsr_sites (HOST arrays owned by the context, valid until its next call). */
int  bm2_bqsr_tables(bm2_ctx *ctx, bm2_bqsr_tables_t *out);

/* ---- Base quality recalibration tables of BAM files (bm2_baserecalibrator) -------------------------------------------------------------
 * The rule of bm2_bqsr_count, with 0x400 read from the input, plus the read group: a record that passes the filters must have an RG:Z tag
 * whose value is one of the map's IDs (checked before the read errors), and it counts into the tables of that ID's covariate.  The
 * reference is the index's packed .pac bytes; the FM index is not needed. */
typedef struct {
    int32_t n_contigs;
    const int64_t *contig_off;             /* each contig's offset in the concatenated reference                                */
    const int32_t *contig_len;             /* and its length                                                                    */
    int64_t l_pac;
    const uint8_t *pac;                    /* (l_pac + 3) / 4 bytes, base i at pac[i >> 2] >> ((~i & 3) << 1) & 3               */
    const int64_t *holes;                  /* the .amb holes as n_holes sorted [beg, end) pairs: N inside them                  */
    int64_t n_holes;
    const uint64_t *covered, *junction;    /* the known-site bitsets of bm2_bqsr_sites, l_pac bits each                         */
    int32_t n_ids;                         /* the headers' @RG IDs (the first of equal IDs is the one matched; at most 32 KiB    */
    const char *const *ids;                /*   with 16 bytes each)                                                             */
    const int32_t *id_cov;                 /* each ID's covariate, 0 .. n_cov - 1                                               */
    int32_t n_cov;                         /* covariates (their tables: about 1.5 MB each on the device)                        */
} bm2_recal_set_t;
/* Device bytes bm2_recal_set and bm2_recal_add need for a reference of l_pac bases, n_cov covariates and windows of window_bytes of records
 * of about 300 bytes, and the bytes free on ctx's device now. */
int  bm2_recal_memory(const bm2_ctx *ctx, int64_t l_pac, int64_t window_bytes, int32_t n_cov, int64_t *needed, int64_t *free_bytes);
/* The reference, the known sites and the read-group map to the context, copied; zeroes the counts.  A reference larger than the free device
 * memory is an error that gives both numbers. */
int  bm2_recal_set(bm2_ctx *ctx, const bm2_recal_set_t *s);
/* One window: recs (HOST, n bytes) holds n_recs records at starts, in any order.  A record that passes the filters and does not lie inside
 * its contig is malformed: 2 is returned, naming it, and nothing is counted.  A read error (no qualities, over 500 cycles after clipping, a
 * quality above 93, no RG tag, an RG tag that is no ID) is not counted; 2 is returned with an error naming the first such read, which
 * bm2_recal_tables reports too (err_kind 1..5). */
int  bm2_recal_add(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs);
/* Covariate cov's counts since bm2_recal_set (HOST arrays owned by the context, valid until its next call; read_group is empty). */
int  bm2_recal_tables(bm2_ctx *ctx, int32_t cov, bm2_bqsr_tables_t *out);

/* ---- Base quality recalibration applied (bm2_applybqsr) ------------------------------------------------------------------------------
 * The rule (csrc/bqsr_device.cuh, csrc/bqsr_report.h) restates GATK 4 ApplyBQSR's BQSRReadTransformer at its defaults: no quantization,
 * qualities below 6 kept, no OQ tag, no global prior; byte equality with GATK is not claimed.  A record's read group is its RG:Z value looked
 * up among the header's @RG IDs; a record without one, of a read group without tables, with l_seq 0 or with QUAL '*' is left unchanged.
 * Any other record's qualities q >= 6 become clamp(fastRound(P[q] + ((0.0 + D_ctx[q][ctx]) + D_cyc[q][cyc])), 1, 93), the context and
 * cycle taken over the whole stored read; a read of more than 500 bases or with a quality above 93 is an error. */
typedef struct {
    int32_t n_rg;                          /* read groups with tables                                                            */
    const double *P, *ctx, *cyc;           /* per read group: P [94], D_ctx [94 * 16], D_cyc [94 * 1001] (cycle + 500)           */
    int32_t n_ids;                         /* the input header's @RG lines                                                       */
    const char *const *ids;                /* their IDs (the first of equal IDs is the one matched)                              */
    const int32_t *id_table;               /* each ID's read group (its PU, else its ID) as an index into the tables, or -1      */
} bm2_bqsr_apply_tables_t;
typedef struct {
    double apply_ms, bgzf_ms;              /* device time of the apply kernel and of BGZF (CUDA events)                          */
    int64_t bases_changed;                 /* bases whose quality changed                                                        */
    int64_t recal_records, kept_records;   /* records recalibrated, records left unchanged                                       */
    int32_t err_kind;                      /* the first read error: 0 none, 1 more than 500 bases, 2 a quality above 93;         */
    int64_t err_index;                     /*   its record's index over all records since bm2_bqsr_apply_set                     */
    const char *err_name;                  /*   and its read name                                                                */
} bm2_bqsr_apply_stats_t;
/* The dense tables and the read-group map to the context (no index needed), copied; resets the counts.  The IDs with their 16-byte entries
 * may take at most 32768 bytes. */
int  bm2_bqsr_apply_set(bm2_ctx *ctx, const bm2_bqsr_apply_tables_t *tables);
/* One window: recs (HOST, n bytes) holds n_recs whole records, the first at 0, each starting where the one before ends, the last ending at n;
 * starts: their offsets.  They are recalibrated on the device and compressed after carry exactly as bm2_bam_sort_compress compresses its
 * sorted records (same members, carry and bm2_sort_rec per record, in input order).  A read error writes nothing and fails with an error
 * naming the read. */
int  bm2_bqsr_apply(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const uint8_t *carry, int64_t carry_len,
                    int last, bm2_sort_out *out);
/* The totals since bm2_bqsr_apply_set (err_name: owned by the context, valid until its next call). */
int  bm2_last_bqsr_apply_stats(bm2_ctx *ctx, bm2_bqsr_apply_stats_t *out);
/* Device bytes bm2_bqsr_apply needs for windows of window_bytes of records of about 300 bytes with n_rg read groups' tables, and the bytes
 * free on ctx's device now. */
int  bm2_bqsr_apply_memory(const bm2_ctx *ctx, int64_t window_bytes, int32_t n_rg, int64_t *needed, int64_t *free_bytes);

/* ---- Duplicate marking of coordinate-sorted BAM files (bm2_markdup) ---------------------------------------------------------------------
 * The rule (csrc/markdup_device.cuh, the host half csrc/markdup_bam.h) restates Picard MarkDuplicates on coordinate-sorted input at its
 * defaults, over the merged records of one or more files; byte equality with Picard is not claimed.  The GPU computes each record's part of
 * it; the mates are paired and the entries resolved (bm2_dup_resolve, bm2_dup_resolve_ex) on the host's side of this ABI. */
enum { BM2_MDB_NONE = 0,           /* no entry: a secondary or supplementary record, or an unmapped primary of no pair */
       BM2_MDB_FRAG = 1,           /* a mapped primary without 0x1, or with 0x8: a fragment */
       BM2_MDB_HALF = 2,           /* a mapped primary with 0x1 and without 0x8: half of a pair */
       BM2_MDB_UNMAPPED_HALF = 3   /* an unmapped primary with 0x1 and without 0x8 (its mate must not claim 0x8 is unset for it) */ };
/* One record: kind; rg, the index of its RG:Z value among bm2_markdup_set's IDs (n_ids without the tag, -1 for a value that is no ID); lib,
 * its library index (unknown_lib without the tag or with a value that is no ID).  A mapped primary: end (dup_end_key) and score (at most
 * 16383); a half (mapped or not) also hash, the 64-bit FNV-1a hash of its QNAME, and a mapped half its location: loc DUP_LOC_HAS or 0,
 * tile, x, y (0 without a location) from its QNAME. */
typedef struct { uint64_t end, hash; int32_t score, kind, rg, lib, tile, x, y, loc; } bm2_markdup_rec;   /* 48 bytes */
/* A half of a pair for bm2_markdup_pair: its QNAME's hash (a half's hash from bm2_markdup_records), read group, and its name's bytes at
 * name_off of the names buffer. */
typedef struct { uint64_t hash; int32_t rg, name_len; int64_t name_off; } bm2_markdup_half;
typedef struct { double records_ms, pair_ms, mark_ms, bgzf_ms; } bm2_markdup_stats_t;
/* The merged header's read groups: ids[i] (n_ids of them, at most 32 KiB with 16 bytes each) belongs to library libs[i] (< n_lib);
 * unknown_lib is the library of records without a known read group.  Zeroes the per-library counts and the times. */
int  bm2_markdup_set(bm2_ctx *ctx, int32_t n_ids, const char *const *ids, const int32_t *libs, int32_t n_lib, int32_t unknown_lib);
/* One window of whole records (HOST, contiguous, each where the one before ends), one warp per record: *out (HOST, n_recs, owned by the
 * context, valid until its next call) gets each record's bm2_markdup_rec.  The per-library counts grow by the window's records. */
int  bm2_markdup_records(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const bm2_markdup_rec **out);
/* The halves of one window, in ordinal order (those carried from earlier windows first): stably sorted by (hash, rg) with cub, then in each
 * run of equal (hash, rg) each half is joined to the first earlier half of the run that is still unjoined and has the same name byte for
 * byte, so a hash collision never joins two reads.  *partner (HOST, n of them, owned by the context, valid until its next call): the index
 * of each half's partner, or -1. */
int  bm2_markdup_pair(bm2_ctx *ctx, const bm2_markdup_half *halves, int64_t n, const uint8_t *names, int64_t names_len, const int32_t **partner);
/* The counts since bm2_markdup_set: counts[2 lib] records with 0x100 or 0x800, counts[2 lib + 1] unmapped primaries (2 n_lib values). */
int  bm2_markdup_counts(bm2_ctx *ctx, int64_t *counts);
/* One window of the second pass: record i is the merged stream's record first + i; its 0x400 is set when that bit of the bitset of bm2_dup_set
 * is set and cleared otherwise.  The stream carry + records is then compressed as bm2_bqsr_apply compresses it (out, carry and index data
 * alike). */
int  bm2_markdup_mark(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, int64_t first, const uint8_t *carry,
                      int64_t carry_len, int last, bm2_sort_out *out);
/* Device ms (CUDA events) since bm2_markdup_set: the record kernel, the pairing (sort and runs), the flag kernel, BGZF of the second pass. */
int  bm2_last_markdup_stats(const bm2_ctx *ctx, bm2_markdup_stats_t *out);
/* Device bytes bm2_markdup_records and bm2_markdup_mark need for windows of window_bytes of records of about 300 bytes, and the bytes free on
 * ctx's device now.  The duplicate bitset and the resolve's buffers come on top. */
int  bm2_markdup_memory(const bm2_ctx *ctx, int64_t window_bytes, int64_t *needed, int64_t *free_bytes);

/* ---- Whole-genome coverage metrics (bm2_wgsmetrics) ----------------------------------------------------------------------------------
 * The rule (csrc/wgs_device.cuh, csrc/wgs_metrics.h) restates Picard CollectWgsMetrics at its defaults (USE_FAST_ALGORITHM=false, no
 * INTERVALS); byte equality with Picard is not claimed.  Records with 0x4, refID -1 or 0x200 count nowhere.  Then the first filter that
 * matches takes a record and its aligned (M / = / X) bases: MAPQ < min_mapq -> EXC_MAPQ, 0x400 -> EXC_DUPE, unless count_unpaired no 0x1 or
 * 0x8 -> EXC_UNPAIRED, 0x100 -> counted nowhere.  Each aligned base of a record that passes, at locus g (contig offset + pos + reference
 * offset): nothing at a no-call locus; quality < min_baseq or base N -> EXC_BASEQ; else EXC_OVERLAP when an earlier record of the same QNAME
 * has such a base at g, else pileup[g] += 1.  Every locus that is not no-call: H[min(pileup, cap)] += 1, EXC_CAPPED += max(0, pileup - cap). */
#define BM2_WGS_MAX_CAP 10000
typedef struct {
    int32_t min_mapq, min_baseq;           /* Picard's MINIMUM_MAPPING_QUALITY and MINIMUM_BASE_QUALITY (20, 20)                 */
    int32_t coverage_cap;                  /* COVERAGE_CAP, 1 .. BM2_WGS_MAX_CAP (250)                                            */
    int32_t count_unpaired;                /* COUNT_UNPAIRED (0)                                                                  */
} bm2_wgs_params_t;
typedef struct {
    const int64_t *hist;                   /* [cap + 1]: loci by min(pileup, cap), no-call loci left out (owned by the context)   */
    int32_t cap;
    int64_t exc[6];                        /* bases excluded: MAPQ, DUPE, UNPAIRED, BASEQ, OVERLAP, CAPPED                        */
    int64_t records, counted_records;      /* records added, records that passed the filters                                     */
    int64_t carried_max;                   /* the most records carried from one window into the next                             */
    double add_ms, finish_ms;              /* device time of the add kernels and of the finish (CUDA events)                     */
} bm2_wgs_result_t;
/* One uint32 counter per reference base (l_pac of them, 4 bytes each) and a no-call bitset (1 bit per base) set over `nocall` (n_nocall
 * sorted [beg, end) pairs: the .amb holes of N, n or .); the contigs' offsets and lengths in the concatenated reference.  Zeroes the counters
 * and the exclusion counts.  Counters larger than the free device memory are an error that gives both numbers. */
int  bm2_wgs_set(bm2_ctx *ctx, const int64_t *contig_off, const int32_t *contig_len, int32_t n_contigs, int64_t l_pac, const int64_t *nocall,
                 int64_t n_nocall, const bm2_wgs_params_t *params);
/* Device bytes bm2_wgs_set and bm2_wgs_add need for a reference of l_pac bases and windows of window_bytes of records of about 300 bytes,
 * and the bytes free on ctx's device now (counting the counters this context already holds). */
int  bm2_wgs_memory(const bm2_ctx *ctx, int64_t l_pac, int64_t window_bytes, int64_t *needed, int64_t *free_bytes);
/* One window: recs (HOST, n bytes) holds n_recs records at starts, in file order, after those of earlier calls.  Every record is checked
 * before anything is counted: a record that is not skipped whose refID is not a contig or whose alignment does not lie inside its contig, or
 * whose CG:B,I CIGAR runs past the record, and a record that passes the filters with l_seq 0, QUAL '*' or a CIGAR whose query length is not
 * l_seq is a read error: the first such record by index is named in the error and 2 is returned, with nothing of the window counted.  The
 * overlap rule is exact across windows: the records a later window may still overlap are carried. */
int  bm2_wgs_add(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs);
/* The pass over every locus: the histogram, the exclusion counts and the totals since bm2_wgs_set.  It may be called again. */
int  bm2_wgs_finish(bm2_ctx *ctx, bm2_wgs_result_t *out);

/* ---- Alignment summary and insert size metrics (bm2_multiplemetrics) -------------------------------------------------------------------
 * The rule (csrc/mm_device.cuh, csrc/mm_metrics.h) restates Picard CollectAlignmentSummaryMetrics and CollectInsertSizeMetrics at their
 * defaults; byte equality with Picard is not claimed.  Records without 0x100 and 0x800 are counted, in three categories: FIRST_OF_PAIR (0x1
 * and 0x40), SECOND_OF_PAIR (0x1 without 0x40) and UNPAIRED.  Per category: read and base counters (the mm_device.cuh enum order), the
 * read-length histogram, the per-read histogram of high-quality mismatch counts and the no-calls by cycle.  Per pair orientation (FR, RF,
 * TANDEM): the insert-size histogram of second reads with both ends mapped, not duplicates, TLEN != 0. */
#define BM2_MM_NCAT 3
#define BM2_MM_NCOUNT 21
typedef struct {
    int64_t counts[BM2_MM_NCAT][BM2_MM_NCOUNT]; /* per category: the counters of mm_device.cuh                                         */
    int32_t max_len;                       /* the longest counted read; the three arrays below are [BM2_MM_NCAT][max_len + 1]        */
    const int64_t *len_hist;               /* reads by l_seq                                                                         */
    const int64_t *mism_hist;              /* high-quality aligned reads by their mismatch count                                     */
    const int64_t *nocall;                 /* read bases N by cycle (0-based, in sequencing order)                                   */
    int32_t max_insert;                    /* the largest insert size below 2^20; insert_hist is [3][max_insert + 1]                 */
    const int64_t *insert_hist;            /* pairs by orientation (FR, RF, TANDEM) and insert size, sizes below 2^20                */
    const uint64_t *insert_big;            /* n_big sizes of 2^20 or more, as orientation << 32 | size, sorted                       */
    int64_t n_big;
    int64_t records;                       /* records added                                                                          */
    double add_ms, finish_ms;              /* device time of the add kernels and of the finish's copies (CUDA events)                */
} bm2_mm_result_t;                         /* the pointers are owned by the context                                                  */
/* The reference: the contigs' offsets and lengths in the concatenated reference, pac ((l_pac + 3) / 4 bytes, base i at
 * pac[i >> 2] >> ((~i & 3) << 1) & 3) and the .amb holes (n_holes sorted, disjoint [beg, end) pairs and their letters, which stand for the
 * reference base inside them).  Uploads the packed bases and a hole bitset (1 bit per base), and zeroes the counters.  A reference larger than
 * the free device memory is an error that gives both numbers. */
int  bm2_mm_set(bm2_ctx *ctx, const int64_t *contig_off, const int32_t *contig_len, int32_t n_contigs, int64_t l_pac, const uint8_t *pac,
                const int64_t *holes, const char *hole_char, int64_t n_holes);
/* Device bytes bm2_mm_set and bm2_mm_add need for a reference of l_pac bases and windows of window_bytes of records of about 300 bytes, and
 * the bytes free on ctx's device now (counting the reference this context already holds). */
int  bm2_mm_memory(const bm2_ctx *ctx, int64_t l_pac, int64_t window_bytes, int64_t *needed, int64_t *free_bytes);
/* One window: recs (HOST, n bytes) holds n_recs records at starts, in any order.  Every record is checked before anything is counted: a
 * counted record with l_seq 0 or above 2^20, and an aligned one (PF, without 0x4) whose CG:B,I CIGAR runs past the record, whose refID is
 * not a contig or whose alignment runs past its contig, or whose CIGAR query length is not l_seq, is a read error: the first such record
 * by index is named in the error and 2 is returned, with nothing of the window counted.  No record is carried between windows. */
int  bm2_mm_add(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs);
/* The counters and histograms since bm2_mm_set, copied back up to their largest keys.  It may be called again. */
int  bm2_mm_finish(bm2_ctx *ctx, bm2_mm_result_t *out);
/* GC bias (Picard CollectGcBiasMetrics at its defaults, csrc/mm_device.cuh's rule, csrc/mm_gcbias.h's formulas; byte equality with Picard is
 * not claimed).  bm2_mm_gc_set, after bm2_mm_set, bins the reference's 100-base windows by GC (windows 1 <= i < L - 100 of each contig, those
 * with more than 4 Ns left out) and turns GC counting on for the bm2_mm_add calls that follow, until the next bm2_mm_set.  With it on, every
 * counted record without 0x4 gets the checks of an aligned record (a read error otherwise), and a record whose window is binned adds a read
 * start, its l_seq and its errors (mismatches plus I and D lengths) to the window's bin.  The contigs must be sorted and disjoint.  Device
 * memory it cannot get is an error that gives the bytes needed and free. */
#define BM2_MM_GC_BINS 101
typedef struct {
    int64_t windows[BM2_MM_GC_BINS];       /* reference windows by GC                                                                */
    int64_t reads[BM2_MM_GC_BINS];         /* read starts by the GC of their window                                                  */
    int64_t bases[BM2_MM_GC_BINS];         /* their l_seq, summed                                                                    */
    int64_t errors[BM2_MM_GC_BINS];        /* their mismatches, I and D lengths, summed                                              */
    int64_t total_clusters;                /* counted records without 0x1 or with 0x40                                               */
    int64_t aligned_reads;                 /* counted records without 0x4                                                            */
    double scan_ms, add_ms;                /* device time of the reference scan, and of the bm2_mm_add kernels since bm2_mm_gc_set   */
} bm2_mm_gc_result_t;
int  bm2_mm_gc_set(bm2_ctx *ctx);
/* Device bytes GC bias adds to bm2_mm_memory's figure for windows of window_bytes. */
int  bm2_mm_gc_memory(const bm2_ctx *ctx, int64_t window_bytes, int64_t *needed);
/* The GC bias counts since bm2_mm_gc_set.  It may be called again. */
int  bm2_mm_gc_finish(bm2_ctx *ctx, bm2_mm_gc_result_t *out);

/* ---- BAM back to FASTQ (bm2_bam2fq) -----------------------------------------------------------------------------------------------------
 * The rule (csrc/bam2fq_device.cuh, the host half csrc/bam2fq.h) follows `samtools fastq` at its defaults where it can; byte equality with
 * samtools is not claimed.  The GPU classifies and checks each record and writes the FASTQ text; the mates are joined by bm2_markdup_pair
 * with one read group, and the host keeps the order of the output. */
enum { BM2_B2F_SKIP = 0, BM2_B2F_READ1 = 1, BM2_B2F_READ2 = 2, BM2_B2F_OTHER = 3 };
/* One record: hash, the 64-bit FNV-1a hash of its QNAME (a READ1 or READ2 only); text_len, the bytes of its text (0 when skipped); kind. */
typedef struct { uint64_t hash; int64_t text_len; int32_t kind, pad; } bm2_bam2fq_rec;   /* 24 bytes */
/* One call's output (HOST, owned by the context, valid until its next call): data, the text, or with compression the BGZF members of the
 * blocks completed; tail, the bytes of the unfinished block (compression without last only); text_len, the text bytes this call formatted. */
typedef struct { const uint8_t *data; int64_t len; const uint8_t *tail; int64_t tail_len, text_len; } bm2_bam2fq_out;
typedef struct { double record_ms, format_ms, bgzf_ms; } bm2_bam2fq_stats_t;
/* One window of whole records (HOST, contiguous, each where the one before ends), one warp per record: *out (HOST, n_recs, owned by the
 * context, valid until its next call) gets each record's bm2_bam2fq_rec, with /1 and /2 counted in text_len when suffixes is set.  A kept
 * record with l_seq 0 or a quality above 93 is a read error: the first by index is named in the error and 2 is returned, with nothing of
 * the window kept.  Otherwise the window stays on the device for the bm2_bam2fq_format calls that follow. */
int  bm2_bam2fq_records(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, int32_t suffixes,
                        const bm2_bam2fq_rec **out);
/* The text of one output stream: list[i] >= 0 is record list[i] of the last bm2_bam2fq_records window, list[i] < 0 record ~list[i] of
 * extra (HOST, n_extra records at extra_starts, such as halves carried from earlier windows).  The lengths come from a device scan and one
 * warp writes each record.  With compress, carry (the tail of the stream's previous call) and the text are cut into blocks of exactly 65280
 * bytes; the full blocks are compressed on the GPU and the rest is the tail, or with last its member too.  Without compress, data is the
 * text. */
int  bm2_bam2fq_format(bm2_ctx *ctx, const int64_t *list, int64_t n_list, const uint8_t *extra, int64_t extra_len, const int64_t *extra_starts,
                       int64_t n_extra, int32_t suffixes, const uint8_t *carry, int64_t carry_len, int32_t compress, int32_t last, bm2_bam2fq_out *out);
/* Device ms (CUDA events) since the context was made: the record kernel, the scan and format kernels, BGZF. */
int  bm2_last_bam2fq_stats(const bm2_ctx *ctx, bm2_bam2fq_stats_t *out);
/* Device bytes bm2_bam2fq_records, bm2_markdup_pair and bm2_bam2fq_format need for windows of window_bytes of records of about 300 bytes,
 * and the bytes free on ctx's device now. */
int  bm2_bam2fq_memory(const bm2_ctx *ctx, int64_t window_bytes, int64_t *needed, int64_t *free_bytes);

/* Staged mate rescue inside bm2_sam_pe (same records, other kernels): the windows mem_matesw (src/bwamem_pair.cpp:150-283) can ask for are
 * listed for all pairs of a wave from the regions before any rescue, aligned as one batch with one window per warp (the job shape of
 * bm2_ksw_align2; the reference batches the same alignments across pairs in its kswv path, src/bwamem_pair.cpp:930-1248, src/kswv.cpp),
 * and the per-pair logic looks them up - it still computes an alignment itself when an earlier rescue of the pair moved the window.
 * on = 0: off; 1: one window per warp (the row of a window split over 32 lanes); 2: one window per thread (the one-thread sweep of the per-pair
 * logic, 32 windows per warp); -1 (default) leaves the choice to the BM2_SAM_STAGED environment variable (unset: off, until the path has GPU numbers). */
int bm2_set_sam_staged(bm2_ctx *ctx, int on);
/* Device times and counters of the last bm2_sam_pe / bm2_sam_se call.  ms[0..3] (CUDA events, summed over waves): job listing, window
 * alignments (both 0 when not staged), the per-pair kernel, the gather.  counts[0..5]: staged mode (0/1/2), jobs listed, alignments looked up,
 * alignments computed in place by the per-pair kernel (staged mode only), of those the ones whose window had moved, waves.  n_ms >= 4, n_counts >= 6. */
int bm2_last_sam_stats(const bm2_ctx *ctx, double *ms, unsigned long long *counts, int n_ms, int n_counts);

/* ---- bm2_index: `bwa-mem2 index` (bwa_idx_build, src/bwtindex.cpp:61-80) in two steps ---- */

/* Step 1, host only: bns_fasta2bntseq(fp, prefix, 1) (src/bntseq.cpp:249-356).  Reads `path` (FASTA or FASTQ as kseq reads them, plain or gzip,
 * every gzip member) and writes <prefix>.pac, .ann and .amb byte for byte as the reference does: ambiguous bases become lrand48() & 3 after
 * srand48(11) (drawn from a private state; the caller's drand48 state is untouched), runs of the same ambiguous byte are holes in .amb.
 * Unlike the reference, a malformed record (kseq_read's -2) and an input without bases (l_pac == 0) are errors (bm2_last_error(NULL)). */
typedef struct bm2_fasta_pack_stats {
    int64_t l_pac, n_seqs, n_holes;
    double seconds;
} bm2_fasta_pack_stats;
int bm2_fasta_pack(const char *path, const char *prefix, bm2_fasta_pack_stats *stats);

/* Step 2, on the GPU: FMI_search::build_index + build_fm_index (src/FMI_search.cpp:83-302, :306-382).  Reads <prefix>.pac and writes
 * <prefix>.0123 and <prefix>.bwt.2bit.64 byte for byte as the reference does, from the suffix array of the forward + reverse-complement text
 * (n = 2 l_pac), which is built on `device` and never held whole: the device keeps the text (2 bits per base) and a 5-byte inverse suffix array,
 * and every other buffer is sized from work_bytes (0: from the free device memory).  Errors (bm2_last_error(NULL)) name the bytes needed and
 * free when the persistent state does not fit. */
typedef struct bm2_index_build_stats {
    int64_t n;                          /* text length 2 l_pac                                                       */
    int64_t peak_device_bytes;          /* the most device memory the build held at once                            */
    int32_t rounds;                     /* prefix-doubling rounds after the 31-mer sort                              */
    int32_t groups, windows;            /* bucket groups of the first pass, row windows of the emit                 */
    int64_t pieces;                     /* refinement pieces over all rounds                                         */
    int64_t unresolved;                 /* suffixes still tied after the 31-mer sort                                 */
    int32_t unresolved_on_host;         /* 1 when the tied positions did not fit on the device                       */
    double load_s, pass1_s, refine_s, emit_s, total_s;
} bm2_index_build_stats;
int bm2_index_build(int device, const char *prefix, int64_t work_bytes, bm2_index_build_stats *stats);

#ifdef __cplusplus
}
#endif
#endif /* BM2_B200_H */
