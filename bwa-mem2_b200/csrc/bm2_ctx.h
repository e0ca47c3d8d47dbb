// bm2_ctx.h — the device context behind the opaque `bm2_ctx*` of the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <string>
#include <type_traits>
#include <vector>
#include <mutex>
#include "bm2_b200.h"

struct DevBuf  { void *p = nullptr; size_t cap = 0; };
struct HostBuf { void *p = nullptr; size_t cap = 0; };

struct DevIndex {                 // FM-index + reference resident in HBM (replicated per GPU)
    int64_t N = 0, l_pac = 0, sentinel = 0;
    int64_t count[5] = {0, 0, 0, 0, 0};
    const bm2_cp_occ *cp_occ = nullptr;
    int occ_layout = 0;                    // FmIndexView::layout of the resident table (1 = half-checkpoint sectors, made at upload)
    const int8_t *sa_ms = nullptr;
    const uint32_t *sa_ls = nullptr;
    const uint8_t *ref = nullptr;          // 2*l_pac codes
    int32_t n_seqs = 0;
    const int64_t *ann_off = nullptr;
    const int32_t *ann_len = nullptr;
    const int32_t *ann_alt = nullptr;
    bool loaded = false;
};

struct bm2_ctx {
    int device = 0, n_sm = 132;
    int fq_n_reads = 0, fq_n_bufs = 0;   // last successful bm2_fastq_encode / bm2_seq_encode (fastq.cu): reads, buffers (0: none)
    cudaStream_t stream = nullptr, own_stream = nullptr, side_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    bm2_mem_opt_t opt;
    std::string err;
    DevIndex idx;
    std::vector<void *> idx_allocs;
    // seam 1
    DevBuf io_pairs, io_ref, io_qer, bsw_jobs, bsw_outs, bsw_scratch;
    // Each x_d / x_h table below holds the scratch and result buffers of one source file, indexed by that file's slot enum; a
    // static_assert there ties the enum to the size here.  A file's results stay valid while other files run on the same context.
    // seam 2 (pipeline.cu)
    DevBuf pipe_d[39];
    HostBuf pipe_h[5];
    std::vector<cudaEvent_t> events;
    std::vector<const char *> stage_names;
    std::vector<float> stage_ms;
    unsigned long long last_n_ext = 0, last_n_lf = 0, last_cells = 0, last_n_retry[2] = {0, 0};
    unsigned long long last_jobs_skipped = 0, last_walk_done = 0;     // lazy extension: jobs never run, reads decided after the first wave
    // seam 2 sub-batches in flight (pipeline.cu run_regs): child contexts with their own streams, events and scratch;
    // they share this context's index (their idx_allocs stay empty)
    int n_lanes = 4, lane_min_reads = 16384;
    std::vector<bm2_ctx *> lanes;
    bm2_ctx *parent = nullptr;                 // set in a lane
    // stage tokens (held by one lane at a time): the sub-batches take turns in the DRAM-bound SMEM stage and in the
    // ALU-bound extension stage, so that at any time DIFFERENT kinds of stages overlap instead of four copies of the same
    std::mutex tok_smem, tok_bsw;
    cudaEvent_t ev_entry = nullptr;
    // seam 3 (cigar.cu), the rescue alignments of bm2_ksw_align2 (ksw.cu), the read batches of bm2_fastq_encode / bm2_fastq_smart_pair /
    // bm2_seq_encode (fastq.cu)
    DevBuf cigar_d[14];
    HostBuf cigar_h[3];
    DevBuf ksw_d[6];
    DevBuf fq_d[38];
    HostBuf fq_h[25];
    // seam 4 (sam.cu): buffers, staged rescue switch (-1: the BM2_SAM_STAGED environment variable decides, default off), events around
    // the stage's kernels, and the last call's times (jobs, window alignments, pairs, gather; ms summed over waves) and counters
    DevBuf sam_d[24];
    HostBuf sam_h[5];
    int sam_staged = -1;
    cudaEvent_t sam_ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    double sam_ms[4] = {0, 0, 0, 0};
    unsigned long long sam_counts[6] = {0, 0, 0, 0, 0, 0};        // staged, jobs, looked up, computed in place, of those: window moved, waves
    // bm2_bgzf_compress (bgzf.cu): buffers, events around its two kernels, the last call's device time and member count
    DevBuf bgzf_d[7];
    HostBuf bgzf_h[2];
    cudaEvent_t bgzf_ev[4] = {nullptr, nullptr, nullptr, nullptr};
    double bgzf_ms = 0;
    int64_t bgzf_members = 0;
    std::vector<int32_t> bgzf_sizes;       // the last call's member sizes
    // bm2_bam_sort_compress (bam_sort.cu): buffers, events around its stages, the last call's device times and outputs
    DevBuf sort_d[16];
    HostBuf sort_h[2];
    cudaEvent_t sort_ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    double sort_ms[4] = {0, 0, 0, 0};
    std::vector<uint8_t> sort_carry;
    std::vector<bm2_sort_rec> sort_recs;
    std::vector<int64_t> sort_tids;        // bm2_bam_sort_compress_ex: the template ids in output order
    // bm2_dup_signatures / bm2_dup_resolve / bm2_dup_set (markdup.cu): buffers, events, the last calls' device times and outputs, the bitset
    DevBuf dup_d[27];
    DevBuf dup_bits;
    int64_t dup_n_bits = 0;
    cudaEvent_t dup_ev[4] = {nullptr, nullptr, nullptr, nullptr};
    double dup_sig_ms = 0, dup_resolve_ms = 0;
    std::vector<bm2_dup_entry> dup_pairs, dup_frags, dup_sorted;
    std::vector<bm2_dup_loc_entry> dup_lpairs, dup_lsorted;   // the _ex calls' located pair entries and sorted entries
    std::vector<int64_t> dup_ids;
    // bm2_bqsr_sites / bm2_bqsr_count / bm2_bqsr_tables (bqsr.cu): buffers, whether bm2_bam_sort_compress_ex counts, events, the device time,
    // the records seen since the sites came, the first read error (kind 0: none), the read group, the last tables
    DevBuf bqsr_d[7];
    bool bqsr_armed = false;
    cudaEvent_t bqsr_ev[2] = {nullptr, nullptr};
    double bqsr_ms = 0;
    int64_t bqsr_n_holes = 0, bqsr_seen = 0, bqsr_err_index = -1;
    uint64_t bqsr_err_word = ~(uint64_t) 0;
    int bqsr_err_kind = 0;
    std::string bqsr_rg, bqsr_err_name;
    std::vector<int64_t> bqsr_tables;
    // bm2_bqsr_apply_set / bm2_bqsr_apply / bm2_last_bqsr_apply_stats (bqsr_apply.cu): buffers, whether tables are set, the read-group map's
    // size, events, the device times and records seen since the tables came, the first read error (kind 0: none), the last call's outputs
    DevBuf bqa_d[8];
    HostBuf bqa_h[1];
    bool bqa_set = false;
    int bqa_n_ids = 0;
    int64_t bqa_map_bytes = 0, bqa_seen = 0, bqa_err_index = -1;
    cudaEvent_t bqa_ev[2] = {nullptr, nullptr};
    double bqa_ms = 0, bqa_bgzf_ms = 0;
    int bqa_err_kind = 0;
    std::string bqa_err_name;
    std::vector<uint8_t> bqa_carry;
    std::vector<bm2_sort_rec> bqa_recs;
    // bm2_wgs_set / bm2_wgs_add / bm2_wgs_finish (wgs.cu): buffers, whether counters are set, the parameters and contigs, events, the
    // records seen and counted since the counters came, the carried records (bytes and starts, on the host), the device times, the histogram
    DevBuf wgs_d[16];
    bool wgs_set = false;
    bm2_wgs_params_t wgs_params{};
    int64_t wgs_l_pac = 0;
    int32_t wgs_n_contigs = 0;
    std::vector<int64_t> wgs_contig_off;
    cudaEvent_t wgs_ev[2] = {nullptr, nullptr};
    int64_t wgs_seen = 0, wgs_counted = 0, wgs_carried_max = 0;
    std::vector<uint8_t> wgs_carry;
    std::vector<int64_t> wgs_carry_starts;
    double wgs_add_ms = 0, wgs_finish_ms = 0;
    std::vector<int64_t> wgs_hist;
    // bm2_mm_set / bm2_mm_add / bm2_mm_finish (mm.cu): buffers, whether a reference is set, its contigs and holes, events, the records seen
    // since, the insert sizes of 2^20 or more (copied back after each window), the device times, the histograms copied back by the finish
    DevBuf mm_d[19];
    bool mm_set = false;
    // bm2_mm_gc_set: GC bias counted by the adds that follow (bm2_mm_set turns it off), the scan's and those adds' device times
    bool mm_gc = false;
    double mm_gc_scan_ms = 0, mm_gc_add_ms = 0;
    int64_t mm_l_pac = 0, mm_n_holes = 0;
    int32_t mm_n_contigs = 0;
    cudaEvent_t mm_ev[2] = {nullptr, nullptr};
    int64_t mm_seen = 0;
    std::vector<uint64_t> mm_big;
    double mm_add_ms = 0, mm_finish_ms = 0;
    std::vector<int64_t> mm_hist;
    // bm2_markdup_set / bm2_markdup_records / bm2_markdup_mark (markdup_bam.cu): buffers, whether read groups are set, the map's size, the
    // libraries, events, the device times, the last call's outputs
    DevBuf mdb_d[14];
    HostBuf mdb_h[1];
    bool mdb_set = false;
    int mdb_n_ids = 0, mdb_n_lib = 0, mdb_unknown_lib = 0;
    int64_t mdb_map_bytes = 0;
    cudaEvent_t mdb_ev[2] = {nullptr, nullptr};
    double mdb_records_ms = 0, mdb_pair_ms = 0, mdb_mark_ms = 0, mdb_bgzf_ms = 0;
    std::vector<bm2_markdup_rec> mdb_recs;
    std::vector<int32_t> mdb_partner;
    std::vector<uint8_t> mdb_carry;
    std::vector<bm2_sort_rec> mdb_srecs;
    // bm2_recal_set / bm2_recal_add / bm2_recal_tables (recal.cu): buffers, whether a reference is set, the contigs' lengths, the reference's
    // size and holes, the map and covariates, events, the device time and records seen since, the first read error (kind 0: none), the last tables
    DevBuf rcl_d[10];
    bool rcl_set = false;
    std::vector<int32_t> rcl_contig_len;
    int64_t rcl_l_pac = 0, rcl_n_holes = 0, rcl_map_bytes = 0, rcl_seen = 0, rcl_err_index = -1;
    int rcl_n_ids = 0, rcl_n_cov = 0, rcl_err_kind = 0;
    cudaEvent_t rcl_ev[2] = {nullptr, nullptr};
    double rcl_ms = 0;
    std::string rcl_err_name;
    std::vector<int64_t> rcl_tables;
    // bm2_bam2fq_records / bm2_bam2fq_format (bam2fq.cu): buffers (the window stays for the format calls), the window's record count,
    // events, the device times, the last calls' outputs
    DevBuf b2f_d[11];
    HostBuf b2f_h[2];
    int64_t b2f_n_recs = 0;
    cudaEvent_t b2f_ev[4] = {nullptr, nullptr, nullptr, nullptr};
    double b2f_record_ms = 0, b2f_format_ms = 0, b2f_bgzf_ms = 0;
    std::vector<bm2_bam2fq_rec> b2f_recs;
    std::vector<uint8_t> b2f_tail;

    int ensure(DevBuf &b, size_t bytes);
    int ensure_host(HostBuf &b, size_t bytes);
    std::vector<DevBuf *> all_dev() {
        std::vector<DevBuf *> v = {&io_pairs, &io_ref, &io_qer, &bsw_jobs, &bsw_outs, &bsw_scratch, &dup_bits};
        append(v, pipe_d); append(v, cigar_d); append(v, sam_d); append(v, ksw_d); append(v, fq_d);
        append(v, bgzf_d); append(v, sort_d); append(v, dup_d); append(v, bqsr_d); append(v, bqa_d); append(v, wgs_d);
        append(v, mm_d); append(v, mdb_d); append(v, rcl_d); append(v, b2f_d);
        return v;
    }
    std::vector<HostBuf *> all_host() {
        std::vector<HostBuf *> v;
        append(v, pipe_h); append(v, cigar_h); append(v, sam_h); append(v, fq_h); append(v, bgzf_h); append(v, sort_h); append(v, bqa_h); append(v, mdb_h); append(v, b2f_h);
        return v;
    }
    template <class B, size_t N> static void append(std::vector<B *> &v, B (&t)[N]) { for (B &x : t) v.push_back(&x); }
};

// bgzf.cu: the members of the nb blocks [starts[b], starts[b+1]) of the device bytes d_in, on ctx's stream (the body of bm2_bgzf_compress),
// gathered into *gather (nullptr: the context's own buffer) before they are copied to the host
int bgzf_compress_device(bm2_ctx *ctx, const uint8_t *d_in, const int64_t *starts, int64_t nb, const uint8_t **out, int64_t *out_len, DevBuf *gather);
// bqsr.cu: bqsr_count_kernel over the n records at d_base + d_starts[i] (device), enqueued on st: n_cov covariates of kBqsrCounts counters
// each at cnt, the read-group map (n_ids entries, map_bytes; n_ids 0: no lookup, covariate 0), the first read error's word into err
struct BqsrView;
int bqsr_count_launch(bm2_ctx *ctx, const uint8_t *d_base, const int64_t *d_starts, int64_t n, const BqsrView &v, const void *d_map, int map_bytes,
                      int n_ids, int n_cov, unsigned long long *cnt, unsigned long long *err, int64_t first, cudaStream_t st);
// bqsr.cu: the covariate counts of the n records at d_base + d_starts[i] (device), enqueued on st; then, once st has finished,
// bqsr_count_done adds the device time and returns 1 (the context's error set, naming the read) when one of these records is a read error
int bqsr_count_device(bm2_ctx *ctx, const uint8_t *d_base, const int64_t *d_starts, int64_t n, cudaStream_t st);
int bqsr_count_done(bm2_ctx *ctx, const uint8_t *d_base, const int64_t *h_starts, int64_t n);
// bam_sort.cu: the tail of bm2_bam_sort_compress and bm2_bqsr_apply.  d_stream (device) holds carry_len bytes of the previous call's
// unfinished block, then the records at carry_len + offs[i], total bytes of them; the stream is cut by bam_sort_layout (which sets each
// record's block and offset in recs, HOST), the full blocks are compressed into *gather, the unfinished one (when !last) is copied to carry_v;
// out gets the members, carry_v and recs_v (the records' bm2_sort_rec, copied from recs)
int bam_compress_stream(bm2_ctx *ctx, const uint8_t *d_stream, int64_t carry_len, const int64_t *offs, int64_t n_recs, int64_t total, int last,
                        bm2_sort_rec *recs, DevBuf *gather, std::vector<uint8_t> &carry_v, std::vector<bm2_sort_rec> &recs_v, bm2_sort_out *out);
// markdup_bam.cu: 0 when the n_recs records at starts (HOST) are whole, each where the one before ends, the last ending at n; otherwise the
// context's error names fn and the record, and 1 is returned
int bam_check_records(bm2_ctx *ctx, const char *fn, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs);
