// sam.cu — seam 4: the SAM stage of a chunk of read pairs (SURVEY §8(f) items 1-3: mate rescue, pairing / MAPQ, records).
//
// Replaces what worker_sam does per pair through mem_sam_pe (reference src/bwamem_pair.cpp:349-552) for all pairs of a chunk: the
// per-pair logic is sam_pe_pair_d / mate_rescue_pair_d (sam_device.cuh, mate_device.cuh: checked on the host against the oracle and
// the unmodified reference), one pair per thread; the scratch of a pair is an arena whose capacities follow from the pair's regions
// and the insert-size statistics (sam_layout.cuh); the records, XA entries, operations and MD bytes go to worst-case stripes and are
// compacted by a gather.  Pairs are processed in waves sized by a scratch budget (worst-case capacities: ≈0.5 MB per typical pair, most of it the MD
// and CIGAR pools - optimistic pools with a second wave for the pairs that overflow are the obvious next step).  The libm values the stage needs (log of small
// integers, the insert-size term of mem_pair) are tabulated on the host with the host's libm, as the reference computes them.
//
// Parity-tested in all three rescue modes (tests/test_zz_sam_gpu.py, tests/test_zzz_sam_staged_gpu.py); `bench.py --workload sam` times it.
//
// Staged rescue (the default; bm2_set_sam_staged / BM2_SAM_STAGED select 0 = per-pair, 1 = warp per window, 2 = thread per window): the local alignments of the rescue - the
// bulk of the stage's arithmetic - leave the per-pair thread.  sam_jobs_kernel lists, from the regions BEFORE any rescue, the windows the
// rescue block of every pair can ask for (mate_jobs_pair_d); sam_ksw_jobs_kernel aligns them one window per warp (ksw_warp.cuh, the mate read
// in place, reverse-complemented by addressing); the per-pair thread then looks its alignments up (MateKswTable) and computes one itself
// only when the table does not hold it (a window that moved, a job that was not listed).  Same records either way - the host
// emulation of exactly this split is tests/test_oracle_sam_pe.py::test_staged_rescue_equals_the_per_pair_block.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "sam_layout.cuh"
#include "ksw_warp.cuh"
#include "mate_stage.cuh"
#include <vector>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>

namespace {
enum { SB_CODES, SB_OFFS, SB_REGS, SB_REGOFF, SB_DESC, SB_ARENA, SB_RECS_W, SB_XA_W, SB_OPS_W, SB_MD_W, SB_CNT, SB_FINAL, SB_LOG, SB_TERM,
       SB_RECS, SB_XA, SB_OPS, SB_MD,
       SJ_PAIRJOBS, SJ_JOBS, SJ_RES, SJ_LISTS, SJ_STATS,          // staged rescue
       SB_ORDER,                                                  // processing order
       SB_COUNT_ };
enum { SH_RECS, SH_XA, SH_OPS, SH_MD, SH_CNT, SH_COUNT_ };
static_assert(SB_COUNT_ == std::extent<decltype(bm2_ctx::sam_d)>::value, "bm2_ctx::sam_d: one buffer per slot");
static_assert(SH_COUNT_ == std::extent<decltype(bm2_ctx::sam_h)>::value, "bm2_ctx::sam_h: one buffer per slot");

struct PairDesc {                 // one pair of a wave
    SamPairCaps caps;
    int64_t arena_off;            // bytes into the wave's arena
    int64_t rec_off, xa_off, ops_off, md_off;      // worst-case stripes of the wave
    int32_t pair;                 // pair index in the batch
};
struct PairCount { int64_t recs, xa, ops, md; int32_t overflow, _pad; };
struct PairFinal { int64_t recs, xa, ops, md; };   // compact offsets (inside the wave)

// ---- staged rescue (mate_stage.cuh) ---------------------------------------------------------------------------------------------
typedef MateStats SamStats;
struct KswMat25 { int8_t m[25]; };
static_assert(sizeof(MateJobRes) == sizeof(bm2_ksw_res), "job results have the layout of bm2_ksw_res");

// stage 1: one pair per thread; the jobs of a pair are consecutive in `jobs` (reserved with one atomicAdd: their order between pairs does
// not matter, the pair finds them through pj[])
__global__ void __launch_bounds__(128)
sam_jobs_kernel(ContigView cv, MatePes pes, int min_seed_len, int pen_unpaired, int max_matesw, const int64_t *__restrict__ offs,
                const bm2_alnreg_t *__restrict__ regs, const int64_t *__restrict__ reg_off, const PairDesc *__restrict__ desc, int n_pairs,
                MateJob *jobs, unsigned int job_cap, PairJobs *pj, SamStats *stats)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_pairs) return;
    const int pair = desc[t].pair;
    const bm2_alnreg_t *a[2]; int n[2], l_seq[2];
    for (int i = 0; i < 2; ++i) {
        const int64_t r = 2LL * pair + i;
        a[i] = regs + reg_off[r]; n[i] = (int) (reg_off[r + 1] - reg_off[r]); l_seq[i] = (int) (offs[r + 1] - offs[r]);
    }
    const int count = mate_jobs_list_d(cv, min_seed_len, pen_unpaired, max_matesw, pes, l_seq, a, n, pair, nullptr);
    PairJobs mine; mine.begin = 0; mine.count = 0;
    if (count) {
        const unsigned int base = atomicAdd(&stats->n_jobs, (unsigned int) count);
        if ((unsigned long long) base + (unsigned int) count <= job_cap) {         // always true with the host's bound; a pair left out computes in place
            mine.begin = (int32_t) base; mine.count = count;
            mate_jobs_list_d(cv, min_seed_len, pen_unpaired, max_matesw, pes, l_seq, a, n, pair, jobs + base);
        }
    }
    pj[t] = mine;
}

// stage 2: one window per warp, grid-stride over the job count stage 1 left on the device (no host round trip in between).
// lists: 2 * lcap ints per warp of the grid (the score-2 list of one window at a time).  res[k].valid = 1: computed.
// With the host's bound every pair fits the table; if the bound had to be clamped, entries below job_cap that no pair wrote (stale bytes) are
// never looked up - the range checks below only keep the warp inside the buffers for them.
template <int TMAX>
__global__ void __launch_bounds__(128)
sam_ksw_jobs_kernel(KswMat25 mat, int a_match, int min_seed_len, int o_del, int e_del, int o_ins, int e_ins, const uint8_t *__restrict__ ref, int64_t ref_len,
                    const uint8_t *__restrict__ codes, const int64_t *__restrict__ offs, int n_reads, const MateJob *__restrict__ jobs, const SamStats *stats,
                    unsigned int job_cap, int32_t *lists, int lcap, MateJobRes *res)
{
    __shared__ int8_t smat[32];                               // the passes index the matrix with data (profile set-up): shared, not a local copy
    if (threadIdx.x < 25) smat[threadIdx.x] = mat.m[threadIdx.x];
    __syncthreads();
    const unsigned int n = stats->n_jobs < job_cap ? stats->n_jobs : job_cap;
    const unsigned int warps = gridDim.x * (blockDim.x >> 5), w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    int32_t *bsc = lists + (size_t) w * 2 * lcap, *bpos = bsc + lcap;
    for (unsigned int k = w; k < n; k += warps) {
        const MateJob jb = jobs[k];
        MateJobRes o; o.score = 0; o.te = -1; o.qe = -1; o.score2 = -1; o.te2 = -1; o.tb = -1; o.qb = -1; o.valid = 0;
        if (jb.pair >= 0 && 2LL * jb.pair + 1 < n_reads && jb.rb >= 0 && jb.re <= ref_len && jb.rb < jb.re) {
            const MateJobQuery q = mate_job_query_d(jb, codes, offs, a_match, min_seed_len);
            if (ksw_lane_fits_d(q.l_ms, TMAX) && ksw_scan_ok_d(e_ins, q.l_ms) && q.tlen / 2 + 2 <= lcap) {
                int overflow = 0;
                const KswRes al = ksw_align2_warp_d<TMAX>(q.l_ms, q.q, q.stride, q.comp, q.tlen, ref + jb.rb, smat, o_del, e_del, o_ins, e_ins, q.xtra, bsc, bpos, lcap, &overflow);
                o.score = al.score; o.te = al.te; o.qe = al.qe; o.score2 = al.score2; o.te2 = al.te2; o.tb = al.tb; o.qb = al.qb; o.valid = overflow ? 0 : 1;
            }
        }
        if (lane == 0) res[k] = o;
        __syncwarp(0xffffffffu);
    }
}

// stage 2, other formulation (staged mode 2): one window per THREAD over the same job table - the one-thread sweep of ksw_device.cuh (the arithmetic the
// per-pair kernel runs) with 32 windows of similar size per warp in lock step.  Per-thread scratch in global memory:
// [3 * (max_l + 16) ints H / E / best row][lcap ints scores][lcap ints rows][tcap bytes reversed target][max_l + 1 bytes reverse complement].
__global__ void __launch_bounds__(128)
sam_ksw_jobs_thread_kernel(KswMat25 mat, int a_match, int min_seed_len, int o_del, int e_del, int o_ins, int e_ins, const uint8_t *__restrict__ ref, int64_t ref_len,
                           const uint8_t *__restrict__ codes, const int64_t *__restrict__ offs, int n_reads, const MateJob *__restrict__ jobs, const SamStats *stats,
                           unsigned int job_cap, uint8_t *scratch, size_t per_thread, int max_l, int lcap, int tcap, MateJobRes *res)
{
    __shared__ int8_t smat[32];
    if (threadIdx.x < 25) smat[threadIdx.x] = mat.m[threadIdx.x];
    __syncthreads();
    const unsigned int n = stats->n_jobs < job_cap ? stats->n_jobs : job_cap;
    const unsigned int T = gridDim.x * blockDim.x, t = blockIdx.x * blockDim.x + threadIdx.x;
    uint8_t *mine = scratch + (size_t) t * per_thread;
    int32_t *ksw = (int32_t *) mine, *bsc = ksw + 3 * (max_l + 16), *bpos = bsc + lcap;
    uint8_t *tmp = (uint8_t *) (bpos + lcap), *rev = tmp + tcap;
    for (unsigned int k = t; k < n; k += T) {
        const MateJob jb = jobs[k];
        MateJobRes o; o.score = 0; o.te = -1; o.qe = -1; o.score2 = -1; o.te2 = -1; o.tb = -1; o.qb = -1; o.valid = 0;
        if (jb.pair >= 0 && 2LL * jb.pair + 1 < n_reads && jb.rb >= 0 && jb.re <= ref_len && jb.rb < jb.re) {
            const MateJobQuery q = mate_job_query_d(jb, codes, offs, a_match, min_seed_len);
            if (q.l_ms > 0 && q.l_ms <= max_l && q.tlen <= tcap && q.tlen / 2 + 2 <= lcap) {
                int overflow = 0;
                const KswRes al = mate_job_align_thread_d(q, ref + jb.rb, smat, o_del, e_del, o_ins, e_ins, ksw, bsc, bpos, lcap, tmp, rev, &overflow);
                o.score = al.score; o.te = al.te; o.qe = al.qe; o.score2 = al.score2; o.te2 = al.te2; o.tb = al.tb; o.qb = al.qb; o.valid = overflow ? 0 : 1;
            }
        }
        res[k] = o;
    }
}

__global__ void __launch_bounds__(64)
sam_kernel(SamParams p, SamTables tb, ContigView cv, MatePes pes, int max_matesw, int rescue, const uint8_t *__restrict__ ref,
           const uint8_t *__restrict__ codes, const int64_t *__restrict__ offs, const bm2_alnreg_t *__restrict__ regs, const int64_t *__restrict__ reg_off,
           const PairDesc *__restrict__ desc, int n_pairs, int paired, int64_t id_base, uint8_t *arena, bm2_sam_rec *recs_w, bm2_sam_xa *xa_w, uint32_t *ops_w,
           char *md_w, PairCount *cnt, const PairJobs *__restrict__ pj, const MateJob *__restrict__ jobs, const MateJobRes *__restrict__ jres, SamStats *stats,
           const int32_t *__restrict__ order)
{
    const int t0 = blockIdx.x * blockDim.x + threadIdx.x;
    if (t0 >= n_pairs) return;
    // order: the wave's pairs sorted by a work key (host): the 32 pairs of a warp run similar code - same number of regions, the same
    // need for a gapped CIGAR - instead of waiting for the one pair that needs a banded DP.  Every per-pair slot is indexed by t, so the
    // output (stripes, counts, the gather) does not depend on the order.
    const int t = order ? order[t0] : t0;
    const PairDesc d = desc[t];
    SamArena ar;
    sam_arena_carve_d(arena + d.arena_off, d.caps, 0, &ar);
    const uint8_t *seq[2] = { codes, codes }; int l_seq[2] = { 0, 0 }, n[2] = { 0, 0 };
    const int64_t read0 = paired ? 2LL * d.pair : d.pair;         // a unit is a pair (reads 2u, 2u+1) or, single-end, one read
    for (int i = 0; i < (paired ? 2 : 1); ++i) {
        const int64_t r = read0 + i;
        seq[i] = codes + offs[r]; l_seq[i] = (int) (offs[r + 1] - offs[r]);
        n[i] = (int) (reg_off[r + 1] - reg_off[r]);
        for (int k = 0; k < n[i]; ++k) reg_copy(&ar.a[i][k], &regs[reg_off[r] + k]);
    }
    int overflow = 0;
    bm2_alnreg_t *ap[2] = { ar.a[0], ar.a[1] }, *bp[2] = { ar.b[0], ar.b[1] };
    if (rescue && paired) {
        if (pj) {             // staged: the alignments were computed by sam_ksw_jobs_kernel
            const PairJobs mine = pj[t];
            MateKswTable look = { jobs + mine.begin, jres + mine.begin, mine.count, { &p.ep, ref, &ar.ms, &overflow }, stats };
            mate_rescue_pair_d(cv, p.ep, p.min_seed_len, p.pen_unpaired, max_matesw, pes, ref, seq, l_seq, ap, n, bp, ar.ms, look, &overflow);
        } else mate_rescue_pair_d(cv, p.ep, p.min_seed_len, p.pen_unpaired, max_matesw, pes, ref, seq, l_seq, ap, n, bp, ar.ms, &overflow);
    }
    PairCount c; c.recs = 0; c.xa = 0; c.ops = 0; c.md = 0; c.overflow = 0; c._pad = 0;
    bm2_sam_rec *recs = recs_w + d.rec_off; bm2_sam_xa *xa = xa_w + d.xa_off; uint32_t *ops = ops_w + d.ops_off; char *md = md_w + d.md_off;
    const SamPairCaps &cp = d.caps;
    auto emit = [&](int i, int k, const SamRec &r, const uint32_t *rops, const char *rmd) {
        const int nmd = r.n_cigar ? r.n_md : 1;
        const int nops = r.n_cigar + r.n_mc;
        if (c.recs >= cp.recs_cap || c.ops + nops > cp.out_ops || c.md + nmd > cp.out_md) { overflow |= BM2_OVF_RECORDS; return; }
        bm2_sam_rec o;
        o.read = (int32_t) read0 + i; o.flag = r.flag; o.rid = r.rid; o.rnext = r.rnext; o.mapq = r.mapq; o.nm = r.nm; o.score = r.score; o.sub = r.sub;
        o.alt_sc = r.alt_sc; o.is_alt = r.is_alt; o.n_mc = r.n_mc; o.reg = r.reg; o.n_cigar = r.n_cigar; o.n_md = nmd; o.pos = r.pos; o.pnext = r.pnext; o.tlen = r.tlen;
        o.cigar_off = c.ops; o.md_off = c.md;
        for (int j = 0; j < nops; ++j) ops[c.ops + j] = rops[j];
        if (r.n_cigar) { for (int j = 0; j < nmd; ++j) md[c.md + j] = rmd[j]; } else md[c.md] = 0;
        recs[c.recs++] = o; c.ops += nops; c.md += nmd;
    };
    auto emit_xa = [&](int i, int reg, const SamAln &e) {
        if (c.xa >= cp.xa_cap || c.ops + e.n_cigar > cp.out_ops) { overflow |= BM2_OVF_RECORDS; return; }
        bm2_sam_xa o;
        o.read = (int32_t) read0 + i; o.reg = reg; o.rid = e.rid; o.is_rev = e.is_rev; o.nm = e.nm; o.n_cigar = e.n_cigar; o.pos = e.pos; o.cigar_off = c.ops;
        for (int j = 0; j < e.n_cigar; ++j) ops[c.ops + j] = e.cigar[j];
        xa[c.xa++] = o; c.ops += e.n_cigar;
    };
    if (paired) sam_pe_pair_d(p, tb, cv, pes, ref, seq, l_seq, ap, n, (int) (id_base + d.pair), ar.sc, emit, emit_xa, &overflow);
    else sam_se_read_d(p, tb, cv, ref, seq[0], l_seq[0], ar.a[0], n[0], id_base + d.pair, ar.sc, emit, emit_xa, &overflow);
    c.overflow = overflow;
    cnt[t] = c;
}

// compaction of one wave: stripes -> dense arrays; offsets become offsets into the batch's result (base_* = what earlier waves produced)
__global__ void sam_gather_kernel(const PairDesc *__restrict__ desc, const PairCount *__restrict__ cnt, const PairFinal *__restrict__ fin, int n_pairs,
                                  const bm2_sam_rec *__restrict__ recs_w, const bm2_sam_xa *__restrict__ xa_w, const uint32_t *__restrict__ ops_w,
                                  const char *__restrict__ md_w, int64_t base_ops, int64_t base_md, bm2_sam_rec *recs, bm2_sam_xa *xa, uint32_t *ops, char *md)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_pairs) return;
    const PairDesc d = desc[t]; const PairCount c = cnt[t]; const PairFinal f = fin[t];
    for (int64_t k = 0; k < c.recs; ++k) {
        bm2_sam_rec o = recs_w[d.rec_off + k];
        o.cigar_off += base_ops + f.ops; o.md_off += base_md + f.md;
        recs[f.recs + k] = o;
    }
    for (int64_t k = 0; k < c.xa; ++k) {
        bm2_sam_xa o = xa_w[d.xa_off + k];
        o.cigar_off += base_ops + f.ops;
        xa[f.xa + k] = o;
    }
    for (int64_t k = 0; k < c.ops; ++k) ops[f.ops + k] = ops_w[d.ops_off + k];
    for (int64_t k = 0; k < c.md; ++k) md[f.md + k] = md_w[d.md_off + k];
}

template <class T> T *P(bm2_ctx *ctx, int b) { return (T *) ctx->sam_d[b].p; }

// pinned host buffer that keeps its content when it grows
int grow_host(bm2_ctx *ctx, HostBuf &b, size_t used, size_t need) {
    bm2_ctx *ctx_for_error = ctx;
    if (b.cap >= need) return 0;
    void *np = nullptr;
    const size_t want = need + need / 2 + 4096;
    BM2_CUDA_OK(cudaMallocHost(&np, want));
    if (used) memcpy(np, b.p, used);
    if (b.p) BM2_CUDA_OK(cudaFreeHost(b.p));
    b.p = np; b.cap = want;
    return 0;
}
}  // namespace

namespace {
// paired: units are pairs (pes4 given); single-end: units are reads (pes4 == nullptr: no orientation has statistics)
int run_sam(bm2_ctx *ctx, const bm2_read_batch *reads, const bm2_alnreg_t *regs, const int64_t *read_off, const bm2_pestat_t *pes4, int64_t id_base,
            bm2_sam_result *out)
{
    bm2_ctx *ctx_for_error = ctx;
    const int paired = pes4 != nullptr;
    if (!ctx || !reads || !out || !read_off) { if (ctx) bm2_set_error(ctx, "bm2_sam_pe / bm2_sam_se: bad arguments"); return 1; }
    if (!ctx->idx.loaded) { bm2_set_error(ctx, "bm2_sam_pe / bm2_sam_se need a context created with an index"); return 1; }
    const int nr = reads->n_reads;
    if (nr < 0 || (paired && (nr & 1))) { bm2_set_error(ctx, "bm2_sam_pe: the batch must hold whole pairs (reads 2i, 2i+1)"); return 1; }
    if (read_off[nr] > 0 && !regs) { bm2_set_error(ctx, "bm2_sam_pe: regs is NULL"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    memset(out, 0, sizeof(*out));
    if (grow_host(ctx, ctx->sam_h[SH_RECS], 0, 64) || grow_host(ctx, ctx->sam_h[SH_XA], 0, 64) || grow_host(ctx, ctx->sam_h[SH_OPS], 0, 64) || grow_host(ctx, ctx->sam_h[SH_MD], 0, 64)) return 1;
    out->recs = (const bm2_sam_rec *) ctx->sam_h[SH_RECS].p; out->xa = (const bm2_sam_xa *) ctx->sam_h[SH_XA].p;
    out->cigar = (const uint32_t *) ctx->sam_h[SH_OPS].p; out->md = (const char *) ctx->sam_h[SH_MD].p;
    const int n_pairs_all = paired ? nr >> 1 : nr;              // units
    if (n_pairs_all == 0) return 0;
    const bm2_mem_opt_t &o = ctx->opt;
    if (o.e_del <= 0 || o.e_ins <= 0 || o.a <= 0) { bm2_set_error(ctx, "bm2_sam_pe: match score and gap extension penalties must be positive"); return 1; }

    // ---- parameters and host-filled tables ----------------------------------------------------------------------------------
    SamParams p;
    p.ep.a = o.a; p.ep.b = o.b; p.ep.o_del = o.o_del; p.ep.e_del = o.e_del; p.ep.o_ins = o.o_ins; p.ep.e_ins = o.e_ins; p.ep.w = o.w;
    p.ep.pen_clip5 = o.pen_clip5; p.ep.pen_clip3 = o.pen_clip3; p.ep.max_chain_gap = o.max_chain_gap; p.ep.mask_level_redun = o.mask_level_redun;
    memcpy(p.ep.mat, o.mat, 25);
    p.T = o.T; p.flag = o.flag; p.min_seed_len = o.min_seed_len; p.pen_unpaired = o.pen_unpaired; p.mask_level = o.mask_level; p.drop_ratio = o.drop_ratio;
    p.mapQ_coef_len = o.mapQ_coef_len; p.mapQ_coef_fac = o.mapQ_coef_fac;
    p.XA_drop_ratio = o.XA_drop_ratio; p.max_XA_hits = o.max_XA_hits; p.max_XA_hits_alt = o.max_XA_hits_alt;
    MatePes pes;
    for (int d = 0; d < 4; ++d) { pes.low[d] = paired ? pes4[d].low : 0; pes.high[d] = paired ? pes4[d].high : 0; pes.failed[d] = paired ? pes4[d].failed : 1; }
    const int n_log = 1 << 16;
    std::vector<double> tab((size_t) n_log);
    for (int k = 0; k < n_log; ++k) tab[(size_t) k] = log((double) k);
    SamTables tb; tb.n_log = n_log;
    size_t term_total = 0, term_at[4];
    for (int d = 0; d < 4; ++d) {
        tb.pair_lo[d] = pes.low[d]; tb.pair_hi[d] = pes.failed[d] ? (int64_t) pes.low[d] - 1 : pes.high[d];
        term_at[d] = term_total;
        if (tb.pair_hi[d] >= tb.pair_lo[d]) term_total += (size_t) (tb.pair_hi[d] - tb.pair_lo[d] + 1);
    }
    if (term_total > ((size_t) 1 << 28)) { bm2_set_error(ctx, "bm2_sam_pe: insert-size bounds span more than 2^28 values"); return 1; }
    std::vector<double> term(term_total + 1);
    for (int d = 0; d < 4; ++d)
        for (int64_t dist = tb.pair_lo[d]; dist <= tb.pair_hi[d]; ++dist) {
            const double ns = (dist - pes4[d].avg) / pes4[d].std;                 // src/bwamem_pair.cpp:320-322
            term[term_at[d] + (size_t) (dist - tb.pair_lo[d])] = .721 * log(2. * erfc(fabs(ns) * M_SQRT1_2)) * o.a;
        }
    if (ctx->ensure(ctx->sam_d[SB_LOG], tab.size() * 8) || ctx->ensure(ctx->sam_d[SB_TERM], term.size() * 8)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->sam_d[SB_LOG].p, tab.data(), tab.size() * 8, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->sam_d[SB_TERM].p, term.data(), term.size() * 8, cudaMemcpyHostToDevice, st));
    tb.log_tab = P<double>(ctx, SB_LOG);
    for (int d = 0; d < 4; ++d) tb.pair_term[d] = P<double>(ctx, SB_TERM) + term_at[d];
    ContigView cv; cv.l_pac = ctx->idx.l_pac; cv.n_seqs = ctx->idx.n_seqs; cv.ann_off = ctx->idx.ann_off; cv.ann_len = ctx->idx.ann_len; cv.ann_alt = ctx->idx.ann_alt;
    const int rescue = paired && !(o.flag & 0x20);
    int staged = ctx->sam_staged;
    // default: staged, one window per warp - byte-identical records (tests/test_zzz_sam_staged_gpu.py) and about 12x the per-pair mode on the 1 Gbp
    // bench workload (H100); BM2_SAM_STAGED / bm2_set_sam_staged select the other modes
    if (staged < 0) { const char *e = getenv("BM2_SAM_STAGED"); staged = e ? atoi(e) : 1; if (staged < 0 || staged > 2) staged = 1; }
    if (!rescue) staged = 0;
    for (double &v : ctx->sam_ms) v = 0;
    for (unsigned long long &v : ctx->sam_counts) v = 0;
    ctx->sam_counts[0] = (unsigned long long) staged;
    for (cudaEvent_t &ev : ctx->sam_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));

    // ---- inputs ------------------------------------------------------------------------------------------------------------
    const int64_t total = reads->offsets[nr], n_regs = read_off[nr];
    if (ctx->ensure(ctx->sam_d[SB_CODES], (size_t) total + 16) || ctx->ensure(ctx->sam_d[SB_OFFS], (size_t) (nr + 1) * 8) ||
        ctx->ensure(ctx->sam_d[SB_REGS], (size_t) (n_regs + 1) * sizeof(bm2_alnreg_t)) || ctx->ensure(ctx->sam_d[SB_REGOFF], (size_t) (nr + 1) * 8)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->sam_d[SB_CODES].p, reads->codes, (size_t) total, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->sam_d[SB_OFFS].p, reads->offsets, (size_t) (nr + 1) * 8, cudaMemcpyHostToDevice, st));
    if (n_regs) BM2_CUDA_OK(cudaMemcpyAsync(ctx->sam_d[SB_REGS].p, regs, (size_t) n_regs * sizeof(bm2_alnreg_t), cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->sam_d[SB_REGOFF].p, read_off, (size_t) (nr + 1) * 8, cudaMemcpyHostToDevice, st));

    // ---- capacities of every pair; waves by budget ---------------------------------------------------------------------------
    std::vector<PairDesc> desc((size_t) n_pairs_all);
    int max_l = 1;
    for (int r = 0; r < nr; ++r) { const int64_t ls = reads->offsets[r + 1] - reads->offsets[r]; if (ls > max_l && ls <= (1 << 24)) max_l = (int) ls; }
    for (int pr = 0; pr < n_pairs_all; ++pr) {
        SamPairShape sh;
        for (int i = 0; i < 2; ++i) {
            if (!paired && i == 1) { sam_shape_read_d(sh, 1, 0, regs, 0, o.w); break; }
            const int r = paired ? 2 * pr + i : pr;
            const int64_t nn = read_off[r + 1] - read_off[r], ls = reads->offsets[r + 1] - reads->offsets[r];
            if (nn < 0 || nn > (1 << 24) || ls < 0 || ls > (1 << 24)) { bm2_set_error(ctx, "bm2_sam_pe / bm2_sam_se: a read with more than 2^24 bases or regions"); return 1; }
            for (int64_t k = read_off[r]; k < read_off[r + 1]; ++k) {
                const long long rl = regs[k].re - regs[k].rb;
                if (rl < 0 || rl > (1 << 24)) { bm2_set_error(ctx, "bm2_sam_pe / bm2_sam_se: a region outside [0, 2^24) reference bases"); return 1; }
            }
            sam_shape_read_d(sh, i, (int) ls, regs + read_off[r], (int) nn, o.w);
        }
        desc[(size_t) pr].caps = sam_pair_caps_d(sh, pes, o.max_matesw, rescue != 0, o.a, o.e_del);
        desc[(size_t) pr].pair = pr;
    }
    // scratch + stripes of one wave (≈0.5 MB per pair of 151-bp reads with 8 regions each): an eighth of the device memory that is free
    // or already held by this context's wave buffers.  Up to four sibling contexts (bm2_mem -p 4) may each hold a wave at once, ensure()
    // adds a quarter on top, and the seed-and-extend buffers of the next chunk need room beside them.
    size_t dev_free = 0, dev_total = 0;
    BM2_CUDA_OK(cudaMemGetInfo(&dev_free, &dev_total));
    for (int b : { SB_ARENA, SB_RECS_W, SB_XA_W, SB_OPS_W, SB_MD_W }) dev_free += ctx->sam_d[b].cap;
    const size_t budget = std::min((size_t) 32 << 30, std::max((size_t) 1 << 30, dev_free / 8));
    size_t used[4] = { 0, 0, 0, 0 };                        // recs, xa, ops, md of the batch so far
    for (int w0 = 0; w0 < n_pairs_all;) {
        size_t arena = 0; int64_t nrec = 0, nxa = 0, nops = 0, nmd = 0; int w1 = w0;
        while (w1 < n_pairs_all && w1 - w0 < (1 << 20)) {
            PairDesc &d = desc[(size_t) w1];
            const size_t add = d.caps.scratch_bytes + (size_t) d.caps.recs_cap * sizeof(bm2_sam_rec) + (size_t) d.caps.xa_cap * sizeof(bm2_sam_xa) +
                               (size_t) d.caps.out_ops * 4 + (size_t) d.caps.out_md;
            const size_t now = arena + (size_t) nrec * sizeof(bm2_sam_rec) + (size_t) nxa * sizeof(bm2_sam_xa) + (size_t) nops * 4 + (size_t) nmd;
            if (w1 > w0 && now + add > budget) break;
            if (add > ((size_t) 100 << 30)) { bm2_set_error(ctx, "bm2_sam_pe: one pair needs more than 100 GB of scratch"); return 1; }
            d.arena_off = (int64_t) arena; d.rec_off = nrec; d.xa_off = nxa; d.ops_off = nops; d.md_off = nmd;
            arena += sam_align16_d(d.caps.scratch_bytes); nrec += d.caps.recs_cap; nxa += d.caps.xa_cap; nops += d.caps.out_ops; nmd += d.caps.out_md;
            ++w1;
        }
        const int np = w1 - w0;
        if (ctx->ensure(ctx->sam_d[SB_DESC], (size_t) np * sizeof(PairDesc)) || ctx->ensure(ctx->sam_d[SB_ARENA], arena + 64) ||
            ctx->ensure(ctx->sam_d[SB_RECS_W], (size_t) (nrec + 1) * sizeof(bm2_sam_rec)) || ctx->ensure(ctx->sam_d[SB_XA_W], (size_t) (nxa + 1) * sizeof(bm2_sam_xa)) ||
            ctx->ensure(ctx->sam_d[SB_OPS_W], (size_t) (nops + 4) * 4) || ctx->ensure(ctx->sam_d[SB_MD_W], (size_t) nmd + 16) ||
            ctx->ensure(ctx->sam_d[SB_CNT], (size_t) np * sizeof(PairCount)) || ctx->ensure(ctx->sam_d[SB_FINAL], (size_t) np * sizeof(PairFinal)) ||
            ctx->ensure_host(ctx->sam_h[SH_CNT], (size_t) np * (sizeof(PairCount) + sizeof(PairFinal)))) return 1;
        BM2_CUDA_OK(cudaMemcpyAsync(ctx->sam_d[SB_DESC].p, desc.data() + w0, (size_t) np * sizeof(PairDesc), cudaMemcpyHostToDevice, st));
        if (ctx->ensure(ctx->sam_d[SJ_STATS], 64)) return 1;
        BM2_CUDA_OK(cudaMemsetAsync(ctx->sam_d[SJ_STATS].p, 0, sizeof(SamStats), st));
        BM2_CUDA_OK(cudaEventRecord(ctx->sam_ev[0], st));
        if (staged) {
            int64_t bound = 0;
            for (int k = w0; k < w1; ++k) bound += mate_jobs_bound_d(read_off[2 * k + 1] - read_off[2 * k], read_off[2 * k + 2] - read_off[2 * k + 1], o.max_matesw);
            if (bound > 0x7fffffff) bound = 0x7fffffff;                       // pairs beyond the table compute in place
            const unsigned int job_cap = (unsigned int) bound;
            // one score-2 list per warp of the alignment kernel's grid: rows of the longest window, neighbours merged
            int lcap = mate_window_max_d(pes, max_l) / 2 + 2;
            int ksw_blocks = ctx->n_sm * 8;
            const size_t list_budget = (size_t) 1 << 30;
            while (ksw_blocks > ctx->n_sm && (size_t) ksw_blocks * 4 * 2 * (size_t) lcap * 4 > list_budget) ksw_blocks >>= 1;
            if ((size_t) ksw_blocks * 4 * 2 * (size_t) lcap * 4 > list_budget) lcap = (int) (list_budget / ((size_t) ksw_blocks * 4 * 2 * 4));   // longer windows: in place
            if (ctx->ensure(ctx->sam_d[SJ_PAIRJOBS], (size_t) np * sizeof(PairJobs)) || ctx->ensure(ctx->sam_d[SJ_JOBS], ((size_t) job_cap + 1) * sizeof(MateJob)) ||
                ctx->ensure(ctx->sam_d[SJ_RES], ((size_t) job_cap + 1) * sizeof(MateJobRes)) ||
                ctx->ensure(ctx->sam_d[SJ_LISTS], (size_t) ksw_blocks * 4 * 2 * (size_t) lcap * 4 + 16)) return 1;
            sam_jobs_kernel<<<(unsigned) ((np + 127) / 128), 128, 0, st>>>(cv, pes, o.min_seed_len, o.pen_unpaired, o.max_matesw, P<int64_t>(ctx, SB_OFFS),
                                                                          P<bm2_alnreg_t>(ctx, SB_REGS), P<int64_t>(ctx, SB_REGOFF), P<PairDesc>(ctx, SB_DESC), np,
                                                                          P<MateJob>(ctx, SJ_JOBS), job_cap, P<PairJobs>(ctx, SJ_PAIRJOBS), P<SamStats>(ctx, SJ_STATS));
            BM2_CUDA_OK(cudaGetLastError());
            BM2_CUDA_OK(cudaEventRecord(ctx->sam_ev[1], st));
            KswMat25 m25; memcpy(m25.m, o.mat, 25);
            if (staged == 2) {               // one window per thread: per-thread scratch instead of per-warp lists
                const int tcap = mate_window_max_d(pes, max_l) + 16;
                const size_t per_thread = sam_align16_d((size_t) 3 * (max_l + 16) * 4 + (size_t) 2 * lcap * 4 + (size_t) tcap + (size_t) max_l + 1);
                int tblocks = ctx->n_sm * 8;
                while (tblocks > ctx->n_sm && (size_t) tblocks * 128 * per_thread > ((size_t) 4 << 30)) tblocks >>= 1;
                if (ctx->ensure(ctx->sam_d[SJ_LISTS], (size_t) tblocks * 128 * per_thread + 16)) return 1;
                sam_ksw_jobs_thread_kernel<<<(unsigned) tblocks, 128, 0, st>>>(m25, o.a, o.min_seed_len, o.o_del, o.e_del, o.o_ins, o.e_ins, ctx->idx.ref, 2 * ctx->idx.l_pac,
                              P<uint8_t>(ctx, SB_CODES), P<int64_t>(ctx, SB_OFFS), nr, P<MateJob>(ctx, SJ_JOBS), P<SamStats>(ctx, SJ_STATS), job_cap,
                              P<uint8_t>(ctx, SJ_LISTS), per_thread, max_l, lcap, tcap, P<MateJobRes>(ctx, SJ_RES));
            } else {
                // the kernel instance whose lanes hold the longest read of the batch; longer reads than any instance holds are aligned in place
#define BM2_SAM_KSW_LAUNCH(T) sam_ksw_jobs_kernel<T><<<(unsigned) ksw_blocks, 128, 0, st>>>(m25, o.a, o.min_seed_len, o.o_del, o.e_del, o.o_ins, o.e_ins, ctx->idx.ref, \
                                  2 * ctx->idx.l_pac, P<uint8_t>(ctx, SB_CODES), P<int64_t>(ctx, SB_OFFS), nr, P<MateJob>(ctx, SJ_JOBS), P<SamStats>(ctx, SJ_STATS), \
                                  job_cap, P<int32_t>(ctx, SJ_LISTS), lcap, P<MateJobRes>(ctx, SJ_RES))
                switch (ksw_kernel_width_d(max_l)) {
                case 5: BM2_SAM_KSW_LAUNCH(5); break;
                case 8: BM2_SAM_KSW_LAUNCH(8); break;
                default: BM2_SAM_KSW_LAUNCH(BM2_KSW_CMAX); break;
                }
#undef BM2_SAM_KSW_LAUNCH
            }
            BM2_CUDA_OK(cudaGetLastError());
        } else BM2_CUDA_OK(cudaEventRecord(ctx->sam_ev[1], st));
        {   // processing order of the per-pair kernel: pairs that need a gapped CIGAR (infer_bw > 0 for the best region of a read: a banded DP
            // with backtrack) apart from those that do not, then by the number of regions (mark_primary / pairing are quadratic in it)
            std::vector<std::pair<int, int32_t>> keyed((size_t) np);
            for (int k = 0; k < np; ++k) {
                const int pr = desc[(size_t) (w0 + k)].pair;
                int gapped = 0; long long nreg = 0;
                for (int i = 0; i < (paired ? 2 : 1); ++i) {
                    const int r = paired ? 2 * pr + i : pr;
                    const int64_t b = read_off[r], e = read_off[r + 1];
                    nreg += e - b;
                    for (int64_t q = b; q < e && q < b + 2; ++q) {
                        const bm2_alnreg_t &a = regs[q];
                        const int l1 = a.qe - a.qb, l2 = (int) (a.re - a.rb);
                        if (sam_infer_bw_d(l1, l2, a.truesc, o.a, o.o_del, o.e_del) > 0 || sam_infer_bw_d(l1, l2, a.truesc, o.a, o.o_ins, o.e_ins) > 0) ++gapped;
                    }
                }
                keyed[(size_t) k] = { gapped * 4096 + (int) (nreg > 4095 ? 4095 : nreg), (int32_t) k };
            }
            // The sorted order was slower in an A/B - the kernel is bound by the
            // latency of its per-thread global-memory DP rows and backtrack bytes (91 stall cycles per issue on long scoreboard, 3 % of the issue
            // slots), and neighbouring pairs share cache lines of regs / reads that the sort scatters.  Off
            // unless BM2_SAM_ORDER=1.
            const char *env = getenv("BM2_SAM_ORDER");
            if (env && env[0] == '1') std::stable_sort(keyed.begin(), keyed.end(), [](const std::pair<int, int32_t> &x, const std::pair<int, int32_t> &y) { return x.first < y.first; });
            std::vector<int32_t> order((size_t) np);
            for (int k = 0; k < np; ++k) order[(size_t) k] = keyed[(size_t) k].second;
            if (ctx->ensure(ctx->sam_d[SB_ORDER], (size_t) np * 4 + 16)) return 1;
            BM2_CUDA_OK(cudaMemcpyAsync(ctx->sam_d[SB_ORDER].p, order.data(), (size_t) np * 4, cudaMemcpyHostToDevice, st));
            BM2_CUDA_OK(cudaStreamSynchronize(st));              // (order is a local vector)
        }
        BM2_CUDA_OK(cudaEventRecord(ctx->sam_ev[2], st));
        sam_kernel<<<(unsigned) ((np + 63) / 64), 64, 0, st>>>(p, tb, cv, pes, o.max_matesw, rescue, ctx->idx.ref, P<uint8_t>(ctx, SB_CODES), P<int64_t>(ctx, SB_OFFS),
                                                              P<bm2_alnreg_t>(ctx, SB_REGS), P<int64_t>(ctx, SB_REGOFF), P<PairDesc>(ctx, SB_DESC), np, paired, id_base,
                                                              P<uint8_t>(ctx, SB_ARENA), P<bm2_sam_rec>(ctx, SB_RECS_W), P<bm2_sam_xa>(ctx, SB_XA_W),
                                                              P<uint32_t>(ctx, SB_OPS_W), P<char>(ctx, SB_MD_W), P<PairCount>(ctx, SB_CNT),
                                                              staged ? P<PairJobs>(ctx, SJ_PAIRJOBS) : nullptr, P<MateJob>(ctx, SJ_JOBS), P<MateJobRes>(ctx, SJ_RES),
                                                              P<SamStats>(ctx, SJ_STATS), P<int32_t>(ctx, SB_ORDER));
        BM2_CUDA_OK(cudaGetLastError());
        BM2_CUDA_OK(cudaEventRecord(ctx->sam_ev[3], st));
        SamStats wave_stats;
        BM2_CUDA_OK(cudaMemcpyAsync(&wave_stats, ctx->sam_d[SJ_STATS].p, sizeof(SamStats), cudaMemcpyDeviceToHost, st));
        PairCount *hc = (PairCount *) ctx->sam_h[SH_CNT].p; PairFinal *hf = (PairFinal *) (hc + np);
        BM2_CUDA_OK(cudaMemcpyAsync(hc, ctx->sam_d[SB_CNT].p, (size_t) np * sizeof(PairCount), cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        PairFinal run = { 0, 0, 0, 0 };
        for (int k = 0; k < np; ++k) {
            if (hc[k].overflow) {
                bm2_set_error(ctx, "bm2_sam_pe: scratch of pair " + std::to_string(w0 + k) + " was too small (BM2_OVF bits " + std::to_string(hc[k].overflow) + ")");
                return 1;
            }
            hf[k] = run;
            run.recs += hc[k].recs; run.xa += hc[k].xa; run.ops += hc[k].ops; run.md += hc[k].md;
        }
        if (ctx->ensure(ctx->sam_d[SB_RECS], (size_t) (run.recs + 1) * sizeof(bm2_sam_rec)) || ctx->ensure(ctx->sam_d[SB_XA], (size_t) (run.xa + 1) * sizeof(bm2_sam_xa)) ||
            ctx->ensure(ctx->sam_d[SB_OPS], (size_t) (run.ops + 4) * 4) || ctx->ensure(ctx->sam_d[SB_MD], (size_t) run.md + 16)) return 1;
        BM2_CUDA_OK(cudaMemcpyAsync(ctx->sam_d[SB_FINAL].p, hf, (size_t) np * sizeof(PairFinal), cudaMemcpyHostToDevice, st));
        sam_gather_kernel<<<(unsigned) ((np + 127) / 128), 128, 0, st>>>(P<PairDesc>(ctx, SB_DESC), P<PairCount>(ctx, SB_CNT), P<PairFinal>(ctx, SB_FINAL), np,
                                                                        P<bm2_sam_rec>(ctx, SB_RECS_W), P<bm2_sam_xa>(ctx, SB_XA_W), P<uint32_t>(ctx, SB_OPS_W),
                                                                        P<char>(ctx, SB_MD_W), (int64_t) (used[2] / 4), (int64_t) used[3], P<bm2_sam_rec>(ctx, SB_RECS),
                                                                        P<bm2_sam_xa>(ctx, SB_XA), P<uint32_t>(ctx, SB_OPS), P<char>(ctx, SB_MD));
        BM2_CUDA_OK(cudaGetLastError());
        const size_t add[4] = { (size_t) run.recs * sizeof(bm2_sam_rec), (size_t) run.xa * sizeof(bm2_sam_xa), (size_t) run.ops * 4, (size_t) run.md };
        const int hb[4] = { SH_RECS, SH_XA, SH_OPS, SH_MD }, db[4] = { SB_RECS, SB_XA, SB_OPS, SB_MD };
        for (int k = 0; k < 4; ++k) {
            if (grow_host(ctx, ctx->sam_h[hb[k]], used[k], used[k] + add[k] + 64)) return 1;
            if (add[k]) BM2_CUDA_OK(cudaMemcpyAsync((char *) ctx->sam_h[hb[k]].p + used[k], ctx->sam_d[db[k]].p, add[k], cudaMemcpyDeviceToHost, st));
            used[k] += add[k];
        }
        BM2_CUDA_OK(cudaEventRecord(ctx->sam_ev[4], st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        for (int k = 0; k < 4; ++k) { float ms = 0; BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->sam_ev[k], ctx->sam_ev[k + 1])); ctx->sam_ms[k] += ms; }
        ctx->sam_counts[1] += wave_stats.n_jobs; ctx->sam_counts[2] += wave_stats.looked_up; ctx->sam_counts[3] += wave_stats.in_place;
        ctx->sam_counts[4] += wave_stats.window_moved; ctx->sam_counts[5] += 1;
        w0 = w1;
    }
    out->n_recs = (int64_t) (used[0] / sizeof(bm2_sam_rec)); out->recs = (const bm2_sam_rec *) ctx->sam_h[SH_RECS].p;
    out->n_xa = (int64_t) (used[1] / sizeof(bm2_sam_xa)); out->xa = (const bm2_sam_xa *) ctx->sam_h[SH_XA].p;
    out->n_ops = (int64_t) (used[2] / 4); out->cigar = (const uint32_t *) ctx->sam_h[SH_OPS].p;
    out->n_md = (int64_t) used[3]; out->md = (const char *) ctx->sam_h[SH_MD].p;
    return 0;
}
}  // namespace

extern "C" int bm2_sam_pe(bm2_ctx *ctx, const bm2_read_batch *reads, const bm2_alnreg_t *regs, const int64_t *read_off, const bm2_pestat_t pes4[4],
                          int64_t id_base, bm2_sam_result *out)
{
    if (!pes4) { if (ctx) bm2_set_error(ctx, "bm2_sam_pe: pes is NULL"); return 1; }
    return run_sam(ctx, reads, regs, read_off, pes4, id_base, out);
}

extern "C" int bm2_sam_se(bm2_ctx *ctx, const bm2_read_batch *reads, const bm2_alnreg_t *regs, const int64_t *read_off, int64_t id_base, bm2_sam_result *out)
{
    return run_sam(ctx, reads, regs, read_off, nullptr, id_base, out);
}
