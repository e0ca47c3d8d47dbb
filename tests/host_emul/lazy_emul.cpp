// lazy_emul.cpp — TEST-ONLY host emulation of the lazy extension of pipeline.cu (BM2_EXT_LAZY, BM2_EXT_WAVES, BM2_EXT_WALK_HEAVY).
//
// lazy_emul_seed_chain_extend is emul_seed_chain_extend (emul.cpp) with the extension run in the kernels' waves: wave 1 extends the
// first seed of every chain, ext_walk_read_d (ext_device.cuh) then decides each read's seeds up to the first kept one not extended yet,
// the last wave extends every reg neither extended nor proved purged.  It also counts what the waves skipped, and the regs that the
// final post-filter keeps without their having been extended (must be none).  Never part of the product.
#include "emul.cpp"      // the stages before the extension (stage_smem_sa, stage_chain) and the views, shared with the eager emulation

// the last lazy_emul_seed_chain_extend call: jobs built, jobs never run, reads decided after the first wave, regs the final post-filter
// kept that were never extended
static int64_t g_ext_stats[4] = {0, 0, 0, 0};

static int env_int(const char *name, int def, int lo, int hi) {     // the knobs of pipeline.cu, same defaults and ranges
    const char *e = getenv(name);
    if (!e || !*e) return def;
    const int v = atoi(e);
    return v < lo ? lo : (v > hi ? hi : v);
}

extern "C" {

void lazy_emul_last_ext_stats(int64_t *v) { for (int i = 0; i < 4; ++i) v[i] = g_ext_stats[i]; }

int lazy_emul_seed_chain_extend(const bm2_index_desc *idx, const bm2_mem_opt_t *o, const bm2_read_batch *rb, bm2_alnreg_t **regs_out,
                                int64_t *n_regs, int64_t **read_off) {
    Views v = make_views(idx, o); Stage1 s1; stage_smem_sa(v, o, rb, s1); Stage2 s2; stage_chain(v, rb, s1, s2);
    const int n = rb->n_reads;
    // reg / job offsets (device: exclusive scans)
    std::vector<int64_t> reg_off(n + 1, 0), left_off(n + 1, 0), right_off(n + 1, 0);
    int max_chain = 1, max_len = 1;
    for (int r = 0; r < n; ++r) {
        int64_t nr = 0;
        for (int64_t c = s2.read_chain_off[r]; c < s2.read_chain_off[r + 1]; ++c) { nr += s2.chains[c].n_seeds; max_chain = std::max(max_chain, s2.chains[c].n_seeds); }
        reg_off[r + 1] = reg_off[r] + nr; left_off[r + 1] = left_off[r] + s2.n_left[r]; right_off[r + 1] = right_off[r] + s2.n_right[r];
        max_len = std::max<int>(max_len, (int) (rb->offsets[r + 1] - rb->offsets[r]));
    }
    std::vector<bm2_alnreg_t> regs(reg_off[n] + 1); std::vector<int32_t> reg_chain(reg_off[n] + 1), reg_seed(reg_off[n] + 1);
    std::vector<ExtJobRec> left(left_off[n] + 1), right(right_off[n] + 1); std::vector<int32_t> left_reg(left_off[n] + 1), right_reg(right_off[n] + 1);
    std::vector<uint64_t> srt(max_chain + 1);
    const int lazy = env_int("BM2_EXT_LAZY", 1, 0, 1), waves = env_int("BM2_EXT_WAVES", 2, 2, 64);
    const int walk_heavy = env_int("BM2_EXT_WALK_HEAVY", 256, 0, 1 << 30);
    std::vector<uint8_t> state(reg_off[n] + 1, EXT_DONE);
    for (int r = 0; r < n; ++r) {
        int64_t cb = s2.read_chain_off[r], ce = s2.read_chain_off[r + 1];
        if (ce == cb) continue;
        // chains of the read address seeds through absolute seed_off: pass seeds base 0
        ext_build_read_d(v.cv, v.ep, s2.chains.data() + cb, (int) (ce - cb), s2.seeds.data(), (int) (rb->offsets[r + 1] - rb->offsets[r]),
                         rb->offsets[r], cb, reg_off[r], regs.data() + reg_off[r], reg_chain.data() + reg_off[r], reg_seed.data() + reg_off[r],
                         left.data() + left_off[r], left_reg.data() + left_off[r], right.data() + right_off[r], right_reg.data() + right_off[r], srt.data(),
                         state.data() + reg_off[r]);
    }
    auto run_phase = [&](std::vector<ExtJobRec> &jobs, std::vector<int32_t> &job_reg, std::vector<int> todo, int is_right) {
        for (int t = 0; t < 2 && !todo.empty(); ++t) {
            int w = o->w << t;
            std::vector<int> retry;
            for (int ji : todo) {
                ExtJobRec &j = jobs[ji];
                bm2_alnreg_t &a = regs[job_reg[ji]];
                if (is_right && t == 0) j.h0 = a.score;
                std::vector<uint8_t> q(j.qlen), tg(j.tlen);
                for (int i = 0; i < j.qlen; ++i) q[i] = rb->codes[j.qoff + (int64_t) i * j.qstride];
                for (int i = 0; i < j.tlen; ++i) tg[i] = idx->ref_string[j.toff + (int64_t) i * j.tstride];
                bm2o_bsw_params bp = { o->a, o->b, o->o_del, o->e_del, o->o_ins, o->e_ins, o->zdrop, is_right ? o->pen_clip3 : o->pen_clip5, 1 };
                int32_t out[6];
                bm2o_bsw_extend(q.data(), j.qlen, tg.data(), j.tlen, w, j.h0, &bp, out);
                const bm2_chain &c = s2.chains[reg_chain[job_reg[ji]]];
                int rd = c.seqid; int l_query = (int) (rb->offsets[rd + 1] - rb->offsets[rd]);
                bool ok = ext_fold_d(v.ep, a, is_right, j.h0, out[0], out[1], out[2], out[3], out[4], out[5], w, t == 1, l_query,
                                     s2.seeds.data() + c.seed_off, c.n_seeds);
                if (!ok) retry.push_back(ji);
            }
            todo.swap(retry);
        }
    };
    std::vector<int32_t> srt2(reg_off[n] + max_chain + 1), he(2 * (max_len + 2)); std::vector<PfBox> box(reg_off[n] + 1);
    g_ext_stats[0] = left_off[n] + right_off[n]; g_ext_stats[1] = g_ext_stats[2] = g_ext_stats[3] = 0;
    if (!lazy) {
        std::vector<int> all_l(left_off[n]), all_r(right_off[n]);
        for (int64_t i = 0; i < left_off[n]; ++i) all_l[i] = (int) i;
        for (int64_t i = 0; i < right_off[n]; ++i) all_r[i] = (int) i;
        run_phase(left, left_reg, all_l, 0);
        run_phase(right, right_reg, all_r, 1);
        std::fill(state.begin(), state.end(), EXT_DONE);
    } else {     // the waves of pipeline.cu: select, left, right, mark, walk; the last wave runs every reg not extended and not purged
        std::vector<PfCursor> cur(n);
        int64_t jobs_run = 0;
        for (int wave = 1; wave <= waves; ++wave) {
            const bool last = wave == waves;
            auto pick = [&](const std::vector<int32_t> &job_reg, int64_t nj) {
                std::vector<int> sel;
                for (int64_t i = 0; i < nj; ++i) { const uint8_t st = state[job_reg[i]]; if (st == EXT_NEED || (last && st == EXT_TODO)) sel.push_back((int) i); }
                return sel;
            };
            std::vector<int> sl = pick(left_reg, left_off[n]), sr = pick(right_reg, right_off[n]);
            run_phase(left, left_reg, sl, 0);
            run_phase(right, right_reg, sr, 1);
            jobs_run += (int64_t) (sl.size() + sr.size());
            for (auto &st : state) if (st == EXT_NEED || (last && st == EXT_TODO)) st = EXT_DONE;
            if (last) break;
            for (int r = 0; r < n; ++r) {
                const int64_t cb = s2.read_chain_off[r], ce = s2.read_chain_off[r + 1];
                const int nreg = (int) (reg_off[r + 1] - reg_off[r]);
                if (ce == cb || nreg > walk_heavy) continue;
                if (wave == 1) { cur[r].ci = 0; cur[r].k = -1; cur[r].lim = 0; cur[r].base = 0; }
                if (cur[r].ci >= (int) (ce - cb)) continue;
                const bool done = ext_walk_read_d(v.ep, s2.chains.data() + cb, (int) (ce - cb), s2.seeds.data(), (int) (rb->offsets[r + 1] - rb->offsets[r]),
                                                  regs.data() + reg_off[r], nreg, reg_seed.data() + reg_off[r], state.data() + reg_off[r],
                                                  srt2.data() + reg_off[r], box.data() + reg_off[r], cur[r]);
                if (done && wave == 1) ++g_ext_stats[2];
            }
        }
        g_ext_stats[1] = g_ext_stats[0] - jobs_run;
    }
    std::vector<bm2_alnreg_t> out; std::vector<int64_t> off(n + 1, 0);
    for (int r = 0; r < n; ++r) {
        int64_t cb = s2.read_chain_off[r], ce = s2.read_chain_off[r + 1];
        int nreg = (int) (reg_off[r + 1] - reg_off[r]);
        int l_query = (int) (rb->offsets[r + 1] - rb->offsets[r]);
        if (ce > cb) {
            ext_postfilter_read_d(v.ep, s2.chains.data() + cb, (int) (ce - cb), s2.seeds.data(), l_query, regs.data() + reg_off[r], nreg,
                                  reg_seed.data() + reg_off[r], srt2.data() + reg_off[r], box.data() + reg_off[r]);
            for (int i = 0; i < nreg; ++i) {
                const bm2_alnreg_t &a = regs[reg_off[r] + i];
                if (!(a.qb == -1 && a.qe == -1) && state[reg_off[r] + i] != EXT_DONE) ++g_ext_stats[3];
            }
            int m = ext_tail_read_d(v.cv, v.ep, idx->ref_string, rb->codes + rb->offsets[r], regs.data() + reg_off[r], nreg, he.data(), srt2.data() + reg_off[r], reinterpret_cast<TailSortKey *>(box.data() + reg_off[r]));
            for (int i = 0; i < m; ++i) out.push_back(regs[reg_off[r] + i]);
        }
        off[r + 1] = (int64_t) out.size();
    }
    *regs_out = (bm2_alnreg_t *) malloc(sizeof(bm2_alnreg_t) * (out.size() + 1)); memcpy(*regs_out, out.data(), sizeof(bm2_alnreg_t) * out.size());
    *read_off = (int64_t *) malloc(8 * (n + 1)); memcpy(*read_off, off.data(), 8 * (n + 1));
    *n_regs = (int64_t) out.size();
    return 0;
}

}
