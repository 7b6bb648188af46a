// TEST INFRASTRUCTURE ONLY.  The CPU oracle's restatement of the reference's constraint-path fold collector,
// `collect_column_oracle_folds` (air/src/lookup/debug/trace/mod.rs:191-207 over run_trace_walk :220-282, filled by the
// column / group / batch handles of DebugTraceBuilder, debug/trace/builder.rs:114-149,234-372), and of the comparison
// the reference makes with it, `assert_prover_matches_oracle` (processor/src/trace/tests/lookup.rs:185-265), as two more
// C entry points beside the oracle's own: the oracle's C API (oracle/capi.cpp, unchanged) is compiled into this library
// with them, and every lookup node is evaluated by the oracle's node evaluator.  The lowered program lists interactions
// only, so the group and batch structure comes as the fold marks of mdn_check_lookup_folds (include/miden_b200.h) and is
// rebuilt here as explicit column -> group -> call -> interaction lists, folded by handle objects like the builder's.
// Single-threaded, like the reference's walk.  tests/test_lookup_folds.py compares mdn_check_lookup_folds with it and
// with a pure-Python restatement.
#include "../../oracle/capi.cpp"

namespace {

struct Call { std::vector<size_t> interactions; };            // one insert / insert_encoded / batch
struct Group { std::vector<Call> calls; };
struct Column { std::vector<Group> groups; };

// DebugTraceBatch: (N, D) from (0, 1)
struct BatchHandle {
    Ef n = Ef(), d = Ef(Fp::raw(1));
    void insert(Fp multiplicity, Ef v_msg) { Ef d_prev = d; n = n * v_msg + d_prev * multiplicity; d = d * v_msg; }
};
// DebugTraceGroup: (V_g, U_g) from (0, 1); insert is the early-returning form, batch the flag-weighted one
struct GroupHandle {
    Ef u = Ef(Fp::raw(1)), v = Ef();
    void insert(Fp flag, Fp multiplicity, Ef v_msg) {
        if (flag.is_zero()) return;
        u += (v_msg - Fp::raw(1)) * flag;
        v += Ef(flag * multiplicity);
    }
    void batch(Fp flag, const BatchHandle& b) { u += (b.d - Fp::raw(1)) * flag; v += b.n * flag; }
};

std::vector<Column> structure_of(const LookupProgram& lp, size_t n_cols, const uint32_t* marks) {
    std::vector<Column> cols(n_cols);
    Group* g = nullptr;
    for (size_t q = 0; q < lp.interactions.size(); q++) {
        uint32_t m = marks ? marks[q] : 3u;
        Column& c = cols.at(lp.interactions[q].column);
        if (m == 3) { c.groups.emplace_back(); g = &c.groups.back(); }
        if (!g || (m != 0 && m != 1 && m != 3)) throw std::runtime_error("folds: bad fold mark");
        if (m & 1) g->calls.emplace_back();
        if (g->calls.empty()) throw std::runtime_error("folds: bad fold mark");
        g->calls.back().interactions.push_back(q);
    }
    return cols;
}

// folds[r * n_cols + c] = (V, U) of AIR `a` over `tr`
std::vector<std::pair<Ef, Ef>> collect(const Statement& s, const AirDesc& a, const Matrix& tr, const std::vector<Ef>& challenges, const uint32_t* marks) {
    const LookupProgram& lp = a.lookup;
    size_t n_cols = a.aux_width;
    std::vector<Column> cols = structure_of(lp, n_cols, marks);
    AirProgram nodes; nodes.nodes = lp.nodes; nodes.consts = lp.consts;   // the node evaluator, no constraints
    size_t N = tr.height, maxp = size_t(1) << a.log_max_period;
    std::vector<Ef> scratch, per(a.n_periodic);
    std::vector<std::pair<Ef, Ef>> folds(N * n_cols);
    for (size_t r = 0; r < N; r++) {
        for (size_t c = 0; c < a.n_periodic; c++) per[c] = Ef(a.periodic[(r % maxp) * a.n_periodic + c]);
        AirPoint pt{};
        pt.main_local = tr.row(r); pt.main_next = tr.row((r + 1) % N);
        pt.publics = s.public_values.data(); pt.challenges = challenges.data(); pt.periodic = per.data();
        air_eval_folded(nodes, pt, Ef(), scratch);
        auto flag_of = [&](size_t q) { const LookupInteraction& it = lp.interactions[q]; return it.flag == LookupProgram::NO_FLAG ? Fp::raw(1) : scratch[it.flag].a; };
        for (size_t c = 0; c < n_cols; c++) {
            Ef v_col = Ef(), u_col = Ef(Fp::raw(1));
            for (const Group& g : cols[c].groups) {
                GroupHandle gh;
                for (const Call& call : g.calls) {
                    size_t q0 = call.interactions[0];
                    if (call.interactions.size() == 1) {
                        const LookupInteraction& it = lp.interactions[q0];
                        gh.insert(flag_of(q0), scratch[it.multiplicity].a, scratch[it.denominator]);
                        continue;
                    }
                    BatchHandle bh;
                    for (size_t q : call.interactions) bh.insert(scratch[lp.interactions[q].multiplicity].a, scratch[lp.interactions[q].denominator]);
                    gh.batch(flag_of(q0), bh);
                }
                Ef v_new = v_col * gh.u + gh.v * u_col;
                u_col = u_col * gh.u; v_col = v_new;
            }
            folds[r * n_cols + c] = {v_col, u_col};
        }
    }
    return folds;
}

std::vector<Ef> challenges_of(const Statement& s, const uint64_t* randomness) {
    size_t max_rand = 0;
    for (auto& a : s.airs) max_rand = std::max(max_rand, a.num_randomness);
    std::vector<Ef> ch;
    for (size_t i = 0; i < max_rand; i++) ch.push_back(Ef(Fp(randomness[2 * i]), Fp(randomness[2 * i + 1])));
    return ch;
}

}  // namespace

extern "C" {

// same layout as mdn_fold_report (include/miden_b200.h)
struct orc_fold_report {
    uint32_t holds, kind, instance, column;
    uint64_t row, fold[4], expected[2], actual[2], failing_rows, zero_u;
    uint32_t n_skipped_airs, reserved;
};

// folds_out[i]: NULL (also for an AIR without lookup) or rows x num_columns x 4 u64.  0, or -1 on malformed input.
int orc_collect_column_folds(const orc_statement* st, const orc_matrix* traces, const uint64_t* randomness,
                             const uint32_t* const* fold_marks, uint64_t* const* folds_out) {
    try {
        Statement s = to_statement(st);
        std::vector<Ef> ch = challenges_of(s, randomness);
        for (size_t i = 0; i < s.airs.size(); i++) {
            if (!s.airs[i].lookup.present() || !folds_out[i]) continue;
            auto folds = collect(s, s.airs[i], to_matrix(traces[i]), ch, fold_marks ? fold_marks[i] : nullptr);
            for (size_t e = 0; e < folds.size(); e++) {
                uint64_t* o = folds_out[i] + 4 * e;
                o[0] = folds[e].first.a.v; o[1] = folds[e].first.b.v; o[2] = folds[e].second.a.v; o[3] = folds[e].second.b.v;
            }
        }
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// aux[i]: host row-major, 2^log_height rows of 2 * aux_width base columns; aux_finals[i]: 2 u64.
int orc_check_lookup_folds(const orc_statement* st, const orc_matrix* traces, const uint64_t* randomness,
                           const uint32_t* const* fold_marks, const orc_matrix* aux, const uint64_t* const* aux_finals,
                           orc_fold_report* out) {
    try {
        Statement s = to_statement(st);
        std::vector<Ef> ch = challenges_of(s, randomness);
        orc_fold_report rep{};
        bool found = false;
        for (size_t i = 0; i < s.airs.size(); i++) {
            const AirDesc& a = s.airs[i];
            if (!a.lookup.present()) { rep.n_skipped_airs++; continue; }
            Matrix tr = to_matrix(traces[i]), ax = to_matrix(aux[i]);
            size_t N = tr.height, C = a.aux_width;
            if (ax.height != N || ax.width != 2 * C) throw std::runtime_error("folds: aux shape mismatch");
            auto folds = collect(s, a, tr, ch, fold_marks ? fold_marks[i] : nullptr);
            auto aux_at = [&](size_t r, size_t c) { return r == N ? Ef(Fp(aux_finals[i][0]), Fp(aux_finals[i][1])) : Ef(ax.row(r)[2 * c], ax.row(r)[2 * c + 1]); };
            for (size_t r = 0; r < N; r++) {
                bool row_bad = false, any_zero = false;
                Ef total = Ef();
                std::vector<Ef> frac(C);
                for (size_t c = 0; c < C; c++) {
                    const Ef& u = folds[r * C + c].second;
                    if (u.is_zero()) { any_zero = true; rep.zero_u++; continue; }
                    frac[c] = folds[r * C + c].first * ef_inv(u);
                    total += frac[c];
                }
                for (size_t c = 0; c < C; c++) {
                    const auto& f = folds[r * C + c];
                    Ef expected = c ? frac[c] : total, actual = c ? aux_at(r, c) : aux_at(r + 1, 0) - aux_at(r, 0);
                    uint32_t kind = 0;
                    if (f.second.is_zero()) kind = 3;
                    else if (!(c == 0 && any_zero) && !(expected == actual)) kind = c ? 1 : 2;
                    if (!kind) continue;
                    row_bad = true;
                    if (found) continue;
                    found = true;
                    rep.kind = kind; rep.instance = (uint32_t)i; rep.column = (uint32_t)c; rep.row = r;
                    rep.fold[0] = f.first.a.v; rep.fold[1] = f.first.b.v; rep.fold[2] = f.second.a.v; rep.fold[3] = f.second.b.v;
                    rep.expected[0] = expected.a.v; rep.expected[1] = expected.b.v; rep.actual[0] = actual.a.v; rep.actual[1] = actual.b.v;
                }
                if (row_bad) rep.failing_rows++;
            }
        }
        rep.holds = rep.failing_rows == 0;
        *out = rep;
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

}  // extern "C"
