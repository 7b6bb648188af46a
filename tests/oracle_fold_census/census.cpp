// TEST INFRASTRUCTURE ONLY.  The census of the CPU oracle's LogUp fold check: tests/oracle_folds/folds.cpp (the oracle's
// C API with orc_collect_column_folds and orc_check_lookup_folds, compiled unchanged) plus two more C entry points over
// its fold walk.  orc_lookup_fold_census keeps every disagreement orc_check_lookup_folds would find, in its walk order;
// orc_logup_aux builds the prover path's aux traces for traces too tall for the Python one.  Single-threaded, like the
// reference's walk.  tests/test_lookup_fold_census.py compares mdn_lookup_fold_census with it and with a pure-Python
// census.
#include "../oracle_folds/folds.cpp"

extern "C" {

// The prover path's aux trace of every lookup AIR (test_lookup_folds.py ref_aux restated for large traces): per row
// and column c >= 1 the sum of m / d over the pushes whose flag is non-zero and whose d is non-zero, column 0 the
// running sum of every column's fractions over the rows before.  aux_out[i]: NULL or 2^log_height x 2 * aux_width u64,
// row-major; finals_out[i]: NULL or 2 u64, the running sum after the last row.
int orc_logup_aux(const orc_statement* st, const orc_matrix* traces, const uint64_t* randomness, uint64_t* const* aux_out,
                  uint64_t* const* finals_out) {
    try {
        Statement s = to_statement(st);
        std::vector<Ef> ch = challenges_of(s, randomness);
        for (size_t i = 0; i < s.airs.size(); i++) {
            const AirDesc& a = s.airs[i];
            if (!a.lookup.present() || !aux_out[i]) continue;
            const LookupProgram& lp = a.lookup;
            Matrix tr = to_matrix(traces[i]);
            AirProgram nodes; nodes.nodes = lp.nodes; nodes.consts = lp.consts;
            size_t N = tr.height, C = a.aux_width, maxp = size_t(1) << a.log_max_period;
            std::vector<Ef> scratch, per(a.n_periodic), frac(C);
            Ef acc = Ef();
            for (size_t r = 0; r < N; r++) {
                for (size_t c = 0; c < a.n_periodic; c++) per[c] = Ef(a.periodic[(r % maxp) * a.n_periodic + c]);
                AirPoint pt{};
                pt.main_local = tr.row(r); pt.main_next = tr.row((r + 1) % N);
                pt.publics = s.public_values.data(); pt.challenges = ch.data(); pt.periodic = per.data();
                air_eval_folded(nodes, pt, Ef(), scratch);
                std::fill(frac.begin(), frac.end(), Ef());
                for (const LookupInteraction& it : lp.interactions) {
                    if (it.flag != LookupProgram::NO_FLAG && scratch[it.flag].a.is_zero()) continue;
                    const Ef& d = scratch[it.denominator];
                    if (d.is_zero()) continue;
                    frac.at(it.column) += Ef(scratch[it.multiplicity].a) * ef_inv(d);
                }
                uint64_t* o = aux_out[i] + 2 * C * r;
                o[0] = acc.a.v; o[1] = acc.b.v;
                for (size_t c = 1; c < C; c++) { o[2 * c] = frac[c].a.v; o[2 * c + 1] = frac[c].b.v; }
                for (size_t c = 0; c < C; c++) acc += frac[c];
            }
            if (finals_out[i]) { finals_out[i][0] = acc.a.v; finals_out[i][1] = acc.b.v; }
        }
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// same layouts as mdn_fold_failure, mdn_fold_tally and mdn_fold_census_report (include/miden_b200.h)
struct orc_fold_failure {
    uint32_t instance, column, kind, reserved;
    uint64_t row, fold[4], expected[2], actual[2];
};
struct orc_fold_tally {
    uint32_t instance, column;
    uint64_t failing_rows, zero_u_rows, first_row, last_row;
    uint32_t first_kind, reserved;
    uint64_t first_expected[2], first_actual[2];
};
struct orc_fold_census_report {
    orc_fold_report first;
    uint64_t disagreements, n_failures, failing_columns, n_tallies;
};

// The census of orc_check_lookup_folds: the same walk keeping every (instance, row, column) of non-zero kind.  failures
// gets the first max_failures in walk order, (instance, row, column); tallies the first max_tallies (instance, column)
// pairs that disagree on at least one row; `first` the first disagreement of the walk, as orc_check_lookup_folds.
int orc_lookup_fold_census(const orc_statement* st, const orc_matrix* traces, const uint64_t* randomness,
                           const uint32_t* const* fold_marks, const orc_matrix* aux, const uint64_t* const* aux_finals,
                           orc_fold_failure* failures, uint64_t max_failures, orc_fold_tally* tallies, uint64_t max_tallies,
                           orc_fold_census_report* out) {
    try {
        Statement s = to_statement(st);
        std::vector<Ef> ch = challenges_of(s, randomness);
        orc_fold_census_report rep{};
        std::vector<orc_fold_tally> all;
        for (size_t i = 0; i < s.airs.size(); i++) {
            const AirDesc& a = s.airs[i];
            if (!a.lookup.present()) { rep.first.n_skipped_airs++; continue; }
            Matrix tr = to_matrix(traces[i]), ax = to_matrix(aux[i]);
            size_t N = tr.height, C = a.aux_width;
            if (ax.height != N || ax.width != 2 * C) throw std::runtime_error("folds: aux shape mismatch");
            auto folds = collect(s, a, tr, ch, fold_marks ? fold_marks[i] : nullptr);
            auto aux_at = [&](size_t r, size_t c) { return r == N ? Ef(Fp(aux_finals[i][0]), Fp(aux_finals[i][1])) : Ef(ax.row(r)[2 * c], ax.row(r)[2 * c + 1]); };
            std::vector<orc_fold_tally> cols(C);
            for (size_t r = 0; r < N; r++) {
                bool row_bad = false, any_zero = false;
                Ef total = Ef();
                std::vector<Ef> frac(C);
                for (size_t c = 0; c < C; c++) {
                    const Ef& u = folds[r * C + c].second;
                    if (u.is_zero()) { any_zero = true; continue; }
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
                    orc_fold_failure fl{};
                    fl.instance = (uint32_t)i; fl.column = (uint32_t)c; fl.kind = kind; fl.row = r;
                    fl.fold[0] = f.first.a.v; fl.fold[1] = f.first.b.v; fl.fold[2] = f.second.a.v; fl.fold[3] = f.second.b.v;
                    fl.expected[0] = expected.a.v; fl.expected[1] = expected.b.v; fl.actual[0] = actual.a.v; fl.actual[1] = actual.b.v;
                    if (rep.disagreements < max_failures) failures[rep.disagreements] = fl;
                    if (rep.disagreements++ == 0) {
                        rep.first.kind = kind; rep.first.instance = fl.instance; rep.first.column = fl.column; rep.first.row = r;
                        std::copy(fl.fold, fl.fold + 4, rep.first.fold);
                        std::copy(fl.expected, fl.expected + 2, rep.first.expected); std::copy(fl.actual, fl.actual + 2, rep.first.actual);
                    }
                    orc_fold_tally& t = cols[c];
                    if (t.failing_rows++ == 0) {
                        t.instance = fl.instance; t.column = fl.column; t.first_row = r; t.first_kind = kind;
                        std::copy(fl.expected, fl.expected + 2, t.first_expected); std::copy(fl.actual, fl.actual + 2, t.first_actual);
                    }
                    t.last_row = r;
                    if (kind == 3) { t.zero_u_rows++; rep.first.zero_u++; }
                }
                if (row_bad) rep.first.failing_rows++;
            }
            for (const orc_fold_tally& t : cols) if (t.failing_rows) all.push_back(t);
        }
        rep.first.holds = rep.first.failing_rows == 0;
        rep.n_failures = std::min<uint64_t>(rep.disagreements, max_failures);
        rep.failing_columns = all.size();
        rep.n_tallies = std::min<uint64_t>(all.size(), max_tallies);
        std::copy(all.begin(), all.begin() + rep.n_tallies, tallies);
        *out = rep;
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

}  // extern "C"
