// TEST INFRASTRUCTURE ONLY.  The CPU oracle's constraint checker (tests/oracle_check, orc_check_constraints) extended
// to keep every violation: orc_constraint_census walks every constraint of every AIR on every trace row exactly as
// orc_check_constraints does -- the oracle's C API (oracle/capi.cpp, unchanged) compiled in, the oracle's challenger,
// LogUp builder or the host callback for the aux traces, the node values of air_eval_folded -- and fills the layout
// of mdn_constraint_census.  tests/test_constraint_census.py pins it on a pure-Python reduction and compares the
// device's mdn_constraint_census with both.
#include "../../oracle/capi.cpp"

extern "C" {

// same layouts as include/miden_b200.h
struct orc_constraint_report { uint32_t holds, kind, instance, constraint; uint64_t row; uint64_t value[2]; uint64_t failing_rows; };
struct orc_constraint_failure { uint32_t instance, constraint; uint64_t row; uint64_t value[2]; };
struct orc_constraint_tally { uint32_t instance, constraint; uint64_t failing_rows, first_row, last_row; uint64_t first_value[2]; };
struct orc_constraint_census_report { orc_constraint_report first; uint64_t violations, n_failures, failing_constraints, n_tallies; };
typedef int (*orc_external_check)(void* ctx, const uint64_t* challenges, uint32_t n_challenges, const uint64_t* const* aux_values,
                                  const uint32_t* n_aux_values, const uint8_t* log_trace_heights, uint32_t n_airs, uint32_t* failed);

// 0 when the census ran (`out` and the first n_failures / n_tallies entries filled), -1 on malformed input or a failing
// callback (orc_last_error).  Arguments as orc_check_constraints plus the two host lists and their capacities.
int orc_constraint_census(const orc_statement* st, const orc_matrix* traces, const orc_matrix* preprocessed,
                          const orc_challenger* challenger, orc_aux_builder cb, void* ctx, orc_external_check ext, void* ext_ctx,
                          uint64_t* randomness_out, orc_constraint_failure* failures, uint64_t max_failures,
                          orc_constraint_tally* tallies, uint64_t max_tallies, orc_constraint_census_report* out) {
    try {
        Statement s = to_statement(st);
        size_t k = s.airs.size();
        if (k == 0) throw std::runtime_error("check: no instances provided");
        std::vector<Matrix> tr, prep(k);
        std::vector<unsigned> lh;
        for (size_t i = 0; i < k; i++) {
            tr.push_back(to_matrix(traces[i]));
            if (tr[i].width != s.airs[i].width) throw std::runtime_error("check: trace width mismatch");
            lh.push_back(traces[i].log_height);
            size_t pw = s.airs[i].preprocessed_width;
            if (!pw) continue;
            if (!preprocessed || preprocessed[i].width != pw || preprocessed[i].log_height != traces[i].log_height)
                throw std::runtime_error("check: preprocessed presence or shape mismatch");
            prep[i] = to_matrix(preprocessed[i]);
        }
        // challenges from the statement and the shape only, no commitment (debug.rs:87-97)
        Challenger ch = to_challenger(challenger);
        for (Fp f : s.observe_felts) ch.observe(f);
        ch.observe(Fp::raw((u64)k));
        for (size_t i = 0; i < k; i++) ch.observe(Fp::raw((u64)lh[i]));
        size_t max_rand = 0;
        for (auto& a : s.airs) max_rand = std::max(max_rand, a.num_randomness);
        std::vector<Ef> randomness;
        for (size_t i = 0; i < max_rand; i++) randomness.push_back(ch.sample_ext());
        if (randomness_out) for (size_t i = 0; i < max_rand; i++) { randomness_out[2 * i] = randomness[i].a.v; randomness_out[2 * i + 1] = randomness[i].b.v; }
        // aux traces with those challenges (debug.rs:99-106)
        std::vector<Matrix> aux(k); std::vector<std::vector<Ef>> auxv(k);
        for (size_t i = 0; i < k; i++) {
            const AirDesc& a = s.airs[i];
            std::vector<Ef> r(randomness.begin(), randomness.begin() + a.num_randomness);
            aux[i] = Matrix(tr[i].height, 2 * a.aux_width);
            auxv[i].assign(a.num_aux_values, Ef());
            if (a.lookup.present()) { build_logup_aux(a, tr[i], r, s.public_values, aux[i], auxv[i]); continue; }
            if (!cb) continue;
            std::vector<uint64_t> rr; for (auto& e : r) { rr.push_back(e.a.v); rr.push_back(e.b.v); }
            rr.push_back(0);
            std::vector<uint64_t> ao(aux[i].v.size() + 1), avo(2 * auxv[i].size() + 1);
            if (cb(ctx, (uint32_t)i, &traces[i], rr.data(), ao.data(), avo.data()) != 0) throw std::runtime_error("aux builder failed");
            for (size_t q = 0; q < aux[i].v.size(); q++) aux[i].v[q] = Fp(ao[q]);
            for (size_t q = 0; q < auxv[i].size(); q++) auxv[i][q] = Ef(Fp(avo[2 * q]), Fp(avo[2 * q + 1]));
        }
        // external assertions first (debug.rs:108-118)
        int ext_rc = 0; uint32_t ext_failed = 0;
        if (ext) {
            std::vector<uint64_t> chal; for (auto& e : randomness) { chal.push_back(e.a.v); chal.push_back(e.b.v); }
            std::vector<std::vector<uint64_t>> vals(k); std::vector<const uint64_t*> vp(k); std::vector<uint32_t> vn(k); std::vector<uint8_t> h8(k);
            for (size_t i = 0; i < k; i++) {
                for (auto& e : auxv[i]) { vals[i].push_back(e.a.v); vals[i].push_back(e.b.v); }
                vp[i] = vals[i].data(); vn[i] = (uint32_t)auxv[i].size(); h8[i] = (uint8_t)lh[i];
            }
            ext_rc = ext(ext_ctx, chal.data(), (uint32_t)randomness.size(), vp.data(), vn.data(), h8.data(), (uint32_t)k, &ext_failed);
            if (ext_rc < 0) throw std::runtime_error("eval_external reported a reduction error");
        }
        // every constraint on every row, every violation kept: failures in (instance, row, constraint) order, one
        // tally per (instance, constraint); the first failure is the first one met, as orc_check_constraints reports it
        orc_constraint_census_report cen{};
        orc_constraint_report& rep = cen.first;
        std::vector<orc_constraint_tally> all;
        std::vector<Ef> scratch, per;
        for (size_t i = 0; i < k; i++) {
            const AirDesc& a = s.airs[i];
            size_t N = tr[i].height, maxp = size_t(1) << a.log_max_period, nc = a.program.constraints.size();
            std::vector<orc_constraint_tally> t(nc);
            for (size_t r = 0; r < N; r++) {
                size_t rn = (r + 1) % N;
                per.assign(a.n_periodic, Ef());
                for (size_t c = 0; c < a.n_periodic; c++) per[c] = Ef(a.periodic[(r % maxp) * a.n_periodic + c]);
                AirPoint pt{};
                pt.main_local = tr[i].row(r); pt.main_next = tr[i].row(rn);
                pt.aux_local = aux[i].row(r); pt.aux_next = aux[i].row(rn);
                pt.publics = s.public_values.data(); pt.challenges = randomness.data(); pt.aux_values = auxv[i].data();
                pt.periodic = per.data();
                if (a.preprocessed_width) { pt.prep_local = prep[i].row(r); pt.prep_next = prep[i].row(rn); }
                pt.is_first = Ef(Fp::raw(r == 0)); pt.is_last = Ef(Fp::raw(r == N - 1)); pt.is_transition = Ef(Fp::raw(r != N - 1));
                air_eval_folded(a.program, pt, Ef(), scratch);
                bool row_fails = false;
                for (size_t c = 0; c < nc; c++) {
                    const Ef& v = scratch[a.program.constraints[c]];
                    if (v.is_zero()) continue;
                    if (rep.kind == 0) { rep.kind = 1; rep.instance = (uint32_t)i; rep.row = r; rep.constraint = (uint32_t)c; rep.value[0] = v.a.v; rep.value[1] = v.b.v; }
                    row_fails = true;
                    if (cen.violations < max_failures)
                        failures[cen.violations] = orc_constraint_failure{(uint32_t)i, (uint32_t)c, (uint64_t)r, {v.a.v, v.b.v}};
                    cen.violations++;
                    if (t[c].failing_rows++ == 0) { t[c].first_row = r; t[c].first_value[0] = v.a.v; t[c].first_value[1] = v.b.v; }
                    t[c].last_row = r;
                }
                rep.failing_rows += row_fails;
            }
            for (size_t c = 0; c < nc; c++) {
                if (!t[c].failing_rows) continue;
                t[c].instance = (uint32_t)i; t[c].constraint = (uint32_t)c;
                all.push_back(t[c]);
            }
        }
        cen.n_failures = std::min<uint64_t>(cen.violations, max_failures);
        cen.failing_constraints = all.size();
        cen.n_tallies = std::min<uint64_t>(all.size(), max_tallies);
        for (uint64_t q = 0; q < cen.n_tallies; q++) tallies[q] = all[q];
        if (ext_rc > 0) { uint64_t fr = rep.failing_rows; rep = orc_constraint_report{}; rep.kind = 2; rep.constraint = ext_failed; rep.failing_rows = fr; }
        rep.holds = rep.kind == 0;
        *out = cen;
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

}  // extern "C"
