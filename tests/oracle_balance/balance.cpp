// TEST INFRASTRUCTURE ONLY.  The CPU oracle's restatement of the reference's LogUp balance debugger,
// `check_trace_balance` (air/src/lookup/debug/trace/mod.rs:169-309: run_trace_walk + finalize; builder.rs:204-208
// track_mutex; the boundary emitter builder.rs:401-415), as one more C entry point beside the oracle's own: the oracle's C
// API (oracle/capi.cpp, unchanged) is compiled into this library with it, so statements and matrices are converted
// exactly as for orc_prove, and every lookup node is evaluated by the oracle's node evaluator (air_eval_folded over the
// lookup program's nodes).  Single-threaded over an ordered map, like the reference's walk over a HashMap.
// tests/test_trace_balance.py pins it on a pure-Python restatement and compares mdn_check_trace_balance with both.
#include "../../oracle/capi.cpp"
#include <map>
#include <set>

extern "C" {

// same layouts as mdn_unmatched / mdn_balance_push / mdn_mutex_violation / mdn_balance_report (include/miden_b200.h)
struct orc_unmatched { uint64_t denom[2], net_multiplicity, n_pushes, first_row; uint32_t first_instance, first_interaction; };
struct orc_balance_push { uint64_t row, multiplicity; uint32_t instance, column, interaction, reserved; };
struct orc_mutex_violation { uint64_t row; uint32_t instance, column, group, active_flags; };
struct orc_balance_report {
    uint32_t holds, contributions_complete;
    uint64_t n_pushes, n_denominators, n_unmatched, n_mutex_violations, n_contributions;
    uint32_t n_skipped_airs, reserved;
    const orc_unmatched* unmatched; const orc_balance_push* contributions; const orc_mutex_violation* mutex_violations;
    uint64_t n_mutex_listed;
};

// 0 when the walk ran (`out` points into this library's storage until the next call), -1 on malformed input.
int orc_check_trace_balance(const orc_statement* st, const orc_matrix* traces, const uint64_t* randomness,
                            const uint64_t* boundary, size_t n_boundary, const uint32_t* const* mutex_sites,
                            uint64_t max_contributions, orc_balance_report* out) {
    static std::vector<orc_unmatched> unmatched;
    static std::vector<orc_balance_push> contributions;
    static std::vector<orc_mutex_violation> mutex;
    try {
        Statement s = to_statement(st);
        size_t k = s.airs.size();
        if (k == 0) throw std::runtime_error("balance: no instances provided");
        size_t max_rand = 0;
        for (auto& a : s.airs) max_rand = std::max(max_rand, a.num_randomness);
        std::vector<Ef> challenges;
        for (size_t i = 0; i < max_rand; i++) challenges.push_back(Ef(Fp(randomness[2 * i]), Fp(randomness[2 * i + 1])));
        // DebugTraceState: balances by encoded denominator, the push log in emission order, mutex violations
        typedef std::pair<u64, u64> Denom;
        std::map<Denom, Fp> balances;
        std::vector<std::pair<Denom, orc_balance_push>> push_log;
        mutex.clear();
        uint32_t skipped = 0;
        for (size_t i = 0; i < k; i++) {
            const AirDesc& a = s.airs[i];
            if (!a.lookup.present()) { skipped++; continue; }
            Matrix tr = to_matrix(traces[i]);
            if (tr.width != a.width) throw std::runtime_error("balance: trace width mismatch");
            const LookupProgram& lp = a.lookup;
            AirProgram nodes; nodes.nodes = lp.nodes; nodes.consts = lp.consts;   // the node evaluator, no constraints
            const uint32_t* ann = mutex_sites ? mutex_sites[i] : nullptr;
            size_t N = tr.height, maxp = size_t(1) << a.log_max_period;
            std::vector<Ef> scratch, per(a.n_periodic);
            for (size_t r = 0; r < N; r++) {
                for (size_t c = 0; c < a.n_periodic; c++) per[c] = Ef(a.periodic[(r % maxp) * a.n_periodic + c]);
                AirPoint pt{};
                pt.main_local = tr.row(r); pt.main_next = tr.row((r + 1) % N);
                pt.publics = s.public_values.data(); pt.challenges = challenges.data(); pt.periodic = per.data();
                air_eval_folded(nodes, pt, Ef(), scratch);
                std::map<std::pair<uint32_t, uint32_t>, std::set<uint32_t>> active_sites;   // (column, group) -> sites
                for (size_t q = 0; q < lp.interactions.size(); q++) {
                    const LookupInteraction& it = lp.interactions[q];
                    Fp flag = it.flag == LookupProgram::NO_FLAG ? Fp::raw(1) : scratch[it.flag].a;
                    if (ann && ann[q] != 0xFFFFFFFFu && !flag.is_zero()) active_sites[{it.column, ann[q] >> 16}].insert(ann[q] & 0xFFFFu);
                    if (flag.is_zero()) continue;
                    const Ef& d = scratch[it.denominator];
                    Fp m = scratch[it.multiplicity].a;
                    Denom key{d.a.v, d.b.v};
                    balances[key] += m;
                    push_log.push_back({key, orc_balance_push{r, m.v, (uint32_t)i, it.column, (uint32_t)q, 0}});
                }
                for (auto& g : active_sites)
                    if (g.second.size() > 1) mutex.push_back(orc_mutex_violation{r, (uint32_t)i, g.first.first, g.first.second, (uint32_t)g.second.size()});
            }
        }
        for (size_t q = 0; q < n_boundary; q++) {
            const uint64_t* b = boundary + 3 * q;
            if (b[0] >= P || b[1] >= P || b[2] >= P) throw std::runtime_error("balance: non-canonical boundary emission");
            Denom key{b[0], b[1]};
            balances[key] += Fp(b[2]);
            push_log.push_back({key, orc_balance_push{~0ull, b[2], 0xFFFFFFFFu, 0xFFFFFFFFu, (uint32_t)q, 0}});
        }
        // finalize: the unmatched denominators in ascending order, each with its pushes in emission order
        unmatched.clear(); contributions.clear();
        std::map<Denom, size_t> rank;
        for (auto& e : balances) {
            if (e.second.is_zero()) continue;
            rank[e.first] = unmatched.size();
            unmatched.push_back(orc_unmatched{{e.first.first, e.first.second}, e.second.v, 0, 0, 0, 0});
        }
        std::vector<std::vector<orc_balance_push>> by_rank(unmatched.size());
        for (auto& p : push_log) {
            auto it = rank.find(p.first);
            if (it == rank.end()) continue;
            orc_unmatched& u = unmatched[it->second];
            if (u.n_pushes++ == 0) { u.first_row = p.second.row; u.first_instance = p.second.instance; u.first_interaction = p.second.interaction; }
            by_rank[it->second].push_back(p.second);
        }
        uint64_t n_contrib = 0;
        for (auto& v : by_rank) n_contrib += v.size();
        bool complete = n_contrib <= max_contributions;
        if (complete) for (auto& v : by_rank) contributions.insert(contributions.end(), v.begin(), v.end());
        orc_balance_report rep{};
        rep.holds = unmatched.empty() && mutex.empty();
        rep.contributions_complete = complete;
        rep.n_pushes = push_log.size(); rep.n_denominators = balances.size(); rep.n_unmatched = unmatched.size();
        rep.n_mutex_violations = mutex.size(); rep.n_contributions = n_contrib; rep.n_skipped_airs = skipped;
        rep.unmatched = unmatched.data(); rep.contributions = complete ? contributions.data() : nullptr;
        rep.mutex_violations = mutex.data(); rep.n_mutex_listed = std::min<uint64_t>(mutex.size(), max_contributions);
        *out = rep;
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

}  // extern "C"
