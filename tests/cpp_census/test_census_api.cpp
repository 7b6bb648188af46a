// TEST INFRASTRUCTURE ONLY.  miden::constraint_census (miden-vm_b200/host/miden_prover.hpp) through the C ABI: a valid
// statement gives an empty census; three faults in two instances are listed per constraint and in row order, with the
// text of check_constraints' panics; truncation keeps the counts.  Prints CENSUS_API_OK.  Built against
// libmiden_b200.so (H100) or the CPU kernel emulator of tests/emu (Makefile).
#include "../../miden-vm_b200/host/miden_prover.hpp"
#include <cstdio>
#include <cstring>

using namespace miden;
#define CHECK(c) do { if (!(c)) { printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

// main[0] * main[1] == 0 and aux[0] == challenge(0) + main[1] (aux built on the host)
static Air air() {
    AirBuilder b;
    b.assert_zero(b.mul(b.main(0, 0), b.main(0, 1)));
    b.assert_zero_ext(b.sub(b.aux(0, 0), b.add(b.challenge(0), b.main(0, 1))));
    Air a; a.width = 2; a.aux_width = 1; a.num_aux_values = 0; a.num_randomness = 1; a.log_quotient_degree = 1;
    a.program = b.finish();
    return a;
}
static RowMajorMatrix trace(uint32_t log_h) {
    std::vector<Felt> v((size_t(1) << log_h) * 2, 0);
    for (size_t r = 0; r < (size_t(1) << log_h); r++) v[2 * r + 1] = r * 3 + 1;
    return RowMajorMatrix(std::move(v), 2);
}

int main() {
    PcsParams params; params.log_final_degree = 2; params.folding_pow_bits = 2; params.deep_pow_bits = 3; params.num_queries = 5; params.query_pow_bits = 4;
    Challenger seed;
    seed.observe_slice({1, 2, 3});
    std::unique_ptr<StarkConfig> config;
    try { config.reset(new StarkConfig(params, seed, 0)); }
    catch (const ProverError& e) {
        if (e.kind == ProverError::NoDevice) { printf("NO_DEVICE %s\n", e.what()); return 3; }
        throw;
    }
    AuxBuilder aux = [](uint32_t, const RowMajorMatrix& main, const std::vector<QuadFelt>& ch, std::vector<Felt>& flat, std::vector<QuadFelt>&) {
        const Felt P = 0xFFFFFFFF00000001ull;
        for (size_t r = 0; r < main.height(); r++) {
            flat[2 * r] = (Felt)(((unsigned __int128)ch[0][0] + main.values[2 * r + 1]) % P);
            flat[2 * r + 1] = ch[0][1];
        }
    };
    Statement st = Statement::with_default_observe({air(), air()}, {});
    {
        ProverStatement ps(st, {trace(6), trace(5)});
        ConstraintCensus c = constraint_census(*config, ps, seed, aux);
        CHECK(c.holds() && c.counts.violations == 0 && c.failures.empty() && c.tallies.empty() && c.to_string().empty());
    }
    ProverStatement ps(st, {trace(6), trace(5)});
    ps.traces[0].values[2 * 3] = 2;                    // instance 0, row 3: 2 * 10
    ps.traces[1].values[2 * 9] = 5;                    // instance 1, rows 9 and 12: 5 * 28, 5 * 37
    ps.traces[1].values[2 * 12] = 5;
    ConstraintCensus c = constraint_census(*config, ps, seed, aux);
    CHECK(!c.holds() && c.first().kind == 1 && c.first().instance == 0 && c.first().row == 3 && c.first().constraint == 0);
    CHECK(c.first().value[0] == 20 && c.first().failing_rows == 3);
    CHECK(c.counts.violations == 3 && c.counts.failing_constraints == 2);
    CHECK(c.failures.size() == 3 && c.failures[1].instance == 1 && c.failures[1].row == 9 && c.failures[1].value[0] == 140);
    CHECK(c.failures[2].row == 12 && c.failures[2].value[0] == 185);
    CHECK(c.tallies.size() == 2 && c.tallies[1].failing_rows == 2 && c.tallies[1].first_row == 9 && c.tallies[1].last_row == 12);
    CHECK(c.tallies[1].first_value[0] == 140 && c.tallies[0].first_value[0] == 20);
    std::string text = c.to_string();
    CHECK(text.find("constraint 0 of instance 1 not satisfied on 2 rows (rows 9 .. 12)") != std::string::npos);
    CHECK(text.find("constraint not satisfied at instance 1, row 12 (constraint 0)") != std::string::npos);
    bool threw = false;                                 // check_constraints panics on the census's first failure
    try { check_constraints(*config, ps, seed, aux); }
    catch (const ConstraintViolation& e) { threw = std::memcmp(&e.report, &c.counts.first, sizeof e.report) == 0; }
    CHECK(threw);
    ConstraintCensus t = constraint_census(*config, ps, seed, aux, 1, 0);
    CHECK(t.failures.size() == 1 && t.failures[0].row == 3 && t.tallies.empty() && t.counts.violations == 3);
    CHECK(std::memcmp(&t.counts.first, &c.counts.first, sizeof t.counts.first) == 0);
    CHECK(t.to_string().find("... 2 more violations") != std::string::npos);
    printf("%s", c.to_string().c_str());
    printf("CENSUS_API_OK\n");
    return 0;
}
