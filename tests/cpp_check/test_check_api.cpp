// TEST INFRASTRUCTURE ONLY.  miden::check_constraints (miden-vm_b200/host/miden_prover.hpp) through the C ABI: a valid
// statement passes; a fault throws ConstraintViolation with debug.rs's panic text and the report; a failing external
// assertion throws with its text; a ReductionError and a failing aux builder throw ProverError.  Prints CHECK_API_OK.
// Built against libmiden_b200.so (H100) or the CPU kernel emulator of tests/emu (Makefile).
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
static int g_ext_mode = 0;
static int ext(void*, const uint64_t*, uint32_t, const uint64_t* const*, const uint32_t*, const uint8_t*, uint32_t, uint32_t* failed) {
    if (g_ext_mode == 1) { *failed = 2; return 1; }
    return g_ext_mode == 2 ? -1 : 0;
}

int main() {
    PcsParams params; params.log_final_degree = 2; params.folding_pow_bits = 2; params.deep_pow_bits = 3; params.num_queries = 5; params.query_pow_bits = 4;
    Challenger seed;                                   // config.challenger() without observe_protocol_params: any seed
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
        check_constraints(*config, ps, seed, aux);     // holds: no throw
    }
    {
        ProverStatement ps(st, {trace(6), trace(5)});
        ps.traces[1].values[2 * 9] = 5;                 // instance 1, row 9: main[0] * main[1] != 0
        bool threw = false;
        try { check_constraints(*config, ps, seed, aux); }
        catch (const ConstraintViolation& e) {
            threw = true;
            CHECK(std::string(e.what()) == "constraint not satisfied at instance 1, row 9");
            CHECK(e.report.kind == 1 && e.report.instance == 1 && e.report.row == 9 && e.report.constraint == 0);
            CHECK(e.report.value[0] == 5 * 28 && e.report.value[1] == 0 && e.report.failing_rows == 1 && e.report.holds == 0);
        }
        CHECK(threw);
        threw = false;                                  // without the aux builder the aux trace is zero: constraint 1 fails on row 0
        try { check_constraints(*config, ps, seed); }
        catch (const ConstraintViolation& e) { threw = e.report.instance == 0 && e.report.row == 0 && e.report.constraint == 1; }
        CHECK(threw);
    }
    {
        ProverStatement ps(st, {trace(6), trace(5)});
        CHECK(mdn_session_set_external_check(config->session(), ext, nullptr) == MDN_OK);
        g_ext_mode = 1;
        bool threw = false;
        try { check_constraints(*config, ps, seed, aux); }
        catch (const ConstraintViolation& e) { threw = std::string(e.what()) == "external assertion 2 is non-zero" && e.report.kind == 2; }
        CHECK(threw);
        g_ext_mode = 2;
        threw = false;
        try { check_constraints(*config, ps, seed, aux); }
        catch (const ProverError& e) { threw = e.kind == ProverError::ExternalAssertion; }
        CHECK(threw);
        g_ext_mode = 0;
        CHECK(mdn_session_set_external_check(config->session(), nullptr, nullptr) == MDN_OK);
        threw = false;
        AuxBuilder bad = [](uint32_t, const RowMajorMatrix&, const std::vector<QuadFelt>&, std::vector<Felt>&, std::vector<QuadFelt>&) { throw std::runtime_error("no"); };
        try { check_constraints(*config, ps, seed, bad); }
        catch (const ProverError& e) { threw = e.kind == ProverError::AuxBuilder; }
        CHECK(threw);
        check_constraints(*config, ps, seed, aux);     // the session is still usable
    }
    printf("CHECK_API_OK\n");
    return 0;
}
