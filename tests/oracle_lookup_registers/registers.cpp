// TEST INFRASTRUCTURE ONLY.  A second lowering of version-2 lookup programs (include/miden_b200.h `mdn_lookup`: LogUp
// columns, then register columns with reg[0] = 0 and reg[r+1] = U(row r, reg[r])), and the aux build on it,
// single-threaded on the CPU and in row order: every row is evaluated once by the oracle's air_eval_folded
// (oracle/air.hpp) with the registers' current values in the aux window, the LogUp fractions are summed as
// build_logup_aux_trace does (air/src/lookup/aux_builder.rs:49-97), and the registers take their update values for the
// next row.  It shares no code with the device path, which splits the program and scans affine row maps; the oracle
// prover proves version-2 AIRs through this library as its aux callback (tests/test_lookup_registers.py).
#include "../../oracle/air.hpp"
#include <string>
#include <vector>

using namespace orc;

namespace {
thread_local std::string g_err;

// words [MAGIC, 2, n_nodes, n_interactions, n_consts, n_registers, nodes (3 each), interactions (4 each),
// update node per register, consts (lo, hi)]
struct Parsed {
    AirProgram nodes;
    std::vector<LookupInteraction> items;
    std::vector<uint32_t> updates;
};
Parsed parse(uint32_t num_columns, const uint32_t* w, size_t n_words, uint32_t width, uint32_t prep_width,
             uint32_t n_periodic, uint32_t n_publics) {
    if (n_words < 6 || w[0] != LookupProgram::MAGIC || w[1] != 2) throw std::runtime_error("lookup program: bad header");
    const size_t nn = w[2], ni = w[3], nk = w[4], nr = w[5];
    if (n_words != 6 + 3 * nn + 4 * ni + nr + 2 * nk) throw std::runtime_error("lookup program: bad length");
    if (nr < 1 || nr > 4) throw std::runtime_error("lookup program: 1..=4 registers");
    Parsed p;
    const uint32_t* q = w + 6;
    std::vector<uint8_t> ext(nn);
    for (size_t i = 0; i < nn; i++, q += 3) {
        const AirNode nd{q[0], q[1], q[2]};
        switch (nd.op) {
            case OP_MAIN: if (nd.a > 1 || nd.b >= width) throw std::runtime_error("lookup program: main column out of range"); break;
            case OP_AUX:
                if (nd.a != 0 || nd.b < num_columns || nd.b >= num_columns + nr) throw std::runtime_error("lookup program: AUX must read a register at offset 0");
                ext[i] = 1; break;
            case OP_PREPROCESSED: if (nd.a > 1 || nd.b >= prep_width) throw std::runtime_error("lookup program: preprocessed column out of range"); break;
            case OP_PERIODIC: if (nd.a >= n_periodic) throw std::runtime_error("lookup program: periodic column out of range"); break;
            case OP_PUBLIC: if (nd.a >= n_publics) throw std::runtime_error("lookup program: public value out of range"); break;
            case OP_CHALLENGE: if (nd.a > 1) throw std::runtime_error("lookup program: challenge out of range"); ext[i] = 1; break;
            case OP_CONST: if (nd.a >= nk) throw std::runtime_error("lookup program: constant out of range"); break;
            case OP_EXT_CONST: if (nd.a + 1 >= nk) throw std::runtime_error("lookup program: constant out of range"); ext[i] = 1; break;
            case OP_ADD: case OP_SUB: case OP_MUL:
                if (nd.a >= i || nd.b >= i) throw std::runtime_error("lookup program: forward reference");
                ext[i] = ext[nd.a] | ext[nd.b]; break;
            case OP_NEG:
                if (nd.a >= i) throw std::runtime_error("lookup program: forward reference");
                ext[i] = ext[nd.a]; break;
            default: throw std::runtime_error("lookup program: op not available to a LookupBuilder");
        }
        p.nodes.nodes.push_back(nd);
    }
    for (size_t i = 0; i < ni; i++, q += 4) {
        const LookupInteraction it{q[0], q[1], q[2], q[3]};
        if (it.column >= num_columns) throw std::runtime_error("lookup program: column out of range");
        if ((it.flag != LookupProgram::NO_FLAG && (it.flag >= nn || ext[it.flag])) || it.multiplicity >= nn || ext[it.multiplicity] || it.denominator >= nn)
            throw std::runtime_error("lookup program: bad interaction");
        p.items.push_back(it);
    }
    for (size_t i = 0; i < nr; i++, q++) {
        if (*q >= nn) throw std::runtime_error("lookup program: bad update node");
        p.updates.push_back(*q);
    }
    for (size_t i = 0; i < nk; i++, q += 2) p.nodes.consts.push_back((u64)q[0] | ((u64)q[1] << 32));
    return p;
}
}  // namespace

extern "C" {

const char* orc_lookup_registers_error() { return g_err.c_str(); }

// The aux trace of one AIR with a version-2 lookup program: main (2^log_height x width) and prep (2^log_height x
// prep_width, or NULL when prep_width is 0) row-major, periodic (2^log_max_period x n_periodic) row-major,
// randomness = alpha, beta as EF pairs.  aux_out row r (2 * (num_columns + n_registers) u64, row-major) = [running sum
// of every column's fraction over the rows before, f_1, ..., f_{C-1}, reg_0[r], ..., reg_{k-1}[r]]; final_out = the
// running sum after the last row.  0, or -1 with orc_lookup_registers_error().
int orc_logup_aux_registers(uint32_t num_columns, const uint32_t* program, size_t program_words,
                            const uint64_t* main, uint32_t log_height, uint32_t width, const uint64_t* prep, uint32_t prep_width,
                            const uint64_t* periodic, uint32_t n_periodic, uint32_t log_max_period,
                            const uint64_t* publics, uint32_t n_publics, const uint64_t* randomness,
                            uint64_t* aux_out, uint64_t* final_out) {
    try {
        const Parsed p = parse(num_columns, program, program_words, width, prep_width, n_periodic, n_publics);
        const size_t N = size_t(1) << log_height, C = num_columns, K = p.updates.size(), A = C + K, maxp = size_t(1) << log_max_period;
        auto row = [&](const uint64_t* m, uint32_t w, size_t r) {
            std::vector<Fp> v(w);
            for (uint32_t c = 0; c < w; c++) v[c] = Fp(m[r * w + c]);
            return v;
        };
        std::vector<Fp> pub(n_publics);
        for (uint32_t i = 0; i < n_publics; i++) pub[i] = Fp(publics[i]);
        const Ef ch[2] = {Ef(Fp(randomness[0]), Fp(randomness[1])), Ef(Fp(randomness[2]), Fp(randomness[3]))};
        std::vector<Ef> scratch, per(n_periodic), frac(C), reg(K);
        std::vector<Fp> aux_row(2 * A);   // the aux window: only the register columns are read
        Ef acc;
        for (size_t r = 0; r < N; r++) {
            const size_t rn = (r + 1) % N;
            const std::vector<Fp> ml = row(main, width, r), mn = row(main, width, rn);
            const std::vector<Fp> pl = prep ? row(prep, prep_width, r) : std::vector<Fp>(), pn = prep ? row(prep, prep_width, rn) : std::vector<Fp>();
            for (uint32_t c = 0; c < n_periodic; c++) per[c] = Ef(Fp(periodic[(r % maxp) * n_periodic + c]));
            for (size_t i = 0; i < K; i++) { aux_row[2 * (C + i)] = reg[i].a; aux_row[2 * (C + i) + 1] = reg[i].b; }
            AirPoint pt{};
            pt.main_local = ml.data(); pt.main_next = mn.data();
            pt.aux_local = aux_row.data(); pt.aux_next = aux_row.data();
            pt.prep_local = pl.data(); pt.prep_next = pn.data();
            pt.publics = pub.data(); pt.challenges = ch; pt.periodic = per.data();
            air_eval_folded(p.nodes, pt, Ef(), scratch);
            std::fill(frac.begin(), frac.end(), Ef());
            for (const LookupInteraction& it : p.items) {
                if (it.flag != LookupProgram::NO_FLAG && scratch[it.flag].a.is_zero()) continue;
                const Ef& d = scratch[it.denominator];
                if (d.is_zero()) throw std::runtime_error("LogUp denominator must be non-zero");
                frac[it.column] += Ef(scratch[it.multiplicity].a) * ef_inv(d);
            }
            uint64_t* o = aux_out + 2 * A * r;
            o[0] = acc.a.v; o[1] = acc.b.v;
            for (size_t c = 1; c < C; c++) { o[2 * c] = frac[c].a.v; o[2 * c + 1] = frac[c].b.v; }
            for (size_t i = 0; i < K; i++) { o[2 * (C + i)] = reg[i].a.v; o[2 * (C + i) + 1] = reg[i].b.v; }
            for (size_t c = 0; c < C; c++) acc += frac[c];
            for (size_t i = 0; i < K; i++) reg[i] = scratch[p.updates[i]];   // every update read the row-r registers
        }
        final_out[0] = acc.a.v; final_out[1] = acc.b.v;
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

}  // extern "C"
