// The C++ host layer (miden-vm_b200/host/miden_prover.hpp) with device-resident column-major traces and a real CUDA aux
// builder: a kernel launched on the session's stream writes the aux trace straight into the library's aux slot.
// The same statement proved from host row-major traces with the equivalent host builder must give the same proof; the
// oracle verifier accepts it and rejects a tampered copy; the constraint check holds, and locates a corrupted aux row.
#include "../../miden-vm_b200/host/miden_prover.hpp"
#include "../../miden-vm_b200/csrc/gl.cuh"
#include <cuda_runtime.h>
#include <cstdio>

extern "C" {
int orc_verify(const void* params, const void* st, const void* proof, const void* challenger);
const char* orc_last_error();
}

using namespace miden;
static const Felt P = 0xFFFFFFFF00000001ULL;

#define CHECK(cond) do { if (!(cond)) { fprintf(stderr, "CHECK failed at line %d: %s (%s)\n", __LINE__, #cond, orc_last_error()); return 1; } } while (0)
#define CUDA_CHECK(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #expr, cudaGetErrorString(e_)); return 2; } } while (0)

static Felt splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

// main[0] * ... * main[8] == 0 (column 0 is zero) and aux[0] == main[1] * challenge 0 (an EF column)
static Air scaled_column_air(uint32_t width) {
    AirBuilder b;
    auto acc = b.constant(1);
    for (uint32_t j = 0; j < 9; j++) acc = b.mul(acc, b.main(0, j));
    b.assert_zero(acc);
    b.assert_zero_ext(b.sub(b.aux(0, 0), b.mul(b.main(0, 1), b.challenge(0))));
    Air a; a.width = width; a.aux_width = 1; a.num_aux_values = 0; a.num_randomness = 2; a.log_quotient_degree = 3;
    a.program = b.finish();
    return a;
}

// aux planes (c0 then c1) of column 0 from column 1 of the column-major main trace
__global__ void k_scaled_column(const Felt* main, uint32_t log_n, Felt c0, Felt c1, Felt* aux, Felt poison_row) {
    size_t n = size_t(1) << log_n, r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    Felt x = main[n + r];
    aux[r] = gl::mul(x, c0);
    aux[n + r] = r == poison_row ? gl::add(gl::mul(x, c1), 1) : gl::mul(x, c1);
}

static Challenger initial_challenger(const PcsParams& p) {
    static const Felt RELATION_DIGEST[4] = {837197885082815666ULL, 17812429367884914ULL, 12945170128166309606ULL, 6547471563106428306ULL};
    Challenger c;
    for (int i = 0; i < 4; i++) c.raw.sponge_state[8 + i] = RELATION_DIGEST[i];
    c.observe_slice({p.num_queries, p.query_pow_bits, p.deep_pow_bits, p.folding_pow_bits, p.log_blowup, p.log_final_degree, Felt(1) << p.log_folding_arity, 0});
    return c;
}

static int verify(const Statement& s, const PcsParams& p, const StarkProofData& pf, const Challenger& ch) {
    detail::Lowered low(s);
    mdn_pcs_params params = p.raw();
    std::vector<Felt> comm;
    for (auto& c : pf.transcript.commitments) comm.insert(comm.end(), c.begin(), c.end());
    mdn_proof proof{pf.log_trace_heights.data(), pf.log_trace_heights.size(), pf.transcript.fields.data(), pf.transcript.fields.size(),
                    comm.data(), pf.transcript.commitments.size()};
    return orc_verify(&params, &low.st, &proof, &ch.raw);
}

int main() {
    PcsParams pcs;
    pcs.log_final_degree = 2; pcs.folding_pow_bits = 2; pcs.deep_pow_bits = 3; pcs.num_queries = 5; pcs.query_pow_bits = 4;
    const uint32_t heights[2] = {9, 6}, widths[2] = {9, 12};
    std::vector<Air> airs;
    std::vector<RowMajorMatrix> host;
    std::vector<Felt*> dev(2, nullptr);
    for (int i = 0; i < 2; i++) {
        size_t n = size_t(1) << heights[i], w = widths[i];
        std::vector<Felt> rm(n * w), cm(n * w);
        for (size_t r = 0; r < n; r++)
            for (size_t c = 0; c < w; c++) {
                Felt x = c ? splitmix64((r * w + c) ^ (77ULL << 40 | (uint64_t)i)) % P : 0;
                rm[r * w + c] = x; cm[c * n + r] = x;
            }
        CUDA_CHECK(cudaMalloc((void**)&dev[i], n * w * sizeof(Felt)));
        CUDA_CHECK(cudaMemcpy(dev[i], cm.data(), n * w * sizeof(Felt), cudaMemcpyHostToDevice));
        host.emplace_back(std::move(rm), (uint32_t)w);
        airs.push_back(scaled_column_air((uint32_t)w));
    }
    Statement st = Statement::with_default_observe(airs, {});
    StarkConfig config(pcs, initial_challenger(pcs));

    // host: row-major traces, the aux column computed on the CPU
    AuxBuilder host_aux = [&](uint32_t inst, const RowMajorMatrix& m, const std::vector<QuadFelt>& ch, std::vector<Felt>& aux, std::vector<QuadFelt>&) {
        for (size_t r = 0; r < m.height(); r++) {
            Felt x = m.values[r * m.width + 1];
            aux[2 * r] = gl::mul(x, ch[0][0]); aux[2 * r + 1] = gl::mul(x, ch[0][1]);
        }
    };
    ProverStatement ps(st, host);
    StarkOutput ref = ProverInstance(config, ps, nullptr, host_aux).prove(config.challenger());
    CHECK(verify(st, pcs, ref.proof, config.challenger()) == 0);

    // device: column-major traces in HBM, the aux column written by a kernel on the session's stream
    Felt poison = ~0ULL;
    DeviceAuxBuilder dev_aux = [&](uint32_t inst, const ColumnMajorDeviceMatrix& m, const std::vector<QuadFelt>& ch, Felt* aux, std::vector<QuadFelt>&, void* stream) {
        if (m.values != dev[inst]) throw std::runtime_error("main is not the caller's buffer");
        k_scaled_column<<<(unsigned)((m.height() + 127) / 128), 128, 0, (cudaStream_t)stream>>>(m.values, m.log_height, ch[0][0], ch[0][1], aux, poison);
        if (cudaGetLastError() != cudaSuccess) throw std::runtime_error("launch failed");
    };
    std::vector<ColumnMajorDeviceMatrix> views;
    for (int i = 0; i < 2; i++) views.push_back(ColumnMajorDeviceMatrix{dev[i], heights[i], widths[i]});
    DeviceProverStatement dps(st, views);
    StarkOutput got = ProverInstance(config, dps, nullptr, dev_aux).prove(config.challenger());
    CHECK(got.proof.log_trace_heights == ref.proof.log_trace_heights);
    CHECK(got.proof.transcript.fields == ref.proof.transcript.fields);
    CHECK(got.proof.transcript.commitments == ref.proof.transcript.commitments);
    CHECK(verify(st, pcs, got.proof, config.challenger()) == 0);
    StarkProofData bad = got.proof;
    bad.transcript.fields[bad.transcript.fields.size() / 2] ^= 1;
    CHECK(verify(st, pcs, bad, config.challenger()) != 0);

    // the constraint check on the same device statement: holds, then finds a corrupted aux row
    check_constraints(config, dps, config.challenger(), dev_aux);
    poison = 17;
    bool caught = false;
    try { check_constraints(config, dps, config.challenger(), dev_aux); }
    catch (const ConstraintViolation& v) { caught = v.report.kind == 1 && v.report.row == 17; }
    CHECK(caught);
    // a proof without a device builder has zero aux traces: the aux constraint fails and the verifier rejects it
    StarkOutput zero = ProverInstance(config, dps, nullptr).prove(config.challenger());
    CHECK(verify(st, pcs, zero.proof, config.challenger()) != 0);
    for (Felt* p : dev) cudaFree(p);
    printf("DEVICE_API_OK\n");
    return 0;
}
