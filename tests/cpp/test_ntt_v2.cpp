// Runs the NTT block functions (miden-vm_b200/csrc/ntt2.cuh, __host__ __device__) ON THE CPU
// with the tables the product builds (ntt_tables.hpp) and compares the inverse transform and every coset of the
// low-degree extension with a textbook transform (itself checked against the O(N^2) definition at small sizes).
// A block function is a sequence of index-parallel loops separated by barriers; the host build runs each loop
// over all indices, the device build over threadIdx.x -- same arithmetic, same shared-memory tile, same tables.
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>
#include "../../miden-vm_b200/csrc/ntt2.cuh"
#include "../../miden-vm_b200/csrc/ntt_tables.hpp"

typedef uint64_t u64;
typedef uint32_t u32;
static u64 rng_state = 0x243F6A8885A308D3ull;
static u64 rnd() { u64 z = (rng_state += 0x9E3779B97F4A7C15ull); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31); }
static u64 rnd_felt() { return rnd() % gl::P; }
static int fails = 0;
#define CHECK(cond, ...) do { if (!(cond)) { if (fails++ < 20) { printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } } while (0)

static u32 brev(u32 x, u32 bits) { u32 r = 0; for (u32 i = 0; i < bits; i++) r |= ((x >> i) & 1u) << (bits - 1 - i); return r; }
// textbook iterative radix-2 DIT, natural in -> natural out: out[k] = sum_j a[j] w^(jk)
static std::vector<u64> ref_ntt(const std::vector<u64>& a, u64 w, u32 n) {
    size_t N = (size_t)1 << n;
    std::vector<u64> x(N);
    for (size_t i = 0; i < N; i++) x[brev((u32)i, n)] = a[i];
    for (u32 s = 0; s < n; s++) {
        size_t h = (size_t)1 << s;
        u64 ws = gl::pow(w, N >> (s + 1));
        for (size_t blk = 0; blk < N; blk += 2 * h) {
            u64 t = 1;
            for (size_t j = 0; j < h; j++) {
                u64 u = x[blk + j], v = gl::mul(x[blk + j + h], t);
                x[blk + j] = gl::add(u, v); x[blk + j + h] = gl::sub(u, v);
                t = gl::mul(t, ws);
            }
        }
    }
    return x;
}
static std::vector<u64> naive_dft(const std::vector<u64>& a, u64 w) {
    size_t N = a.size();
    std::vector<u64> o(N);
    for (size_t k = 0; k < N; k++) {
        u64 acc = 0, wk = gl::pow(w, k), x = 1;
        for (size_t j = 0; j < N; j++) { acc = gl::add(acc, gl::mul(a[j], x)); x = gl::mul(x, wk); }
        o[k] = acc;
    }
    return o;
}

// `specialised` = the instantiation with the split as compile-time constants that kernels.cu launches for this size
// (NTT_SPECIALISED there); otherwise the run-time schedules.  Both must give the same words.
template <int N1C, int N2C>
static void run_intt_t(std::vector<u64>& col, const mk::NttTables& T, std::vector<u64>& sm) {
    u32 N1 = 1u << T.n1, N2 = 1u << T.n2;
    size_t N = (size_t)1 << T.n;
    if (T.n1 > 0) {
        u32 log_c = T.n1 >= 12 ? 0 : 12 - T.n1; if (log_c > T.n2) log_c = T.n2;      // launch_intt (kernels.cu)
        sm.assign(ntt2::smem_words_strided(T.n1, log_c), 0xDEADBEEFDEADBEEFull);
        for (u32 bx = 0; bx < (N2 >> log_c); bx++) ntt2::intt_strided_block<N1C, N2C>(bx, 0, sm.data(), col.data(), N, T, log_c);
    }
    sm.assign(ntt2::smem_words_contig_inv(T.n2), 0xDEADBEEFDEADBEEFull);
    for (u32 bx = 0; bx < N1; bx++) ntt2::intt_contig_block<N2C>(bx, 0, sm.data(), col.data(), N, T);
}
template <int N1C, int N2C>
static void run_fwd_t(const std::vector<mk::FwdItem>& items, const mk::NttTables& T, const mk::PremulTables& Pm, std::vector<u64>& sm) {
    u32 N1 = 1u << T.n1, N2 = 1u << T.n2;
    sm.assign(ntt2::smem_words_contig_fwd(T.n2), 0xDEADBEEFDEADBEEFull);
    for (u32 by = 0; by < items.size(); by++)
        for (u32 bx = 0; bx < N1; bx++) ntt2::fwd_contig_block<N1C, N2C>(bx, by, sm.data(), items.data(), T, Pm);
    if (T.n1 > 0) {
        u32 log_c = T.n1 >= 12 ? 0 : 12 - T.n1; if (log_c > T.n2) log_c = T.n2;      // launch_fwd_ntt (kernels.cu)
        sm.assign(ntt2::smem_words_strided(T.n1, log_c), 0xDEADBEEFDEADBEEFull);
        for (u32 by = 0; by < items.size(); by++)
            for (u32 bx = 0; bx < (N2 >> log_c); bx++) ntt2::fwd_strided_block<N1C, N2C>(bx, by, sm.data(), items.data(), T, log_c);
    }
}
#define NTT_SPECIALISED(X) X(8, 8) X(8, 9) X(9, 9) X(9, 10) X(10, 10) X(10, 11) X(11, 11)
static bool g_generic_only = false;
static void run_intt(std::vector<u64>& col, const mk::NttTables& T, std::vector<u64>& sm) {
#define X(a, b) if (!g_generic_only && T.n1 == a && T.n2 == b) { run_intt_t<a, b>(col, T, sm); return; }
    NTT_SPECIALISED(X)
#undef X
    run_intt_t<-1, -1>(col, T, sm);
}
static void run_fwd(const std::vector<mk::FwdItem>& items, const mk::NttTables& T, const mk::PremulTables& Pm, std::vector<u64>& sm) {
#define X(a, b) if (!g_generic_only && T.n1 == a && T.n2 == b) { run_fwd_t<a, b>(items, T, Pm, sm); return; }
    NTT_SPECIALISED(X)
#undef X
    run_fwd_t<-1, -1>(items, T, Pm, sm);
}

static void test_size(u32 n, u32 log_blowup) {
    size_t N = (size_t)1 << n;
    u32 B = 1u << log_blowup;
    ntt_tables::NttHost nh = ntt_tables::build_ntt(n);
    mk::NttTables T = nh.view(nh.data.data());
    // bases of the trace LDE (session.cu premul_trace) plus two arbitrary ones (the quotient uses other bases)
    std::vector<u64> bases(B + 2);
    u64 s = gl::lde_shift(n + log_blowup), wl = gl::two_adic_generator(n + log_blowup), xx = s;
    for (u32 t = 0; t < B; t++) { bases[t] = xx; xx = gl::mul(xx, wl); }
    bases[B] = rnd_felt() | 1; bases[B + 1] = 1;
    ntt_tables::PremulHost ph = ntt_tables::build_premul(bases, n);
    mk::PremulTables Pm = ph.view(ph.data.data());

    std::vector<u64> col(N), work;
    for (auto& v : col) v = rnd_felt();
    col[0] = gl::P - 1; if (N > 1) col[1] = 0;
    work = col;
    std::vector<u64> sm;
    run_intt(work, T, sm);
    u64 w = gl::two_adic_generator(n), wi = gl::inv(w);
    std::vector<u64> nc = ref_ntt(col, wi, n);                  // N * c[j]
    for (size_t p = 0; p < N; p++) CHECK(work[p] == nc[brev((u32)p, n)], "n=%u inverse slot %zu", n, p);
    if (n <= 9) { std::vector<u64> nv = naive_dft(col, wi); for (size_t j = 0; j < N; j++) CHECK(nv[j] == nc[j], "reference self-check n=%u", n); }

    std::vector<u64> out((B + 2) * N, 0xAAAAAAAAAAAAAAAAull);
    std::vector<mk::FwdItem> items;
    for (u32 t = 0; t < B + 2; t++) items.push_back(mk::FwdItem{work.data(), out.data() + (size_t)t * N, t, 0});
    run_fwd(items, T, Pm, sm);
    u64 n_inv = gl::inv((u64)N % gl::P);
    for (u32 t = 0; t < B + 2; t++) {
        std::vector<u64> a(N);
        u64 g = bases[t], gp = 1;
        for (size_t j = 0; j < N; j++) { a[j] = gl::mul(gl::mul(nc[j], n_inv), gp); gp = gl::mul(gp, g); }
        std::vector<u64> want = ref_ntt(a, w, n);
        for (size_t r = 0; r < N; r++) CHECK(out[(size_t)t * N + r] == want[r], "n=%u coset %u row %zu", n, t, r);
    }
    for (size_t i = 0; i < work.size(); i++) CHECK(work[i] < gl::P, "non-canonical coefficient");
    for (size_t i = 0; i < out.size(); i++) CHECK(out[i] < gl::P, "non-canonical evaluation");
}

// The tables ntt_tables.hpp builds for session.cu: every NttTables member and the premultiplication table tab_b against
// their definitions, and where tab_b and tab_c sit in the premultiplication block (tab_c itself is checked by test_size).
static void test_table_layout(u32 n) {
    u32 n1, n2;
    if (n <= 11) { n1 = 0; n2 = n; } else { n1 = n / 2; n2 = n - n1; }
    size_t N1 = (size_t)1 << n1, N2 = (size_t)1 << n2;
    ntt_tables::NttHost nh = ntt_tables::build_ntt(n);
    mk::NttTables T = nh.view(nh.data.data());
    CHECK(T.n == n && T.n1 == n1 && T.n2 == n2 && T.lo_bits == (n + 1) / 2, "split of 2^%u", n);
    u64 w = gl::two_adic_generator(n), wi = gl::inv(w), w1 = gl::two_adic_generator(n1), w2 = gl::two_adic_generator(n2);
    for (size_t i = 0; i < (n1 ? N1 / 2 : 1); i++) { CHECK(T.tw_n1[i] == gl::pow(w1, i), "tw_n1"); CHECK(T.twi_n1[i] == gl::pow(gl::inv(w1), i), "twi_n1"); }
    for (size_t i = 0; i < (n2 ? N2 / 2 : 1); i++) CHECK(T.twi_n2[i] == gl::pow(gl::inv(w2), i), "twi_n2");
    for (size_t i = 0; i < ((size_t)1 << T.lo_bits); i += 37) { CHECK(T.w_lo[i] == gl::pow(w, i), "w_lo"); CHECK(T.wi_lo[i] == gl::pow(wi, i), "wi_lo"); }
    for (size_t i = 0; i < ((size_t)1 << (n - T.lo_bits)); i += 13) { CHECK(T.w_hi[i] == gl::pow(w, i << T.lo_bits), "w_hi"); CHECK(T.wi_hi[i] == gl::pow(wi, i << T.lo_bits), "wi_hi"); }
    std::vector<u64> bases = {gl::lde_shift(n + 3), rnd_felt() | 1, 1};
    ntt_tables::PremulHost ph = ntt_tables::build_premul(bases, n);
    mk::PremulTables Pm = ph.view(ph.data.data());
    CHECK(Pm.tab_b == ph.data.data() && Pm.tab_c == ph.data.data() + bases.size() * N1, "premul offsets");
    u64 n_inv = gl::inv((u64)1 << n);
    for (size_t b = 0; b < bases.size(); b++) {
        for (size_t j1 = 0; j1 < N1; j1 += 7) CHECK(Pm.tab_b[b * N1 + j1] == gl::mul(n_inv, gl::pow(bases[b], j1)), "tab_b");
    }
}

int main(int argc, char** argv) {
    u32 max_n = argc > 1 ? (u32)atoi(argv[1]) : 16;
    for (u32 n = 1; n <= 22; n++) test_table_layout(n);
    for (u32 n = 1; n <= max_n; n++) test_size(n, n % 3 == 0 ? 2 : 3);
    // sizes with a specialised instantiation once more through the run-time schedules
    g_generic_only = true;
    for (u32 n = 16; n <= max_n; n++) test_size(n, 3);
    g_generic_only = false;
    if (fails) { printf("NTT_V2_FAILED %d\n", fails); return 1; }
    printf("NTT_V2_OK up to 2^%u\n", max_n);
    return 0;
}
