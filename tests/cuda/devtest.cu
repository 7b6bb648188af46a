// Test-only library: the product's __host__ __device__ field arithmetic, Poseidon2 and NTT kernels run on the device and,
// from the same source, on the host (the #else branches), so tests/test_device_units.py can compare the two bit for bit
// and both with plain integer references.  The product headers are included unchanged and kernels.cu is compiled into
// this library, so the NTT and batch-permutation entry points call the product's own launchers.
//
// Every entry point returns 0 on success.  A device entry point returns DT_NO_DEVICE when no CUDA device is present,
// so a CPU-only machine can load the library and run the host half.
#include "../../miden-vm_b200/csrc/kernels.cuh"
#include "../../miden-vm_b200/csrc/poseidon2.cuh"
#include "../../miden-vm_b200/csrc/poseidon2_fast2.cuh"
#include "../../miden-vm_b200/csrc/ntt2.cuh"
#include "../../miden-vm_b200/csrc/ntt_tables.hpp"
#include <cstring>
#include <vector>

using gl::u64;
using gl::u32;

enum { DT_OK = 0, DT_NO_DEVICE = -1, DT_CUDA_ERROR = -2, DT_BAD_ARG = -3 };

// ---- scalar operations ---------------------------------------------------------------------------------------------
// One row: DT_IN input words, DT_OUT output words.  Wide values W = (lo, hi) and Acc160 = (lo, mid, hi) occupy
// consecutive words; E2 values (a, b) too.  Unused output words are left zero.
static constexpr int DT_IN = 6, DT_OUT = 4;
#define DT_OPS(X)                                                                                                       \
    X(glf_addc64) X(glf_subb64) X(glf_mul_eps) X(glf_mul) X(glf_sqr) X(glf_red128) X(glf_add_const) X(glf_canon)     \
    X(glf_canon_cc) X(glf_csub) X(glf_cadd) X(glf_cmul) X(glf_half) X(glf_div2k2) X(glf_div2k3) X(glf_wsum)           \
    X(glf_wadd_u64) X(glf_wadd_w) X(glf_wsub) X(glf_wshl) X(glf_wtriple) X(glf_wred) X(glf_wshl96) X(glf_wshr96)      \
    X(glf_whalf) X(glf_wdiv2k2) X(glf_wdiv2k3) X(gl_fast_addc64) X(gl_fast_subb64) X(gl_add) X(gl_sub) X(gl_neg)      \
    X(gl_mul) X(gl_half) X(gl_pow) X(gl_inv) X(gl_e2_mul) X(gl_e2_sqr) X(gl_e2_inv) X(gl_e2_pow) X(acc_mul)          \
    X(acc_reduce) X(acc_sum)
#define X(name) OP_##name,
enum DtOp { DT_OPS(X) OP_COUNT };
#undef X
#define X(name) #name,
static const char* const OP_NAMES[] = {DT_OPS(X)};
#undef X

static GL_HD glf::W wide_of(const u64* a) { glf::W w; w.lo = a[0]; w.hi = (u32)a[1]; return w; }
static GL_HD void put_w(u64* o, glf::W w) { o[0] = w.lo; o[1] = w.hi; }
static GL_HD void put_acc(u64* o, const glf::Acc160& A) { o[0] = A.lo; o[1] = A.mid; o[2] = A.hi; }

static GL_HD void apply(int op, const u64* a, u64* o) {
    u64 r; u32 c;
    glf::W w;
    switch (op) {
    case OP_glf_addc64: glf::addc64(a[0], a[1], r, c); o[0] = r; o[1] = c; break;
    case OP_glf_subb64: glf::subb64(a[0], a[1], r, c); o[0] = r; o[1] = c; break;
    case OP_glf_mul_eps: o[0] = glf::mul_eps((u32)a[0]); break;
    case OP_glf_mul: o[0] = glf::mul(a[0], a[1]); break;
    case OP_glf_sqr: o[0] = glf::sqr(a[0]); break;
    case OP_glf_red128: o[0] = glf::red128(a[0], a[1]); break;
    case OP_glf_add_const: o[0] = glf::add_const(a[0], a[1]); break;
    case OP_glf_canon: o[0] = glf::canon(a[0]); break;
    case OP_glf_canon_cc: o[0] = glf::canon_cc(a[0]); break;
    case OP_glf_csub: o[0] = glf::csub(a[0], a[1]); break;
    case OP_glf_cadd: o[0] = glf::cadd(a[0], a[1]); break;
    case OP_glf_cmul: o[0] = glf::cmul(a[0], a[1]); break;
    case OP_glf_half: o[0] = glf::half(a[0]); break;
    case OP_glf_div2k2: o[0] = glf::div2k<2>(a[0]); break;
    case OP_glf_div2k3: o[0] = glf::div2k<3>(a[0]); break;
    case OP_glf_wsum: put_w(o, glf::wsum(a[0], a[1])); break;
    case OP_glf_wadd_u64: w = wide_of(a); glf::wadd(w, a[2]); put_w(o, w); break;
    case OP_glf_wadd_w: w = wide_of(a); glf::wadd(w, wide_of(a + 2)); put_w(o, w); break;
    case OP_glf_wsub: w = wide_of(a); glf::wsub(w, wide_of(a + 2)); put_w(o, w); break;
    case OP_glf_wshl: put_w(o, glf::wshl(a[0], (int)a[1])); break;
    case OP_glf_wtriple: put_w(o, glf::wtriple(a[0])); break;
    case OP_glf_wred: o[0] = glf::wred(wide_of(a)); break;
    case OP_glf_wshl96: put_w(o, glf::wshl96(wide_of(a), (int)a[2])); break;
    case OP_glf_wshr96: put_w(o, glf::wshr96(wide_of(a), (int)a[2])); break;
    case OP_glf_whalf: put_w(o, glf::whalf(wide_of(a))); break;
    case OP_glf_wdiv2k2: put_w(o, glf::wdiv2k<2>(wide_of(a))); break;
    case OP_glf_wdiv2k3: put_w(o, glf::wdiv2k<3>(wide_of(a))); break;
    case OP_gl_fast_addc64: { unsigned cc; gl::fast_addc64(a[0], a[1], r, cc); o[0] = r; o[1] = cc; break; }
    case OP_gl_fast_subb64: { unsigned mm; gl::fast_subb64(a[0], a[1], r, mm); o[0] = r; o[1] = mm; break; }
    case OP_gl_add: o[0] = gl::add(a[0], a[1]); break;
    case OP_gl_sub: o[0] = gl::sub(a[0], a[1]); break;
    case OP_gl_neg: o[0] = gl::neg(a[0]); break;
    case OP_gl_mul: o[0] = gl::mul(a[0], a[1]); break;
    case OP_gl_half: o[0] = gl::half(a[0]); break;
    case OP_gl_pow: o[0] = gl::pow(a[0], a[1]); break;
    case OP_gl_inv: o[0] = gl::inv(a[0]); break;
    case OP_gl_e2_mul: { gl::E2 e = gl::e2_mul(gl::e2(a[0], a[1]), gl::e2(a[2], a[3])); o[0] = e.a; o[1] = e.b; break; }
    case OP_gl_e2_sqr: { gl::E2 e = gl::e2_sqr(gl::e2(a[0], a[1])); o[0] = e.a; o[1] = e.b; break; }
    case OP_gl_e2_inv: { gl::E2 e = gl::e2_inv(gl::e2(a[0], a[1])); o[0] = e.a; o[1] = e.b; break; }
    case OP_gl_e2_pow: { gl::E2 e = gl::e2_pow(gl::e2(a[0], a[1]), a[2]); o[0] = e.a; o[1] = e.b; break; }
    case OP_acc_mul: { glf::Acc160 A{a[0], a[1], (u32)a[2]}; glf::acc_mul(A, a[3], a[4]); put_acc(o, A); break; }
    case OP_acc_reduce: { glf::Acc160 A{a[0], a[1], (u32)a[2]}; o[0] = glf::acc_reduce(A); break; }
    case OP_acc_sum: {   // a[2] products a[0] * a[1] accumulated from zero: the reduced value and the accumulator
        glf::Acc160 A{0, 0, 0};
        for (u64 i = 0; i < a[2]; i++) glf::acc_mul(A, a[0], a[1]);
        put_acc(o, A); o[3] = glf::acc_reduce(A); break;
    }
    default: break;
    }
}

__global__ void k_scalar(int op, const u64* __restrict__ in, u64* __restrict__ out, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u64 a[DT_IN], o[DT_OUT] = {0, 0, 0, 0};
    for (int k = 0; k < DT_IN; k++) a[k] = in[i * DT_IN + k];
    apply(op, a, o);
    for (int k = 0; k < DT_OUT; k++) out[i * DT_OUT + k] = o[k];
}

// ---- Poseidon2 -----------------------------------------------------------------------------------------------------
enum { P2_FAST_PERMUTE = 0, P2_FAST_EXTERNAL = 1, P2_CANONICAL_PERMUTE = 2 };
static GL_HD void apply_p2(int op, u64* s) {
    if (op == P2_FAST_PERMUTE) p2f::permute(s);
    else if (op == P2_FAST_EXTERNAL) p2f::external_layer(s);
    else p2::permute(s);
}
__global__ void k_p2(int op, u64* st, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u64 s[12];
    for (int k = 0; k < 12; k++) s[k] = st[i * 12 + k];
    apply_p2(op, s);
    for (int k = 0; k < 12; k++) st[i * 12 + k] = s[k];
}
// The sponge of k_leaf_hash: from the zero state, lanes 0..7 are overwritten with data[8 j .. 8 j + 8) before permutation
// j; lanes 8..11 carry the permutation's representatives from one permutation to the next.  Raw state out.
static GL_HD void p2_chain(const u64* data, u32 n_perms, u64* s) {
    for (int k = 0; k < 12; k++) s[k] = 0;
    for (u32 j = 0; j < n_perms; j++) {
        for (int k = 0; k < 8; k++) s[k] = data[8 * j + k];
        p2f::permute(s);
    }
}
__global__ void k_p2_chain(const u64* data, u32 n_perms, u64* out) {
    if (blockIdx.x == 0 && threadIdx.x == 0) p2_chain(data, n_perms, out);
}

// ---- plumbing ------------------------------------------------------------------------------------------------------
static bool have_device() {
    int n = 0;
    return cudaGetDeviceCount(&n) == cudaSuccess && n > 0;
}
static bool g_uploaded = false;
// Round constants into both translation units' __constant__ arrays: this file's (p2::permute, p2f::permute in the
// kernels above) and kernels.cu's (mk::upload_constants, for launch_poseidon2_batch).
static int prepare() {
    if (!have_device()) return DT_NO_DEVICE;
    if (!g_uploaded) {
        if (cudaMemcpyToSymbol(p2::D_RC_EXT_INITIAL, p2::P2_RC_EXT_INITIAL, sizeof(u64) * 48) != cudaSuccess ||
            cudaMemcpyToSymbol(p2::D_RC_INTERNAL, p2::P2_RC_INTERNAL, sizeof(u64) * 22) != cudaSuccess ||
            cudaMemcpyToSymbol(p2::D_RC_EXT_TERMINAL, p2::P2_RC_EXT_TERMINAL, sizeof(u64) * 48) != cudaSuccess)
            return DT_CUDA_ERROR;
        mk::upload_constants();
        if (cudaDeviceSynchronize() != cudaSuccess) return DT_CUDA_ERROR;
        g_uploaded = true;
    }
    return DT_OK;
}
struct Dev {   // device buffer freed on scope exit
    void* p = nullptr;
    bool alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 8) == cudaSuccess; }
    ~Dev() { if (p) cudaFree(p); }
    template <class T> T* as() const { return (T*)p; }
};
static int finish() {
    if (cudaGetLastError() != cudaSuccess) return DT_CUDA_ERROR;
    return cudaDeviceSynchronize() == cudaSuccess ? DT_OK : DT_CUDA_ERROR;
}
#define DT_TRY(x) do { if ((x) != cudaSuccess) return DT_CUDA_ERROR; } while (0)
#define DT_ALLOC(buf, bytes) do { if (!(buf).alloc(bytes)) return DT_CUDA_ERROR; } while (0)

// ---- NTT on the host: the block functions of the launchers' kernels, one block after another -----------------------
static u32 ntt_log_c(const mk::NttTables& T) { u32 lc = T.n1 >= 12 ? 0 : 12 - T.n1; return lc > T.n2 ? T.n2 : lc; }   // = kernels.cu
static void host_intt(u64* cols, size_t col_stride, u32 n_cols, const mk::NttTables& T) {
    u32 N1 = 1u << T.n1, N2 = 1u << T.n2, log_c = ntt_log_c(T);
    std::vector<u64> sm;
    for (u32 by = 0; by < n_cols; by++) {
        if (T.n1 > 0) {
            sm.assign(ntt2::smem_words_strided(T.n1, log_c), 0);
            for (u32 bx = 0; bx < (N2 >> log_c); bx++) ntt2::intt_strided_block<-1, -1>(bx, by, sm.data(), cols, col_stride, T, log_c);
        }
        sm.assign(ntt2::smem_words_contig_inv(T.n2), 0);
        for (u32 bx = 0; bx < N1; bx++) ntt2::intt_contig_block<-1>(bx, by, sm.data(), cols, col_stride, T);
    }
}
static void host_fwd(const std::vector<mk::FwdItem>& items, const mk::NttTables& T, const mk::PremulTables& Pm) {
    u32 N1 = 1u << T.n1, N2 = 1u << T.n2, log_c = ntt_log_c(T);
    std::vector<u64> sm(ntt2::smem_words_contig_fwd(T.n2));
    for (u32 by = 0; by < items.size(); by++)
        for (u32 bx = 0; bx < N1; bx++) ntt2::fwd_contig_block<-1, -1>(bx, by, sm.data(), items.data(), T, Pm);
    if (T.n1 > 0) {
        sm.assign(ntt2::smem_words_strided(T.n1, log_c), 0);
        for (u32 by = 0; by < items.size(); by++)
            for (u32 bx = 0; bx < (N2 >> log_c); bx++) ntt2::fwd_strided_block<-1, -1>(bx, by, sm.data(), items.data(), T, log_c);
    }
}

extern "C" {

int dt_op_count() { return OP_COUNT; }
const char* dt_op_name(int op) { return op >= 0 && op < OP_COUNT ? OP_NAMES[op] : nullptr; }
int dt_has_device() { return have_device() ? 1 : 0; }

// n rows of DT_IN words -> n rows of DT_OUT words through operation `op`
int dt_scalar(int op, const u64* in, u64* out, size_t n, int on_device) {
    if (op < 0 || op >= OP_COUNT) return DT_BAD_ARG;
    if (!on_device) {
        for (size_t i = 0; i < n; i++) {
            u64 o[DT_OUT] = {0, 0, 0, 0};
            apply(op, in + i * DT_IN, o);
            memcpy(out + i * DT_OUT, o, sizeof o);
        }
        return DT_OK;
    }
    int rc = prepare(); if (rc) return rc;
    if (!n) return DT_OK;
    Dev d_in, d_out;
    DT_ALLOC(d_in, n * DT_IN * 8); DT_ALLOC(d_out, n * DT_OUT * 8);
    DT_TRY(cudaMemcpy(d_in.p, in, n * DT_IN * 8, cudaMemcpyHostToDevice));
    k_scalar<<<(unsigned)((n + 127) / 128), 128>>>(op, d_in.as<u64>(), d_out.as<u64>(), n);
    if ((rc = finish())) return rc;
    DT_TRY(cudaMemcpy(out, d_out.p, n * DT_OUT * 8, cudaMemcpyDeviceToHost));
    return DT_OK;
}

// n states of 12 words in place: op 0 p2f::permute, 1 p2f::external_layer (raw representatives out), 2 p2::permute
int dt_p2(int op, u64* states, size_t n, int on_device) {
    if (op < 0 || op > 2) return DT_BAD_ARG;
    if (!on_device) { for (size_t i = 0; i < n; i++) apply_p2(op, states + 12 * i); return DT_OK; }
    int rc = prepare(); if (rc) return rc;
    if (!n) return DT_OK;
    Dev d; DT_ALLOC(d, n * 96);
    DT_TRY(cudaMemcpy(d.p, states, n * 96, cudaMemcpyHostToDevice));
    k_p2<<<(unsigned)((n + 127) / 128), 128>>>(op, d.as<u64>(), n);
    if ((rc = finish())) return rc;
    DT_TRY(cudaMemcpy(states, d.p, n * 96, cudaMemcpyDeviceToHost));
    return DT_OK;
}

// the leaf sponge: 8 * n_perms data words -> the raw 12-word state
int dt_p2_chain(const u64* data, u32 n_perms, u64* out, int on_device) {
    if (!on_device) { p2_chain(data, n_perms, out); return DT_OK; }
    int rc = prepare(); if (rc) return rc;
    Dev d_data, d_out;
    DT_ALLOC(d_data, (size_t)n_perms * 64); DT_ALLOC(d_out, 96);
    DT_TRY(cudaMemcpy(d_data.p, data, (size_t)n_perms * 64, cudaMemcpyHostToDevice));
    k_p2_chain<<<1, 32>>>(d_data.as<u64>(), n_perms, d_out.as<u64>());
    if ((rc = finish())) return rc;
    DT_TRY(cudaMemcpy(out, d_out.p, 96, cudaMemcpyDeviceToHost));
    return DT_OK;
}

// In-place inverse NTT (mk::launch_intt) of n_cols columns of 2^log_n words, col_stride words apart; the words between
// columns are copied through unchanged, so a test can see a write outside a column.
int dt_intt(u64* cols, size_t col_stride, u32 n_cols, u32 log_n, int on_device) {
    if (log_n < 1 || log_n > 22 || col_stride < ((size_t)1 << log_n) || !n_cols) return DT_BAD_ARG;
    ntt_tables::NttHost nh = ntt_tables::build_ntt(log_n);
    size_t words = col_stride * n_cols;
    if (!on_device) { host_intt(cols, col_stride, n_cols, nh.view(nh.data.data())); return DT_OK; }
    int rc = prepare(); if (rc) return rc;
    Dev d_tab, d_cols;
    DT_ALLOC(d_tab, nh.data.size() * 8 + 16); DT_ALLOC(d_cols, words * 8);
    DT_TRY(cudaMemcpy(d_tab.p, nh.data.data(), nh.data.size() * 8, cudaMemcpyHostToDevice));
    DT_TRY(cudaMemcpy(d_cols.p, cols, words * 8, cudaMemcpyHostToDevice));
    mk::launch_intt(d_cols.as<u64>(), col_stride, n_cols, nh.view(d_tab.as<u64>()), 0);
    if ((rc = finish())) return rc;
    DT_TRY(cudaMemcpy(cols, d_cols.p, words * 8, cudaMemcpyDeviceToHost));
    return DT_OK;
}

// Forward coset NTTs (mk::launch_fwd_ntt) of n_cols bit-reversed coefficient columns (2^log_n words each, contiguous)
// on n_bases coset bases, premultiplication tables from ntt_tables::build_premul.  out[(c * n_bases + b) << log_n + r]
// = column c evaluated at bases[b] * w^r.
int dt_fwd(const u64* src, u32 n_cols, u32 log_n, const u64* bases, u32 n_bases, u64* out, int on_device) {
    if (log_n < 1 || log_n > 22 || !n_cols || !n_bases) return DT_BAD_ARG;
    size_t N = (size_t)1 << log_n, n_out = (size_t)n_cols * n_bases * N;
    ntt_tables::NttHost nh = ntt_tables::build_ntt(log_n);
    ntt_tables::PremulHost ph = ntt_tables::build_premul(std::vector<u64>(bases, bases + n_bases), log_n);
    auto items_on = [&](const u64* s, u64* o) {
        std::vector<mk::FwdItem> items;
        for (u32 c = 0; c < n_cols; c++)
            for (u32 b = 0; b < n_bases; b++) items.push_back(mk::FwdItem{s + c * N, o + ((size_t)c * n_bases + b) * N, b, 0});
        return items;
    };
    if (!on_device) { host_fwd(items_on(src, out), nh.view(nh.data.data()), ph.view(ph.data.data())); return DT_OK; }
    int rc = prepare(); if (rc) return rc;
    Dev d_tab, d_pm, d_src, d_out, d_items;
    std::vector<mk::FwdItem> items;
    DT_ALLOC(d_tab, nh.data.size() * 8 + 16); DT_ALLOC(d_pm, ph.data.size() * 8 + 16);
    DT_ALLOC(d_src, n_cols * N * 8); DT_ALLOC(d_out, n_out * 8);
    items = items_on(d_src.as<u64>(), d_out.as<u64>());
    DT_ALLOC(d_items, items.size() * sizeof(mk::FwdItem));
    DT_TRY(cudaMemcpy(d_tab.p, nh.data.data(), nh.data.size() * 8, cudaMemcpyHostToDevice));
    DT_TRY(cudaMemcpy(d_pm.p, ph.data.data(), ph.data.size() * 8, cudaMemcpyHostToDevice));
    DT_TRY(cudaMemcpy(d_src.p, src, n_cols * N * 8, cudaMemcpyHostToDevice));
    DT_TRY(cudaMemcpy(d_items.p, items.data(), items.size() * sizeof(mk::FwdItem), cudaMemcpyHostToDevice));
    DT_TRY(cudaMemset(d_out.p, 0xAA, n_out * 8));
    mk::launch_fwd_ntt(d_items.as<mk::FwdItem>(), (u32)items.size(), nh.view(d_tab.as<u64>()), ph.view(d_pm.as<u64>()), 0);
    if ((rc = finish())) return rc;
    DT_TRY(cudaMemcpy(out, d_out.p, n_out * 8, cudaMemcpyDeviceToHost));
    return DT_OK;
}

}  // extern "C"
