// Runs the product's device arithmetic (miden-vm_b200/csrc/poseidon2_fast2.cuh, every function
// __host__ __device__) ON THE CPU and compares it with the canonical restatement in poseidon2.cuh and
// with the reference's known-answer test (crates/crypto/src/hash/algebraic_sponge/poseidon2/test.rs:7-39).
// The device build differs only in the five carry primitives, which use the PTX carry flag there.
// Inputs include non-canonical representatives (>= p, up to 2^64 - 1): the lazy arithmetic accepts any u64.
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include "../../miden-vm_b200/csrc/poseidon2.cuh"
#include "../../miden-vm_b200/csrc/poseidon2_fast2.cuh"

typedef uint64_t u64;
static u64 rng_state = 0x9E3779B97F4A7C15ull;
static u64 rnd() { u64 z = (rng_state += 0x9E3779B97F4A7C15ull); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31); }
static u64 edge(int i) {
    static const u64 E[] = {0, 1, 2, 7, 8, 0xFFFFFFFFull, 0x100000000ull, 0xFFFFFFFF00000000ull, 0xFFFFFFFF00000001ull,
                            0xFFFFFFFF00000002ull, 0xFFFFFFFFFFFFFFFFull, 0xFFFFFFFFFFFFFFFEull, 0xFFFFFFFFFFFFFFF9ull,
                            0xFFFFFFFFFFFFFFF8ull, 0x7FFFFFFF80000000ull, 0x7FFFFFFF80000001ull, 0x8000000000000000ull,
                            0xFFFFFFFEFFFFFFFFull, 0xFFFFFFFF00000000ull - 1, 3, 4, 5, 6, 0xFFFFFFFFFFFFFFFDull};
    return E[i % (int)(sizeof(E) / sizeof(E[0]))];
}
static u64 pick(int i) { return (i & 3) == 0 ? edge(i >> 2) : ((i & 3) == 1 ? rnd() | 0xFFFFFFFF00000000ull : rnd()); }
static u64 cn(u64 x) { return x >= gl::P ? x - gl::P : x; }
static int fails = 0;
#define CHECK(cond, ...) do { if (!(cond)) { if (fails++ < 20) { printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } } while (0)

int main() {
    // scalar primitives against 128-bit integer arithmetic
    for (int i = 0; i < 400000; i++) {
        u64 a = pick(i), b = pick(i * 7 + 3);
        unsigned __int128 q = (unsigned __int128)a * b;
        u64 want = (u64)(q % gl::P);
        CHECK(cn(glf::mul(a, b)) == want, "mul %llx %llx", (unsigned long long)a, (unsigned long long)b);
        CHECK(cn(glf::sqr(a)) == (u64)(((unsigned __int128)a * a) % gl::P), "sqr %llx", (unsigned long long)a);
        CHECK(glf::cmul(cn(a), cn(b)) == want, "cmul");
        CHECK(glf::cadd(cn(a), cn(b)) == (u64)(((unsigned __int128)cn(a) + cn(b)) % gl::P), "cadd");
        CHECK(glf::csub(cn(a), cn(b)) == (u64)(((unsigned __int128)cn(a) + gl::P - cn(b)) % gl::P), "csub");
        CHECK(glf::canon_cc(a) == cn(a), "canon_cc");
        CHECK(cn(glf::add_const(a, cn(b))) == (u64)(((unsigned __int128)cn(a) + cn(b)) % gl::P), "add_const");
        CHECK(gl::mul(cn(glf::half(a)), 2) == cn(a), "half %llx", (unsigned long long)a);
        CHECK(gl::mul(cn(glf::div2k<2>(a)), 4) == cn(a), "div4 %llx", (unsigned long long)a);
        CHECK(gl::mul(cn(glf::div2k<3>(a)), 8) == cn(a), "div8 %llx", (unsigned long long)a);
        glf::W w = glf::wsum(a, b); glf::wadd(w, a); glf::wadd(w, glf::wshl(b, 2)); glf::wadd(w, glf::wtriple(a));
        unsigned __int128 ww = (unsigned __int128)a * 5 + (unsigned __int128)b * 5;
        CHECK(cn(glf::wred(w)) == (u64)(ww % gl::P), "wide add");
        glf::W p8; p8.lo = glf::P8_LO; p8.hi = glf::P8_HI; glf::wadd(w, p8); glf::wsub(w, glf::wtriple(b));
        CHECK(cn(glf::wred(w)) == (u64)(((unsigned __int128)a * 5 + (unsigned __int128)b * 2) % gl::P), "wide sub");
    }
    // the external layer and the permutation against the canonical implementation
    for (int it = 0; it < 20000; it++) {
        u64 s[12], c[12];
        for (int k = 0; k < 12; k++) { s[k] = pick(it * 12 + k); c[k] = cn(s[k]); }
        u64 a[12], b[12];
        for (int k = 0; k < 12; k++) { a[k] = s[k]; b[k] = c[k]; }
        p2f::external_layer(a); p2::external_layer(b);
        for (int k = 0; k < 12; k++) CHECK(cn(a[k]) == b[k], "external layer word %d", k);
        for (int k = 0; k < 12; k++) { a[k] = s[k]; b[k] = c[k]; }
        p2f::permute(a); p2::permute(b);
        for (int k = 0; k < 12; k++) CHECK(cn(a[k]) == b[k], "permutation word %d", k);
    }
    // 96-bit helpers of the lazy internal rounds against 128-bit integer arithmetic
    for (int i = 0; i < 400000; i++) {
        glf::W w; w.lo = pick(i); w.hi = (unsigned)(rnd() >> (32 + (i % 29)));         // any high word up to 2^32 - 1 >> small shifts
        unsigned __int128 v = ((unsigned __int128)w.hi << 64) | w.lo;
        auto val = [](glf::W x) { return ((unsigned __int128)x.hi << 64) | x.lo; };
        if (w.hi < (1u << 29)) {
            CHECK(val(glf::wshl96(w, 1)) == v * 2 && val(glf::wshl96(w, 2)) == v * 4, "wshl96");
            glf::W h = glf::whalf(w);
            CHECK(val(h) * 2 % gl::P == v % gl::P && val(h) <= (v + gl::P) / 2, "whalf");
            glf::W q = glf::wdiv2k<2>(w), e = glf::wdiv2k<3>(w);
            CHECK(val(q) * 4 % gl::P == v % gl::P && val(q) <= v / 4 + gl::P, "wdiv4");
            CHECK(val(e) * 8 % gl::P == v % gl::P && val(e) <= v / 8 + gl::P, "wdiv8");
        }
        CHECK(cn(glf::wred(w)) == (u64)(v % gl::P), "wred of a 96-bit value");
    }
    // the offset table: OFF_j = ceil(4 M_j / p) p, M_(j+1) = 2^64 + 11 M_j + max(4 M_j, OFF_j) < 2^96 for the 8 rounds of a block
    {
        unsigned __int128 M = (unsigned __int128)1 << 64, lim = (unsigned __int128)1 << 96;
        for (int j = 0; j < 8; j++) {
            unsigned __int128 C = (4 * M + gl::P - 1) / gl::P, OFF = C * gl::P, S = ((unsigned __int128)1 << 64) + 11 * M;
            CHECK((u64)OFF == p2f::H_OFF_LO[j] && (unsigned)(OFF >> 64) == p2f::H_OFF_HI[j], "offset table entry %d", j);
            CHECK(OFF >= 4 * M && S + OFF < lim && 4 * M + S < lim, "bound of round %d", j);
            M = S + (OFF > 4 * M ? OFF : 4 * M);
        }
    }
    // worst-case drivers for the bound: every lane at 2^64 - 1 and at p - 1 on entry
    for (int it = 0; it < 2000; it++) {
        u64 a[12], b[12];
        for (int k = 0; k < 12; k++) { a[k] = (it & 1) ? 0xFFFFFFFFFFFFFFFFull : (it & 2) ? gl::P - 1 : pick(it + k) | 0xFFFFFFFF00000000ull; b[k] = cn(a[k]); }
        a[0] = pick(it); b[0] = cn(a[0]);
        p2f::permute(a); p2::permute(b);
        for (int k = 0; k < 12; k++) CHECK(cn(a[k]) == b[k], "permutation (large lanes) word %d", k);
    }
#ifdef P2F_TRACK_BOUNDS
    printf("lazy internal rounds: largest lane high word seen 2^%.2f (limit 2^32)\n", p2f::p2f_max_hi ? __builtin_log2((double)p2f::p2f_max_hi) : 0.0);
#endif
    // reference KAT: input 0..11 (test.rs:7-39)
    static const u64 KAT[12] = {0xf292ab67c0f14b03ull, 0x0a32f1b37656544cull, 0x053c61ab895498deull, 0x02ff92e55b196ffbull,
                                0x58176e8f6f58cab2ull, 0xb0aa1206e7aec0f8ull, 0xe90c13f3dce83ca4ull, 0xf4da15333edf39c2ull,
                                0x23b701c053c2ca6cull, 0xd233d593dcdfbf58ull, 0x4effa5f9516fb52eull, 0x0aaf4489f1f40166ull};
    u64 s[12];
    for (int k = 0; k < 12; k++) s[k] = k;
    p2f::permute(s);
    for (int k = 0; k < 12; k++) CHECK(cn(s[k]) == KAT[k], "KAT word %d: %016llx", k, (unsigned long long)cn(s[k]));
    if (fails) { printf("ARITH_V2_FAILED %d\n", fails); return 1; }
    printf("ARITH_V2_OK\n");
    return 0;
}
