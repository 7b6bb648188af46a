// Goldilocks field (p = 2^64 - 2^32 + 1) and its quadratic extension F_p[u]/(u^2 - 7) for
// device and host code of the product.  All values are canonical u64 (< p).
//
// Reference definitions being reproduced: `Felt` = p3 Goldilocks (crates/field/src/native/mod.rs:58),
// `QuadFelt` = binomial extension with W = 7 (air/src/constraints/ext_field.rs:11-12,
// crates/field/src/native/mod.rs:394-425).  64-bit modular integer arithmetic: tensor cores do
// not apply; the multiplier is the 32-bit IMAD pipe (mul.lo/mul.hi.u64 expand to IMADs).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace gl {

typedef uint64_t u64;
typedef unsigned int u32;

#define GL_HD __host__ __device__ __forceinline__

static constexpr u64 P = 0xFFFFFFFF00000001ULL;
static constexpr u64 EPS = 0xFFFFFFFFULL;  // 2^64 mod p = 2^32 - 1

// add / sub / mul of the kernels that use gl:: directly (constraint interpreter, LogUp rows, DEEP tail, OOD, FRI fold) on
// the carry flag and one 128-bit product, like poseidon2_fast2.cuh: canonical operands for add / sub, canonical results
// everywhere, the same PTX templates, unsigned __int128 on the host.
GL_HD void fast_subb64(u64 a, u64 b, u64& r, unsigned& m) {
#ifdef __CUDA_ARCH__
    asm("sub.cc.u64 %0, %2, %3;\n\tsubc.u32 %1, 0, 0;" : "=l"(r), "=r"(m) : "l"(a), "l"(b));
#else
    r = a - b; m = a < b ? 0xFFFFFFFFu : 0u;
#endif
}
GL_HD void fast_addc64(u64 a, u64 b, u64& r, unsigned& c) {
#ifdef __CUDA_ARCH__
    asm("add.cc.u64 %0, %2, %3;\n\taddc.u32 %1, 0, 0;" : "=l"(r), "=r"(c) : "l"(a), "l"(b));
#else
    unsigned __int128 s = (unsigned __int128)a + b; r = (u64)s; c = (unsigned)(s >> 64);
#endif
}
GL_HD u64 sub(u64 a, u64 b) { u64 d; unsigned m; fast_subb64(a, b, d, m); return d - (u64)m; }
GL_HD u64 add(u64 a, u64 b) { return sub(a, P - b); }
GL_HD u64 neg(u64 a) { return a ? P - a : 0; }
GL_HD u64 dbl(u64 a) { return add(a, a); }

GL_HD u64 mul(u64 a, u64 b) {
    unsigned __int128 q = (unsigned __int128)a * b;
    u64 lo = (u64)q, hi = (u64)(q >> 64);
    unsigned x2 = (unsigned)hi, x3 = (unsigned)(hi >> 32), m, c;
    u64 t, r, e;
    fast_subb64(lo, (u64)x3, t, m);
    t -= (u64)m;
#ifdef __CUDA_ARCH__
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(e) : "r"(x2), "r"(0xFFFFFFFFu));
#else
    e = (u64)x2 * EPS;
#endif
    fast_addc64(t, e, r, c);
    r = (u64)c * EPS + r;
    fast_subb64(r, P, t, m);
    return t - (u64)m;
}
GL_HD u64 sqr(u64 a) { return mul(a, a); }

// Halve: a/2 mod p.
GL_HD u64 half(u64 a) { return (a >> 1) + ((a & 1) ? 0x7FFFFFFF80000001ULL : 0); }

GL_HD u64 pow(u64 b, u64 e) {
    u64 r = 1;
    while (e) { if (e & 1) r = mul(r, b); b = sqr(b); e >>= 1; }
    return r;
}
GL_HD u64 exp_pow2(u64 a, unsigned k) { while (k--) a = sqr(a); return a; }

// a^(p-2) with the standard 2^32-structured addition chain (72 multiplications).
GL_HD u64 inv(u64 a) {
    // p - 2 = 0xFFFFFFFE_FFFFFFFF = (2^32 - 2) * 2^32 + (2^32 - 1)
    u64 t2 = mul(sqr(a), a);              // a^3          (2 bits)
    u64 t3 = mul(sqr(t2), a);             // a^7          (3 bits)
    u64 t6 = mul(exp_pow2(t3, 3), t3);    // 2^6 - 1
    u64 t12 = mul(exp_pow2(t6, 6), t6);   // 2^12 - 1
    u64 t24 = mul(exp_pow2(t12, 12), t12);// 2^24 - 1
    u64 t30 = mul(exp_pow2(t24, 6), t6);  // 2^30 - 1
    u64 t31 = mul(sqr(t30), a);           // 2^31 - 1
    u64 t32 = mul(sqr(t31), a);           // 2^32 - 1
    // exponent = (2^31 - 1) * 2^33 + (2^32 - 1):  high part 2^32 - 2 = (2^31 - 1) * 2
    u64 r = exp_pow2(t31, 33);
    return mul(r, t32);
}

static constexpr u64 ROOT_2_32 = 1753635133440165772ULL;   // 7^((p-1)/2^32)
GL_HD u64 two_adic_generator(unsigned bits) { return exp_pow2(ROOT_2_32, 32 - bits); }
// canonical LDE coset shift 7^(2^(32 - log_lde))  (crates/lifted-stark/src/domain.rs:358-361)
GL_HD u64 lde_shift(unsigned log_lde) { return exp_pow2(7, 32 - log_lde); }

struct E2 { u64 a, b; };   // a + b*u, u^2 = 7

GL_HD E2 e2(u64 a, u64 b) { E2 r; r.a = a; r.b = b; return r; }
GL_HD E2 e2_add(E2 x, E2 y) { return e2(add(x.a, y.a), add(x.b, y.b)); }
GL_HD E2 e2_sub(E2 x, E2 y) { return e2(sub(x.a, y.a), sub(x.b, y.b)); }
GL_HD E2 e2_neg(E2 x) { return e2(neg(x.a), neg(x.b)); }
GL_HD u64 mul7(u64 x) { u64 x2 = dbl(x), x4 = dbl(x2); return sub(add(x4, x4), x); }  // 8x - x
GL_HD E2 e2_mul(E2 x, E2 y) {
    // Karatsuba: 3 base multiplications
    u64 aa = mul(x.a, y.a), bb = mul(x.b, y.b);
    u64 cross = sub(sub(mul(add(x.a, x.b), add(y.a, y.b)), aa), bb);
    return e2(add(aa, mul7(bb)), cross);
}
GL_HD E2 e2_sqr(E2 x) {
    u64 ab = mul(x.a, x.b);
    return e2(add(sqr(x.a), mul7(sqr(x.b))), dbl(ab));
}
GL_HD E2 e2_mulf(E2 x, u64 s) { return e2(mul(x.a, s), mul(x.b, s)); }
GL_HD E2 e2_inv(E2 x) {
    u64 n = sub(sqr(x.a), mul7(sqr(x.b)));
    u64 ni = inv(n);
    return e2(mul(x.a, ni), neg(mul(x.b, ni)));
}
GL_HD bool e2_eq(E2 x, E2 y) { return x.a == y.a && x.b == y.b; }
GL_HD E2 e2_exp_pow2(E2 x, unsigned k) { while (k--) x = e2_sqr(x); return x; }
GL_HD E2 e2_pow(E2 b, u64 e) {
    E2 r = e2(1, 0);
    while (e) { if (e & 1) r = e2_mul(r, b); b = e2_sqr(b); e >>= 1; }
    return r;
}

GL_HD u32 bitrev32(u32 x, unsigned bits) {
#ifdef __CUDA_ARCH__
    return bits ? (__brev(x) >> (32 - bits)) : 0;
#else
    u32 r = 0;
    for (unsigned i = 0; i < bits; i++) r |= ((x >> i) & 1u) << (bits - 1 - i);
    return r;
#endif
}

}  // namespace gl
