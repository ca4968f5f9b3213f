// 128-bit prime field arithmetic for sm_90a, values kept canonical (< M) in two 64-bit registers.
//
//   M = 2^128 - 45*2^40 + 1          (/root/reference/src/math/field.rs:11)
//   C = 2^128 mod M = 45*2^40 - 1    (a 46-bit constant)  =>  x*2^128 == x*C (mod M)
//
// The reference reduces with two 128x64 partial products (field.rs:38-73); here the full 256-bit product is formed with
// 32-bit multiply-add chains (IMAD) and folded twice through C (Solinas-style), which maps onto the integer pipes of
// the SM without any division.  Results are the canonical representatives, so every value is bit-identical to the
// reference's `field::{add,sub,mul}` (checked against the oracle and Python integers in tests/test_gpu_blocks.py).
#pragma once
#include <cstdint>

namespace dg {

struct __align__(16) fe {
    unsigned long long lo, hi;
};

#define DG_M_LO 0xffffd30000000001ULL
#define DG_M_HI 0xffffffffffffffffULL
#define DG_C_LO 0x00002cffffffffffULL   // C = 45*2^40 - 1

__host__ __device__ __forceinline__ fe fe_make(unsigned long long lo, unsigned long long hi = 0) { fe r; r.lo = lo; r.hi = hi; return r; }
__host__ __device__ __forceinline__ bool fe_is_zero(fe a) { return (a.lo | a.hi) == 0; }
__host__ __device__ __forceinline__ bool fe_eq(fe a, fe b) { return a.lo == b.lo && a.hi == b.hi; }


// ---------------------------------------------------------------------------------------------------------------------
// portable restatement of the same folding (plain C++): the host path (table setup, unit tests of the logic on the CPU
// box) and the cross-check for the PTX path in tests/test_gpu_blocks.py
// ---------------------------------------------------------------------------------------------------------------------
namespace portable {

typedef unsigned __int128 dg_u128;
__host__ __device__ inline dg_u128 fe_to_u128(fe a) { return ((dg_u128)a.hi << 64) | a.lo; }
__host__ __device__ inline fe fe_from_u128(dg_u128 v) { return fe_make((unsigned long long)v, (unsigned long long)(v >> 64)); }
__host__ __device__ inline fe fe_add(fe a, fe b) {
    dg_u128 x = fe_to_u128(a), y = fe_to_u128(b), s = x + y;
    bool c1 = s < x;
    dg_u128 t = s + DG_C_LO;
    bool c2 = t < s;
    return fe_from_u128((c1 || c2) ? t : s);
}
__host__ __device__ inline fe fe_sub(fe a, fe b) {
    dg_u128 x = fe_to_u128(a), y = fe_to_u128(b), d = x - y;
    return fe_from_u128(x < y ? d - DG_C_LO : d);
}
__host__ __device__ inline fe fe_neg(fe a) { return fe_sub(fe_make(0, 0), a); }
__host__ __device__ inline fe fe_reduce256(unsigned long long t0, unsigned long long t1, unsigned long long t2, unsigned long long t3) {
    dg_u128 p0 = (dg_u128)t2 * 45, p1 = (dg_u128)t3 * 45;
    unsigned long long u0 = (unsigned long long)p0, p0h = (unsigned long long)(p0 >> 64), p1l = (unsigned long long)p1, p1h = (unsigned long long)(p1 >> 64);
    unsigned long long u1 = p0h + p1l, u2 = p1h + (u1 < p1l ? 1ULL : 0ULL);
    unsigned long long s0 = u0 << 40, s1 = (u1 << 40) | (u0 >> 24), s2 = (u2 << 40) | (u1 >> 24);
    dg_u128 lo = ((dg_u128)t1 << 64) | t0, s = ((dg_u128)s1 << 64) | s0, hi = ((dg_u128)t3 << 64) | t2;
    dg_u128 v = lo + s;
    unsigned long long v2 = s2 + (v < lo ? 1ULL : 0ULL);
    dg_u128 v_ = v - hi;
    if (v < hi) v2 -= 1;
    dg_u128 w = (dg_u128)v2 * DG_C_LO;
    dg_u128 r = v_ + w;
    bool cy = r < v_;
    dg_u128 q = r + DG_C_LO;
    bool cy2 = q < r;
    return fe_from_u128((cy || cy2) ? q : r);
}
__host__ __device__ inline fe fe_mul(fe a, fe b) {
    dg_u128 p00 = (dg_u128)a.lo * b.lo, p01 = (dg_u128)a.lo * b.hi, p10 = (dg_u128)a.hi * b.lo, p11 = (dg_u128)a.hi * b.hi;
    dg_u128 mid = (p00 >> 64) + (unsigned long long)p01 + (unsigned long long)p10;
    dg_u128 hi = p11 + (p01 >> 64) + (p10 >> 64) + (mid >> 64);
    return fe_reduce256((unsigned long long)p00, (unsigned long long)mid, (unsigned long long)hi, (unsigned long long)(hi >> 64));
}
__host__ __device__ inline fe fe_sqr(fe a) { return fe_mul(a, a); }
__host__ __device__ inline fe fe_pow_u128(fe a, unsigned long long e_lo, unsigned long long e_hi) {
    fe r = fe_make(1, 0);
    for (int i = 127; i >= 0; i--) {
        r = fe_sqr(r);
        unsigned long long bit = i >= 64 ? (e_hi >> (i - 64)) & 1ULL : (e_lo >> i) & 1ULL;
        if (bit) r = fe_mul(r, a);
    }
    return r;
}
__host__ __device__ inline fe fe_pow_u64(fe a, unsigned long long e) { return fe_pow_u128(a, e, 0); }
__host__ __device__ inline fe fe_inv(fe a) { return fe_pow_u128(a, DG_M_LO - 2ULL, DG_M_HI); }
// the companion of a twiddle for fe_mul_tw: w * 2^64 mod M
__host__ __device__ inline fe fe_tw_companion(fe w) { return fe_mul(w, fe_make(0, 1)); }
// a0*w + a1*w_c mod M for a = a1*2^64 + a0: a*w when w_c is w's companion
__host__ __device__ inline fe fe_mul_tw(fe a, fe w, fe w_c) {
    return fe_add(fe_mul(fe_make(a.lo, 0), w), fe_mul(fe_make(a.hi, 0), w_c));
}


}  // namespace portable

// unreduced accumulators (see the ptx namespace): 288-bit sums of products / one 256-bit product
struct fe_wide { unsigned int r[9]; };
struct fe_prod { unsigned int r[8]; };

#ifdef __CUDA_ARCH__
namespace ptx {

// fe_add: select-based (13 ALU instructions).  A mask-based variant with an out-of-line path for sums in [M, 2^128) is
// shorter but puts a call site into every addition: measured slower inside the NTT / constraint kernels, removed.
__device__ __forceinline__ fe fe_add(fe a, fe b) {
    unsigned long long s0, s1, t0, t1;
    unsigned int c1, c2;
    asm("{\n\t"
        "add.cc.u64  %0, %6, %8;\n\t"
        "addc.cc.u64 %1, %7, %9;\n\t"
        "addc.u32    %4, 0, 0;\n\t"
        "add.cc.u64  %2, %0, %10;\n\t"
        "addc.cc.u64 %3, %1, 0;\n\t"
        "addc.u32    %5, 0, 0;\n\t"
        "}"
        : "=&l"(s0), "=&l"(s1), "=&l"(t0), "=&l"(t1), "=&r"(c1), "=&r"(c2)
        : "l"(a.lo), "l"(a.hi), "l"(b.lo), "l"(b.hi), "l"(DG_C_LO));
    bool wrap = (c1 | c2) != 0;      // a + b >= M  <=>  a + b + C >= 2^128
    fe r; r.lo = wrap ? t0 : s0; r.hi = wrap ? t1 : s1;
    return r;
}

// a - b: subtract, then subtract C when the difference borrowed (a - b + M = a - b - C mod 2^128); always canonical
__device__ __forceinline__ fe fe_sub(fe a, fe b) {
    unsigned int d0, d1, d2, d3, m, c1;
    (void)m; (void)c1;
    asm("sub.cc.u32  %0, %6, %10;\n\t"
        "subc.cc.u32 %1, %7, %11;\n\t"
        "subc.cc.u32 %2, %8, %12;\n\t"
        "subc.cc.u32 %3, %9, %13;\n\t"
        "subc.u32    %4, 0, 0;\n\t"            // m = 0xffffffff on borrow, else 0
        "and.b32     %5, %4, 0x00002cff;\n\t"
        "sub.cc.u32  %0, %0, %4;\n\t"
        "subc.cc.u32 %1, %1, %5;\n\t"
        "subc.cc.u32 %2, %2, 0;\n\t"
        "subc.u32    %3, %3, 0;"
        : "=&r"(d0), "=&r"(d1), "=&r"(d2), "=&r"(d3), "=&r"(m), "=&r"(c1)
        : "r"((unsigned int)a.lo), "r"((unsigned int)(a.lo >> 32)), "r"((unsigned int)a.hi), "r"((unsigned int)(a.hi >> 32)),
          "r"((unsigned int)b.lo), "r"((unsigned int)(b.lo >> 32)), "r"((unsigned int)b.hi), "r"((unsigned int)(b.hi >> 32)));
    fe r;
    r.lo = ((unsigned long long)d1 << 32) | d0;
    r.hi = ((unsigned long long)d3 << 32) | d2;
    return r;
}

__device__ __forceinline__ fe fe_neg(fe a) { return fe_sub(fe_make(0, 0), a); }

// 256-bit product of two 128-bit values as eight 32-bit limbs (schoolbook, carry chains on the IMAD pipe)
__device__ __forceinline__ void mul_wide_4x4(const unsigned int a[4], const unsigned int b[4], unsigned int r[8]) {
    // row 0
    asm("mul.lo.u32 %0, %4, %5;\n\t"
        "mul.hi.u32 %1, %4, %5;\n\t"
        "mul.lo.u32 %2, %4, %6;\n\t"   // placeholders overwritten below
        "mul.hi.u32 %3, %4, %6;"
        : "=&r"(r[0]), "=&r"(r[1]), "=&r"(r[2]), "=&r"(r[3]) : "r"(a[0]), "r"(b[0]), "r"(b[2]));
    // r[0] = lo(a0 b0); r[1] = hi(a0 b0); r[2] = lo(a0 b2); r[3] = hi(a0 b2)
    asm("mad.lo.cc.u32  %0, %4, %5, %0;\n\t"     // r1 += lo(a0 b1)
        "madc.hi.cc.u32 %1, %4, %5, %1;\n\t"     // r2 += hi(a0 b1) + c
        "madc.lo.cc.u32 %2, %4, %6, %2;\n\t"     // r3 += lo(a0 b3) + c
        "madc.hi.u32    %3, %4, %6, 0;"          // r4  = hi(a0 b3) + c
        : "+r"(r[1]), "+r"(r[2]), "+r"(r[3]), "=&r"(r[4]) : "r"(a[0]), "r"(b[1]), "r"(b[3]));
#pragma unroll
    for (int i = 1; i < 4; i++) {
        // even columns of row i: lo(ai b0)->r[i], hi(ai b0)->r[i+1], lo(ai b2)->r[i+2], hi(ai b2)->r[i+3], carry->r[i+4]
        asm("mad.lo.cc.u32  %0, %5, %6, %0;\n\t"
            "madc.hi.cc.u32 %1, %5, %6, %1;\n\t"
            "madc.lo.cc.u32 %2, %5, %7, %2;\n\t"
            "madc.hi.cc.u32 %3, %5, %7, %3;\n\t"
            "addc.u32       %4, 0, 0;"
            : "+r"(r[i]), "+r"(r[i + 1]), "+r"(r[i + 2]), "+r"(r[i + 3]), "=&r"(r[i + 4])
            : "r"(a[i]), "r"(b[0]), "r"(b[2]));
        // odd columns of row i: lo(ai b1)->r[i+1], hi(ai b1)->r[i+2], lo(ai b3)->r[i+3], hi(ai b3)->r[i+4]
        asm("mad.lo.cc.u32  %0, %4, %5, %0;\n\t"
            "madc.hi.cc.u32 %1, %4, %5, %1;\n\t"
            "madc.lo.cc.u32 %2, %4, %6, %2;\n\t"
            "madc.hi.u32    %3, %4, %6, %3;"
            : "+r"(r[i + 1]), "+r"(r[i + 2]), "+r"(r[i + 3]), "+r"(r[i + 4])
            : "r"(a[i]), "r"(b[1]), "r"(b[3]));
    }
}

// reduce a 256-bit value (t0..t3 little-endian 64-bit limbs) modulo M
__device__ __forceinline__ fe fe_reduce256(unsigned long long t0, unsigned long long t1, unsigned long long t2, unsigned long long t3) {
    // fold 1: v = lo + hi*C = lo + ((hi*45) << 40) - hi         (hi = t3:t2, 128 bits)
    // u = hi * 45  (134 bits: u2:u1:u0)
    unsigned long long u0, u1, u2;
    {
        unsigned long long p0l = t2 * 45ULL, p0h = __umul64hi(t2, 45ULL);
        unsigned long long p1l = t3 * 45ULL, p1h = __umul64hi(t3, 45ULL);
        u0 = p0l;
        u1 = p0h + p1l;                    // cannot lose a carry into u2 beyond what we add next
        u2 = p1h + (u1 < p1l ? 1ULL : 0ULL);
    }
    // s = u << 40 (174 bits: s2:s1:s0)
    unsigned long long s0 = u0 << 40;
    unsigned long long s1 = (u1 << 40) | (u0 >> 24);
    unsigned long long s2 = (u2 << 40) | (u1 >> 24);
    // v = lo + s - hi   (192-bit arithmetic, result non-negative and < 2^175)
    unsigned long long v0, v1, v2;
    asm("{\n\t"
        "add.cc.u64  %0, %3, %5;\n\t"
        "addc.cc.u64 %1, %4, %6;\n\t"
        "addc.u64    %2, %7, 0;\n\t"
        "sub.cc.u64  %0, %0, %8;\n\t"
        "subc.cc.u64 %1, %1, %9;\n\t"
        "subc.u64    %2, %2, 0;\n\t"
        "}"
        : "=&l"(v0), "=&l"(v1), "=&l"(v2)
        : "l"(t0), "l"(t1), "l"(s0), "l"(s1), "l"(s2), "l"(t2), "l"(t3));
    // fold 2: w = v2 * C  (v2 < 2^47, C < 2^46 => w < 2^93)
    unsigned long long w0 = v2 * DG_C_LO, w1 = __umul64hi(v2, DG_C_LO);
    unsigned long long r0, r1, q0, q1;
    unsigned int cy, cy2;
    asm("{\n\t"
        "add.cc.u64  %0, %6, %8;\n\t"
        "addc.cc.u64 %1, %7, %9;\n\t"
        "addc.u32    %4, 0, 0;\n\t"
        "add.cc.u64  %2, %0, %10;\n\t"      // q = r + C  (used when r wrapped 2^128 or r >= M)
        "addc.cc.u64 %3, %1, 0;\n\t"
        "addc.u32    %5, 0, 0;\n\t"
        "}"
        : "=&l"(r0), "=&l"(r1), "=&l"(q0), "=&l"(q1), "=&r"(cy), "=&r"(cy2)
        : "l"(v0), "l"(v1), "l"(w0), "l"(w1), "l"(DG_C_LO));
    // if r wrapped (cy): true value = r + 2^128 == r + C (< M because r is tiny after a wrap)
    // else if r >= M (cy2): r - M = r + C - 2^128 = q
    bool use_q = (cy | cy2) != 0;
    fe r; r.lo = use_q ? q0 : r0; r.hi = use_q ? q1 : r1;
    return r;
}

__device__ __forceinline__ fe fe_mul_v1(fe a, fe b) {
    unsigned int x[4] = { (unsigned int)a.lo, (unsigned int)(a.lo >> 32), (unsigned int)a.hi, (unsigned int)(a.hi >> 32) };
    unsigned int y[4] = { (unsigned int)b.lo, (unsigned int)(b.lo >> 32), (unsigned int)b.hi, (unsigned int)(b.hi >> 32) };
    unsigned int r[8];
    mul_wide_4x4(x, y, r);
    return fe_reduce256(((unsigned long long)r[1] << 32) | r[0], ((unsigned long long)r[3] << 32) | r[2],
                        ((unsigned long long)r[5] << 32) | r[4], ((unsigned long long)r[7] << 32) | r[6]);
}

// 256-bit product with separate even-column / odd-column 64-bit accumulators: every (lo, hi) pair below is a dedicated
// register pair, so ptxas fuses each mad.lo/madc.hi couple into one IMAD.WIDE.U32 (carry-out / .X carry-in forms) without
// the register shuffles that overlapping pairs cause.  E = columns 0,2,4,6 ; O = columns 1,3,5,7.
__device__ __forceinline__ void mul_wide_eo(const unsigned int a[4], const unsigned int b[4], unsigned int r[8]) {
    unsigned int e0, e1, e2, e3, e4, e5, e6, e7, o1, o2, o3, o4, o5, o6, o7;
    // row 0: E0 = a0 b0, E2 = a0 b2, O1 = a0 b1, O3 = a0 b3
    asm("mul.lo.u32 %0, %8, %9;\n\t"  "mul.hi.u32 %1, %8, %9;\n\t"
        "mul.lo.u32 %2, %8, %11;\n\t" "mul.hi.u32 %3, %8, %11;\n\t"
        "mul.lo.u32 %4, %8, %10;\n\t" "mul.hi.u32 %5, %8, %10;\n\t"
        "mul.lo.u32 %6, %8, %12;\n\t" "mul.hi.u32 %7, %8, %12;"
        : "=&r"(e0), "=&r"(e1), "=&r"(e2), "=&r"(e3), "=&r"(o1), "=&r"(o2), "=&r"(o3), "=&r"(o4)
        : "r"(a[0]), "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]));
    // row 1: O1 += a1 b0 ; O3 += a1 b2 + c ; O5 = c        E2 += a1 b1 ; E4 = a1 b3 + c
    asm("mad.lo.cc.u32  %0, %9, %10, %0;\n\t"  "madc.hi.cc.u32 %1, %9, %10, %1;\n\t"
        "madc.lo.cc.u32 %2, %9, %12, %2;\n\t"  "madc.hi.cc.u32 %3, %9, %12, %3;\n\t"
        "addc.u32       %4, 0, 0;\n\t"
        "mad.lo.cc.u32  %5, %9, %11, %5;\n\t"  "madc.hi.cc.u32 %6, %9, %11, %6;\n\t"
        "madc.lo.cc.u32 %7, %9, %13, 0;\n\t"   "madc.hi.u32    %8, %9, %13, 0;"
        : "+r"(o1), "+r"(o2), "+r"(o3), "+r"(o4), "=&r"(o5), "+r"(e2), "+r"(e3), "=&r"(e4), "=&r"(e5)
        : "r"(a[1]), "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]));
    // row 2: E2 += a2 b0 ; E4 += a2 b2 + c ; E6 = c        O3 += a2 b1 ; O5:O6 = a2 b3 + O5 + c
    asm("mad.lo.cc.u32  %0, %9, %10, %0;\n\t" "madc.hi.cc.u32 %1, %9, %10, %1;\n\t"
        "madc.lo.cc.u32 %2, %9, %12, %2;\n\t" "madc.hi.cc.u32 %3, %9, %12, %3;\n\t"
        "addc.u32       %4, 0, 0;\n\t"
        "mad.lo.cc.u32  %5, %9, %11, %5;\n\t" "madc.hi.cc.u32 %6, %9, %11, %6;\n\t"
        "madc.lo.cc.u32 %7, %9, %13, %7;\n\t" "madc.hi.u32    %8, %9, %13, 0;"
        : "+r"(e2), "+r"(e3), "+r"(e4), "+r"(e5), "=&r"(e6), "+r"(o3), "+r"(o4), "+r"(o5), "=&r"(o6)
        : "r"(a[2]), "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]));
    // row 3: O3 += a3 b0 ; O5 += a3 b2 + c ; O7 = c        E4 += a3 b1 ; E6:E7 = a3 b3 + E6 + c
    asm("mad.lo.cc.u32  %0, %9, %10, %0;\n\t" "madc.hi.cc.u32 %1, %9, %10, %1;\n\t"
        "madc.lo.cc.u32 %2, %9, %12, %2;\n\t" "madc.hi.cc.u32 %3, %9, %12, %3;\n\t"
        "addc.u32       %4, 0, 0;\n\t"
        "mad.lo.cc.u32  %5, %9, %11, %5;\n\t" "madc.hi.cc.u32 %6, %9, %11, %6;\n\t"
        "madc.lo.cc.u32 %7, %9, %13, %7;\n\t" "madc.hi.u32    %8, %9, %13, 0;"
        : "+r"(o3), "+r"(o4), "+r"(o5), "+r"(o6), "=&r"(o7), "+r"(e4), "+r"(e5), "+r"(e6), "=&r"(e7)
        : "r"(a[3]), "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]));
    // result = E + (O << 32)
    r[0] = e0;
    asm("add.cc.u32  %0, %7, %14;\n\t"
        "addc.cc.u32 %1, %8, %15;\n\t"
        "addc.cc.u32 %2, %9, %16;\n\t"
        "addc.cc.u32 %3, %10, %17;\n\t"
        "addc.cc.u32 %4, %11, %18;\n\t"
        "addc.cc.u32 %5, %12, %19;\n\t"
        "addc.u32    %6, %13, %20;"
        : "=&r"(r[1]), "=&r"(r[2]), "=&r"(r[3]), "=&r"(r[4]), "=&r"(r[5]), "=&r"(r[6]), "=&r"(r[7])
        : "r"(e1), "r"(e2), "r"(e3), "r"(e4), "r"(e5), "r"(e6), "r"(e7), "r"(o1), "r"(o2), "r"(o3), "r"(o4), "r"(o5), "r"(o6), "r"(o7));
}

// ---- variant 3: reduction built from IMAD.WIDE chains (FMA pipe) instead of 64-bit add/shift sequences (ALU pipe) --------------
//   hi*C = ((hi * 45*2^8) << 32) - hi ;  the "<< 32" is a limb rename, the additions of the low limbs ride on the wide
//   multiply-adds (multiplier 1), so the only ALU work left is two borrow chains and the final canonicalisation.
#define DG_HAVE_V3 1
__device__ __forceinline__ unsigned long long wmad(unsigned int a, unsigned int b, unsigned long long c) {
    unsigned long long d;
    asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(d) : "r"(a), "r"(b), "l"(c));
    return d;
}
__device__ __forceinline__ fe fe_reduce_v3(const unsigned int r[8]) {
    const unsigned int K = 11520u;   // 45 * 2^8
    // V = lo + ((hi * K) << 32)   (6 limbs)
    unsigned long long t0 = wmad(r[4], K, (unsigned long long)r[1]);
    unsigned long long t1 = wmad(r[2], 1u, wmad(r[5], K, t0 >> 32));
    unsigned long long t2 = wmad(r[3], 1u, wmad(r[6], K, t1 >> 32));
    unsigned long long t3 = wmad(r[7], K, t2 >> 32);
    unsigned int v0 = r[0], v1 = (unsigned int)t0, v2 = (unsigned int)t1, v3 = (unsigned int)t2, v4 = (unsigned int)t3, v5 = (unsigned int)(t3 >> 32);
    // V -= hi
    asm("sub.cc.u32  %0, %0, %6;\n\t"
        "subc.cc.u32 %1, %1, %7;\n\t"
        "subc.cc.u32 %2, %2, %8;\n\t"
        "subc.cc.u32 %3, %3, %9;\n\t"
        "subc.cc.u32 %4, %4, 0;\n\t"
        "subc.u32    %5, %5, 0;"
        : "+r"(v0), "+r"(v1), "+r"(v2), "+r"(v3), "+r"(v4), "+r"(v5) : "r"(r[4]), "r"(r[5]), "r"(r[6]), "r"(r[7]));
    // fold the 47-bit top T = v5:v4 :  T*C = ((T*K) << 32) - T ;  T*K < 2^61
    unsigned long long w0 = wmad(v4, K, 0ULL);
    unsigned long long w1 = wmad(v5, K, w0 >> 32);
    unsigned int a1 = (unsigned int)w0, a2 = (unsigned int)w1, a3 = (unsigned int)(w1 >> 32);
    unsigned int cy, bw;
    asm("add.cc.u32  %0, %0, %5;\n\t"
        "addc.cc.u32 %1, %1, %6;\n\t"
        "addc.cc.u32 %2, %2, %7;\n\t"
        "addc.u32    %3, 0, 0;\n\t"
        "sub.cc.u32  %4, %4, %8;\n\t"
        "subc.cc.u32 %0, %0, %9;\n\t"
        "subc.cc.u32 %1, %1, 0;\n\t"
        "subc.cc.u32 %2, %2, 0;\n\t"
        "subc.u32    %3, %3, 0;"
        : "+r"(v1), "+r"(v2), "+r"(v3), "=&r"(cy), "+r"(v0) : "r"(a1), "r"(a2), "r"(a3), "r"(v4), "r"(v5));
    // cy is now carry - borrow in {0, 1} (the value is non-negative and < 2^128 + 2^93)
    (void)bw;
    // canonical form: q = r + C; take q when r overflowed 2^128 or r >= M
    unsigned int q0, q1, q2, q3, g;
    asm("add.cc.u32  %0, %5, 0xffffffff;\n\t"
        "addc.cc.u32 %1, %6, 0x00002cff;\n\t"
        "addc.cc.u32 %2, %7, 0;\n\t"
        "addc.cc.u32 %3, %8, 0;\n\t"
        "addc.u32    %4, 0, 0;"
        : "=&r"(q0), "=&r"(q1), "=&r"(q2), "=&r"(q3), "=&r"(g) : "r"(v0), "r"(v1), "r"(v2), "r"(v3));
    const bool use_q = (cy | g) != 0;
    fe out;
    out.lo = ((unsigned long long)(use_q ? q1 : v1) << 32) | (use_q ? q0 : v0);
    out.hi = ((unsigned long long)(use_q ? q3 : v3) << 32) | (use_q ? q2 : v2);
    return out;
}
__device__ __forceinline__ fe fe_mul_v3(fe a, fe b) {
    unsigned int x[4] = { (unsigned int)a.lo, (unsigned int)(a.lo >> 32), (unsigned int)a.hi, (unsigned int)(a.hi >> 32) };
    unsigned int y[4] = { (unsigned int)b.lo, (unsigned int)(b.lo >> 32), (unsigned int)b.hi, (unsigned int)(b.hi >> 32) };
    unsigned int r[8];
    mul_wide_eo(x, y, r);
    return fe_reduce_v3(r);
}
// ---- variant 4: v3 with less work on the arithmetic pipe ---------------------------------------------------------------------------
// The NTT and constraint kernels issue more of their work to the ALU pipe (IADD3 / SEL / LOP3) than to the FMA pipe, so v4 moves work off it.
//   * the second fold adds (T*K) << 32 through a multiply-add chain instead of an add-with-carry sequence;
//   * the result needs the final "subtract M" only if it overflowed 2^128 or its top limb is all ones (probability ~2^-32 for
//     uniform values), so that case is an out-of-line slow path behind one predicate.  In the sm_90a build a product is 41 ALU-pipe
//     instructions (30 IADD3, 8 SEL, 2 ISETP, 1 LOP3) next to 38 IMAD.
// (Keeping the "x*1 + c" limb additions on the FMA pipe with an opaque multiplier was tried: ptxas splits them into IMAD + IADD3.)
#define DG_HAVE_V4 1
static __device__ __forceinline__ fe fe_canon_inline(unsigned int v0, unsigned int v1, unsigned int v2, unsigned int v3, unsigned int cy);
static __device__ __noinline__ fe fe_canon_slow(unsigned int v0, unsigned int v1, unsigned int v2, unsigned int v3, unsigned int cy) {
    unsigned int q0, q1, q2, q3, g;
    asm("add.cc.u32  %0, %5, 0xffffffff;\n\t"
        "addc.cc.u32 %1, %6, 0x00002cff;\n\t"
        "addc.cc.u32 %2, %7, 0;\n\t"
        "addc.cc.u32 %3, %8, 0;\n\t"
        "addc.u32    %4, 0, 0;"
        : "=&r"(q0), "=&r"(q1), "=&r"(q2), "=&r"(q3), "=&r"(g) : "r"(v0), "r"(v1), "r"(v2), "r"(v3));
    const bool use_q = (cy | g) != 0;
    fe out;
    out.lo = ((unsigned long long)(use_q ? q1 : v1) << 32) | (use_q ? q0 : v0);
    out.hi = ((unsigned long long)(use_q ? q3 : v3) << 32) | (use_q ? q2 : v2);
    return out;
}
template <bool NESTED_CALL>
__device__ __forceinline__ fe fe_reduce_v4(const unsigned int r[8]) {
    const unsigned int K = 11520u;   // 45 * 2^8 : C = K * 2^32 - 1
    const unsigned int one = 1u;
    // V = lo + ((hi * K) << 32)   (6 limbs), all on multiply-add chains
    unsigned long long t0 = wmad(r[4], K, (unsigned long long)r[1]);
    unsigned long long t1 = wmad(r[2], one, wmad(r[5], K, t0 >> 32));
    unsigned long long t2 = wmad(r[3], one, wmad(r[6], K, t1 >> 32));
    unsigned long long t3 = wmad(r[7], K, t2 >> 32);
    unsigned int v0 = r[0], v1 = (unsigned int)t0, v2 = (unsigned int)t1, v3 = (unsigned int)t2, v4 = (unsigned int)t3, v5 = (unsigned int)(t3 >> 32);
    // V -= hi
    asm("sub.cc.u32  %0, %0, %6;\n\t"
        "subc.cc.u32 %1, %1, %7;\n\t"
        "subc.cc.u32 %2, %2, %8;\n\t"
        "subc.cc.u32 %3, %3, %9;\n\t"
        "subc.cc.u32 %4, %4, 0;\n\t"
        "subc.u32    %5, %5, 0;"
        : "+r"(v0), "+r"(v1), "+r"(v2), "+r"(v3), "+r"(v4), "+r"(v5) : "r"(r[4]), "r"(r[5]), "r"(r[6]), "r"(r[7]));
    // fold the 47-bit top T = v5:v4 :  + (T*K) << 32 on a multiply-add chain (T*K < 2^61), then - T
    unsigned long long u1 = wmad(v4, K, (unsigned long long)v1);
    unsigned long long u2 = wmad(v2, one, wmad(v5, K, u1 >> 32));
    unsigned long long u3 = wmad(v3, one, u2 >> 32);
    v1 = (unsigned int)u1; v2 = (unsigned int)u2; v3 = (unsigned int)u3;
    unsigned int cy = (unsigned int)(u3 >> 32);
    asm("sub.cc.u32  %0, %0, %5;\n\t"
        "subc.cc.u32 %1, %1, %6;\n\t"
        "subc.cc.u32 %2, %2, 0;\n\t"
        "subc.cc.u32 %3, %3, 0;\n\t"
        "subc.u32    %4, %4, 0;"
        : "+r"(v0), "+r"(v1), "+r"(v2), "+r"(v3), "+r"(cy) : "r"(v4), "r"(v5));
    // cy is now carry - borrow in {0, 1}: the value is non-negative and < 2^128 + 2^93.  It is canonical unless it overflowed or
    // lies in [2^128 - 2^96, 2^128)
    if (__builtin_expect((cy != 0u) | (v3 == 0xffffffffu), 0)) {
        if (NESTED_CALL) return fe_canon_slow(v0, v1, v2, v3, cy);
        return fe_canon_inline(v0, v1, v2, v3, cy);        // inside an out-of-line multiply: a plain branch, no nested call frame
    }
    fe out;
    out.lo = ((unsigned long long)v1 << 32) | v0;
    out.hi = ((unsigned long long)v3 << 32) | v2;
    return out;
}
static __device__ __forceinline__ fe fe_canon_inline(unsigned int v0, unsigned int v1, unsigned int v2, unsigned int v3, unsigned int cy) {
    unsigned int q0, q1, q2, q3, g;
    asm volatile("add.cc.u32  %0, %5, 0xffffffff;\n\t"
        "addc.cc.u32 %1, %6, 0x00002cff;\n\t"
        "addc.cc.u32 %2, %7, 0;\n\t"
        "addc.cc.u32 %3, %8, 0;\n\t"
        "addc.u32    %4, 0, 0;"
        : "=&r"(q0), "=&r"(q1), "=&r"(q2), "=&r"(q3), "=&r"(g) : "r"(v0), "r"(v1), "r"(v2), "r"(v3));
    const bool use_q = (cy | g) != 0;
    fe out;
    out.lo = ((unsigned long long)(use_q ? q1 : v1) << 32) | (use_q ? q0 : v0);
    out.hi = ((unsigned long long)(use_q ? q3 : v3) << 32) | (use_q ? q2 : v2);
    return out;
}
template <bool NESTED_CALL>
__device__ __forceinline__ fe fe_mul_v4t(fe a, fe b) {
    unsigned int x[4] = { (unsigned int)a.lo, (unsigned int)(a.lo >> 32), (unsigned int)a.hi, (unsigned int)(a.hi >> 32) };
    unsigned int y[4] = { (unsigned int)b.lo, (unsigned int)(b.lo >> 32), (unsigned int)b.hi, (unsigned int)(b.hi >> 32) };
    unsigned int r[8];
    mul_wide_eo(x, y, r);
    return fe_reduce_v4<NESTED_CALL>(r);
}
__device__ __forceinline__ fe fe_mul_v4(fe a, fe b) { return fe_mul_v4t<true>(a, b); }
// ---- product with a fixed twiddle w and its companion w_c = w * 2^64 mod M (fe_tw_companion) -----------------------------------------
// For a = a1*2^64 + a0:  a*w == a0*w + a1*w_c (mod M).  Both products are 64 x 128 bits, so the 16 IMAD.WIDE of a full product sum
// into columns 0..6 only (a0*w + a1*w_c < 2^193), and the reduction is v4's second fold alone, widened to a 65-bit top.
// tools/model_mul_tw.py restates every chain below and checks its bounds against Python integers.
template <bool NESTED_CALL>
__device__ __forceinline__ fe fe_mul_twt(fe a, fe w, fe w_c) {
    const unsigned int x0 = (unsigned int)a.lo, x1 = (unsigned int)(a.lo >> 32), x2 = (unsigned int)a.hi, x3 = (unsigned int)(a.hi >> 32);
    const unsigned int y0 = (unsigned int)w.lo, y1 = (unsigned int)(w.lo >> 32), y2 = (unsigned int)w.hi, y3 = (unsigned int)(w.hi >> 32);
    const unsigned int z0 = (unsigned int)w_c.lo, z1 = (unsigned int)(w_c.lo >> 32), z2 = (unsigned int)w_c.hi, z3 = (unsigned int)(w_c.hi >> 32);
    // E = even columns 0, 2, 4, 6 ; O = odd columns 1, 3, 5 (64-bit accumulators as in mul_wide_eo)
    unsigned int e0, e1, e2, e3, e4, e5, e6, o1, o2, o3, o4, o5;
    // x0 * w at column 0: E0 = x0 y0, E2 = x0 y2, O1 = x0 y1, O3 = x0 y3
    asm("mul.lo.u32 %0, %8, %9;\n\t"  "mul.hi.u32 %1, %8, %9;\n\t"
        "mul.lo.u32 %2, %8, %11;\n\t" "mul.hi.u32 %3, %8, %11;\n\t"
        "mul.lo.u32 %4, %8, %10;\n\t" "mul.hi.u32 %5, %8, %10;\n\t"
        "mul.lo.u32 %6, %8, %12;\n\t" "mul.hi.u32 %7, %8, %12;"
        : "=&r"(e0), "=&r"(e1), "=&r"(e2), "=&r"(e3), "=&r"(o1), "=&r"(o2), "=&r"(o3), "=&r"(o4)
        : "r"(x0), "r"(y0), "r"(y1), "r"(y2), "r"(y3));
    // x2 * w_c at column 0: E0 += x2 z0 ; E2 += x2 z2 + c ; E4 = c        O1 += x2 z1 ; O3 += x2 z3 + c ; O5 = c
    asm("mad.lo.cc.u32  %0, %10, %11, %0;\n\t" "madc.hi.cc.u32 %1, %10, %11, %1;\n\t"
        "madc.lo.cc.u32 %2, %10, %13, %2;\n\t" "madc.hi.cc.u32 %3, %10, %13, %3;\n\t"
        "addc.u32       %4, 0, 0;\n\t"
        "mad.lo.cc.u32  %5, %10, %12, %5;\n\t" "madc.hi.cc.u32 %6, %10, %12, %6;\n\t"
        "madc.lo.cc.u32 %7, %10, %14, %7;\n\t" "madc.hi.cc.u32 %8, %10, %14, %8;\n\t"
        "addc.u32       %9, 0, 0;"
        : "+r"(e0), "+r"(e1), "+r"(e2), "+r"(e3), "=&r"(e4), "+r"(o1), "+r"(o2), "+r"(o3), "+r"(o4), "=&r"(o5)
        : "r"(x2), "r"(z0), "r"(z1), "r"(z2), "r"(z3));
    // x1 * w at column 1: O1 += x1 y0 ; O3 += x1 y2 + c ; O5 += c         E2 += x1 y1 ; E4:E5 = x1 y3 + E4 + c
    asm("mad.lo.cc.u32  %0, %9, %10, %0;\n\t" "madc.hi.cc.u32 %1, %9, %10, %1;\n\t"
        "madc.lo.cc.u32 %2, %9, %12, %2;\n\t" "madc.hi.cc.u32 %3, %9, %12, %3;\n\t"
        "addc.u32       %4, %4, 0;\n\t"
        "mad.lo.cc.u32  %5, %9, %11, %5;\n\t" "madc.hi.cc.u32 %6, %9, %11, %6;\n\t"
        "madc.lo.cc.u32 %7, %9, %13, %7;\n\t" "madc.hi.u32    %8, %9, %13, 0;"
        : "+r"(o1), "+r"(o2), "+r"(o3), "+r"(o4), "+r"(o5), "+r"(e2), "+r"(e3), "+r"(e4), "=&r"(e5)
        : "r"(x1), "r"(y0), "r"(y1), "r"(y2), "r"(y3));
    // x3 * w_c at column 1: O1 += x3 z0 ; O3 += x3 z2 + c ; O5 += c       E2 += x3 z1 ; E4 += x3 z3 + c ; E6 = c
    asm("mad.lo.cc.u32  %0, %10, %11, %0;\n\t" "madc.hi.cc.u32 %1, %10, %11, %1;\n\t"
        "madc.lo.cc.u32 %2, %10, %13, %2;\n\t" "madc.hi.cc.u32 %3, %10, %13, %3;\n\t"
        "addc.u32       %4, %4, 0;\n\t"
        "mad.lo.cc.u32  %5, %10, %12, %5;\n\t" "madc.hi.cc.u32 %6, %10, %12, %6;\n\t"
        "madc.lo.cc.u32 %7, %10, %14, %7;\n\t" "madc.hi.cc.u32 %8, %10, %14, %8;\n\t"
        "addc.u32       %9, 0, 0;"
        : "+r"(o1), "+r"(o2), "+r"(o3), "+r"(o4), "+r"(o5), "+r"(e2), "+r"(e3), "+r"(e4), "+r"(e5), "=&r"(e6)
        : "r"(x3), "r"(z0), "r"(z1), "r"(z2), "r"(z3));
    // r = E + (O << 32): columns 0..6, r6 <= 1 because the sum is < 2^193
    unsigned int r1, r2, r3, r4, r5, r6;
    asm("add.cc.u32  %0, %6, %12;\n\t"
        "addc.cc.u32 %1, %7, %13;\n\t"
        "addc.cc.u32 %2, %8, %14;\n\t"
        "addc.cc.u32 %3, %9, %15;\n\t"
        "addc.cc.u32 %4, %10, %16;\n\t"
        "addc.u32    %5, %11, 0;"
        : "=&r"(r1), "=&r"(r2), "=&r"(r3), "=&r"(r4), "=&r"(r5), "=&r"(r6)
        : "r"(e1), "r"(e2), "r"(e3), "r"(e4), "r"(e5), "r"(e6), "r"(o1), "r"(o2), "r"(o3), "r"(o4), "r"(o5));
    // fold the 65-bit top T = r6:r5:r4:  + (T*K) << 32 on a multiply-add chain (T*K < 2^79), then - T.  The result is non-negative and
    // < 2^128 + 2^111: cy below is carry - borrow in {0, 1}
    const unsigned int K = 11520u, one = 1u;
    unsigned int v0 = e0;
    unsigned long long u1 = wmad(r4, K, (unsigned long long)r1);
    unsigned long long u2 = wmad(r2, one, wmad(r5, K, u1 >> 32));
    unsigned long long u3 = wmad(r3, one, wmad(r6, K, u2 >> 32));
    unsigned int v1 = (unsigned int)u1, v2 = (unsigned int)u2, v3 = (unsigned int)u3, cy = (unsigned int)(u3 >> 32);
    asm("sub.cc.u32  %0, %0, %5;\n\t"
        "subc.cc.u32 %1, %1, %6;\n\t"
        "subc.cc.u32 %2, %2, %7;\n\t"
        "subc.cc.u32 %3, %3, 0;\n\t"
        "subc.u32    %4, %4, 0;"
        : "+r"(v0), "+r"(v1), "+r"(v2), "+r"(v3), "+r"(cy) : "r"(r4), "r"(r5), "r"(r6));
    // canonical unless it overflowed 2^128 or lies in [2^128 - 2^96, 2^128): the same rare path as fe_reduce_v4
    if (__builtin_expect((cy != 0u) | (v3 == 0xffffffffu), 0)) {
        if (NESTED_CALL) return fe_canon_slow(v0, v1, v2, v3, cy);
        return fe_canon_inline(v0, v1, v2, v3, cy);
    }
    fe out;
    out.lo = ((unsigned long long)v1 << 32) | v0;
    out.hi = ((unsigned long long)v3 << 32) | v2;
    return out;
}
// ---- unreduced accumulation: sums of up to 128 products are kept as 288-bit integers and reduced once ------------------------------
// A dot product sum_j a_j b_j costs, per term, one 256-bit product (16 IMAD.WIDE + 13 ALU) and one 9-limb addition (9 ALU) instead of a
// full modular multiplication and a modular addition (31 + 13 ALU); the single reduction at the end is the v4 fold extended by one limb
// (tools/model_reduce9.py checks every intermediate bound of it against Python integers).
__device__ __forceinline__ fe_prod fe_mul_wide(fe a, fe b) {
    unsigned int x[4] = { (unsigned int)a.lo, (unsigned int)(a.lo >> 32), (unsigned int)a.hi, (unsigned int)(a.hi >> 32) };
    unsigned int y[4] = { (unsigned int)b.lo, (unsigned int)(b.lo >> 32), (unsigned int)b.hi, (unsigned int)(b.hi >> 32) };
    fe_prod p;
    mul_wide_eo(x, y, p.r);
    return p;
}
__device__ __forceinline__ void wide_set(fe_wide &w, const fe_prod &p) {
#pragma unroll
    for (int i = 0; i < 8; i++) w.r[i] = p.r[i];
    w.r[8] = 0;
}
__device__ __forceinline__ void wide_add(fe_wide &w, const fe_prod &p) {
    asm("add.cc.u32  %0, %0, %9;\n\t"
        "addc.cc.u32 %1, %1, %10;\n\t"
        "addc.cc.u32 %2, %2, %11;\n\t"
        "addc.cc.u32 %3, %3, %12;\n\t"
        "addc.cc.u32 %4, %4, %13;\n\t"
        "addc.cc.u32 %5, %5, %14;\n\t"
        "addc.cc.u32 %6, %6, %15;\n\t"
        "addc.cc.u32 %7, %7, %16;\n\t"
        "addc.u32    %8, %8, 0;"
        : "+r"(w.r[0]), "+r"(w.r[1]), "+r"(w.r[2]), "+r"(w.r[3]), "+r"(w.r[4]), "+r"(w.r[5]), "+r"(w.r[6]), "+r"(w.r[7]), "+r"(w.r[8])
        : "r"(p.r[0]), "r"(p.r[1]), "r"(p.r[2]), "r"(p.r[3]), "r"(p.r[4]), "r"(p.r[5]), "r"(p.r[6]), "r"(p.r[7]));
}
// w (< 128 M^2, i.e. r[8] < 128) modulo M, canonical
__device__ __forceinline__ fe fe_reduce_wide(const fe_wide &w) {
    const unsigned int K = 11520u;
    const unsigned int *r = w.r;
    // V = lo + ((H * K) << 32) - H,  H = r[4..8]
    unsigned long long t0 = wmad(r[4], K, (unsigned long long)r[1]);
    unsigned long long t1 = wmad(r[2], 1u, wmad(r[5], K, t0 >> 32));
    unsigned long long t2 = wmad(r[3], 1u, wmad(r[6], K, t1 >> 32));
    unsigned long long t3 = wmad(r[7], K, t2 >> 32);
    unsigned long long t4 = wmad(r[8], K, t3 >> 32);
    unsigned int v0 = r[0], v1 = (unsigned int)t0, v2 = (unsigned int)t1, v3 = (unsigned int)t2, v4 = (unsigned int)t3, v5 = (unsigned int)t4;
    asm("sub.cc.u32  %0, %0, %6;\n\t"
        "subc.cc.u32 %1, %1, %7;\n\t"
        "subc.cc.u32 %2, %2, %8;\n\t"
        "subc.cc.u32 %3, %3, %9;\n\t"
        "subc.cc.u32 %4, %4, %10;\n\t"
        "subc.u32    %5, %5, 0;"
        : "+r"(v0), "+r"(v1), "+r"(v2), "+r"(v3), "+r"(v4), "+r"(v5) : "r"(r[4]), "r"(r[5]), "r"(r[6]), "r"(r[7]), "r"(r[8]));
    // the limb above v5 is zero (V < 2^181); fold T = v5:v4 (< 2^53)
    unsigned long long u1 = wmad(v4, K, (unsigned long long)v1);
    unsigned long long u2 = wmad(v2, 1u, wmad(v5, K, u1 >> 32));
    unsigned long long u3 = wmad(v3, 1u, u2 >> 32);
    v1 = (unsigned int)u1; v2 = (unsigned int)u2; v3 = (unsigned int)u3;
    unsigned int cy = (unsigned int)(u3 >> 32);
    asm("sub.cc.u32  %0, %0, %5;\n\t"
        "subc.cc.u32 %1, %1, %6;\n\t"
        "subc.cc.u32 %2, %2, 0;\n\t"
        "subc.cc.u32 %3, %3, 0;\n\t"
        "subc.u32    %4, %4, 0;"
        : "+r"(v0), "+r"(v1), "+r"(v2), "+r"(v3), "+r"(cy) : "r"(v4), "r"(v5));
    if (__builtin_expect((cy != 0u) | (v3 == 0xffffffffu), 0)) return fe_canon_inline(v0, v1, v2, v3, cy);
    fe out;
    out.lo = ((unsigned long long)v1 << 32) | v0;
    out.hi = ((unsigned long long)v3 << 32) | v2;
    return out;
}
// the multiply used by every kernel (tools/bench_modmul.cu on an H100 SXM, 700 W: v1 204, v3 249, v4 266 G modmul/s; butterfly mix 163 / 183 / 200 G/s;
// fe_mul_tw above, for fixed twiddles with companions: 340 G modmul/s, 244 G butterflies/s)
#ifdef DG_MUL_CALL
// out-of-line variant for kernels whose fully inlined code would not fit the instruction caches
static __device__ __noinline__ fe fe_mul_call(fe a, fe b) { return fe_mul_v4t<false>(a, b); }
__device__ __forceinline__ fe fe_mul(fe a, fe b) { return fe_mul_call(a, b); }
#else
__device__ __forceinline__ fe fe_mul(fe a, fe b) { return fe_mul_v4(a, b); }
#endif
__device__ __forceinline__ fe fe_sqr(fe a) { return fe_mul(a, a); }

// multiply by a small constant (< 2^32)
__device__ __forceinline__ fe fe_mul_small(fe a, unsigned int k) {
    unsigned long long p0l = a.lo * (unsigned long long)k, p0h = __umul64hi(a.lo, (unsigned long long)k);
    unsigned long long p1l = a.hi * (unsigned long long)k, p1h = __umul64hi(a.hi, (unsigned long long)k);
    unsigned long long t1 = p0h + p1l;
    unsigned long long t2 = p1h + (t1 < p1l ? 1ULL : 0ULL);
    return fe_reduce256(p0l, t1, t2, 0ULL);
}

// a^e for a 64-bit exponent (square-and-multiply, MSB first)
__device__ __forceinline__ fe fe_pow_u64(fe a, unsigned long long e) {
    fe r = fe_make(1, 0);
    if (e == 0) return r;
    int top = 63 - __clzll((long long)e);
    for (int i = top; i >= 0; i--) {
        r = fe_sqr(r);
        if ((e >> i) & 1ULL) r = fe_mul(r, a);
    }
    return r;
}
// a^e for a 128-bit exponent
__device__ __forceinline__ fe fe_pow_u128(fe a, unsigned long long e_lo, unsigned long long e_hi) {
    if (e_hi == 0) return fe_pow_u64(a, e_lo);
    fe r = fe_pow_u64(a, e_hi);
    for (int i = 63; i >= 0; i--) {
        r = fe_sqr(r);
        if ((e_lo >> i) & 1ULL) r = fe_mul(r, a);
    }
    return r;
}
// multiplicative inverse by Fermat (inv(0) = 0, as field::inv, field.rs:84)
__device__ __forceinline__ fe fe_inv(fe a) { return fe_pow_u128(a, DG_M_LO - 2ULL, DG_M_HI); }

__device__ __forceinline__ fe fe_cube(fe a) { return fe_mul(fe_sqr(a), a); }


}  // namespace ptx
#endif

// ---- public entry points: PTX path on the device, portable path on the host ------------------------------------------
#ifdef __CUDA_ARCH__
#define DG_IMPL ptx
#else
#define DG_IMPL portable
#endif
__host__ __device__ __forceinline__ fe fe_add(fe a, fe b) { return DG_IMPL::fe_add(a, b); }
__host__ __device__ __forceinline__ fe fe_sub(fe a, fe b) { return DG_IMPL::fe_sub(a, b); }
__host__ __device__ __forceinline__ fe fe_neg(fe a) { return DG_IMPL::fe_neg(a); }
__host__ __device__ __forceinline__ fe fe_mul(fe a, fe b) { return DG_IMPL::fe_mul(a, b); }
__host__ __device__ __forceinline__ fe fe_sqr(fe a) { return DG_IMPL::fe_sqr(a); }
__host__ __device__ __forceinline__ fe fe_pow_u64(fe a, unsigned long long e) { return DG_IMPL::fe_pow_u64(a, e); }
__host__ __device__ __forceinline__ fe fe_pow_u128(fe a, unsigned long long lo, unsigned long long hi) { return DG_IMPL::fe_pow_u128(a, lo, hi); }
__host__ __device__ __forceinline__ fe fe_inv(fe a) { return DG_IMPL::fe_inv(a); }
__host__ __device__ __forceinline__ fe fe_cube(fe a) { return fe_mul(fe_sqr(a), a); }
__host__ __device__ __forceinline__ fe fe_tw_companion(fe w) { return portable::fe_tw_companion(w); }
__host__ __device__ __forceinline__ fe fe_mul_tw(fe a, fe w, fe w_c) {
#ifdef __CUDA_ARCH__
    return ptx::fe_mul_twt<true>(a, w, w_c);
#else
    return portable::fe_mul_tw(a, w, w_c);
#endif
}
__host__ __device__ __forceinline__ fe fe_mul_small(fe a, unsigned int k) {
#ifdef __CUDA_ARCH__
    return ptx::fe_mul_small(a, k);
#else
    return portable::fe_mul(a, fe_make(k, 0));
#endif
}
#undef DG_IMPL

// ---- unreduced dot products: device = 288-bit accumulation (ptx::), host = the same values through reduced arithmetic ----------------
#ifdef __CUDA_ARCH__
#ifdef DG_MUL_CALL
static __device__ __noinline__ fe_prod fe_mul_wide_call(fe a, fe b) { return ptx::fe_mul_wide(a, b); }
static __device__ __noinline__ fe fe_reduce_wide_call(fe_wide w) { return ptx::fe_reduce_wide(w); }
#define DG_MUL_WIDE fe_mul_wide_call
#define DG_REDUCE_WIDE fe_reduce_wide_call
#else
#define DG_MUL_WIDE ptx::fe_mul_wide
#define DG_REDUCE_WIDE ptx::fe_reduce_wide
#endif
__device__ __forceinline__ void wide_set(fe_wide &w, const fe_prod &p) { ptx::wide_set(w, p); }
__device__ __forceinline__ void wide_add(fe_wide &w, const fe_prod &p) { ptx::wide_add(w, p); }
#else
// host pass: a product is carried already reduced in its low four limbs
inline fe_prod fe_mul_wide_host(fe a, fe b) {
    fe m = portable::fe_mul(a, b);
    fe_prod p = {{(unsigned int)m.lo, (unsigned int)(m.lo >> 32), (unsigned int)m.hi, (unsigned int)(m.hi >> 32), 0, 0, 0, 0}};
    return p;
}
inline fe fe_reduce_wide_host(fe_wide w) { return fe_make(((unsigned long long)w.r[1] << 32) | w.r[0], ((unsigned long long)w.r[3] << 32) | w.r[2]); }
#define DG_MUL_WIDE fe_mul_wide_host
#define DG_REDUCE_WIDE fe_reduce_wide_host
inline void wide_set(fe_wide &w, const fe_prod &p) { for (int i = 0; i < 8; i++) w.r[i] = p.r[i]; w.r[8] = 0; }
inline void wide_add(fe_wide &w, const fe_prod &p) {
    fe s = portable::fe_add(fe_reduce_wide_host(w), fe_make(((unsigned long long)p.r[1] << 32) | p.r[0], ((unsigned long long)p.r[3] << 32) | p.r[2]));
    w.r[0] = (unsigned int)s.lo; w.r[1] = (unsigned int)(s.lo >> 32); w.r[2] = (unsigned int)s.hi; w.r[3] = (unsigned int)(s.hi >> 32);
}
#endif
// sum_j a[j] * b[j], N <= 128 terms (compile-time N: fully unrolled)
template <int N>
__host__ __device__ __forceinline__ fe fe_dot(const fe *a, const fe *b) {
    fe_wide w;
    wide_set(w, DG_MUL_WIDE(a[0], b[0]));
#pragma unroll
    for (int j = 1; j < N; j++) wide_add(w, DG_MUL_WIDE(a[j], b[j]));
    return DG_REDUCE_WIDE(w);
}


}  // namespace dg
