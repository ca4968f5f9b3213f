// The inverse S-box x^INV_ALPHA of Rescue (crypto/hash.rs:238-244) and of the sponge and hasher rounds of the VM (utils/sponge.rs:13-30,
// utils/hasher.rs:28-40): shared by the algebraic hashes (alghash.cu) and the VM interpreter (vm.cu).  Include after fp128.cuh with
// DG_MUL_CALL defined, as both do: the multiplies are out-of-line calls.  `inline` gives the translation units one shared definition.
#pragma once
#include "fp128.cuh"

namespace dg {

// x^INV_ALPHA, hex digits of the exponent from the most significant: 20 x 'a', '8', 'c', 9 x 'a', 'b'
__device__ __noinline__ inline fe alg_inv_sbox(fe x) {
    const fe x2 = fe_sqr(x), x4 = fe_sqr(x2), x8 = fe_sqr(x4);
    const fe xa = fe_mul(x8, x2), xb = fe_mul(xa, x), xc = fe_mul(x8, x4);
    fe acc = xa;
#pragma unroll 1
    for (int d = 1; d < 32; d++) {
        acc = fe_sqr(acc); acc = fe_sqr(acc); acc = fe_sqr(acc); acc = fe_sqr(acc);
        const fe m = d == 20 ? x8 : (d == 21 ? xc : (d == 31 ? xb : xa));
        acc = fe_mul(acc, m);
    }
    return acc;
}

}  // namespace dg
