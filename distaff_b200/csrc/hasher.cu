// utils::hasher::digest (hasher.rs:12-40) on the GPU: the hash of the VM's RESCR op and of the Merkle paths its smpath / pmpath operations
// verify, over 64-byte messages, in two layouts (poly.h, HASHER_WIDE_MIN): a thread per message for wide batches, and 8 lanes per message
// for batches too small to fill the GPU, such as the top levels of a tree.  alg_hash64 / alg_merkle_build (alghash.cu) run it as hash 3.
// Its own translation unit: the out-of-line multiply of a unit is shared by all its kernels, so these kernels beside alghash.cu's would
// change the code ptxas gives those.
#define DG_MUL_CALL 1
#include "common.cuh"
#include "alg_sbox.cuh"
#include "poly.h"
#include "vm.h"

namespace dg {

// A 6-wide Rescue over the reversed state: elements 0..3 of a message go to state[5..2], state[1..0] = 0, 10 rounds with ARK column r, and
// the digest is (state[5], state[4]).  The round constants and MDS are the VM's own __constant__ tables (vm.cu, vm_upload_constants).
extern __constant__ fe c_vm_hasher_ark[192];
extern __constant__ fe c_vm_hasher_mds[36];

__device__ __forceinline__ void alg_mds6(fe st[6], const fe *m) {
    fe r[6];
#pragma unroll
    for (int i = 0; i < 6; i++) {
        fe acc = fe_mul(m[i * 6], st[0]);
#pragma unroll
        for (int j = 1; j < 6; j++) acc = fe_add(acc, fe_mul(m[i * 6 + j], st[j]));
        r[i] = acc;
    }
#pragma unroll
    for (int i = 0; i < 6; i++) st[i] = r[i];
}

// wide layout: one thread per message, the round of vm.cu's hasher_round with its six inverse S-boxes one after another
__global__ void __launch_bounds__(128) hasher_digest_kernel(const fe *__restrict__ in, fe *__restrict__ out, unsigned long long n) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe s[6];
    s[0] = fe_make(0, 0); s[1] = fe_make(0, 0);
#pragma unroll
    for (int q = 0; q < 4; q++) s[5 - q] = in[4 * i + q];
#pragma unroll 1
    for (int r = 0; r < 10; r++) {
#pragma unroll
        for (int j = 0; j < 6; j++) s[j] = fe_cube(fe_add(s[j], c_vm_hasher_ark[j * 16 + r]));
        alg_mds6(s, c_vm_hasher_mds);
#pragma unroll
        for (int j = 0; j < 6; j++) s[j] = alg_inv_sbox(fe_add(s[j], c_vm_hasher_ark[(6 + j) * 16 + r]));
        alg_mds6(s, c_vm_hasher_mds);
    }
    out[2 * i] = s[5];
    out[2 * i + 1] = s[4];
}

// narrow layout: 8 lanes per message, lane e < 6 holding state element e (lanes 6 and 7 repeat lane 5), so the six inverse S-boxes of a
// round run side by side; the MDS gathers the state by shuffles within the 8 lanes.  A message's latency is one S-box chain per round
// instead of six, which is what the narrow levels of a tree, too few digests to fill the GPU, are bound by.
__device__ __forceinline__ fe hasher_lanes_mds(fe s, unsigned e) {
    fe acc = fe_make(0, 0);
#pragma unroll
    for (int j = 0; j < 6; j++) {
        fe t;
        t.lo = __shfl_sync(0xffffffffu, s.lo, j, 8);
        t.hi = __shfl_sync(0xffffffffu, s.hi, j, 8);
        acc = j == 0 ? fe_mul(c_vm_hasher_mds[e * 6], t) : fe_add(acc, fe_mul(c_vm_hasher_mds[e * 6 + j], t));
    }
    return acc;
}
__global__ void __launch_bounds__(128) hasher_digest_lanes_kernel(const fe *__restrict__ in, fe *__restrict__ out, unsigned long long n) {
    const unsigned long long g = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const unsigned long long i = g < n ? g : n - 1;         // the spare groups of the last warp repeat the last message: every lane shuffles
    const unsigned k = threadIdx.x & 7u, e = k < 5u ? k : 5u;
    fe s = e >= 2 ? in[4 * i + 5 - e] : fe_make(0, 0);
#pragma unroll 1
    for (int r = 0; r < 10; r++) {
        s = hasher_lanes_mds(fe_cube(fe_add(s, c_vm_hasher_ark[e * 16 + r])), e);
        s = hasher_lanes_mds(alg_inv_sbox(fe_add(s, c_vm_hasher_ark[(6 + e) * 16 + r])), e);
    }
    if (g < n && (k == 4 || k == 5)) out[2 * i + 5 - k] = s;
}

static void hasher_digest_wide(Context &c, const void *in, void *out, unsigned long long n) {
    if (n == 0) return;
    vm_upload_constants(c);
    hasher_digest_kernel<<<(unsigned)((n + 127) / 128), 128, 0, c.stream>>>((const fe *)in, (fe *)out, n);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}
static void hasher_digest_narrow(Context &c, const void *in, void *out, unsigned long long n) {
    if (n == 0) return;
    vm_upload_constants(c);
    hasher_digest_lanes_kernel<<<(unsigned)((8 * n + 127) / 128), 128, 0, c.stream>>>((const fe *)in, (fe *)out, n);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}
void hasher_digest(Context &c, const void *in, void *out, unsigned long long n) {
    if (n < HASHER_WIDE_MIN) hasher_digest_narrow(c, in, out, n);
    else hasher_digest_wide(c, in, out, n);
}

}  // namespace dg
