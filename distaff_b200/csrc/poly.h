// Polynomial / scan / gather kernels (poly.cu) and FRI kernels (fri.cu).
#pragma once
#include <array>
#include "common.cuh"

namespace dg {

// two-level table of powers of an arbitrary base: base^e = lo[e & (2^lo_bits - 1)] * hi[e >> lo_bits],  e < len
struct PowRef { const fe *lo, *hi; int lo_bits; };
// `batch` tables of one length in one launch: table q from the device pair base_step[2q] = base, base_step[2q + 1] = step(base, len)
struct PowTables {
    DevBuf lo, hi;
    int lo_bits = 0;
    unsigned long long lo_n = 0, hi_n = 0;
    PowTables(Context &c, const fe *base_step, int batch, unsigned long long len);
    static fe step(fe base, unsigned long long len);          // the second entry of a table's pair
    // the pairs of the tables of x and of 1 / x, both of length len, at pairs[0..2) and pairs[inv_at .. inv_at + 2)
    static void pack_point(fe *pairs, size_t inv_at, fe x, unsigned long long len);
    static unsigned long long entries(unsigned long long len);   // lo_n + hi_n of one table
    PowRef ref(int q) const { PowRef r; r.lo = lo.as<fe>() + q * lo_n; r.hi = hi.as<fe>() + q * hi_n; r.lo_bits = lo_bits; return r; }
};

// synthetic division of `batch` vectors in one launch: vector q reads in + q in_stride, writes out + q out_stride, uses the power tables
// moved by q * (lo, hi) strides and subtracts sub0[q] (device) from its constant coefficient
void syn_div(Context &c, int batch, const fe *in, unsigned long long in_stride, fe *out, unsigned long long out_stride, unsigned long long len,
             const PowRef &b_pows, unsigned long long b_lo_stride, unsigned long long b_hi_stride, const PowRef &binv_pows,
             unsigned long long binv_lo_stride, unsigned long long binv_hi_stride, const fe *sub0);
// batch > 1: a, add0, add1 of vector q at q * in_stride, out at q * out_stride; scratch holds batch * len elements
void syn_div_expanded_sum(Context &c, const fe *a, fe *scratch, const fe *add0, const fe *add1, fe *out, unsigned long long n, unsigned long long len, fe e,
                          int batch = 1, unsigned long long in_stride = 0, unsigned long long out_stride = 0);
// cols_per_proof < cols: the columns of several proofs, proof q's powers of z at zt moved by q * (lo, hi) strides; col_proof (device, one
// entry per column, may be null) names each column's proof instead, for proofs of several widths
void eval_polys_at(Context &c, const fe *polys, unsigned long long n, int cols, const PowRef &zt, const TwiddleRef &gt, bool two_points, fe *out,
                   int cols_per_proof = 1 << 30, unsigned long long zt_stride_lo = 0, unsigned long long zt_stride_hi = 0,
                   const unsigned *col_proof = nullptr);
// one opened row computed from the trace polynomials: the w columns from column `col` on, at LDE position pos (out: set by eval_trace_rows)
struct TraceRow { unsigned long long pos, out; unsigned col, w; };
// rows of the trace extension computed from the trace polynomials (column stride n): point m's values P_j(w_N^pos), j < w, at out + the
// widths of the points before it; one launch for all points (plus the reduction of the tile sums)
void eval_trace_rows(Context &c, const fe *polys, unsigned long long n, std::vector<TraceRow> points, int log_N, fe *out);
// `batch` proofs: polys, coef, ic / fc of proof q at q * the strides, its constants KiA, KiB, KfA, KfB = K[4q .. 4q + 4) on the device.
// cols (device, may be null): proofs of several widths, proof q's polynomials the cols[q].y columns from column cols[q].x on
void boundary_coeffs(Context &c, int batch, const fe *polys, unsigned long long poly_stride, unsigned long long n, int nb, const fe *coef,
                     unsigned long long coef_stride, const fe *K, fe *ic, fe *fc, unsigned long long out_stride, const uint2 *cols = nullptr);
// finishes the coset-by-coset interpolation of 8n evaluations: b = [8][n] size-n inverse transforms of the cosets -> 8n coefficients;
// batch > 1: vector q at b + q b_stride, out + q out_stride
void coset_interp_finish(Context &c, const fe *b, fe *out, int log_n, int batch = 1, unsigned long long b_stride = 0, unsigned long long out_stride = 0);
// batch > 1: proof q's polynomials w n elements after proof q - 1's (or, with cols, the cols[q].y columns from column cols[q].x on), its
// coefficients at q cc_stride, outputs at q t_stride
void lincomb2(Context &c, const fe *polys, unsigned long long n, int w, const fe *cc1, const fe *cc2, fe *t1, fe *t2, int batch = 1,
              unsigned long long cc_stride = 0, unsigned long long t_stride = 0, const uint2 *cols = nullptr);
// `batch` proofs: t1q / t2q at q t_stride, cq / comp at q len, k1, k2, kc = ks[3q .. 3q + 3) on the device
void compose(Context &c, int batch, const fe *t1q, const fe *t2q, unsigned long long t_stride, const fe *cq, fe *comp, unsigned long long n,
             unsigned long long len, unsigned long long inc, const fe *ks);

// ---- hashing (hash.cu) ----
// ext: the cosets [c0, c0 + nc) of every column ([w][nc][n], column stride nc n; nc = 0: all 2^log_blowup); the row of coset c at step k
// is leaf (k << log_blowup) + c.  batch > 1: `batch` matrices ext_stride elements apart, their leaves leaf_stride digests apart (0: N);
// cols (device, may be null): matrices of several widths, matrix q the cols[q].y columns from column cols[q].x on (w, ext_stride unused)
void hash_trace_rows(Context &c, const fe *ext, void *leaves, int w, int log_n, int log_blowup, int batch = 1, unsigned long long ext_stride = 0,
                     unsigned c0 = 0, unsigned nc = 0, unsigned long long leaf_stride = 0, const uint2 *cols = nullptr);
// digests of the rows of a plain column-major [w][rows] matrix
void hash_rows_plain(Context &c, const fe *cols, void *digests, int w, unsigned long long rows);
void hash64_contiguous(Context &c, const void *in, void *out, unsigned long long count);
// `batch` trees of L leaves (L a power of two >= 2): tree q's leaves and nodes q * L digests after tree 0's
void merkle_build(Context &c, const void *leaves, void *nodes, unsigned long long L, int batch = 1);
// levels of a heap-layout tree from L/2 nodes down to (and including) the level with `stop` nodes
void merkle_levels_down_to(Context &c, const void *leaves, void *nodes, unsigned long long L, unsigned long long stop);
void merkle_finish(Context &c, void *nodes, unsigned long long m);     // level with m nodes already at nodes[m..2m)
// alghash.cu: blake3 / rescue / poseidon / the VM's hasher over 64-byte messages, and Merkle trees with them
void alg_hash64(Context &c, int hash_id, const void *in, void *out, unsigned long long n);
// hasher::digest of n messages of 4 elements (64 bytes) into 2 elements (32 bytes) each: fewer than HASHER_WIDE_MIN messages run the
// narrow layout (8 lanes per message), more the wide one (a thread per message)
constexpr unsigned long long HASHER_WIDE_MIN = 1ULL << 16;     // measured crossover on an H100 (DESIGN.md section 7j)
void hasher_digest(Context &c, const void *in, void *out, unsigned long long n);
void alg_merkle_build(Context &c, int hash_id, const void *leaves, void *nodes, unsigned long long L);
// the smallest proof-of-work nonce >= 1 of every seed for its own grinding factor (grinding[i] of seeds[i]), one kernel per round for
// all of them; result i belongs to seeds[i]
std::vector<unsigned long long> pow_search_batch(Context &c, const std::vector<std::array<uint8_t, 32>> &seeds, const std::vector<unsigned> &grinding);
void pow_hash(const uint8_t seed[32], unsigned long long nonce, uint8_t out[32]);

// ---- FRI (fri.cu) ----
// storage layout of a vector of D = 2^log_d evaluations: natural (log_b < 0) or coset-major with 2^log_b cosets:
// logical index i = (k << log_b) + c  lives at  (c << (log_d - log_b)) + k
struct Layout {
    int log_d, log_b;
    __host__ __device__ unsigned long long phys(unsigned long long i) const {
        if (log_b < 0) return i;
        return ((i & ((1ULL << log_b) - 1ULL)) << (log_d - log_b)) + (i >> log_b);
    }
    __host__ __device__ unsigned long long logical(unsigned long long p) const {
        if (log_b < 0) return p;
        const int log_k = log_d - log_b;
        return ((p & ((1ULL << log_k) - 1ULL)) << log_b) + (p >> log_k);
    }
};
// leaves[r] = blake3(v[r], v[r+R], v[r+2R], v[r+3R]),  R = D/4   (fri/prover.rs:16-17, fri/utils.rs:16-21)
// batch > 1: `batch` layers values_stride elements apart, leaves R = D/4 digests apart
void fri_hash_rows(Context &c, const fe *values, Layout in, Layout rows, void *leaves, int batch = 1, unsigned long long values_stride = 0);
// next[r] = f_r(alpha), f_r = cubic through (x_r t^j, v[r + jR])   (fri/prover.rs:26-32, quartic.rs:20-135)
// alpha: device pointer (derived on the device by fri_alpha, or uploaded by the host when RNG callbacks are registered)
// batch > 1: `batch` layers values_stride elements apart, next R elements apart, folding point alpha[q] for layer q
void fri_fold(Context &c, const fe *values, Layout in, fe *next, Layout out, const fe *alpha, const TwiddleRef &inv_root_table, int log_n_total,
              fe tau_inv, fe inv4, int batch = 1, unsigned long long values_stride = 0);
// the layout of the layer that folding a layer of layout `in` produces (the layout of its row hashes): D / 4 values, coset-major while
// at least 2^log_b of them remain, natural below
Layout fri_next_layout(Layout in);
// what fri_fold and fri_fold_local take besides the layer: 1 / tau (tau the 4th root of unity) and 1 / 4
struct FoldConstants { fe tau_inv, inv4; };
FoldConstants fri_fold_constants();
// alpha_dev[0] = field::prng(root) (fri/prover.rs:29); root_copy_dev receives the 32 root bytes (collected for one host copy at the end)
// batch > 1: the roots root_stride_bytes apart -> alpha_dev[q], root_copy_dev + 32 q
void fri_alpha(Context &c, const void *root_dev, fe *alpha_dev, void *root_copy_dev, int batch = 1, unsigned long long root_stride_bytes = 0);
// coset-sharded variants (a rank holds cosets [c0, c0 + 2^log_nc) of the layer as [c - c0][k]); items in ShardedTree order [k'][c - c0]
void fri_hash_rows_local(Context &c, const fe *values_local, int log_d, int log_b, int log_nc, void *items_local);
void fri_fold_local(Context &c, const fe *values_local, int log_d, int log_b, int log_nc, unsigned c0, fe *next_local, const fe *alpha,
                    const TwiddleRef &inv_root_table, int log_n_total, fe tau_inv, fe inv4);

}  // namespace dg
