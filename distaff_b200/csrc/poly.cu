// Polynomial kernels of the prove pipeline (coefficient-domain steps 4 and 6 of /root/reference/src/stark/prover.rs):
//   polynom::syn_div_in_place            /root/reference/src/math/polynom.rs:190-197   -> weighted suffix scan
//   polynom::syn_div_expanded_in_place   /root/reference/src/math/polynom.rs:202-236   -> strided suffix sums + 2-tap stencil
//   polynom::eval (Horner)               /root/reference/src/math/polynom.rs:9-17       -> dot product with a power table
//   parallel::mul_acc / add_in_place     /root/reference/src/math/parallel.rs           -> fused element-wise kernels
//
// The sequential recurrences of the reference are re-expressed as parallel scans.  With q[i] = sum_{j>i} a[j] b^(j-i-1)
// (exactly what the synthetic-division loop leaves in a[i], remainder dropped) one has
//      q[i] = b^-(i+1) * sum_{j>i} a[j] b^j
// i.e. an element-wise scaling, a plain (addition-only) exclusive suffix sum, and another scaling.  Field arithmetic is
// exact, so the coefficients are identical to the reference's.
#include "poly.h"

namespace dg {

__device__ __forceinline__ fe pw(const PowRef &t, unsigned long long e) {
    return fe_mul(t.lo[e & ((1ULL << t.lo_bits) - 1ULL)], t.hi[e >> t.lo_bits]);
}

// table q = blockIdx.y: (base, step) = bs[2q], bs[2q + 1], written to lo + q lo_n and hi + q hi_n
__global__ void pow_fill_batch_kernel(fe *lo, unsigned long long lo_n, fe *hi, unsigned long long hi_n, const fe *__restrict__ bs) {
    const fe base = bs[2 * blockIdx.y], step = bs[2 * blockIdx.y + 1];
    lo += blockIdx.y * lo_n;
    hi += blockIdx.y * hi_n;
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < lo_n) lo[i] = fe_pow_u64(base, i);
    else if (i < lo_n + hi_n) hi[i - lo_n] = fe_pow_u64(step, i - lo_n);
}

static int pow_lo_bits(unsigned long long len) {
    int lo_bits = 1;
    while ((1ULL << (2 * lo_bits)) < len) lo_bits++;
    return lo_bits;
}
static unsigned long long pow_hi_n(unsigned long long len) {
    const unsigned long long lo_n = 1ULL << pow_lo_bits(len);
    return (len + lo_n - 1) / lo_n + 1;
}

fe PowTables::step(fe base, unsigned long long len) { return fe_pow_u64(base, 1ULL << pow_lo_bits(len)); }
void PowTables::pack_point(fe *pairs, size_t inv_at, fe x, unsigned long long len) {
    const fe xi = host_inv(x);
    pairs[0] = x;
    pairs[1] = step(x, len);
    pairs[inv_at] = xi;
    pairs[inv_at + 1] = step(xi, len);
}
unsigned long long PowTables::entries(unsigned long long len) { return (1ULL << pow_lo_bits(len)) + pow_hi_n(len); }

PowTables::PowTables(Context &c, const fe *base_step, int batch, unsigned long long len) {
    DG_REQUIRE(batch >= 1 && batch <= 65535, "power table batch out of range");
    lo_bits = pow_lo_bits(len);
    lo_n = 1ULL << lo_bits;
    hi_n = pow_hi_n(len);
    lo.alloc(lo_n * batch * sizeof(fe));
    hi.alloc(hi_n * batch * sizeof(fe));
    pow_fill_batch_kernel<<<dim3((unsigned)((lo_n + hi_n + 127) / 128), (unsigned)batch), 128, 0, c.stream>>>(lo.as<fe>(), lo_n, hi.as<fe>(), hi_n, base_step);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

// ---- exclusive suffix sum (plain additions) -----------------------------------------------------------------------------------------
static const int SCAN_THREADS = 256, SCAN_PER_THREAD = 4, SCAN_BLOCK = SCAN_THREADS * SCAN_PER_THREAD;

__device__ __forceinline__ fe shfl_down_fe(fe v, int d) {
    fe r;
    r.lo = __shfl_down_sync(0xffffffffu, v.lo, d);
    r.hi = __shfl_down_sync(0xffffffffu, v.hi, d);
    return r;
}

// block-wide inclusive suffix sum of one value per thread; returns (inclusive suffix over threads >= tid); total in *block_total
__device__ __forceinline__ fe block_suffix_inclusive(fe v, fe *s_warp, fe *block_total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        fe o = shfl_down_fe(v, d);
        if (lane + d < 32) v = fe_add(v, o);
    }
    if (lane == 0) s_warp[warp] = v;
    __syncthreads();
    fe above = fe_make(0, 0);
    for (int w2 = warp + 1; w2 < nwarps; w2++) above = fe_add(above, s_warp[w2]);
    if (block_total) {
        fe tot = fe_make(0, 0);
        for (int w2 = 0; w2 < nwarps; w2++) tot = fe_add(tot, s_warp[w2]);
        *block_total = tot;
    }
    __syncthreads();
    return fe_add(v, above);
}

// ---- synthetic division by (x - b) ----------------------------------------------------------------------------------------------------
// Single-pass form (decoupled look-back, "chained scan"): one kernel reads every coefficient once and writes every quotient once.
// Blocks take tickets in launch order and work from the top of the vector downwards; a block publishes the sum of its scaled
// coefficients, then its first warp walks the descriptors of the blocks above it (32 at a time) until it meets one whose inclusive
// suffix is known.  One launch, where scale + block sums + recursive scan + apply + scale take 7-9 launches and ~9 passes over the vector.
struct __align__(16) ScanDesc { fe agg; fe incl; int status; int pad[3]; };     // status: 0 nothing, 1 aggregate published, 2 inclusive suffix published

__device__ __forceinline__ fe ld_cg_fe(const fe *p) {
    uint4 v = __ldcg(reinterpret_cast<const uint4 *>(p));
    fe r; r.lo = ((unsigned long long)v.y << 32) | v.x; r.hi = ((unsigned long long)v.w << 32) | v.z;
    return r;
}
__device__ __forceinline__ void st_cg_fe(fe *p, fe v) {
    __stcg(reinterpret_cast<uint4 *>(p), make_uint4((unsigned)v.lo, (unsigned)(v.lo >> 32), (unsigned)v.hi, (unsigned)(v.hi >> 32)));
}

// `batch` vectors in one launch (SynDivBatch strides); one ticket counter over all their blocks, ticket t = (vector t / nblocks,
// block nblocks - 1 - t % nblocks): a block only waits on blocks of its own vector with smaller tickets, so the look-back keeps its
// forward-progress guarantee.
struct SynDivBatch { unsigned long long in_stride, out_stride, b_stride_lo, b_stride_hi, binv_stride_lo, binv_stride_hi; const fe *sub0; };
__global__ void __launch_bounds__(SCAN_THREADS) syn_div_chained_kernel(const fe *__restrict__ in, fe *__restrict__ out, unsigned long long len, PowRef bp,
                                                                       PowRef binvp, ScanDesc *desc, unsigned *ticket, unsigned nblocks, SynDivBatch sb) {
    __shared__ fe s_warp[SCAN_THREADS / 32];
    __shared__ fe s_carry;
    __shared__ unsigned s_ticket;
    if (threadIdx.x == 0) s_ticket = atomicAdd(ticket, 1u);
    __syncthreads();
    unsigned t = s_ticket;
    const unsigned q = t / nblocks;
    t -= q * nblocks;
    in += q * sb.in_stride; out += q * sb.out_stride;
    bp.lo += q * sb.b_stride_lo; bp.hi += q * sb.b_stride_hi;
    binvp.lo += q * sb.binv_stride_lo; binvp.hi += q * sb.binv_stride_hi;
    const fe sub0 = sb.sub0[q];
    desc += (unsigned long long)q * nblocks;
    const unsigned blk = nblocks - 1u - t;
    const unsigned long long base = (unsigned long long)blk * SCAN_BLOCK + (unsigned long long)threadIdx.x * SCAN_PER_THREAD;
    fe x[SCAN_PER_THREAD];
    fe v = fe_make(0, 0);
#pragma unroll
    for (int u = 0; u < SCAN_PER_THREAD; u++) {
        const unsigned long long i = base + u;
        x[u] = fe_make(0, 0);
        if (i < len) {
            fe a = in[i];
            if (i == 0) a = fe_sub(a, sub0);
            x[u] = fe_mul(a, pw(bp, i));
        }
        v = fe_add(v, x[u]);
    }
    fe total;
    const fe incl = block_suffix_inclusive(v, s_warp, &total);
    if (threadIdx.x < 32) {
        const unsigned lane = threadIdx.x;
        ScanDesc *me = desc + blk;
        fe carry = fe_make(0, 0);
        if (blk == nblocks - 1u) {
            if (lane == 0) { st_cg_fe(&me->incl, total); __threadfence(); *(volatile int *)&me->status = 2; }
        } else {
            if (lane == 0) { st_cg_fe(&me->agg, total); __threadfence(); *(volatile int *)&me->status = 1; }
            for (unsigned first = blk + 1u;; first += 32u) {
                const unsigned b2 = first + lane;
                int st = 2;
                fe val = fe_make(0, 0);
                if (b2 < nblocks) {
                    const ScanDesc *d = desc + b2;
                    do { st = *(const volatile int *)&d->status; } while (st == 0);
                    __threadfence();
                    val = ld_cg_fe(st == 2 ? &d->incl : &d->agg);
                }
                const unsigned done = __ballot_sync(0xffffffffu, st == 2);
                const unsigned upto = done ? (unsigned)(__ffs((int)done) - 1) : 31u;         // first lane with a complete suffix
                if (lane > upto) val = fe_make(0, 0);
#pragma unroll
                for (int dd = 16; dd >= 1; dd >>= 1) val = fe_add(val, shfl_down_fe(val, dd));
                val.lo = __shfl_sync(0xffffffffu, val.lo, 0); val.hi = __shfl_sync(0xffffffffu, val.hi, 0);
                carry = fe_add(carry, val);
                if (done) break;
            }
            if (lane == 0) { st_cg_fe(&me->incl, fe_add(total, carry)); __threadfence(); *(volatile int *)&me->status = 2; }
        }
        if (lane == 0) s_carry = carry;
    }
    __syncthreads();
    fe run = fe_add(fe_sub(incl, v), s_carry);               // everything strictly above this thread's elements
#pragma unroll
    for (int u = SCAN_PER_THREAD - 1; u >= 0; u--) {
        const unsigned long long i = base + u;
        if (i < len) out[i] = fe_mul(run, pw(binvp, i + 1));
        run = fe_add(run, x[u]);
    }
}

// out[i] = sum_{j>i} (in[j] - [j==0] sub0) b^(j-i-1) for each vector.  in may equal out.
void syn_div(Context &c, int batch, const fe *in, unsigned long long in_stride, fe *out, unsigned long long out_stride, unsigned long long len,
             const PowRef &b_pows, unsigned long long b_lo_stride, unsigned long long b_hi_stride, const PowRef &binv_pows,
             unsigned long long binv_lo_stride, unsigned long long binv_hi_stride, const fe *sub0) {
    const unsigned long long nblk = (len + SCAN_BLOCK - 1) / SCAN_BLOCK;
    DG_REQUIRE(nblk * batch < (1ULL << 31), "division batch too large for one launch");
    DevBuf d((size_t)nblk * batch * sizeof(ScanDesc) + 16);
    DG_CUDA(cudaMemsetAsync(d.p, 0, d.bytes, c.stream));
    ScanDesc *desc = d.as<ScanDesc>();
    unsigned *ticket = reinterpret_cast<unsigned *>(desc + nblk * batch);
    const SynDivBatch sb{in_stride, out_stride, b_lo_stride, b_hi_stride, binv_lo_stride, binv_hi_stride, sub0};
    syn_div_chained_kernel<<<(unsigned)(nblk * batch), SCAN_THREADS, 0, c.stream>>>(in, out, len, b_pows, binv_pows, desc, ticket, (unsigned)nblk, sb);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

// ---- division by (x^n - 1) / (x - e) -----------------------------------------------------------------------------------------------------
// s[i + m n] = sum_{m' >= m} a[i + m' n]
// blockIdx.y = vector of a batch, a_stride / s_stride elements apart
__global__ void strided_suffix_kernel(const fe *__restrict__ a, fe *__restrict__ s, unsigned long long n, int blocks_m, unsigned long long a_stride,
                                      unsigned long long s_stride) {
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    a += blockIdx.y * a_stride;
    s += blockIdx.y * s_stride;
    fe run = fe_make(0, 0);
    for (int m = blocks_m - 1; m >= 0; m--) {
        run = fe_add(run, a[i + (unsigned long long)m * n]);
        s[i + (unsigned long long)m * n] = run;
    }
}
// out[idx] = s[idx+n-1] - e * s[idx+n]  for idx <= len-n (with s[len] = 0), else 0 ; optionally accumulated: out = base0 + base1 + that
// blockIdx.y = vector of a batch: s at s_stride, add0 / add1 at in_stride, out at out_stride elements apart
__global__ void expanded_stencil_kernel(const fe *__restrict__ s, const fe *__restrict__ add0, const fe *__restrict__ add1, fe *__restrict__ out,
                                        unsigned long long n, unsigned long long len, fe e, unsigned long long s_stride, unsigned long long in_stride,
                                        unsigned long long out_stride) {
    unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= len) return;
    s += blockIdx.y * s_stride;
    if (add0) add0 += blockIdx.y * in_stride;
    if (add1) add1 += blockIdx.y * in_stride;
    out += blockIdx.y * out_stride;
    fe v = fe_make(0, 0);
    if (idx <= len - n) {
        v = s[idx + n - 1];
        if (idx + n < len) v = fe_sub(v, fe_mul(e, s[idx + n]));
    }
    if (add0) v = fe_add(v, add0[idx]);
    if (add1) v = fe_add(v, add1[idx]);
    out[idx] = v;
}
void syn_div_expanded_sum(Context &c, const fe *a, fe *scratch, const fe *add0, const fe *add1, fe *out, unsigned long long n, unsigned long long len, fe e,
                          int batch, unsigned long long in_stride, unsigned long long out_stride) {
    DG_REQUIRE(batch >= 1 && batch <= 65535, "division batch out of range");
    strided_suffix_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)batch), 256, 0, c.stream>>>(a, scratch, n, (int)(len / n), in_stride, len);
    c.launches++;
    expanded_stencil_kernel<<<dim3((unsigned)((len + 255) / 256), (unsigned)batch), 256, 0, c.stream>>>(scratch, add0, add1, out, n, len, e, len, in_stride,
                                                                                                        out_stride);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

// ---- evaluation of many polynomials at two points (DEEP values) -----------------------------------------------------------------------------
// partial[(col*2 + p) * chunks + chunk] = sum_{k in chunk} poly[col][k] * x_p^k,  x_0 = z (table zt), x_1 = z*g (zt * gt)
static const int EVAL_CHUNK = 4096;
// columns of a batch: column col uses the table of its proof col / cols_per_proof, or col_proof[col] (a batch of several widths),
// zt_stride_lo / zt_stride_hi elements apart
__global__ void __launch_bounds__(256) eval2_partial_kernel(const fe *__restrict__ polys, unsigned long long n, PowRef zt, TwiddleRef gt, fe *__restrict__ partial,
                                                            int two_points, unsigned cols_per_proof, unsigned long long zt_stride_lo,
                                                            unsigned long long zt_stride_hi, const unsigned *__restrict__ col_proof) {
    __shared__ fe s_warp[2][8];
    const unsigned long long col = blockIdx.y, chunk = blockIdx.x, chunks = gridDim.x;
    const fe *p = polys + col * n;
    const unsigned q = col_proof ? col_proof[blockIdx.y] : blockIdx.y / cols_per_proof;
    zt.lo += q * zt_stride_lo;
    zt.hi += q * zt_stride_hi;
    fe a0 = fe_make(0, 0), a1 = fe_make(0, 0);
    for (int u = 0; u < EVAL_CHUNK / 256; u++) {
        unsigned long long k = chunk * EVAL_CHUNK + (unsigned long long)u * 256 + threadIdx.x;
        if (k < n) {
            fe v = p[k];
            fe zk = pw(zt, k);
            fe t = fe_mul(v, zk);
            a0 = fe_add(a0, t);
            if (two_points) {
                unsigned ee = (unsigned)k & gt.mask;
                fe gk = fe_mul(gt.lo[ee & ((1u << gt.lo_bits) - 1u)], gt.hi[ee >> gt.lo_bits]);
                a1 = fe_add(a1, fe_mul(t, gk));
            }
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) { a0 = fe_add(a0, shfl_down_fe(a0, d)); a1 = fe_add(a1, shfl_down_fe(a1, d)); }
    if (lane == 0) { s_warp[0][warp] = a0; s_warp[1][warp] = a1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        fe t0 = fe_make(0, 0), t1 = fe_make(0, 0);
        for (int w2 = 0; w2 < 8; w2++) { t0 = fe_add(t0, s_warp[0][w2]); t1 = fe_add(t1, s_warp[1][w2]); }
        partial[(col * 2 + 0) * chunks + chunk] = t0;
        partial[(col * 2 + 1) * chunks + chunk] = t1;
    }
}
__global__ void reduce_partials_kernel(const fe *__restrict__ partial, fe *__restrict__ out, unsigned long long chunks) {
    // one block of 32 threads per output
    const unsigned long long o = blockIdx.x;
    fe a = fe_make(0, 0);
    for (unsigned long long i = threadIdx.x; i < chunks; i += 32) a = fe_add(a, partial[o * chunks + i]);
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) a = fe_add(a, shfl_down_fe(a, d));
    if (threadIdx.x == 0) out[o] = a;
}
// out[col*2 + p] = poly_col(x_p)
void eval_polys_at(Context &c, const fe *polys, unsigned long long n, int cols, const PowRef &zt, const TwiddleRef &gt, bool two_points, fe *out,
                   int cols_per_proof, unsigned long long zt_stride_lo, unsigned long long zt_stride_hi, const unsigned *col_proof) {
    const unsigned chunks = (unsigned)((n + EVAL_CHUNK - 1) / EVAL_CHUNK);
    DG_REQUIRE(cols >= 1 && cols <= 65535 && cols_per_proof >= 1, "too many polynomials for one launch");
    DevBuf partial((size_t)cols * 2 * chunks * sizeof(fe));
    eval2_partial_kernel<<<dim3(chunks, cols), 256, 0, c.stream>>>(polys, n, zt, gt, partial.as<fe>(), two_points ? 1 : 0, (unsigned)cols_per_proof,
                                                                   zt_stride_lo, zt_stride_hi, col_proof); c.launches++;
    reduce_partials_kernel<<<cols * 2, 32, 0, c.stream>>>(partial.as<fe>(), out, chunks); c.launches++;
    DG_CUDA(cudaGetLastError());
}

// ---- trace rows at LDE positions (openings outside the retained cosets) -------------------------------------------------------------------
// Row `pos` of the trace extension is (P_0(x), ..., P_{w-1}(x)) at x = w_N^pos.  Block (m, y) evaluates the w columns of point m's proof
// on the tiles y, y + gridDim.y, ... of ROW_TILE coefficients: the tile's powers x^k = w_N^(pos k mod N) go to shared memory once (two-level
// table, one product each) and are shared by all w columns; warp v sums columns v, v + 8, ..., each lane ROW_TILE / 32 = 64 products
// accumulated unreduced (288 bits, < 128 products) and reduced once, then the warp's lanes are added into the column's shared sum.
// partial[(out + j) * gridDim.y + y] = the block's sum for column j, out = point m's first output (the widths of the points before it).
static const int ROW_TILE = 2048, ROW_MAX_BLOCKS = 64;
__global__ void __launch_bounds__(256) eval_rows_partial_kernel(const fe *__restrict__ polys, unsigned long long n, const TraceRow *__restrict__ pts,
                                                                TwiddleRef twN, fe *__restrict__ partial) {
    __shared__ fe s_pw[ROW_TILE];
    __shared__ fe s_acc[128];
    const TraceRow pt = pts[blockIdx.x];
    const int w = (int)pt.w;
    const fe *p = polys + (unsigned long long)pt.col * n;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j = threadIdx.x; j < w; j += blockDim.x) s_acc[j] = fe_make(0, 0);
    const unsigned long long tile = n < (unsigned long long)ROW_TILE ? n : (unsigned long long)ROW_TILE;
    for (unsigned long long k0 = (unsigned long long)blockIdx.y * tile; k0 < n; k0 += (unsigned long long)gridDim.y * tile) {
        __syncthreads();                                             // the previous tile's powers are no longer read
        for (unsigned i = threadIdx.x; i < tile; i += blockDim.x) {
            const unsigned e = (unsigned)((pt.pos * (k0 + i)) & twN.mask);
            s_pw[i] = fe_mul(twN.lo[e & ((1u << twN.lo_bits) - 1u)], twN.hi[e >> twN.lo_bits]);
        }
        __syncthreads();
        for (int j = warp; j < w; j += 8) {
            const fe *col = p + (unsigned long long)j * n + k0;
            fe v = fe_make(0, 0);
            if (lane < tile) {
                fe_wide acc;
                wide_set(acc, DG_MUL_WIDE(col[lane], s_pw[lane]));
                for (unsigned i = lane + 32; i < tile; i += 32) wide_add(acc, DG_MUL_WIDE(col[i], s_pw[i]));
                v = DG_REDUCE_WIDE(acc);
            }
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) v = fe_add(v, shfl_down_fe(v, d));
            if (lane == 0) s_acc[j] = fe_add(s_acc[j], v);
        }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < w; j += blockDim.x) partial[(pt.out + j) * gridDim.y + blockIdx.y] = s_acc[j];
}
void eval_trace_rows(Context &c, const fe *polys, unsigned long long n, std::vector<TraceRow> points, int log_N, fe *out) {
    DG_REQUIRE(!points.empty() && points.size() < (1ULL << 31), "opened-row evaluation out of range");
    unsigned long long values = 0;
    for (TraceRow &pt : points) {
        DG_REQUIRE(pt.w >= 1 && pt.w <= 128, "opened-row evaluation out of range");
        pt.out = values;
        values += pt.w;
    }
    DevBuf d_pts(points.size() * sizeof(TraceRow));
    DG_CUDA(cudaMemcpyAsync(d_pts.p, points.data(), d_pts.bytes, cudaMemcpyHostToDevice, c.stream));
    const unsigned tiles = (unsigned)((n + ROW_TILE - 1) / ROW_TILE), by = std::min<unsigned>(tiles, ROW_MAX_BLOCKS);
    DevBuf partial(values * by * sizeof(fe));
    // the points run on x, so the blocks of one tile and many points are resident together and share its coefficients through L2
    eval_rows_partial_kernel<<<dim3((unsigned)points.size(), by), 256, 0, c.stream>>>(polys, n, d_pts.as<TraceRow>(), c.twiddle(log_N, false),
                                                                                    partial.as<fe>()); c.launches++;
    reduce_partials_kernel<<<(unsigned)values, 32, 0, c.stream>>>(partial.as<fe>(), out, by); c.launches++;
    DG_CUDA(cudaGetLastError());
}

// ---- linear combinations ------------------------------------------------------------------------------------------------------------------
// t1[k] = sum_i cc1[i] P_i[k],  t2[k] = sum_i cc2[i] P_i[k]
// blockIdx.y = proof of a batch: polys w n, cc1 / cc2 cc_stride, t1 / t2 t_stride elements apart; with a column table, proof q's
// polynomials are the cols[q].y columns from column cols[q].x on
__global__ void lincomb2_kernel(const fe *__restrict__ polys, unsigned long long n, int w, const fe *__restrict__ cc1, const fe *__restrict__ cc2,
                                fe *__restrict__ t1, fe *__restrict__ t2, unsigned long long cc_stride, unsigned long long t_stride,
                                const uint2 *__restrict__ cols) {
    unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    if (cols) {
        const uint2 t = cols[blockIdx.y];
        polys += (unsigned long long)t.x * n;
        w = (int)t.y;
    } else {
        polys += blockIdx.y * (unsigned long long)w * n;
    }
    cc1 += blockIdx.y * cc_stride; cc2 += blockIdx.y * cc_stride;
    t1 += blockIdx.y * t_stride; t2 += blockIdx.y * t_stride;
    // w < 128 products per sum: accumulated unreduced (288 bits), one reduction each (fp128.cuh: fe_wide)
    fe_wide a, b;
    for (int i = 0; i < w; i++) {
        const fe v = polys[(unsigned long long)i * n + k];
        if (i == 0) { wide_set(a, DG_MUL_WIDE(v, cc1[0])); wide_set(b, DG_MUL_WIDE(v, cc2[0])); }
        else { wide_add(a, DG_MUL_WIDE(v, cc1[i])); wide_add(b, DG_MUL_WIDE(v, cc2[i])); }
    }
    t1[k] = DG_REDUCE_WIDE(a); t2[k] = DG_REDUCE_WIDE(b);
}
void lincomb2(Context &c, const fe *polys, unsigned long long n, int w, const fe *cc1, const fe *cc2, fe *t1, fe *t2, int batch,
              unsigned long long cc_stride, unsigned long long t_stride, const uint2 *cols) {
    DG_REQUIRE(batch >= 1 && batch <= 65535, "linear combination batch out of range");
    lincomb2_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)batch), 256, 0, c.stream>>>(polys, n, w, cc1, cc2, t1, t2, cc_stride, t_stride,
                                                                                             cols);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

// Boundary-constraint numerators in coefficient form.  The reference evaluates, at every point x of the 8n-point constraint domain,
//   I(x) = sum_j (T_j(x) - in_j) (a_j + b_j x^adj)            (evaluator.rs:181-326, adj = 6n + 2)
// and interpolates the evaluations afterwards (constraint_poly.rs).  I has degree n - 1 + adj < 8n, so the interpolant IS the polynomial
//   I = (sum_j a_j T_j - Ka) + x^adj (sum_j b_j T_j - Kb),     Ka = sum_j a_j in_j,  Kb = sum_j b_j in_j
// whose coefficients are two linear combinations of the trace polynomials' coefficients: n*nb multiplications instead of 8n*nb.
// coef = [a_init | b_init | a_final | b_final], nb entries each; ic / fc receive the 8n coefficients of the first / last step numerators.
// blockIdx.y = proof of a batch: polys poly_stride, coef coef_stride, ic / fc out_stride elements apart, its constants
// KiA, KiB, KfA, KfB = K[4 y .. 4 y + 4).  With a column table, proof q's polynomials are the cols[q].y columns from column cols[q].x on,
// and only the first min(nb, cols[q].y) coefficients of each vector are read: the vectors are padded with zeros to the batch's largest
// count nb, which a narrower proof's registers do not reach (a zero coefficient adds nothing to the unreduced sums)
__global__ void boundary_coeffs_kernel(const fe *__restrict__ polys, unsigned long long n, int nb, const fe *__restrict__ coef, unsigned long long adj,
                                       fe *__restrict__ ic, fe *__restrict__ fc, const fe *__restrict__ K, unsigned long long poly_stride,
                                       unsigned long long coef_stride, unsigned long long out_stride, const uint2 *__restrict__ cols) {
    const unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    int regs = nb;
    if (cols) {
        const uint2 t = cols[blockIdx.y];
        polys += (unsigned long long)t.x * n;
        regs = min(nb, (int)t.y);
    } else {
        polys += blockIdx.y * poly_stride;
    }
    coef += blockIdx.y * coef_stride;
    ic += blockIdx.y * out_stride; fc += blockIdx.y * out_stride;
    const fe KiA = K[4 * blockIdx.y], KiB = K[4 * blockIdx.y + 1], KfA = K[4 * blockIdx.y + 2], KfB = K[4 * blockIdx.y + 3];
    // nb < 128 products per sum: accumulated unreduced (288 bits), one reduction each
    fe_wide wa, wb, wc, wd;
    for (int j = 0; j < regs; j++) {
        const fe v = polys[(unsigned long long)j * n + k];
        if (j == 0) {
            wide_set(wa, DG_MUL_WIDE(v, coef[0])); wide_set(wb, DG_MUL_WIDE(v, coef[nb])); wide_set(wc, DG_MUL_WIDE(v, coef[2 * nb]));
            wide_set(wd, DG_MUL_WIDE(v, coef[3 * nb]));
        } else {
            wide_add(wa, DG_MUL_WIDE(v, coef[j])); wide_add(wb, DG_MUL_WIDE(v, coef[nb + j])); wide_add(wc, DG_MUL_WIDE(v, coef[2 * nb + j]));
            wide_add(wd, DG_MUL_WIDE(v, coef[3 * nb + j]));
        }
    }
    fe ia = DG_REDUCE_WIDE(wa), ib = DG_REDUCE_WIDE(wb), fa = DG_REDUCE_WIDE(wc), fb = DG_REDUCE_WIDE(wd);
    if (k == 0) { ia = fe_sub(ia, KiA); ib = fe_sub(ib, KiB); fa = fe_sub(fa, KfA); fb = fe_sub(fb, KfB); }
    const fe zero = fe_make(0, 0);
    ic[k] = ia; fc[k] = fa;
    ic[adj + k] = ib; fc[adj + k] = fb;
    // the gaps [n, adj) and [adj + n, 8n): 5n + 2 + (n - 2) = 6n entries, six per thread
    for (unsigned long long q = n + k; q < 8 * n; q += n)
        if (q < adj || q >= adj + n) { ic[q] = zero; fc[q] = zero; }
}
void boundary_coeffs(Context &c, int batch, const fe *polys, unsigned long long poly_stride, unsigned long long n, int nb, const fe *coef,
                     unsigned long long coef_stride, const fe *K, fe *ic, fe *fc, unsigned long long out_stride, const uint2 *cols) {
    DG_REQUIRE(batch >= 1 && batch <= 65535, "boundary batch out of range");
    boundary_coeffs_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)batch), 256, 0, c.stream>>>(polys, n, nb, coef, 6 * n + 2, ic, fc, K, poly_stride,
                                                                                                   coef_stride, out_stride, cols);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

// Interpolation of 8n evaluations given coset by coset (the constraint kernel's layout): e[8k + c] = P(w_E^(8k + c)), E = 8n.
// With m = m0 + n*m1:  e_c[k] = sum_m0 w_n^(k m0) * [ w_E^(c m0) * sum_m1 a[m0 + n m1] w_8^(c m1) ], so each coset is inverted by a size-n
// inverse transform (b_c = iNTT_n(e_c), done by the caller; it shards by coset), and this kernel finishes: for every m0 it undoes the
// factor w_E^(c m0) and runs the 8-point inverse DFT across the cosets.  Output: the 8n coefficients in natural order, exactly what
// interpolate_fft of the natural-order evaluation vector returns (constraint_table.rs:54-63) -- no transposition, no 8n-point transform.
// b: [8][n]; tw: powers of w_E^-1; w8i[j] = w_8^-j, j = 1..3; inv8 = 1/8.
// blockIdx.y = vector of a batch: b b_stride, out out_stride elements apart
__global__ void coset_interp_finish_kernel(const fe *__restrict__ b, fe *__restrict__ out, unsigned long long n, TwiddleRef tw, fe w8i1, fe w8i2, fe w8i3, fe inv8,
                                           unsigned long long b_stride, unsigned long long out_stride) {
    const unsigned long long m0 = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (m0 >= n) return;
    b += blockIdx.y * b_stride;
    out += blockIdx.y * out_stride;
    fe x[8];
    x[0] = fe_mul(b[m0], inv8);
#pragma unroll
    for (int c = 1; c < 8; c++) {
        const unsigned e = (unsigned)((unsigned long long)c * m0) & (unsigned)tw.mask;
        const fe t = fe_mul(fe_mul(tw.lo[e & ((1u << tw.lo_bits) - 1u)], tw.hi[e >> tw.lo_bits]), inv8);
        x[c] = fe_mul(b[(unsigned long long)c * n + m0], t);
    }
    // decimation in frequency with w = w_8^-1: X[m1] = sum_c x_c w^(c m1)
    fe u[4], v[4];
    const fe wp[4] = {fe_make(1, 0), w8i1, w8i2, w8i3};
#pragma unroll
    for (int c = 0; c < 4; c++) {
        u[c] = fe_add(x[c], x[c + 4]);
        v[c] = fe_sub(x[c], x[c + 4]);
        if (c) v[c] = fe_mul(v[c], wp[c]);
    }
    fe X[8];
    {   // even outputs from u, odd outputs from v, 4-point transforms with w^2
        fe p0 = fe_add(u[0], u[2]), p1 = fe_add(u[1], u[3]), q0 = fe_sub(u[0], u[2]), q1 = fe_mul(fe_sub(u[1], u[3]), w8i2);
        X[0] = fe_add(p0, p1); X[4] = fe_sub(p0, p1); X[2] = fe_add(q0, q1); X[6] = fe_sub(q0, q1);
        p0 = fe_add(v[0], v[2]); p1 = fe_add(v[1], v[3]); q0 = fe_sub(v[0], v[2]); q1 = fe_mul(fe_sub(v[1], v[3]), w8i2);
        X[1] = fe_add(p0, p1); X[5] = fe_sub(p0, p1); X[3] = fe_add(q0, q1); X[7] = fe_sub(q0, q1);
    }
#pragma unroll
    for (int m1 = 0; m1 < 8; m1++) out[m0 + n * (unsigned long long)m1] = X[m1];
}
void coset_interp_finish(Context &c, const fe *b, fe *out, int log_n, int batch, unsigned long long b_stride, unsigned long long out_stride) {
    const unsigned long long n = 1ULL << log_n;
    const fe w8i = host_inv(host_root_of_unity(3));
    const fe w8i2 = fe_mul(w8i, w8i);
    DG_REQUIRE(batch >= 1 && batch <= 65535, "interpolation batch out of range");
    coset_interp_finish_kernel<<<dim3((unsigned)((n + 127) / 128), (unsigned)batch), 128, 0, c.stream>>>(
        b, out, n, c.twiddle(log_n + 3, true), w8i, w8i2, fe_mul(w8i2, w8i), host_inv(fe_make(8, 0)), b_stride, out_stride);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

// composition polynomial (trace_table.rs:241-258, constraint_poly.rs:49):
//   comp[k] = cq[k]*kc + [k < n] (t1q[k]+t2q[k])*k1 + [inc <= k < inc+n] (t1q[k-inc]+t2q[k-inc])*k2
// blockIdx.y = proof of a batch: t1q / t2q t_stride, cq / comp len elements apart, its k1, k2, kc = ks[3 y ..]
__global__ void compose_kernel(const fe *__restrict__ t1q, const fe *__restrict__ t2q, const fe *__restrict__ cq, fe *__restrict__ comp,
                               unsigned long long n, unsigned long long len, unsigned long long inc, const fe *__restrict__ ks, unsigned long long t_stride) {
    unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= len) return;
    t1q += blockIdx.y * t_stride; t2q += blockIdx.y * t_stride;
    cq += blockIdx.y * len; comp += blockIdx.y * len;
    const fe k1 = ks[3 * blockIdx.y], k2 = ks[3 * blockIdx.y + 1], kc = ks[3 * blockIdx.y + 2];
    fe v = fe_mul(cq[k], kc);
    if (k < n) v = fe_add(v, fe_mul(fe_add(t1q[k], t2q[k]), k1));
    if (k >= inc && k < inc + n) v = fe_add(v, fe_mul(fe_add(t1q[k - inc], t2q[k - inc]), k2));
    comp[k] = v;
}
void compose(Context &c, int batch, const fe *t1q, const fe *t2q, unsigned long long t_stride, const fe *cq, fe *comp, unsigned long long n,
             unsigned long long len, unsigned long long inc, const fe *ks) {
    DG_REQUIRE(batch >= 1 && batch <= 65535, "composition batch out of range");
    compose_kernel<<<dim3((unsigned)((len + 255) / 256), (unsigned)batch), 256, 0, c.stream>>>(t1q, t2q, cq, comp, n, len, inc, ks, t_stride);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

}  // namespace dg
