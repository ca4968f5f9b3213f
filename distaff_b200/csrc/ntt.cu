// Batched radix-2 NTT / inverse NTT and coset low-degree extension over F_M for sm_90a.
//
// Replaces, for the prove hot path, the reference's recursive in-place FFT + bit-reversal permutation
//   /root/reference/src/math/fft.rs:16-79, /root/reference/src/math/polynom.rs:34-41,93-103
// and the zero-padded extension loop of /root/reference/src/stark/trace/trace_table.rs:143-169.
// Contract (pinned by fft.rs:117-157): natural-order input -> natural-order DFT  X[k] = sum_j x[j] w^(jk).
//
// Design: a transform of size n = 2^log_n is split into at most three passes of <= 1024-point sub-transforms that run
// entirely in shared memory (decimation in frequency, twiddles for the in-block stages staged in shared memory).  Every
// pass streams HBM once with 16-byte vector accesses; a block owns a tile of T neighbouring "lanes" (independent
// sub-transforms whose elements are adjacent in memory) so that global reads and writes are T*16-byte contiguous
// segments.  Inter-pass twiddles w^(lane*k) come from a two-level power table (2 loads + 1 multiply).
//
// Low-degree extension does not zero-pad: evaluating P (n coefficients) on the LDE domain of size N = b*n is done as b
// independent size-n transforms of the coset-scaled coefficients p[m] * w_N^(c*m); the result is stored coset-major
// ([c][k] <-> LDE index b*k + c), which is the layout every later kernel (leaf hashing, constraint evaluation, FRI)
// consumes with unit-stride reads.  This removes log2(b) of the log2(N) butterfly levels and all work on zeros.
// The fully unrolled rounds are far larger than the 32 KB instruction cache; with the field multiplication out of line
// (one shared 80-instruction body) the pass kernels are much smaller.  The large transforms use inlined multiplies with small
// register rounds instead (ntt_inl.cu): the small rounds keep the unrolled code near the instruction-cache size without a call per multiply.
// Each kernel is specialised at compile time for one pass kind (PassKind, ntt_pass.cuh), so it holds only its own input and output
// paths; with 4-element register rounds, 512 threads and 64 registers the kernels of the 2^20-step proof do not spill.
#define DG_MUL_CALL 1
#include "ntt_pass.cuh"

namespace dg {

// the kernel specialisation of a pass, from the flags run_transform sets
static int pass_kind(const PassGeom &g) {
    if (!g.lane_major) {
        DG_REQUIRE(g.tw_on && !g.has_scale, "strided NTT pass without inter-pass twiddle");
        if (g.coset_fast) return g.tw_full ? PK_COSET_TWFULL : PK_COSET_TW;
        return g.coset_on ? PK_FOLD_TW : PK_TW;
    }
    DG_REQUIRE(!g.tw_on, "contiguous NTT pass with inter-pass twiddle");
    if (g.coset_on) {
        DG_REQUIRE(!g.has_scale, "scaled coset transform");
        return g.coset_fast ? PK_COSET_ONE : PK_FOLD_ONE;
    }
    return g.has_scale ? PK_LAST_SCALE : PK_LAST;
}

// Pass kernel shape (ntt_pass.cuh: PASS_RMAX, PASS_THREADS, PASS_INLINE_LOG_L) and tile size.  H100 SXM 80 GB (700 W power limit),
// stage 1 of the 2^20-step proof (26 columns, LDE x32), ms (A = strided first / middle passes, B = contiguous last pass, AF = fold-8
// first passes):
//   inline multiply, 4-element units (rmax 2), 512 threads, 4096-element tiles: 52.7 (no spills at the 64-register cap)
//   A = B = 8-element units (rmax 3), 512 threads: 56.9 (150-570 bytes of spills per kernel at the 64-register cap)
//   measured before the kernels were specialised per pass kind (every kind's path in one kernel, a call per multiply):
//   rmax 3 for A and B 60.8 - 61.3;  A = 256 threads 68.0;  A = 1024 threads + 8192-element tiles 71.7;  B = 256 threads 62.5;
//   AF = 8-element units or 256 threads: no change in stages 5 / 6
// The other shapes were removed after this measurement.
static const int TILE = 4096;                    // elements per block = 64 KB

static void launch_pass(Context &c, int log_l, PassGeom g, const fe *src, fe *dst, unsigned blocks_x, unsigned by, unsigned bz) {
    const int L = 1 << log_l, T = 1 << g.log_t;
    const size_t data = g.lane_major ? (size_t)T * (L + (L >> 3) + 1) : (size_t)L * T;
    const size_t smem = ((size_t)L + data) * sizeof(fe);
    const int kind = pass_kind(g);
    const PassKernel k = log_l >= PASS_INLINE_LOG_L ? pass_kernel_inline(kind, log_l)
                                                    : pass_kernel_of<PASS_RMAX, PASS_THREADS, PASS_MINB, 0, 1, PASS_INLINE_LOG_L - 1>(kind, log_l);
    DG_REQUIRE(k, "unsupported sub-transform size");
    int threads = (L * T) >> (log_l < PASS_RMAX ? log_l : PASS_RMAX);           // one unit per thread in the largest round
    if (threads > PASS_THREADS) threads = PASS_THREADS;
    if (threads < 32) threads = 32;
    set_func_smem(c, (const void *)k, 200 * 1024);
    DG_REQUIRE(by <= 65535 && bz <= 65535, "batch too large for one launch");
    // (folding the vector index into blockIdx.x so that all columns of a (tile, coset) share the streamed twiddles in L2 spills at the
    //  64-register cap: rejected)
    k<<<dim3(blocks_x, by, bz), threads, smem, c.stream>>>(src, dst, g); c.launches++;
    DG_CUDA(cudaGetLastError());
}

static int lanes_log(int log_l, long long available) {
    int lt = 4;                                   // 16 lanes
    while ((1 << (log_l + lt)) > TILE && lt > 0) lt--;
    while ((1LL << lt) > available && lt > 0) lt--;
    return lt;
}

// split log_n into 1..3 pass sizes (outermost first)
static int split_passes(int log_n, int l[3]) {
    if (log_n <= MAX_LOG_L) { l[0] = log_n; return 1; }
    if (log_n <= 2 * MAX_LOG_L) { l[0] = (log_n + 1) / 2; l[1] = log_n / 2; return 2; }
    DG_REQUIRE(log_n <= 3 * MAX_LOG_L, "transform too large");
    l[0] = (log_n + 2) / 3; l[1] = (log_n + 1) / 3; l[2] = log_n / 3;
    return 3;
}

struct CosetSpec { bool on; int log_blowup; int fold; unsigned coset0; };

// table[c][k * R1 + lane] = w_N^(lane * (k * b + c)): the twiddle the first LDE pass applies to output k of lane `lane` on coset c.
// It depends on the shape only (n, b, first pass size), so it is built once per shape and kept: N elements (512 MB for 2^20 x 32).
__global__ void lde_twiddle_fill_kernel(fe *table, TwiddleRef cw, int log_n, int log_r1, int log_b) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >> (log_n + log_b)) return;
    const unsigned long long c = i >> log_n, pos = i & ((1ULL << log_n) - 1);
    const unsigned long long lane = pos & ((1ULL << log_r1) - 1), k = pos >> log_r1;
    table[i] = tw_lookup(cw, lane * ((k << log_b) + c));
}
static const fe *lde_twiddle_table(Context &c, int log_n, int log_b, int l0) {
    const size_t bytes = ((size_t)16 << (log_n + log_b));
    if (bytes > ((size_t)1 << 30)) return nullptr;         // over 1 GiB (2^22 steps x 32): the pass uses the two-level table instead
    const long long key = ((long long)log_n << 16) | (log_b << 8) | l0;
    auto it = c.lde_twiddles.find(key);
    if (it == c.lde_twiddles.end()) {
        DevBuf t;
        t.alloc(bytes, true);
        const unsigned long long cnt = 1ULL << (log_n + log_b);
        lde_twiddle_fill_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, c.stream>>>(t.as<fe>(), c.twiddle(log_n + log_b, false), log_n, log_n - l0, log_b);
        c.launches++;
        DG_CUDA(cudaGetLastError());
        it = c.lde_twiddles.emplace(key, std::move(t)).first;
    }
    return it->second.as<fe>();
}

// Runs the passes of one batched transform.  `by` = number of y-batches (cosets for the LDE, else 1), `bz` = vectors.
// src strides: vector stride src_stride (z), y stride 0 for the LDE (every coset reads the same coefficients).
static void run_transform(Context &c, const fe *src, fe *dst, int log_n, bool inverse, unsigned by, unsigned bz, long long src_stride_z,
                          long long dst_stride_y, long long dst_stride_z, CosetSpec cs) {
    int l[3];
    const int np = split_passes(log_n, l);
    const long long n = 1LL << log_n;
    fe scale = fe_make(1, 0);
    if (inverse) scale = host_inv(fe_make((unsigned long long)n, 0));

    PassGeom base;
    memset(&base, 0, sizeof base);
    if (cs.on) {
        base.coset_on = 1;
        base.fold = cs.fold;
        base.fold_stride = n;
        base.cw = c.twiddle(log_n + cs.log_blowup, false);
        base.log_blowup = cs.log_blowup;
        base.coset0 = cs.coset0;
        if (cs.fold == 1) {
            // order of w_N^in_point where in_point = n / N1 (first pass) : N / in_point = N1 << log_blowup
            const int log_order = l[0] + cs.log_blowup;
            base.coset_fast = 1;
            base.cw_point = c.single_table(log_order);
            base.cw_point_mask = (1u << log_order) - 1u;
        }
    }

    fe *tmp = nullptr;
    long long tmp_stride_y = n, tmp_stride_z = n * by;
    if (np > 1) {
        c.ntt_tmp.ensure((size_t)n * by * bz * sizeof(fe), true);
        tmp = c.ntt_tmp.as<fe>();
    }

    if (np == 1) {
        PassGeom g = base;
        g.log_t = 0; g.num_tiles = 1;
        g.in_point = 1; g.out_point = 1; g.in_lane = 0; g.out_lane = 0;
        g.in_batch_y = 0; g.in_batch_z = src_stride_z; g.out_batch_y = dst_stride_y; g.out_batch_z = dst_stride_z;
        g.lane_major = 1; g.tw_on = 0;
        g.has_scale = inverse; g.scale = scale;
        g.roots = c.roots(l[0], inverse);
        launch_pass(c, l[0], g, src, dst, 1, by, bz);
        return;
    }

    const long long N1 = 1LL << l[0];
    const long long R1 = n >> l[0];
    {   // pass 1: N1-point transforms over j1 (stride R1), twiddle w_n^(j' * k1)
        PassGeom g = base;
        g.log_t = lanes_log(l[0], R1);
        g.num_tiles = (unsigned)(R1 >> g.log_t);
        g.in_point = R1; g.in_lane = 1; g.out_point = R1; g.out_lane = 1;
        g.in_batch_y = 0; g.in_batch_z = src_stride_z; g.out_batch_y = tmp_stride_y; g.out_batch_z = tmp_stride_z;
        g.lane_major = 0;
        g.tw_on = 1; g.tw = c.twiddle(log_n, inverse);
        if (g.coset_fast) { g.tw_full = lde_twiddle_table(c, log_n, cs.log_blowup, l[0]); g.tw_full_stride = n; }
        g.roots = c.roots(l[0], inverse);
        launch_pass(c, l[0], g, src, tmp, g.num_tiles, by, bz);
    }
    long long N2 = 1;
    if (np == 3) {   // pass 2: within every row k1, N2-point transforms over ja (stride N3), twiddle w_R1^(jb * ka)
        N2 = 1LL << l[1];
        const long long N3 = 1LL << l[2];
        PassGeom g;
        memset(&g, 0, sizeof g);
        g.log_t = lanes_log(l[1], N3);
        g.num_tiles = (unsigned)(N3 >> g.log_t);
        g.in_point = N3; g.in_lane = 1; g.in_outer = R1; g.out_point = N3; g.out_lane = 1; g.out_outer = R1;
        g.in_batch_y = tmp_stride_y; g.in_batch_z = tmp_stride_z; g.out_batch_y = tmp_stride_y; g.out_batch_z = tmp_stride_z;
        g.lane_major = 0;
        g.tw_on = 1; g.tw = c.twiddle(log_n - l[0], inverse);
        g.roots = c.roots(l[1], inverse);
        launch_pass(c, l[1], g, tmp, tmp, (unsigned)(g.num_tiles * N1), by, bz);
    }
    {   // last pass: contiguous NL-point transforms; output index k1 + N1*ka + N1*N2*kb
        const int ll = l[np - 1];
        PassGeom g;
        memset(&g, 0, sizeof g);
        g.log_t = lanes_log(ll, N1);
        g.num_tiles = (unsigned)(N1 >> g.log_t);
        g.in_point = 1; g.in_lane = R1; g.in_outer = (np == 3) ? (1LL << ll) : 0;
        g.out_lane = 1; g.out_outer = (np == 3) ? N1 : 0; g.out_point = N1 * N2;
        g.in_batch_y = tmp_stride_y; g.in_batch_z = tmp_stride_z; g.out_batch_y = dst_stride_y; g.out_batch_z = dst_stride_z;
        g.lane_major = 1; g.tw_on = 0;
        g.has_scale = inverse; g.scale = scale;
        g.roots = c.roots(ll, inverse);
        launch_pass(c, ll, g, tmp, dst, (unsigned)(g.num_tiles * N2), by, bz);
    }
}

void ntt_batch(Context &c, const fe *src, fe *dst, int log_n, int batch, size_t src_stride, size_t dst_stride, bool inverse) {
    DG_REQUIRE(log_n >= 1 && log_n <= 30, "log_n out of range");
    const size_t n = (size_t)1 << log_n;
    // bound the scratch: process vectors in chunks of at most ~1 GiB of scratch
    size_t max_chunk = std::max<size_t>(1, ((size_t)1 << 30) / (n * sizeof(fe)));
    if (max_chunk > 65535) max_chunk = 65535;
    for (size_t b0 = 0; b0 < (size_t)batch; b0 += max_chunk) {
        size_t nb = std::min(max_chunk, (size_t)batch - b0);
        run_transform(c, src + b0 * src_stride, dst + b0 * dst_stride, log_n, inverse, 1, (unsigned)nb, (long long)src_stride, 0,
                      (long long)dst_stride, CosetSpec{false, 0, 1, 0});
    }
}

// ---- fold-8 input transform for all cosets at once -----------------------------------------------------------------------------------
// Extending a polynomial with 8n coefficients (constraint / composition polynomial) over all b cosets needs, for every coefficient
// position j < n and coset c, the value  w_N^(c j) * sum_{f<8} p[j + f n] * zeta^(c f),  zeta = w_N^n = w_b.  Inside the pass kernel that
// is a Horner evaluation per (coset, position): 9 multiplications per input element, as much as the whole transform that follows.
// For all cosets together the inner sums are a b-point DFT of the zero-padded 8-vector: with c = (b/8) q + r it is, per residue r, a
// twist by zeta^(r f) (7 multiplications) and an 8-point DFT over q (5 multiplications); the outer factor is a geometric progression in
// q.  One thread per (r, j): 29 multiplications for 8 outputs instead of 72.  The result feeds b plain size-n transforms.
// blockIdx.y = vector of a batch: src + y * src_stride in, dst + y * (b n) out.
__global__ void __launch_bounds__(256) prefold8_kernel(const fe *__restrict__ src, fe *__restrict__ dst, int log_n, int log_b, const fe *__restrict__ zeta,
                                                       TwiddleRef twN, fe w8, fe w8_2, fe w8_3, unsigned long long src_stride) {
    src += blockIdx.y * src_stride;
    dst += (unsigned long long)blockIdx.y << (log_n + log_b);
    const unsigned long long n = 1ULL << log_n;
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >> (log_n + log_b - 3)) return;
    const unsigned long long j = t & (n - 1);
    const unsigned r = (unsigned)(t >> log_n);                 // residue of the coset index modulo b/8
    const unsigned bmask = (1u << log_b) - 1u, step = 1u << (log_b - 3);
    fe x[8];
#pragma unroll
    for (int f = 0; f < 8; f++) x[f] = src[j + (unsigned long long)f * n];
    if (r) {
#pragma unroll
        for (int f = 1; f < 8; f++) x[f] = fe_mul(x[f], zeta[(r * (unsigned)f) & bmask]);
    }
    // 8-point DFT X[q] = sum_f x[f] w8^(q f), decimation in frequency, outputs in natural order
    fe u[4], v[4];
    const fe wp[4] = {fe_make(1, 0), w8, w8_2, w8_3};
#pragma unroll
    for (int i = 0; i < 4; i++) {
        u[i] = fe_add(x[i], x[i + 4]);
        v[i] = fe_sub(x[i], x[i + 4]);
        if (i) v[i] = fe_mul(v[i], wp[i]);
    }
    fe X[8];
    {
        fe p0 = fe_add(u[0], u[2]), p1 = fe_add(u[1], u[3]), q0 = fe_sub(u[0], u[2]), q1 = fe_mul(fe_sub(u[1], u[3]), w8_2);
        X[0] = fe_add(p0, p1); X[4] = fe_sub(p0, p1); X[2] = fe_add(q0, q1); X[6] = fe_sub(q0, q1);
        p0 = fe_add(v[0], v[2]); p1 = fe_add(v[1], v[3]); q0 = fe_sub(v[0], v[2]); q1 = fe_mul(fe_sub(v[1], v[3]), w8_2);
        X[1] = fe_add(p0, p1); X[5] = fe_sub(p0, p1); X[3] = fe_add(q0, q1); X[7] = fe_sub(q0, q1);
    }
    // outer factor w_N^(c j), c = step q + r: w_N^(r j) * (w_N^(step j))^q
    fe cur = tw_lookup(twN, (unsigned long long)r * j);
    const fe rho = tw_lookup(twN, (unsigned long long)step * j);
#pragma unroll
    for (int q = 0; q < 8; q++) {
        dst[((unsigned long long)(step * (unsigned)q + r) << log_n) + j] = fe_mul(X[q], cur);
        if (q < 7) cur = fe_mul(cur, rho);
    }
}

void lde_batch(Context &c, const fe *src, fe *dst, int log_n, int log_blowup, int fold, int batch, size_t src_stride, size_t dst_stride,
               unsigned coset0, unsigned ncosets) {
    DG_REQUIRE(log_n >= 1 && log_n + log_blowup <= 30, "LDE domain too large");
    const size_t n = (size_t)1 << log_n;
    DG_REQUIRE(log_blowup >= 0 && log_blowup <= 16 && fold >= 1, "bad LDE shape");
    const unsigned b = 1u << log_blowup, cosets = ncosets ? ncosets : b;
    // any sub-range works (blockIdx.y = coset - coset0 indexes the streamed twiddles and dst); a range beyond the domain does not
    DG_REQUIRE(coset0 < b && cosets <= b - coset0, "coset range out of bounds");
    if (fold == 8 && cosets == (1u << log_blowup) && log_blowup >= 3 && log_blowup <= 8 && (batch == 1 || dst_stride == n * cosets) &&
        batch <= 65535) {
        // all cosets: input transform for every coset in one kernel, then b plain transforms (H100 SXM, 700 W, 2^20-step proof: stage 5 5.35 -> 3.83 ms, stage 6 5.83 -> 4.30 ms);
        // a batch of vectors whose outputs are contiguous runs both steps once for all of them
        DevBuf pre((size_t)n * cosets * batch * sizeof(fe));
        const fe w8 = host_root_of_unity(3), w8_2 = fe_mul(w8, w8);
        const unsigned long long threads = (unsigned long long)n << (log_blowup - 3);
        prefold8_kernel<<<dim3((unsigned)((threads + 255) / 256), (unsigned)batch), 256, 0, c.stream>>>(
            src, pre.as<fe>(), log_n, log_blowup, c.single_table(log_blowup), c.twiddle(log_n + log_blowup, false), w8, w8_2, fe_mul(w8_2, w8),
            (unsigned long long)src_stride); c.launches++;
        DG_CUDA(cudaGetLastError());
        ntt_batch(c, pre.as<fe>(), dst, log_n, (int)cosets * batch, n, n, false);
        return;
    }
    // scratch of the two-pass transforms: one intermediate of n * cosets elements per vector; more vectors per launch = fewer passes over
    // the streamed first-pass twiddles (at most 4 GiB of scratch)
    size_t max_chunk = std::max<size_t>(1, ((size_t)4 << 30) / (n * cosets * sizeof(fe)));
    if (max_chunk > 65535) max_chunk = 65535;
    for (size_t b0 = 0; b0 < (size_t)batch; b0 += max_chunk) {
        size_t nb = std::min(max_chunk, (size_t)batch - b0);
        run_transform(c, src + b0 * src_stride, dst + b0 * dst_stride, log_n, false, cosets, (unsigned)nb, (long long)src_stride,
                      (long long)n, (long long)dst_stride, CosetSpec{true, log_blowup, fold, coset0});
    }
}

}  // namespace dg
