// BLAKE3 commitment kernels: trace-row leaf hashing, Merkle level sweeps, proof-of-work grinding.
//
//   leaf hashing   /root/reference/src/stark/trace/trace_table.rs:174-185  (hash(as_bytes(row)) for every LDE row)
//   tree building  /root/reference/src/crypto/merkle.rs:269-294            (heap layout, nodes[0] = 0, root = nodes[1])
//   PoW grinding   /root/reference/src/stark/utils/proof_of_work.rs:4-32   (smallest nonce >= 1)
//
// Leaf hashing reads the extended trace in its coset-major layout ([column][coset][k]): a warp's 32 threads hash 32
// neighbouring k of one coset, so each column read is one 512-byte contiguous request; the 32-byte digest is written to
// its logical row position (one full 32-byte sector per thread).  The column->row "gather" that the reference performs
// on the CPU therefore costs no extra memory pass.
#include "common.cuh"
#include "blake3.cuh"
#include <algorithm>

namespace dg {

// ---- trace rows -----------------------------------------------------------------------------------------------------
// ext: [w][N] coset-major (N = rows of the slab: its cosets c0, c0 + 1, ... of n = 2^log_n rows each), leaves in logical row order: the row
// of coset c at step k is leaf (k << log_blowup) + c; blockIdx.y = matrix of a batch, ext_stride elements / 2 leaf_stride uint4 apart, or,
// with a column table, matrix q = the cols[q].y columns from column cols[q].x on (a batch of several widths)
__global__ void __launch_bounds__(256) hash_rows_kernel(const fe *__restrict__ ext, uint4 *__restrict__ leaves, int w, unsigned long long N,
                                                        int log_n, int log_blowup, uint32_t one, unsigned long long ext_stride, unsigned c0,
                                                        unsigned long long leaf_stride, const uint2 *__restrict__ cols) {
    const unsigned long long p = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    if (cols) {
        const uint2 t = cols[blockIdx.y];
        ext += (unsigned long long)t.x * N;
        w = (int)t.y;
    } else {
        ext += blockIdx.y * ext_stride;
    }
    leaves += blockIdx.y * 2 * leaf_stride;
    const unsigned long long n_mask = (1ULL << log_n) - 1ULL;
    const unsigned long long k = p & n_mask, c = (p >> log_n) + c0;
    const unsigned long long row = (k << log_blowup) + c;
    const uint4 *col = reinterpret_cast<const uint4 *>(ext) + p;

    const int total_bytes = w * 16;
    uint32_t cv[8], cv0[8];
    int chunk_start_col = 0;
    const bool two_chunks = total_bytes > 1024;
    for (int chunk = 0; chunk < (two_chunks ? 2 : 1); chunk++) {
        const int chunk_cols = two_chunks ? (chunk == 0 ? 64 : w - 64) : w;
        const int nblocks = (chunk_cols + 3) >> 2;
        b3::iv(cv);
        for (int b = 0; b < nblocks; b++) {
            uint32_t m[16];
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int j = b * 4 + q;
                uint4 v = make_uint4(0, 0, 0, 0);
                if (j < chunk_cols) v = col[(unsigned long long)(chunk_start_col + j) * N];
                m[4 * q] = v.x; m[4 * q + 1] = v.y; m[4 * q + 2] = v.z; m[4 * q + 3] = v.w;
            }
            const int rem = chunk_cols * 16 - b * 64;
            uint32_t flags = 0;
            if (b == 0) flags |= b3::CHUNK_START;
            if (b == nblocks - 1) { flags |= b3::CHUNK_END; if (!two_chunks) flags |= b3::ROOT; }
            b3::compress_fma(cv, m, (uint64_t)chunk, rem < 64 ? rem : 64, flags, one);
        }
        if (two_chunks && chunk == 0) {
#pragma unroll
            for (int i = 0; i < 8; i++) cv0[i] = cv[i];
            chunk_start_col = 64;
        }
    }
    if (two_chunks) {
        uint32_t m[16];
#pragma unroll
        for (int i = 0; i < 8; i++) { m[i] = cv0[i]; m[8 + i] = cv[i]; }
        b3::iv(cv);
        b3::compress(cv, m, 0, 64, b3::PARENT | b3::ROOT);
    }
    leaves[2 * row] = make_uint4(cv[0], cv[1], cv[2], cv[3]);
    leaves[2 * row + 1] = make_uint4(cv[4], cv[5], cv[6], cv[7]);
}

void hash_trace_rows(Context &c, const fe *ext, void *leaves, int w, int log_n, int log_blowup, int batch, unsigned long long ext_stride, unsigned c0,
                     unsigned nc, unsigned long long leaf_stride, const uint2 *cols) {
    const unsigned long long all = 1ULL << (log_n + log_blowup);
    const unsigned long long rows = nc ? (unsigned long long)nc << log_n : all;
    DG_REQUIRE(batch >= 1 && batch <= 65535, "row hashing batch out of range");
    DG_REQUIRE(c0 + (rows >> log_n) <= (1ULL << log_blowup), "coset range out of bounds");
    const dim3 grid((unsigned)((rows + 255) / 256), (unsigned)batch);
    // FMA-pipe additions: trace tree 10.3 -> 8.8 ms at 2^25 rows x 26 columns (H100 SXM, 700 W)
    hash_rows_kernel<<<grid, 256, 0, c.stream>>>(ext, (uint4 *)leaves, w, rows, log_n, log_blowup, 1u, ext_stride, c0, leaf_stride ? leaf_stride : all,
                                                 cols);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

// rows of a plain column-major matrix (no coset permutation): physical position == logical row
void hash_rows_plain(Context &c, const fe *cols, void *digests, int w, unsigned long long rows) {
    hash_rows_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, c.stream>>>(cols, (uint4 *)digests, w, rows, 63, 0, 1u, 0, 0u, 0, nullptr);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

// ---- Merkle levels ----------------------------------------------------------------------------------------------------
// out[i] = H(in[2i] || in[2i+1]),  i < count; blockIdx.y = tree of a batch, `stride` uint4 apart (in and out)
__global__ void __launch_bounds__(256) merkle_level_kernel(const uint4 *__restrict__ in, uint4 *__restrict__ out, unsigned long long count,
                                                           unsigned long long in_stride, unsigned long long out_stride) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    in += blockIdx.y * in_stride;
    out += blockIdx.y * out_stride;
    uint32_t m[16], cv[8];
#pragma unroll
    for (int q = 0; q < 4; q++) {
        uint4 v = in[4 * i + q];
        m[4 * q] = v.x; m[4 * q + 1] = v.y; m[4 * q + 2] = v.z; m[4 * q + 3] = v.w;
    }
    b3::hash64(m, cv);
    out[2 * i] = make_uint4(cv[0], cv[1], cv[2], cv[3]);
    out[2 * i + 1] = make_uint4(cv[4], cv[5], cv[6], cv[7]);
}

// finishes a tree whose level with `count` (<= 1024, power of two) nodes sits at nodes[count .. 2*count): computes
// nodes[count/2 .. count), ..., nodes[1] in one block, and zeroes nodes[0]; block b finishes the tree `stride` uint4 after block b - 1's
__global__ void __launch_bounds__(512) merkle_top_kernel(uint4 *__restrict__ nodes, unsigned count, unsigned long long stride) {
    __shared__ uint32_t s[2048 * 8 / 2];     // up to 1024 digests
    const unsigned tid = threadIdx.x;
    nodes += blockIdx.x * stride;
    for (unsigned i = tid; i < count * 2; i += blockDim.x) {
        uint4 v = nodes[2 * count + i];
        s[4 * i] = v.x; s[4 * i + 1] = v.y; s[4 * i + 2] = v.z; s[4 * i + 3] = v.w;
    }
    __syncthreads();
    for (unsigned m = count / 2; m >= 1; m >>= 1) {
        // level with m nodes from 2m children held in s[0 .. 2m*8)
        uint32_t cv[8];
        uint32_t msg[16];
        const bool active = tid < m;
        if (active) {
#pragma unroll
            for (int q = 0; q < 16; q++) msg[q] = s[16 * tid + q];
            b3::hash64(msg, cv);
        }
        __syncthreads();
        if (active) {
#pragma unroll
            for (int q = 0; q < 8; q++) s[8 * tid + q] = cv[q];
            nodes[2 * (m + tid)] = make_uint4(cv[0], cv[1], cv[2], cv[3]);
            nodes[2 * (m + tid) + 1] = make_uint4(cv[4], cv[5], cv[6], cv[7]);
        }
        __syncthreads();
    }
    if (tid == 0) { nodes[0] = make_uint4(0, 0, 0, 0); nodes[1] = make_uint4(0, 0, 0, 0); }
}

// computes the levels count/2, count/4, ... down to and including the level with `stop` nodes (stop >= 1, a power of two) from the
// input level `in` (count nodes) into the heap `nodes` (a level with m nodes sits at nodes[m .. 2m)).  One launch per level while a
// level has more than 1024 nodes -- BLAKE3 is ALU-bound with long dependency chains, so the per-level kernel at full occupancy is the
// fastest form (a fused variant that keeps 8 -> 4 -> 2 -> 1 nodes per thread in registers for 11 levels per launch needs far more
// registers, hence fewer resident warps) -- then the last <= 1024 nodes level by level inside one block.
// `batch` trees at once: tree q reads in + q * in_stride and writes nodes + q * nodes_stride (uint4 units)
static void tree_levels(Context &c, const uint4 *in, uint4 *nodes, unsigned long long count, unsigned long long stop, int batch = 1,
                        unsigned long long in_stride = 0, unsigned long long nodes_stride = 0) {
    DG_REQUIRE(batch >= 1 && batch <= 65535, "tree batch out of range");
    while (count > stop) {
        const unsigned long long m = count / 2;
        if (stop == 1 && count <= 1024 && count >= 2 && in == nodes + 2 * count) {     // the rest of a complete tree: one block per tree
            merkle_top_kernel<<<batch, 512, 0, c.stream>>>(nodes, (unsigned)count, nodes_stride); c.launches++;
            DG_CUDA(cudaGetLastError());
            return;
        }
        merkle_level_kernel<<<dim3((unsigned)((m + 255) / 256), (unsigned)batch), 256, 0, c.stream>>>(in, nodes + 2 * m, m, in_stride, nodes_stride);
        c.launches++;
        DG_CUDA(cudaGetLastError());
        count = m;
        in = nodes + 2 * m;
        in_stride = nodes_stride;
    }
}

// `batch` trees of L leaves each (L power of two >= 2), L digests of nodes each (heap layout): leaves and nodes of tree q at q * L digests
// from the first
void merkle_build(Context &c, const void *leaves, void *nodes, unsigned long long L, int batch) {
    DG_REQUIRE(L >= 2 && (L & (L - 1)) == 0, "number of leaves must be a power of 2 and >= 2");
    uint4 *nd = (uint4 *)nodes;
    tree_levels(c, (const uint4 *)leaves, nd, L, 1, batch, 2 * L, 2 * L);
    DG_CUDA(cudaMemset2DAsync(nd, L * 32, 0, 32, batch, c.stream));     // nodes[0] = 0 (merkle.rs:273)
}

// completes a tree whose level with m nodes (m a power of two) already sits at nodes[m .. 2m)
void merkle_finish(Context &c, void *nodes, unsigned long long m) {
    uint4 *nd = (uint4 *)nodes;
    tree_levels(c, nd + 2 * m, nd, m, 1);
    DG_CUDA(cudaMemsetAsync(nd, 0, 32, c.stream));
}

// levels of a heap-layout tree from L/2 nodes down to (and including) the level with `stop` nodes
void merkle_levels_down_to(Context &c, const void *leaves, void *nodes, unsigned long long L, unsigned long long stop) {
    tree_levels(c, (const uint4 *)leaves, (uint4 *)nodes, L, stop);
}

// ---- generic 64-byte hashing (tests / FRI rows given contiguously) ------------------------------------------------------
void hash64_contiguous(Context &c, const void *in, void *out, unsigned long long count) {
    merkle_level_kernel<<<(unsigned)((count + 255) / 256), 256, 0, c.stream>>>((const uint4 *)in, (uint4 *)out, count, 0, 0); c.launches++;
    DG_CUDA(cudaGetLastError());
}

// ---- proof of work ------------------------------------------------------------------------------------------------------
// does blake3(seed || nonce) have >= grinding trailing zero bits in its first 8 bytes
__device__ __forceinline__ bool pow_hit(const uint32_t *__restrict__ seed, unsigned long long nonce, unsigned grinding) {
    uint32_t m[16], cv[8];
#pragma unroll
    for (int i = 0; i < 8; i++) m[i] = seed[i];
    m[8] = (uint32_t)nonce; m[9] = (uint32_t)(nonce >> 32);
#pragma unroll
    for (int i = 10; i < 16; i++) m[i] = 0;
    b3::hash64(m, cv);
    const unsigned long long o0 = ((unsigned long long)cv[1] << 32) | cv[0];
    const unsigned tz = o0 == 0 ? 64u : (unsigned)(__ffsll((long long)o0) - 1);
    return tz >= grinding;
}

// one window [start, start + count) of nonces for each unfinished proof active[blockIdx.y]: seeds [proof][8 words], grinding [proof],
// best [proof]
__global__ void __launch_bounds__(256) pow_batch_kernel(const uint32_t *__restrict__ seeds, const unsigned *__restrict__ grinding,
                                                        const unsigned *__restrict__ active, unsigned long long start,
                                                        unsigned long long count, unsigned long long *best) {
    const unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= count) return;
    const unsigned p = active[blockIdx.y];
    const unsigned long long nonce = start + g;
    if (pow_hit(seeds + 8 * p, nonce, grinding[p])) atomicMin(best + p, nonce);
}

// For each of K seeds, the smallest nonce >= 1 whose hash has >= grinding[p] trailing zero bits in its first 8 bytes.  Each round scans
// the same window of nonces for every proof that has no hit yet (one launch, one copy of the K results back).  A proof finishes in the
// first window where it has a hit, and the window's smallest hit is its smallest nonce; proofs of low grinding factors drop out early.
// One proof scans a 2^22 window per round.  A batch scans 2^22 / K nonces per proof and round (one 2^22-nonce round in all), but at least
// 2^(g - 2) for the largest grinding factor g, a quarter of its expected search (clamped to 2^10 .. 2^22): large batches run more rounds
// but hash little past each proof's first hit, small ones keep few rounds.  Measured on an H100 at 400 W, grinding 20, PoW
// stage of a batch of 16 / 64 / 256 proofs: 2^16: 1.17 / 3.02 / 11.7 ms; 2^18: 0.76 / 2.57 / 10.9; 2^19: 0.74 / 2.75 / 12.2; 2^20: 0.86 /
// 3.30 / 14.8; 2^21: 1.34 / 4.84 / 21.2; 2^22: 2.24 / 8.87 / 36.3 ms.
std::vector<unsigned long long> pow_search_batch(Context &c, const std::vector<std::array<uint8_t, 32>> &seeds,
                                                 const std::vector<unsigned> &grinding) {
    const unsigned K = (unsigned)seeds.size();
    std::vector<unsigned long long> best(K, ~0ULL);
    if (K == 0) return best;
    DG_REQUIRE(K <= 65535, "too many proof-of-work seeds for one launch");
    DG_REQUIRE(grinding.size() == K, "one grinding factor per proof-of-work seed");
    // one upload: the seeds [K][8 words], then the grinding factors [K]
    std::vector<uint32_t> in((size_t)9 * K);
    memcpy(in.data(), seeds.data(), (size_t)32 * K);
    std::copy(grinding.begin(), grinding.end(), in.begin() + (size_t)8 * K);
    DevBuf d_seeds(in.size() * 4), d_best((size_t)8 * K), d_active((size_t)4 * K);
    DG_CUDA(cudaMemcpyAsync(d_seeds.p, in.data(), in.size() * 4, cudaMemcpyHostToDevice, c.stream));
    DG_CUDA(cudaMemcpyAsync(d_best.p, best.data(), (size_t)8 * K, cudaMemcpyHostToDevice, c.stream));
    unsigned long long window = 1ULL << 22;
    if (K > 1) {
        int log_k = 0;
        while ((1u << log_k) < K) log_k++;
        const unsigned gmax = *std::max_element(grinding.begin(), grinding.end());
        window = 1ULL << std::max(10, std::min(22, std::max((int)gmax - 2, 22 - log_k)));
    }
    std::vector<unsigned> active(K);
    for (unsigned p = 0; p < K; p++) active[p] = p;
    bool upload = true;
    for (unsigned long long start = 1; start < (1ULL << 42); start += window) {
        if (upload) DG_CUDA(cudaMemcpyAsync(d_active.p, active.data(), (size_t)4 * active.size(), cudaMemcpyHostToDevice, c.stream));
        pow_batch_kernel<<<dim3((unsigned)(window / 256), (unsigned)active.size()), 256, 0, c.stream>>>(
            d_seeds.as<uint32_t>(), d_seeds.as<unsigned>() + (size_t)8 * K, d_active.as<unsigned>(), start, window, d_best.as<unsigned long long>());
        c.launches++;
        DG_CUDA(cudaGetLastError());
        DG_CUDA(cudaMemcpyAsync(best.data(), d_best.p, (size_t)8 * K, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
        std::vector<unsigned> still;
        for (unsigned p : active) if (best[p] == ~0ULL) still.push_back(p);
        if (still.empty()) return best;
        upload = still.size() != active.size();
        active.swap(still);
    }
    throw Error(-4, "proof-of-work search exhausted");
}

// host-side BLAKE3 of the 64-byte proof-of-work input seed || nonce_le || 0^24 (proof_of_work.rs:12-24)
void pow_hash(const uint8_t seed[32], unsigned long long nonce, uint8_t out[32]) {
    uint32_t m[16], cv[8];
    memcpy(m, seed, 32);
    m[8] = (uint32_t)nonce; m[9] = (uint32_t)(nonce >> 32);
    for (int i = 10; i < 16; i++) m[i] = 0;
    b3::hash64(m, cv);
    memcpy(out, cv, 32);
}
}  // namespace dg
