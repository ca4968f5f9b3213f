// extern "C" surface declared in include/distaff_gpu.h.  Every entry point catches dg::Error and returns a code.
#include "../../include/distaff_gpu.h"
#include "common.cuh"
#include "prover.h"
#include "host_fs.h"
#include "shard.h"
#include "poly.h"
#include "air.h"
#include "tree.h"
#include <memory>
#include <thread>

using namespace dg;

static thread_local std::string t_last_error;
static thread_local std::vector<std::string> t_batch_messages;     // per trace / proof of the calling thread's last batched call

template <typename F>
static int guarded(F &&f) {
    try {
        f();
        return DG_OK;
    } catch (const dg::Error &e) {
        t_last_error = e.what();
        return e.code;
    } catch (const std::exception &e) {
        t_last_error = e.what();
        return DG_ERR_INVALID;
    }
}

// ---- helper kernels ------------------------------------------------------------------------------------------------------
__global__ void coset_to_logical_kernel(const fe *__restrict__ in, fe *__restrict__ out, int log_n, int log_blowup) {
    const unsigned long long p = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long N = 1ULL << (log_n + log_blowup);
    if (p >= N) return;
    const unsigned long long k = p & ((1ULL << log_n) - 1ULL), c = p >> log_n;
    out[(unsigned long long)blockIdx.y * N + (k << log_blowup) + c] = in[(unsigned long long)blockIdx.y * N + p];
}

__global__ void field_op_kernel(int op, int impl, const fe *a, const fe *b, fe *out, unsigned long long n) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (op == 5) {                    // unreduced dot product of groups of 6: out[i] = sum_j a[6i+j] * b[6i+j]; impl 0 = 288-bit accumulation, 1 = reduced
        if (6 * i + 6 > n) return;
        fe xs[6], ys[6];
#pragma unroll
        for (int j = 0; j < 6; j++) { xs[j] = a[6 * i + j]; ys[j] = b[6 * i + j]; }
        if (impl == 0) out[i] = fe_dot<6>(xs, ys);
        else { fe acc = portable::fe_mul(xs[0], ys[0]); for (int j = 1; j < 6; j++) acc = portable::fe_add(acc, portable::fe_mul(xs[j], ys[j])); out[i] = acc; }
        return;
    }
    fe x = a[i], y = b ? b[i] : fe_make(0, 0), r;
    if (op == 6) {                    // a * b through fe_mul_tw, the companion of b computed as the twiddle tables compute it
        out[i] = impl == 0 ? fe_mul_tw(x, y, fe_tw_companion(y)) : portable::fe_mul_tw(x, y, portable::fe_tw_companion(y));
        return;
    }
    if ((impl == 2 || impl == 3) && op == 2) {
#ifdef __CUDA_ARCH__
        r = impl == 2 ? ptx::fe_mul_v1(x, y) : ptx::fe_mul_v3(x, y);      // earlier multiplies, kept for differential tests
#endif
    } else if (impl == 0) {
        switch (op) {
            case 0: r = fe_add(x, y); break;
            case 1: r = fe_sub(x, y); break;
            case 2: r = fe_mul(x, y); break;
            case 3: r = fe_inv(x); break;
            default: r = fe_is_zero(x) ? fe_make(0, 0) : fe_pow_u128(x, y.lo, y.hi); break;
        }
    } else {
        switch (op) {
            case 0: r = portable::fe_add(x, y); break;
            case 1: r = portable::fe_sub(x, y); break;
            case 2: r = portable::fe_mul(x, y); break;
            case 3: r = portable::fe_inv(x); break;
            default: r = fe_is_zero(x) ? fe_make(0, 0) : portable::fe_pow_u128(x, y.lo, y.hi); break;
        }
    }
    out[i] = r;
}

// out[i] = sum_j a[len i + j] * b[len i + j] for a runtime len (1..128): the 288-bit accumulation of the constraint kernel's Acc and of
// the per-register linear combinations, reduced once
__global__ void field_dot_kernel(const fe *a, const fe *b, fe *out, unsigned long long groups, unsigned len) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= groups) return;
    const fe *x = a + i * len, *y = b + i * len;
    fe_wide w;
    wide_set(w, DG_MUL_WIDE(x[0], y[0]));
    for (unsigned j = 1; j < len; j++) wide_add(w, DG_MUL_WIDE(x[j], y[j]));
    out[i] = DG_REDUCE_WIDE(w);
}

__global__ void fill_kernel(uint4 *p, size_t n, unsigned v) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = make_uint4(v, v + 1, v + 2, v + 3);
}

// Single-process multi-GPU (dg_init_devices): the proof is sharded exactly as in the one-process-per-GPU mode, but the ranks are host
// threads of this process, each bound to its own device context and NCCL communicator.  Rank 0 runs on the calling thread.
template <typename F>
static Proof *prove_on_all_devices(F &&prove_rank, dg_prove_stats_t *stats) {
    const int n = ctx_device_count();
    std::vector<Proof *> res(n, nullptr);
    std::vector<int> codes(n, 0);
    std::vector<std::string> msgs(n);
    auto run = [&](int g) {
        try {
            Context &cg = ctx_of(g);
            ctx_bind(&cg);
            res[g] = prove_rank(cg, g == 0 ? stats : nullptr);
        } catch (const dg::Error &e) { codes[g] = e.code; msgs[g] = e.what(); }
        catch (const std::exception &e) { codes[g] = DG_ERR_INVALID; msgs[g] = e.what(); }
    };
    std::vector<std::thread> th;
    for (int g = 1; g < n; g++) th.emplace_back(run, g);
    run(0);
    for (auto &t : th) t.join();
    ctx_bind(&ctx_of(0));
    for (int g = 0; g < n; g++)
        if (codes[g] != 0) {
            for (auto *p : res) delete p;
            throw Error(codes[g], "rank " + std::to_string(g) + ": " + msgs[g]);
        }
    for (int g = 1; g < n; g++) {
        const bool same = res[g] && res[g]->bytes == res[0]->bytes;
        delete res[g];
        if (!same) { delete res[0]; throw Error(DG_ERR_CUDA, "ranks produced different proofs"); }
    }
    return res[0];
}

extern "C" {

int dg_init(int device) { return guarded([&] { ctx_init(device); }); }
int dg_init_devices(int n_devices) {
    return guarded([&] {
        DG_REQUIRE(n_devices == 1 || ctx().mem_limit == 0, "a memory limit applies to one GPU: clear it (dg_set_memory_limit(0)) before spanning several");
        ctx_init_devices(n_devices);
    });
}
const char *dg_last_error(void) { return t_last_error.c_str(); }

int dg_device_info(char *name, size_t cap, int *sm_count, size_t *total_mem) {
    return guarded([&] {
        Context &c = ctx();
        cudaDeviceProp prop;
        DG_CUDA(cudaGetDeviceProperties(&prop, c.device));
        if (name && cap) { strncpy(name, prop.name, cap - 1); name[cap - 1] = 0; }
        if (sm_count) *sm_count = prop.multiProcessorCount;
        if (total_mem) *total_mem = prop.totalGlobalMem;
    });
}

// ---- device memory -------------------------------------------------------------------------------------------------------
int dg_dev_alloc(void **ptr, size_t bytes) { return guarded([&] { ctx(); DG_CUDA(cudaMalloc(ptr, bytes)); }); }
int dg_dev_free(void *ptr) { return guarded([&] { ctx(); DG_CUDA(cudaFree(ptr)); }); }
int dg_dev_upload(void *dst, const void *src, size_t bytes) {
    return guarded([&] { Context &c = ctx(); DG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c.stream)); DG_CUDA(cudaStreamSynchronize(c.stream)); });
}
int dg_dev_download(void *dst, const void *src, size_t bytes) {
    return guarded([&] { Context &c = ctx(); DG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c.stream)); DG_CUDA(cudaStreamSynchronize(c.stream)); });
}
int dg_dev_sync(void) { return guarded([&] { DG_CUDA(cudaStreamSynchronize(ctx().stream)); }); }
int dg_dev_flush_l2(void) {
    return guarded([&] {
        Context &c = ctx();
        const size_t bytes = (size_t)256 << 20;
        c.l2_scratch.ensure(bytes, true);
        fill_kernel<<<(unsigned)(bytes / 16 / 256), 256, 0, c.stream>>>(c.l2_scratch.as<uint4>(), bytes / 16, 7u); c.launches++;
        DG_CUDA(cudaGetLastError());
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}

// ---- device-resident building blocks ----------------------------------------------------------------------------------------
int dg_dev_ntt(void *d_values, uint32_t log_n, uint32_t batch, int inverse, float *ms) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        c.twiddle(log_n, inverse != 0);       // table setup outside the timed region
        if (log_n > 20) c.twiddle(log_n - (log_n + 2) / 3, inverse != 0);
        c.ntt_tmp.ensure(((size_t)16 << log_n) * std::min<size_t>(batch, std::max<size_t>(1, ((size_t)1 << 30) / ((size_t)16 << log_n))), true);
        EventTimer t(c.stream, ms);
        ntt_batch(c, (const fe *)d_values, (fe *)d_values, log_n, batch, (size_t)1 << log_n, (size_t)1 << log_n, inverse != 0);
        t.stop();
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
int dg_dev_lde(const void *d_polys, void *d_ext, uint32_t log_n, uint32_t log_blowup, uint32_t batch, float *ms) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        c.twiddle(log_n + log_blowup, false);
        c.twiddle(log_n, false);
        if (log_n > 20) c.twiddle(log_n - (log_n + 2) / 3, false);
        EventTimer t(c.stream, ms);
        lde_batch(c, (const fe *)d_polys, (fe *)d_ext, log_n, log_blowup, 1, batch, (size_t)1 << log_n, (size_t)1 << (log_n + log_blowup));
        t.stop();
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
int dg_dev_merkle_build(const void *d_leaves, uint64_t n_leaves, void *d_nodes, float *ms) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        EventTimer t(c.stream, ms);
        merkle_build(c, d_leaves, d_nodes, n_leaves);
        t.stop();
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
int dg_dev_merkle_build_with(int hash, const void *d_leaves, uint64_t n_leaves, void *d_nodes, float *ms) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        EventTimer t(c.stream, ms);
        alg_merkle_build(c, hash, d_leaves, d_nodes, n_leaves);
        t.stop();
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
int dg_dev_hash_rows(const void *d_ext, uint32_t width, uint32_t log_n, uint32_t log_blowup, void *d_leaves, float *ms) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(width >= 1 && width < 128, "width must be in 1..127");
        EventTimer t(c.stream, ms);
        hash_trace_rows(c, (const fe *)d_ext, d_leaves, (int)width, (int)log_n, (int)log_blowup);
        t.stop();
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}

// ---- host-memory building blocks -----------------------------------------------------------------------------------------------
int dg_ntt(uint8_t *values, uint32_t log_n, uint32_t batch, int inverse) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(values, "null buffer");
        DG_REQUIRE(log_n >= 1 && log_n <= 30 && batch >= 1, "invalid transform size");
        const size_t bytes = ((size_t)16 << log_n) * batch;
        DevBuf d(bytes);
        DG_CUDA(cudaMemcpyAsync(d.p, values, bytes, cudaMemcpyHostToDevice, c.stream));
        ntt_batch(c, d.as<fe>(), d.as<fe>(), log_n, batch, (size_t)1 << log_n, (size_t)1 << log_n, inverse != 0);
        DG_CUDA(cudaMemcpyAsync(values, d.p, bytes, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
int dg_lde(const uint8_t *values, uint8_t *extended, uint32_t log_n, uint32_t log_blowup, uint32_t batch) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(values && extended, "null buffer");
        DG_REQUIRE(log_n >= 1 && log_blowup >= 1 && log_n + log_blowup <= 30 && batch >= 1 && batch <= 65535, "invalid extension size");
        const size_t n = (size_t)1 << log_n, N = n << log_blowup;
        DevBuf d_in(n * batch * 16), d_ext(N * batch * 16), d_out(N * batch * 16);
        DG_CUDA(cudaMemcpyAsync(d_in.p, values, n * batch * 16, cudaMemcpyHostToDevice, c.stream));
        ntt_batch(c, d_in.as<fe>(), d_in.as<fe>(), log_n, batch, n, n, true);                 // interpolate (trace_table.rs:158)
        lde_batch(c, d_in.as<fe>(), d_ext.as<fe>(), log_n, log_blowup, 1, batch, n, N);       // evaluate over the LDE domain (:165)
        coset_to_logical_kernel<<<dim3((unsigned)((N + 255) / 256), batch), 256, 0, c.stream>>>(d_ext.as<fe>(), d_out.as<fe>(), log_n, log_blowup); c.launches++;
        DG_CUDA(cudaGetLastError());
        DG_CUDA(cudaMemcpyAsync(extended, d_out.p, N * batch * 16, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
int dg_merkle_build(const uint8_t *leaves, uint64_t n_leaves, uint8_t *nodes) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(leaves && nodes, "null buffer");
        DG_REQUIRE(n_leaves >= 2 && (n_leaves & (n_leaves - 1)) == 0, "number of leaves must be a power of 2 and >= 2");
        DevBuf d_l(n_leaves * 32), d_n(n_leaves * 32);
        DG_CUDA(cudaMemcpyAsync(d_l.p, leaves, n_leaves * 32, cudaMemcpyHostToDevice, c.stream));
        merkle_build(c, d_l.p, d_n.p, n_leaves);
        DG_CUDA(cudaMemcpyAsync(nodes, d_n.p, n_leaves * 32, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
// the VM's hasher takes field elements only (a tape value >= M fails its execution): rejects the first of n items of `width` little-endian
// u128 elements that holds one
static void require_canonical(const uint8_t *items, uint64_t n, unsigned width, const char *what) {
    DG_REQUIRE(items, "null buffer");
    for (uint64_t k = 0; k < n * width; k++) {
        uint64_t lo, hi;
        memcpy(&lo, items + 16 * k, 8);
        memcpy(&hi, items + 16 * k + 8, 8);
        if (hi == DG_M_HI && lo >= DG_M_LO)
            throw dg::Error(DG_ERR_INVALID, std::string(what) + " " + std::to_string(k / width) + " element " + std::to_string(k % width) +
                                                " is not a field element (>= M)");
    }
}
int dg_hash64(int hash, const uint8_t *messages64, uint64_t n, uint8_t *digests32) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(hash >= 0 && hash <= 3, "hash id must be 0 (blake3), 1 (rescue), 2 (poseidon) or 3 (hasher)");
        if (n == 0) return;
        DG_REQUIRE(messages64 && digests32, "null buffer");
        if (hash == DG_HASH_HASHER) require_canonical(messages64, n, 4, "message");
        DevBuf d_in(n * 64), d_out(n * 32);
        DG_CUDA(cudaMemcpyAsync(d_in.p, messages64, n * 64, cudaMemcpyHostToDevice, c.stream));
        alg_hash64(c, hash, d_in.p, d_out.p, n);
        DG_CUDA(cudaMemcpyAsync(digests32, d_out.p, n * 32, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
int dg_merkle_build_with(int hash, const uint8_t *leaves, uint64_t n_leaves, uint8_t *nodes) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(n_leaves >= 2 && (n_leaves & (n_leaves - 1)) == 0, "number of leaves must be a power of 2 and >= 2");
        if (hash == DG_HASH_HASHER) require_canonical(leaves, n_leaves, 2, "leaf");
        DevBuf d_l(n_leaves * 32), d_n(n_leaves * 32);
        DG_CUDA(cudaMemcpyAsync(d_l.p, leaves, n_leaves * 32, cudaMemcpyHostToDevice, c.stream));
        alg_merkle_build(c, hash, d_l.p, d_n.p, n_leaves);
        DG_CUDA(cudaMemcpyAsync(nodes, d_n.p, n_leaves * 32, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}

// ---- Merkle trees that stay on the GPU (tree.cu) ---------------------------------------------------------------------------------------
static void require_tree_shape(int hash, uint64_t n_leaves) {
    DG_REQUIRE(hash >= 0 && hash <= 3, "hash id must be 0 (blake3), 1 (rescue), 2 (poseidon) or 3 (hasher)");
    DG_REQUIRE(n_leaves >= 2 && (n_leaves & (n_leaves - 1)) == 0, "number of leaves must be a power of 2 and >= 2");
}
static void require_tree_indexes(const Tree &t, const uint64_t *indexes, uint32_t count) {
    for (uint32_t k = 0; k < count; k++)
        if (indexes[k] >= t.L)
            throw Error(DG_ERR_INVALID, "index " + std::to_string(indexes[k]) + " (entry " + std::to_string(k) + ") is not a leaf of a tree of " +
                                            std::to_string(t.L) + " leaves");
}
// a new tree on the primary context, its buffers from the pool; `fill` copies the leaves in
static Tree *new_tree(int hash, uint64_t n_leaves, const std::function<void(Context &, Tree &)> &fill) {
    Context &c = ctx();
    std::lock_guard<std::mutex> lk(c.mu);
    std::unique_ptr<Tree> t(new Tree());
    t->hash = hash;
    t->L = n_leaves;
    t->leaves.alloc(n_leaves * 32, true);
    t->nodes.alloc(n_leaves * 32, true);
    fill(c, *t);
    tree_build(c, *t);
    return t.release();
}
int dg_tree_new(int hash, const uint8_t *leaves32, uint64_t n_leaves, dg_tree_t **tree) {
    return guarded([&] {
        DG_REQUIRE(tree && leaves32, "null argument");
        *tree = nullptr;
        require_tree_shape(hash, n_leaves);
        if (hash == DG_HASH_HASHER) require_canonical(leaves32, n_leaves, 2, "leaf");
        *tree = (dg_tree_t *)new_tree(hash, n_leaves, [&](Context &c, Tree &t) {
            DG_CUDA(cudaMemcpyAsync(t.leaves.p, leaves32, n_leaves * 32, cudaMemcpyHostToDevice, c.stream));
        });
    });
}
int dg_tree_new_device(int hash, const void *d_leaves32, uint64_t n_leaves, dg_tree_t **tree) {
    return guarded([&] {
        DG_REQUIRE(tree && d_leaves32, "null argument");
        *tree = nullptr;
        require_tree_shape(hash, n_leaves);
        *tree = (dg_tree_t *)new_tree(hash, n_leaves, [&](Context &c, Tree &t) {
            DG_CUDA(cudaMemcpyAsync(t.leaves.p, d_leaves32, n_leaves * 32, cudaMemcpyDeviceToDevice, c.stream));
        });
    });
}
int dg_tree_info(const dg_tree_t *tree, int *hash, uint64_t *n_leaves, uint8_t root32[32]) {
    return guarded([&] {
        DG_REQUIRE(tree, "null tree");
        const Tree &t = *(const Tree *)tree;
        if (hash) *hash = t.hash;
        if (n_leaves) *n_leaves = t.L;
        if (root32) memcpy(root32, t.root, 32);
    });
}
int dg_tree_paths(const dg_tree_t *tree, const uint64_t *indexes, uint32_t count, uint8_t *paths32) {
    return guarded([&] {
        DG_REQUIRE(tree, "null tree");
        DG_REQUIRE(count == 0 || (indexes && paths32), "null buffer");
        const Tree &t = *(const Tree *)tree;
        require_tree_indexes(t, indexes, count);
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        tree_paths(c, t, indexes, count, paths32);
    });
}
int dg_tree_membership_inputs(const dg_tree_t *tree, int program, const uint64_t *indexes, uint32_t count, void *d_values, uint64_t cap,
                              dg_device_inputs_t *out) {
    return guarded([&] {
        DG_REQUIRE(tree && out, "null argument");
        DG_REQUIRE(program == DG_PATH_SMPATH || program == DG_PATH_PMPATH, "program must be DG_PATH_SMPATH (0) or DG_PATH_PMPATH (1)");
        DG_REQUIRE(count == 0 || indexes, "null buffer");
        const Tree &t = *(const Tree *)tree;
        DG_REQUIRE(t.hash == DG_HASH_HASHER, "membership inputs are paths of the VM's hash: a tree of hash 3 (hasher), not " + std::to_string(t.hash));
        require_tree_indexes(t, indexes, count);
        const bool pm = program == DG_PATH_PMPATH;
        const uint64_t d = (uint64_t)ceil_log2(t.L), per = pm ? 2 * d + 3 : 4 * d + 2;
        out->n_values = per * count;
        if (!d_values) return;
        DG_REQUIRE(cap >= out->n_values, "d_values holds " + std::to_string(cap) + " values, the inputs need " + std::to_string(out->n_values));
        DG_REQUIRE(((uintptr_t)d_values & 15) == 0, "d_values is not 16-byte aligned");
        DG_REQUIRE(out->public_first && out->n_public && out->secret_a_first && out->n_secret_a && out->secret_b_first && out->n_secret_b,
                   "null offset or count array in out");
        uint64_t *pf = (uint64_t *)out->public_first, *af = (uint64_t *)out->secret_a_first, *bf = (uint64_t *)out->secret_b_first;
        uint32_t *np = (uint32_t *)out->n_public;
        uint64_t *na = (uint64_t *)out->n_secret_a, *nb = (uint64_t *)out->n_secret_b;
        const uint64_t tape = pm ? d + 1 : 2 * d + 1, pub = pm ? 1 : 0;
        for (uint32_t k = 0; k < count; k++) {
            pf[k] = k * per; np[k] = (uint32_t)pub;
            af[k] = k * per + pub; na[k] = tape;
            bf[k] = k * per + pub + tape; nb[k] = tape;
        }
        out->d_values = d_values;
        if (count == 0) return;
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        require_device_memory(c, d_values, "d_values");
        tree_membership_inputs(c, t, pm, indexes, count, (fe *)d_values);
    });
}
int dg_tree_update(dg_tree_t *tree, const uint64_t *indexes, const uint8_t *leaves32, uint32_t count, uint8_t root32[32]) {
    return guarded([&] {
        DG_REQUIRE(tree, "null tree");
        DG_REQUIRE(count == 0 || (indexes && leaves32), "null buffer");
        Tree &t = *(Tree *)tree;
        require_tree_indexes(t, indexes, count);
        if (t.hash == DG_HASH_HASHER && count) require_canonical(leaves32, count, 2, "leaf");
        if (count) {
            const TreePlan plan = plan_tree_update(indexes, count, t.L);
            Context &c = ctx();
            std::lock_guard<std::mutex> lk(c.mu);
            tree_update(c, t, plan, leaves32);
        }
        if (root32) memcpy(root32, t.root, 32);
    });
}
int dg_tree_read(const dg_tree_t *tree, uint8_t *leaves32, uint8_t *nodes32) {
    return guarded([&] {
        DG_REQUIRE(tree, "null tree");
        const Tree &t = *(const Tree *)tree;
        if (!leaves32 && !nodes32) return;
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        if (leaves32) DG_CUDA(cudaMemcpyAsync(leaves32, t.leaves.p, t.L * 32, cudaMemcpyDeviceToHost, c.stream));
        if (nodes32) DG_CUDA(cudaMemcpyAsync(nodes32, t.nodes.p, t.L * 32, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
void dg_tree_free(dg_tree_t *tree) {
    if (!tree) return;
    guarded([&] {                         // a tree exists only on a context, so ctx() does not throw here
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        delete (Tree *)tree;              // the buffers go back to the pool in stream order
    });
}

// ---- batch proofs of a tree, and verification of paths and batch proofs (tree.cu) ------------------------------------------------------
// prove_batch's panics in the crate's order: map_indexes asserts index <= L, then that no index repeats; an index of L then fails the
// slice index, named here as map_indexes names the others
static void require_batch_indexes(const uint64_t *indexes, uint32_t count, uint64_t L) {
    for (uint32_t k = 0; k < count; k++)
        if (indexes[k] > L) throw Error(DG_ERR_INVALID, "invalid index " + std::to_string(indexes[k]));
    std::vector<uint64_t> sorted(indexes, indexes + count);
    std::sort(sorted.begin(), sorted.end());
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) throw Error(DG_ERR_INVALID, "repeating indexes detected");
    if (count && sorted.back() == L) throw Error(DG_ERR_INVALID, "invalid index " + std::to_string(L));
}
int dg_tree_prove_batch(const dg_tree_t *tree, const uint64_t *indexes, uint32_t count, uint8_t *proof_out, size_t cap, size_t *len) {
    return guarded([&] {
        DG_REQUIRE(tree && len, "null argument");
        DG_REQUIRE(count == 0 || indexes, "null buffer");
        const Tree &t = *(const Tree *)tree;
        require_batch_indexes(indexes, count, t.L);
        const fs::BatchPlan plan = fs::plan_batch_proof(std::vector<uint64_t>(indexes, indexes + count), t.L);
        *len = batch_proof_len(plan);
        if (!proof_out) return;
        if (cap < *len) throw Error(DG_ERR_INVALID, "proof buffer too small: the proof has " + std::to_string(*len) + " bytes");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        tree_prove_batch(c, t, plan, proof_out);
    });
}

// the first of n little-endian u128 elements that is >= M, or -1
static int64_t first_noncanonical(const uint8_t *elements, size_t n) {
    for (size_t k = 0; k < n; k++) {
        uint64_t lo, hi;
        memcpy(&lo, elements + 16 * k, 8);
        memcpy(&hi, elements + 16 * k + 8, 8);
        if (hi == DG_M_HI && lo >= DG_M_LO) return (int64_t)k;
    }
    return -1;
}
static std::string noncanonical_message(const std::string &what, int64_t k) {
    return what + " element " + std::to_string(k) + " is not a field element (>= M)";
}
static void require_hash_id(int hash) {
    DG_REQUIRE(hash >= 0 && hash <= 3, "hash id must be 0 (blake3), 1 (rescue), 2 (poseidon) or 3 (hasher)");
}
int dg_merkle_verify_paths(int hash, const uint8_t *roots32, uint32_t n_roots, const uint64_t *indexes, const uint8_t *paths32,
                           uint32_t entries, uint32_t count, int *status) {
    return guarded([&] {
        require_hash_id(hash);
        DG_REQUIRE(entries >= 2 && entries <= 64, "a path has 2 to 64 entries");
        DG_REQUIRE(n_roots == 1 || n_roots == count, "n_roots must be 1 or count");
        DG_REQUIRE(roots32 && indexes && paths32 && status, "null array");
        t_batch_messages.assign(count, std::string());
        if (count == 0) return;
        // the algebraic hashes take field elements only: a path with an entry element >= M is malformed input.  Its digests are computed with
        // the others (the kernels' addresses do not depend on the values) and its verdict is replaced.
        std::vector<uint8_t> valid(count, 1);
        if (hash != DG_HASH_BLAKE3)
            for (uint32_t k = 0; k < count; k++) {
                const int64_t e = first_noncanonical(paths32 + (size_t)32 * entries * k, 2 * (size_t)entries);
                if (e < 0) continue;
                valid[k] = 0;
                t_batch_messages[k] = noncanonical_message("entry " + std::to_string(e / 2), e % 2);
            }
        std::vector<uint8_t> accepted(count);
        {
            Context &c = ctx();
            std::lock_guard<std::mutex> lk(c.mu);
            merkle_verify_paths(c, hash, roots32, n_roots != 1, indexes, paths32, entries, count, accepted.data());
        }
        for (uint32_t k = 0; k < count; k++) {
            status[k] = !valid[k] ? DG_ERR_INVALID : accepted[k] ? DG_OK : DG_ERR_REJECTED;
            if (valid[k] && !accepted[k]) t_batch_messages[k] = "the path does not lead to the root";
        }
    });
}
int dg_merkle_verify_batch(int hash, uint32_t count, const uint8_t *roots32, const uint64_t *const *indexes, const uint32_t *n_indexes,
                           const uint8_t *const *proofs, const size_t *proof_lens, int *status) {
    return guarded([&] {
        require_hash_id(hash);
        DG_REQUIRE(roots32 && indexes && n_indexes && proofs && proof_lens && status, "null array");
        t_batch_messages.assign(count, std::string());
        // host: parse, check the elements, plan; the entries decided here never reach the device
        std::vector<BatchMerkleProof> parsed(count);
        std::vector<BatchCheck> checks;
        std::vector<uint32_t> of;
        std::vector<const uint8_t *> roots;
        for (uint32_t i = 0; i < count; i++) {
            std::string &msg = t_batch_messages[i];
            BatchMerkleProof &p = parsed[i];
            status[i] = DG_ERR_INVALID;
            if ((n_indexes[i] && !indexes[i]) || (proof_lens[i] && !proofs[i])) { msg = "null indexes or proof bytes"; continue; }
            if (!read_batch_proof(proofs[i], proof_lens[i], p)) {
                msg = "malformed proof bytes (bincode layout of BatchMerkleProof, merkle.rs:14-18)";
                continue;
            }
            if (p.depth > 63) { msg = "attempt to multiply with overflow"; continue; }           // usize::pow(2, depth)
            if (hash != DG_HASH_BLAKE3) {
                for (size_t v = 0; v < p.values.size() && msg.empty(); v++) {
                    const int64_t e = first_noncanonical(p.values[v].data(), 2);
                    if (e >= 0) msg = noncanonical_message("value " + std::to_string(v), e);
                }
                for (size_t s = 0; s < p.nodes.size() && msg.empty(); s++)
                    for (size_t j = 0; j < p.nodes[s].size() && msg.empty(); j++) {
                        const int64_t e = first_noncanonical(p.nodes[s][j].data(), 2);
                        if (e >= 0) msg = noncanonical_message("node " + std::to_string(j) + " of slot " + std::to_string(s), e);
                    }
                if (!msg.empty()) continue;
            }
            std::vector<uint32_t> bases;
            uint32_t next = (uint32_t)p.values.size();
            for (auto &slot : p.nodes) { bases.push_back(next); next += (uint32_t)slot.size(); }
            MerklePlan plan = plan_verify_batch(std::vector<uint64_t>(indexes[i], indexes[i] + n_indexes[i]), p.depth, p.values.size(), 0, p.nodes,
                                                bases, next, 0, 63);
            if (!plan.ok) {
                status[i] = plan.panic ? DG_ERR_INVALID : DG_ERR_REJECTED;
                msg = plan.why;
                continue;
            }
            checks.push_back(BatchCheck{&p, std::move(plan)});
            of.push_back(i);
            roots.push_back(roots32 + (size_t)32 * i);
        }
        if (checks.empty()) return;
        std::vector<uint8_t> accepted(checks.size());
        {
            Context &c = ctx();
            std::lock_guard<std::mutex> lk(c.mu);
            merkle_verify_batch(c, hash, checks, roots.data(), accepted.data());
        }
        for (size_t j = 0; j < checks.size(); j++) {
            status[of[j]] = accepted[j] ? DG_OK : DG_ERR_REJECTED;
            if (!accepted[j]) t_batch_messages[of[j]] = "the proof does not lead to the root";
        }
    });
}

int dg_hash_rows(const uint8_t *columns, uint32_t width, uint64_t rows, uint8_t *digests) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(columns && digests, "null buffer");
        DG_REQUIRE(width >= 1 && width < 128 && rows >= 1, "invalid matrix shape");
        DevBuf d_c((size_t)width * rows * 16), d_d(rows * 32);
        DG_CUDA(cudaMemcpyAsync(d_c.p, columns, (size_t)width * rows * 16, cudaMemcpyHostToDevice, c.stream));
        // reuse the trace-row kernel with a single "coset": physical position == logical row
        hash_rows_plain(c, d_c.as<fe>(), d_d.p, (int)width, rows);
        DG_CUDA(cudaMemcpyAsync(digests, d_d.p, rows * 32, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
int dg_find_pow_nonce(const uint8_t seed[32], uint32_t grinding_factor, uint64_t *nonce, uint8_t new_seed[32]) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(seed && nonce, "null argument");
        DG_REQUIRE(grinding_factor <= 32, "grinding factor cannot be greater than 32");
        std::array<uint8_t, 32> s;
        memcpy(s.data(), seed, 32);
        const unsigned long long n = pow_search_batch(c, {s}, {grinding_factor})[0];
        *nonce = n;
        if (new_seed) pow_hash(seed, n, new_seed);
    });
}
int dg_field_op(int op, int impl, const uint8_t *a, const uint8_t *b, uint8_t *out, uint64_t n) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(a && out && n >= 1 && op >= 0 && op <= 6, "invalid argument");
        DG_REQUIRE(b || op == 3, "second operand missing");
        DevBuf da(n * 16), db(n * 16), dout(n * 16);
        DG_CUDA(cudaMemcpyAsync(da.p, a, n * 16, cudaMemcpyHostToDevice, c.stream));
        if (b) DG_CUDA(cudaMemcpyAsync(db.p, b, n * 16, cudaMemcpyHostToDevice, c.stream));
        field_op_kernel<<<(unsigned)((n + 127) / 128), 128, 0, c.stream>>>(op, impl, da.as<fe>(), b ? db.as<fe>() : nullptr, dout.as<fe>(), n); c.launches++;
        DG_CUDA(cudaGetLastError());
        DG_CUDA(cudaMemcpyAsync(out, dout.p, n * 16, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
int dg_field_dot(const uint8_t *a, const uint8_t *b, uint8_t *out, uint64_t groups, uint32_t len) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(a && b && out && groups >= 1, "invalid argument");
        DG_REQUIRE(len >= 1 && len <= 128, "group length must be in 1..128");
        const size_t n = groups * len;
        DevBuf da(n * 16), db(n * 16), dout(groups * 16);
        DG_CUDA(cudaMemcpyAsync(da.p, a, n * 16, cudaMemcpyHostToDevice, c.stream));
        DG_CUDA(cudaMemcpyAsync(db.p, b, n * 16, cudaMemcpyHostToDevice, c.stream));
        field_dot_kernel<<<(unsigned)((groups + 127) / 128), 128, 0, c.stream>>>(da.as<fe>(), db.as<fe>(), dout.as<fe>(), groups, len); c.launches++;
        DG_CUDA(cudaGetLastError());
        DG_CUDA(cudaMemcpyAsync(out, dout.p, groups * 16, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    });
}
int dg_eval_transitions(const uint8_t *ext16, uint32_t count, uint32_t ctx_depth, uint32_t loop_depth, uint32_t stack_depth, uint32_t log_n,
                        uint32_t log_blowup, const uint8_t *seeds32, const uint8_t *coefs16, int check, uint8_t *out16, uint32_t *first_violation) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(ext16 && out16 && first_violation && (seeds32 || coefs16), "null argument");
        DG_REQUIRE(count >= 1 && count <= 65535, "count must be in 1..65535");
        DG_REQUIRE(TraceShape::in_range(ctx_depth, loop_depth, stack_depth), "register shape out of range");
        DG_REQUIRE(log_n >= 4 && log_blowup >= 4 && log_blowup <= 8 && log_n + log_blowup <= 20, "trace length or extension factor out of range");
        const TraceShape shape(ctx_depth, loop_depth, stack_depth);
        const int w = shape.w, T = shape.T;
        const size_t n = (size_t)1 << log_n, b = (size_t)1 << log_blowup, N = n << log_blowup, E = 8 * n;

        // per entry [coefA | coefB] in evaluation order, drawn as the prover draws them (no public inputs or outputs) or given
        std::vector<fe> coef((size_t)count * 2 * T);
        if (coefs16) {
            memcpy(coef.data(), coefs16, coef.size() * 16);
        } else {
            const fe no_hash[2] = {fe_make(0, 0), fe_make(0, 0)};
            for (uint32_t q = 0; q < count; q++) {
                fs::ConstraintCoefficients cc = fs::draw_constraint_coefficients(seeds32 + 32 * (size_t)q, shape, {}, {}, fe_make(0, 0), no_hash);
                std::copy(cc.coefA.begin(), cc.coefA.end(), coef.begin() + (size_t)q * 2 * T);
                std::copy(cc.coefB.begin(), cc.coefB.end(), coef.begin() + (size_t)q * 2 * T + T);
            }
        }
        // logical LDE order (index k * b + c) -> the prover's coset-major slab ([c][k])
        std::vector<fe> slab((size_t)count * w * N);
        for (size_t col = 0; col < (size_t)count * w; col++)
            for (size_t k = 0; k < n; k++)
                for (size_t cs = 0; cs < b; cs++) memcpy(&slab[col * N + cs * n + k], ext16 + (col * N + k * b + cs) * 16, 16);

        const fe *periodic = periodic_table(c);
        DevBuf d_ext(slab.size() * 16), d_coef(coef.size() * 16), d_out((size_t)count * E * 16), d_violation((size_t)4 * count);
        DG_CUDA(cudaMemcpyAsync(d_ext.p, slab.data(), slab.size() * 16, cudaMemcpyHostToDevice, c.stream));
        DG_CUDA(cudaMemcpyAsync(d_coef.p, coef.data(), coef.size() * 16, cudaMemcpyHostToDevice, c.stream));
        DG_CUDA(cudaMemsetAsync(d_violation.p, 0, (size_t)4 * count, c.stream));
        AirParams P = shape.air_params(n);
        P.log_blowup = log_blowup;
        P.ext = d_ext.as<fe>(); P.col_stride = N;
        P.c8_base = 0; P.num_c8 = 8;
        P.t_ev = d_out.as<fe>();
        P.periodic = periodic;
        P.coefA = d_coef.as<fe>(); P.coefB = d_coef.as<fe>() + T;
        P.twN = c.twiddle(log_n + log_blowup, false);
        P.violation = d_violation.as<unsigned>();
        P.verify_mode = check ? 0 : 1;          // verify mode: no trace-domain check, a value at every step
        P.ext_stride = (size_t)w * N; P.t_ev_stride = E; P.coef_stride = 2 * T;
        launch_constraint_eval(c, P, (int)count);

        std::vector<fe> t_ev((size_t)count * E);
        std::vector<unsigned> violation(count);
        DG_CUDA(cudaMemcpyAsync(t_ev.data(), d_out.p, t_ev.size() * 16, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaMemcpyAsync(violation.data(), d_violation.p, (size_t)4 * count, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
        // coset-major [c8][k] -> step order s = 8 k + c8
        for (size_t q = 0; q < count; q++)
            for (size_t c8 = 0; c8 < 8; c8++)
                for (size_t k = 0; k < n; k++) memcpy(out16 + (q * E + 8 * k + c8) * 16, &t_ev[q * E + c8 * n + k], 16);
        for (uint32_t q = 0; q < count; q++) first_violation[q] = violation[q] ? (uint32_t)violation_step(violation[q]) + 1 : 0;
    });
}

// ---- prover ------------------------------------------------------------------------------------------------------------------------
// the options of a call: one set for every entry (per_entry false), or options[i] for entry i, each checked on the host with `what i: `
// before the message (dg_*_with_options)
static std::vector<dg_options_t> call_options(const dg_options_t *options, uint32_t count, bool per_entry, const char *what) {
    if (!per_entry) return std::vector<dg_options_t>(count, *options);
    for (uint32_t i = 0; i < count; i++) {
        try {
            check_options(options[i]);
        } catch (const Error &e) {
            throw Error(e.code, std::string(what) + " " + std::to_string(i) + ": " + e.what());
        }
    }
    return std::vector<dg_options_t>(options, options + count);
}

// A prove or trace-check call as its entry received it: every trace host (dg_trace_t columns) or every trace on the device, and trace
// i's n_inputs[i] public inputs at inputs16[i] and n_outputs[i] outputs at outputs16[i] (16 bytes each; a null count array: none).
// one_shape: how the messages of a call of one shape name it ("batch" or "call": dg_prove, dg_prove_device, dg_prove_batch*,
// dg_check_traces*); null for the per-trace calls (dg_prove_traces*), whose traces may differ in shape and whose messages name the trace.
struct ProveCall {
    std::vector<TraceRef> traces;
    bool host;
    const char *one_shape;
    const uint8_t *const *inputs16;
    const uint32_t *n_inputs;
    const uint8_t *const *outputs16;
    const uint32_t *n_outputs;
};

// Every prove and trace-check entry runs this once, before it touches the device.  Each trace in input order: the form of a host trace
// (the shape of trace 0 in a call of one shape, columns, 16..127 registers), its length, its register shape (TraceShape::of_trace), its
// registers and its public inputs / outputs; then the options of a prove call, one set or one per trace (per_trace).  A failure is
// DG_ERR_INVALID, with `trace i: ` before the message of a per-trace call's trace and of per-trace options.  Returns every trace's options.
static std::vector<dg_options_t> check_prove_call(const ProveCall &x, const dg_options_t *options = nullptr, bool per_trace = false) {
    const TraceRef &t0 = x.traces[0];
    for (uint32_t i = 0; i < x.traces.size(); i++) {
        const TraceRef &t = x.traces[i];
        try {
            if (x.host) {
                if (x.one_shape)
                    DG_REQUIRE(t.shape() == t0.shape() && t.length == t0.length,
                               std::string("all traces of a ") + x.one_shape + " must have the same width, length, context depth and loop depth");
                DG_REQUIRE(t.host_cols && t.width >= 16 && t.width < 128, "invalid trace");
            }
            DG_REQUIRE(t.length >= 16 && (t.length & (t.length - 1)) == 0 && t.length <= (1ULL << 30),
                       "execution trace length must be a power of 2 and at least 16");
            TraceShape::of_trace(t.width, t.ctx_depth, t.loop_depth);
            if (x.host)
                for (uint32_t j = 0; j < t.width; j++) DG_REQUIRE(t.host_cols[j] != nullptr, "null register column");
            else
                DG_REQUIRE(t.d_regs, "null registers");
            const uint32_t ni = x.n_inputs ? x.n_inputs[i] : 0, no = x.n_outputs ? x.n_outputs[i] : 0;
            DG_REQUIRE(ni <= 8 && no <= 8, "cannot have more than 8 public inputs / outputs");
            DG_REQUIRE((ni == 0 || (x.inputs16 && x.inputs16[i])) && (no == 0 || (x.outputs16 && x.outputs16[i])), "null public inputs / outputs");
        } catch (const Error &e) {
            if (x.one_shape) throw;
            throw Error(e.code, "trace " + std::to_string(i) + ": " + e.what());
        }
    }
    if (!options) return {};
    if (!per_trace) check_options(*options);
    return call_options(options, (uint32_t)x.traces.size(), per_trace, "trace");
}

// the traces of a host call
static std::vector<TraceRef> host_traces(const dg_trace_t *traces, uint32_t count) {
    std::vector<TraceRef> refs(count);
    for (uint32_t i = 0; i < count; i++) {
        const dg_trace_t &t = traces[i];
        refs[i].width = t.width; refs[i].length = t.length; refs[i].ctx_depth = t.ctx_depth; refs[i].loop_depth = t.loop_depth;
        refs[i].host_cols = t.columns;
    }
    return refs;
}
// the traces of a per-trace device call: trace i's registers at d_registers[i]
static std::vector<TraceRef> device_traces(const void *const *d_registers, const uint32_t *width, const uint64_t *length, const uint32_t *ctx_depth,
                                           const uint32_t *loop_depth, uint32_t count) {
    std::vector<TraceRef> refs(count);
    for (uint32_t i = 0; i < count; i++) {
        refs[i].width = width[i]; refs[i].length = length[i]; refs[i].ctx_depth = ctx_depth[i]; refs[i].loop_depth = loop_depth[i];
        refs[i].d_regs = (const fe *)d_registers[i];
    }
    return refs;
}

// Checks a prove call (check_prove_call) and proves it.  A batched call (batch) writes every trace's proof and status, and its message to
// the thread's dg_batch_message list.  dg_prove / dg_prove_device put the one proof in proofs_out[0] or throw its failure; when the
// library spans several devices every device proves it, sharded.
static void prove_call(const ProveCall &x, const dg_options_t *options, bool per_trace, bool batch, dg_proof_t **proofs_out, int *status,
                       dg_prove_stats_t *stats) {
    const std::vector<dg_options_t> opts = check_prove_call(x, options, per_trace);
    Context &c = ctx();
    std::lock_guard<std::mutex> lk(c.mu);
    if (batch) {
        t_batch_messages.clear();
        prove_traces(c, x.traces, x.inputs16, x.n_inputs, x.outputs16, x.n_outputs, opts, true, (Proof **)proofs_out, status, t_batch_messages,
                     stats);
        return;
    }
    auto prove = [&](Context &cg, dg_prove_stats_t *st) {
        Proof *proof = nullptr;
        int one = DG_OK;
        std::vector<std::string> messages;
        prove_traces(cg, x.traces, x.inputs16, x.n_inputs, x.outputs16, x.n_outputs, opts, false, &proof, &one, messages, st);
        if (one != DG_OK) throw Error(one, messages[0]);
        return proof;
    };
    *proofs_out = (dg_proof_t *)(ctx_device_count() > 1 ? prove_on_all_devices(prove, stats) : prove(c, stats));
}

int dg_prove(const dg_trace_t *trace, const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16, uint32_t n_outputs,
             const dg_options_t *options, dg_proof_t **proof_out, dg_prove_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(trace && options && proof_out, "null argument");
        prove_call({host_traces(trace, 1), true, "call", &inputs16, &n_inputs, &outputs16, &n_outputs},
                   options, false, false, proof_out, nullptr, stats);
    });
}
int dg_prove_device(const void *d_registers, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                    const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16, uint32_t n_outputs,
                    const dg_options_t *options, dg_proof_t **proof_out, dg_prove_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(d_registers && options && proof_out, "null argument");
        // several devices: the trace lives on device 0; the other devices read their columns over NVLink (peer access)
        prove_call({one_shape_traces((const fe *)d_registers, 1, width, length, ctx_depth, loop_depth), false, "call", &inputs16, &n_inputs,
                    &outputs16, &n_outputs}, options, false, false, proof_out, nullptr, stats);
    });
}
int dg_prove_batch(const dg_trace_t *traces, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                   const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t *options, dg_proof_t **proofs_out,
                   int *status, dg_prove_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "batch must hold at least one trace");
        DG_REQUIRE(traces && options && proofs_out && status, "null argument");
        prove_call({host_traces(traces, count), true, "batch", inputs16, n_inputs, outputs16, n_outputs},
                   options, false, true, proofs_out, status, stats);
    });
}
int dg_prove_batch_device(const void *d_registers, uint32_t count, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                          const uint8_t *const *inputs16, const uint32_t *n_inputs, const uint8_t *const *outputs16, const uint32_t *n_outputs,
                          const dg_options_t *options, dg_proof_t **proofs_out, int *status, dg_prove_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "batch must hold at least one trace");
        DG_REQUIRE(d_registers && options && proofs_out && status, "null argument");
        prove_call({one_shape_traces((const fe *)d_registers, count, width, length, ctx_depth, loop_depth), false, "batch", inputs16, n_inputs,
                    outputs16, n_outputs}, options, false, true, proofs_out, status, stats);
    });
}
int dg_prove_traces(const dg_trace_t *traces, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                    const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t *options, dg_proof_t **proofs_out,
                    int *status, dg_prove_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "batch must hold at least one trace");
        DG_REQUIRE(traces && options && proofs_out && status, "null argument");
        prove_call({host_traces(traces, count), true, nullptr, inputs16, n_inputs, outputs16, n_outputs},
                   options, false, true, proofs_out, status, stats);
    });
}
int dg_prove_traces_with_options(const dg_trace_t *traces, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                                 const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t *options, dg_proof_t **proofs_out,
                                 int *status, dg_prove_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "batch must hold at least one trace");
        DG_REQUIRE(traces && options && proofs_out && status, "null argument");
        prove_call({host_traces(traces, count), true, nullptr, inputs16, n_inputs, outputs16, n_outputs},
                   options, true, true, proofs_out, status, stats);
    });
}
int dg_prove_traces_device(const void *const *d_registers, const uint32_t *width, const uint64_t *length, const uint32_t *ctx_depth,
                           const uint32_t *loop_depth, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                           const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t *options, dg_proof_t **proofs_out,
                           int *status, dg_prove_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "batch must hold at least one trace");
        DG_REQUIRE(d_registers && width && length && ctx_depth && loop_depth && options && proofs_out && status, "null argument");
        prove_call({device_traces(d_registers, width, length, ctx_depth, loop_depth, count), false, nullptr, inputs16, n_inputs, outputs16,
                    n_outputs}, options, false, true, proofs_out, status, stats);
    });
}
int dg_prove_traces_device_with_options(const void *const *d_registers, const uint32_t *width, const uint64_t *length, const uint32_t *ctx_depth,
                                        const uint32_t *loop_depth, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                                        const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t *options,
                                        dg_proof_t **proofs_out, int *status, dg_prove_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "batch must hold at least one trace");
        DG_REQUIRE(d_registers && width && length && ctx_depth && loop_depth && options && proofs_out && status, "null argument");
        prove_call({device_traces(d_registers, width, length, ctx_depth, loop_depth, count), false, nullptr, inputs16, n_inputs, outputs16,
                    n_outputs}, options, true, true, proofs_out, status, stats);
    });
}
int dg_check_traces(const dg_trace_t *traces, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                    const uint8_t *const *outputs16, const uint32_t *n_outputs, const uint8_t *program_hashes32, dg_trace_report_t *reports,
                    uint32_t *step_masks) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "at least one trace must be checked");
        DG_REQUIRE(traces && reports, "null argument");
        const ProveCall x{host_traces(traces, count), true, "call", inputs16, n_inputs, outputs16, n_outputs};
        check_prove_call(x);
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        check_traces(c, x.traces, inputs16, n_inputs, outputs16, n_outputs, program_hashes32, reports, step_masks, nullptr);
    });
}
int dg_check_traces_device(const void *d_registers, uint32_t count, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                           const uint8_t *const *inputs16, const uint32_t *n_inputs, const uint8_t *const *outputs16, const uint32_t *n_outputs,
                           const uint8_t *program_hashes32, dg_trace_report_t *reports, uint32_t *d_step_masks) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "at least one trace must be checked");
        DG_REQUIRE(d_registers && reports, "null argument");
        const ProveCall x{one_shape_traces((const fe *)d_registers, count, width, length, ctx_depth, loop_depth), false, "call", inputs16, n_inputs,
                          outputs16, n_outputs};
        check_prove_call(x);
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        check_traces(c, x.traces, inputs16, n_inputs, outputs16, n_outputs, program_hashes32, reports, nullptr, d_step_masks);
    });
}
static void run_trace_programs(const ExecutionCall &x, dg_execution_info_t *info, uint8_t *const *registers_out, int *status,
                               dg_execution_stats_t *vm_stats) {
    DG_REQUIRE(x.count >= 1, "at least one execution is needed");
    DG_REQUIRE(x.programs && x.program_of && (x.inputs || x.device_inputs) && status, "null argument");
    check_execution_call(x);
    Context &c = ctx();
    std::lock_guard<std::mutex> lk(c.mu);
    t_batch_messages.clear();
    trace_programs(c, x, info, registers_out, status, t_batch_messages, vm_stats);
}
int dg_trace_programs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                      const dg_program_inputs_t *inputs, uint64_t max_steps, dg_execution_info_t *info, uint8_t *const *registers_out,
                      int *status, dg_execution_stats_t *vm_stats) {
    return guarded([&] {
        run_trace_programs(ExecutionCall{programs, n_programs, count, program_of, inputs, max_steps}, info, registers_out, status, vm_stats);
    });
}
static void run_execute_programs(const ExecutionCall &x, const uint32_t *num_outputs, const dg_options_t *options, bool per_execution,
                                 dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *stats, dg_execution_stats_t *vm_stats) {
    DG_REQUIRE(x.count >= 1, "at least one execution is needed");
    DG_REQUIRE(x.programs && x.program_of && (x.inputs || x.device_inputs) && options && proofs_out && status, "null argument");
    check_execution_call(x, OutputCounts{num_outputs, outputs16});
    const std::vector<dg_options_t> opts = call_options(options, x.count, per_execution, "execution");
    Context &c = ctx();
    std::lock_guard<std::mutex> lk(c.mu);
    t_batch_messages.clear();
    execute_programs(c, x, num_outputs, opts.data(), (Proof **)proofs_out, outputs16, status, t_batch_messages, stats, vm_stats);
}
int dg_execute_programs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                        const dg_program_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, const dg_options_t *options,
                        dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *stats, dg_execution_stats_t *vm_stats) {
    return guarded([&] {
        run_execute_programs(ExecutionCall{programs, n_programs, count, program_of, inputs, max_steps}, num_outputs, options, false, proofs_out,
                             outputs16, status, stats, vm_stats);
    });
}
int dg_execute_programs_with_options(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                     const dg_program_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, const dg_options_t *options,
                                     dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *stats,
                                     dg_execution_stats_t *vm_stats) {
    return guarded([&] {
        run_execute_programs(ExecutionCall{programs, n_programs, count, program_of, inputs, max_steps}, num_outputs, options, true, proofs_out,
                             outputs16, status, stats, vm_stats);
    });
}
// the one-program case: program_of all 0
int dg_trace_batch(const dg_program_t *program, uint32_t count, const dg_program_inputs_t *inputs, uint64_t max_steps,
                   dg_execution_info_t *info, uint8_t *const *registers_out, int *status) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "at least one execution is needed");
        DG_REQUIRE(program && inputs && status, "null argument");
        const std::vector<uint32_t> of(count, 0);
        const ExecutionCall x{program, 1, count, of.data(), inputs, max_steps};
        check_execution_call(x);
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        t_batch_messages.clear();
        trace_programs(c, x, info, registers_out, status, t_batch_messages, nullptr);
    });
}
int dg_execute_batch(const dg_program_t *program, uint32_t count, const dg_program_inputs_t *inputs, uint32_t num_outputs, uint64_t max_steps,
                     const dg_options_t *options, dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "at least one execution is needed");
        DG_REQUIRE(program && inputs && options && proofs_out && status, "null argument");
        const std::vector<uint32_t> of(count, 0), n_out(count, num_outputs);
        const ExecutionCall x{program, 1, count, of.data(), inputs, max_steps};
        check_execution_call(x, OutputCounts{n_out.data(), outputs16});
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        t_batch_messages.clear();
        std::vector<uint8_t> outs((size_t)count * 8 * 16);
        const std::vector<dg_options_t> opts(count, *options);
        execute_programs(c, x, n_out.data(), opts.data(), (Proof **)proofs_out, outs.data(), status, t_batch_messages, stats, nullptr);
        if (num_outputs)     // num_outputs elements per execution
            for (uint32_t i = 0; i < count; i++) memcpy(outputs16 + (size_t)16 * num_outputs * i, outs.data() + (size_t)128 * i, (size_t)16 * num_outputs);
    });
}
// dg_trace_one's stats from its dg_trace_many call's: after the fallback, the batch path's shape and write passes
static void one_stats(dg_trace_one_stats_t *stats, const dg_many_stats_t &m) {
    if (!stats) return;
    memset(stats, 0, sizeof *stats);
    const bool fb = m.fallback_programs > 0;
    stats->table_ms = m.table_ms;
    stats->sequential_ms = fb ? m.fallback.shape_ms : m.sequential_ms;
    stats->segment_ms = fb ? m.fallback.write_ms : m.segment_ms;
    stats->table_rounds = m.table_rounds;
    stats->table_entries = m.table_entries;
    stats->table_levels = m.table_levels;
    stats->sequential_launches = m.sequential_launches;
    stats->checkpoints = m.checkpoints;
    stats->segments = m.segments;
    stats->logged = m.logged;
    stats->segment_steps = m.segment_steps;
    stats->fallback = fb ? 1 : 0;
}
// dg_trace_one / dg_execute_one: many(status, messages, many_stats) runs the execution as dg_trace_many / dg_execute_many with count 1.
// Its stats reach `stats` also when it throws, and a failed execution throws with its message.  The messages stay local, so that these
// calls leave the thread's dg_batch_message list as it was.
static void run_one(dg_trace_one_stats_t *stats, const std::function<void(int *, std::vector<std::string> &, dg_many_stats_t *)> &many) {
    dg_many_stats_t m;
    memset(&m, 0, sizeof m);
    int status = DG_OK;
    std::vector<std::string> messages;
    try {
        many(&status, messages, &m);
    } catch (...) {
        one_stats(stats, m);
        throw;
    }
    one_stats(stats, m);
    if (status != DG_OK) throw Error(status, messages[0]);
}
int dg_trace_one(const dg_program_t *program, const dg_program_inputs_t *inputs, uint64_t max_steps, uint64_t segment_steps,
                 dg_execution_info_t *info, uint8_t *registers_out, dg_trace_one_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(program && inputs, "null argument");
        const uint32_t of = 0;
        const ExecutionCall x{program, 1, 1, &of, inputs, max_steps};
        check_execution_call(x, std::nullopt, segment_steps);
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        uint8_t *const outs[1] = {registers_out};
        dg_execution_info_t one;          // reaches info only when the call succeeds
        run_one(stats, [&](int *status, std::vector<std::string> &messages, dg_many_stats_t *m) {
            trace_many(c, x, segment_steps, &one, registers_out ? outs : nullptr, status, messages, m);
        });
        if (info) *info = one;
    });
}
int dg_execute_one(const dg_program_t *program, const dg_program_inputs_t *inputs, uint32_t num_outputs, uint64_t max_steps,
                   uint64_t segment_steps, const dg_options_t *options, dg_proof_t **proof_out, uint8_t *outputs16, dg_execution_info_t *info,
                   dg_prove_stats_t *prove_stats, dg_trace_one_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(program && inputs && options && proof_out, "null argument");
        *proof_out = nullptr;
        const uint32_t of = 0;
        const ExecutionCall x{program, 1, 1, &of, inputs, max_steps};
        check_execution_call(x, OutputCounts{&num_outputs, outputs16}, segment_steps);
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        uint8_t outs[8 * 16];             // execute_many writes 8 elements; the caller's buffer holds num_outputs
        dg_execution_info_t one;
        run_one(stats, [&](int *status, std::vector<std::string> &messages, dg_many_stats_t *m) {
            execute_many(c, x, &num_outputs, segment_steps, options, (Proof **)proof_out, outs, &one, status, messages, prove_stats, m);
        });
        if (num_outputs) memcpy(outputs16, outs, (size_t)16 * num_outputs);
        if (info) *info = one;
    });
}
static void run_trace_many(const ExecutionCall &x, uint64_t segment_steps, dg_execution_info_t *info, uint8_t *const *registers_out, int *status,
                           dg_many_stats_t *stats) {
    DG_REQUIRE(x.count >= 1, "at least one execution is needed");
    DG_REQUIRE(x.programs && x.program_of && (x.inputs || x.device_inputs) && status, "null argument");
    check_execution_call(x, std::nullopt, segment_steps);
    Context &c = ctx();
    std::lock_guard<std::mutex> lk(c.mu);
    t_batch_messages.clear();
    trace_many(c, x, segment_steps, info, registers_out, status, t_batch_messages, stats);
}
int dg_trace_many(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                  const dg_program_inputs_t *inputs, uint64_t max_steps, uint64_t segment_steps, dg_execution_info_t *info,
                  uint8_t *const *registers_out, int *status, dg_many_stats_t *stats) {
    return guarded([&] {
        run_trace_many(ExecutionCall{programs, n_programs, count, program_of, inputs, max_steps}, segment_steps, info, registers_out, status, stats);
    });
}
static void run_execute_many(const ExecutionCall &x, const uint32_t *num_outputs, uint64_t segment_steps, const dg_options_t *options,
                             bool per_execution, dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *prove_stats,
                             dg_many_stats_t *stats) {
    DG_REQUIRE(x.count >= 1, "at least one execution is needed");
    DG_REQUIRE(x.programs && x.program_of && (x.inputs || x.device_inputs) && options && proofs_out && status, "null argument");
    check_execution_call(x, OutputCounts{num_outputs, outputs16}, segment_steps);
    const std::vector<dg_options_t> opts = call_options(options, x.count, per_execution, "execution");
    Context &c = ctx();
    std::lock_guard<std::mutex> lk(c.mu);
    t_batch_messages.clear();
    execute_many(c, x, num_outputs, segment_steps, opts.data(), (Proof **)proofs_out, outputs16, nullptr, status, t_batch_messages, prove_stats,
                 stats);
}
int dg_execute_many(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                    const dg_program_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, uint64_t segment_steps,
                    const dg_options_t *options, dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *prove_stats,
                    dg_many_stats_t *stats) {
    return guarded([&] {
        run_execute_many(ExecutionCall{programs, n_programs, count, program_of, inputs, max_steps}, num_outputs, segment_steps, options, false,
                         proofs_out, outputs16, status, prove_stats, stats);
    });
}
int dg_execute_many_with_options(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                 const dg_program_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, uint64_t segment_steps,
                                 const dg_options_t *options, dg_proof_t **proofs_out, uint8_t *outputs16, int *status,
                                 dg_prove_stats_t *prove_stats, dg_many_stats_t *stats) {
    return guarded([&] {
        run_execute_many(ExecutionCall{programs, n_programs, count, program_of, inputs, max_steps}, num_outputs, segment_steps, options, true,
                         proofs_out, outputs16, status, prove_stats, stats);
    });
}

// ---- program inputs in device memory: the calls above with ExecutionCall::device_inputs ----------------------------------------------
static ExecutionCall device_call(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                 const dg_device_inputs_t *inputs, uint64_t max_steps) {
    DG_REQUIRE(inputs, "null device inputs");
    return ExecutionCall{programs, n_programs, count, program_of, nullptr, max_steps, inputs};
}
int dg_trace_programs_device_inputs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                    const dg_device_inputs_t *inputs, uint64_t max_steps, dg_execution_info_t *info, uint8_t *const *registers_out,
                                    int *status, dg_execution_stats_t *vm_stats) {
    return guarded([&] {
        run_trace_programs(device_call(programs, n_programs, count, program_of, inputs, max_steps), info, registers_out, status, vm_stats);
    });
}
int dg_execute_programs_device_inputs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                      const dg_device_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, const dg_options_t *options,
                                      dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *stats,
                                      dg_execution_stats_t *vm_stats) {
    return guarded([&] {
        run_execute_programs(device_call(programs, n_programs, count, program_of, inputs, max_steps), num_outputs, options, true, proofs_out,
                             outputs16, status, stats, vm_stats);
    });
}
int dg_trace_many_device_inputs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                const dg_device_inputs_t *inputs, uint64_t max_steps, uint64_t segment_steps, dg_execution_info_t *info,
                                uint8_t *const *registers_out, int *status, dg_many_stats_t *stats) {
    return guarded([&] {
        run_trace_many(device_call(programs, n_programs, count, program_of, inputs, max_steps), segment_steps, info, registers_out, status, stats);
    });
}
int dg_execute_many_device_inputs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                  const dg_device_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, uint64_t segment_steps,
                                  const dg_options_t *options, dg_proof_t **proofs_out, uint8_t *outputs16, int *status,
                                  dg_prove_stats_t *prove_stats, dg_many_stats_t *stats) {
    return guarded([&] {
        run_execute_many(device_call(programs, n_programs, count, program_of, inputs, max_steps), num_outputs, segment_steps, options, true,
                         proofs_out, outputs16, status, prove_stats, stats);
    });
}
int dg_batch_message(uint32_t index, char *message, size_t cap) {
    return guarded([&] {
        DG_REQUIRE(message && cap, "null argument");
        DG_REQUIRE(index < t_batch_messages.size(), "no such trace or proof in this thread's last batched call");
        strncpy(message, t_batch_messages[index].c_str(), cap - 1);
        message[cap - 1] = 0;
    });
}
// ---- device memory ------------------------------------------------------------------------------------------------------------
static void require_one_gpu(const Context &c) {
    DG_REQUIRE(c.world == 1 && ctx_device_count() == 1, "memory limits and plans apply to one GPU: the library was initialised for several (dg_init_devices / dg_comm_init)");
}
int dg_set_memory_limit(size_t bytes) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        if (bytes) require_one_gpu(c);
        memory_set_limit(c, bytes);
    });
}
int dg_memory_usage(size_t *held, size_t *peak) {
    return guarded([&] {
        DG_REQUIRE(held || peak, "null argument");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        memory_usage(c, held, peak);
    });
}
int dg_plan_prove(uint32_t width, uint64_t length, uint32_t count, const dg_options_t *options, dg_prove_plan_t *plan) {
    return guarded([&] {
        DG_REQUIRE(options && plan, "null argument");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        require_one_gpu(c);
        const ProvePlan P = plan_prove(c, width, length, options->extension_factor, count);
        plan->layout = P.full ? DG_LAYOUT_FULL : DG_LAYOUT_EVAL_COSETS;
        plan->group = (uint32_t)P.group;
        plan->coset_chunk = P.chunk;
        plan->retained_cosets = P.full ? options->extension_factor : 8;
        plan->bytes_per_proof = P.per_proof;
        plan->fixed_bytes = P.fixed;
        plan->available_bytes = P.available;
    });
}

int dg_set_rng_callbacks(const dg_rng_callbacks_t *callbacks) {
    return guarded([&] {
        if (!callbacks) { fs::set_rng_hooks(nullptr); return; }
        fs::RngHooks h{callbacks->user, callbacks->draw_field, callbacks->draw_positions};
        fs::set_rng_hooks(&h);
    });
}
int dg_verify(const uint8_t program_hash[32], const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16, uint32_t n_outputs,
              const uint8_t *proof_bytes, size_t proof_len, char *message, size_t message_cap) {
    if (message && message_cap) message[0] = 0;
    return guarded([&] {
        DG_REQUIRE(program_hash && proof_bytes, "null argument");
        DG_REQUIRE((n_inputs == 0 || inputs16) && (n_outputs == 0 || outputs16), "null public inputs / outputs");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        std::vector<int> status;
        std::vector<std::string> messages;
        verify_proofs(c, {VerifyRequest{program_hash, inputs16, n_inputs, outputs16, n_outputs, proof_bytes, proof_len}}, status, messages, nullptr);
        if (status[0] == DG_OK) return;
        if (status[0] == DG_ERR_REJECTED && message && message_cap) {
            strncpy(message, messages[0].c_str(), message_cap - 1);
            message[message_cap - 1] = 0;
        }
        throw Error(status[0], messages[0]);
    });
}
int dg_verify_batch(uint32_t count, const uint8_t *const *program_hashes, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                    const uint8_t *const *outputs16, const uint32_t *n_outputs, const uint8_t *const *proof_bytes, const size_t *proof_lens,
                    int *status, dg_verify_stats_t *stats) {
    return guarded([&] {
        DG_REQUIRE(count >= 1, "batch must hold at least one proof");
        DG_REQUIRE(program_hashes && inputs16 && n_inputs && outputs16 && n_outputs && proof_bytes && proof_lens && status, "null argument");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        std::vector<VerifyRequest> req(count);
        for (uint32_t i = 0; i < count; i++)
            req[i] = VerifyRequest{program_hashes[i], inputs16[i], n_inputs[i], outputs16[i], n_outputs[i], proof_bytes[i], proof_lens[i]};
        std::vector<int> st;
        std::vector<std::string> messages;
        verify_proofs(c, req, st, messages, stats);
        std::copy(st.begin(), st.end(), status);
        t_batch_messages = std::move(messages);
    });
}
int dg_proof_serialized_len(const dg_proof_t *proof, size_t *len) {
    return guarded([&] { DG_REQUIRE(proof && len, "null argument"); *len = ((const Proof *)proof)->bytes.size(); });
}
int dg_proof_serialize(const dg_proof_t *proof, uint8_t *buf, size_t cap) {
    return guarded([&] {
        DG_REQUIRE(proof && buf, "null argument");
        const Proof *p = (const Proof *)proof;
        DG_REQUIRE(cap >= p->bytes.size(), "buffer too small");
        memcpy(buf, p->bytes.data(), p->bytes.size());
    });
}
int dg_proof_digest(const dg_proof_t *proof, int which, uint8_t out32[32]) {
    return guarded([&] {
        DG_REQUIRE(proof && out32 && which >= 0 && which <= 2, "invalid argument");
        const Proof *p = (const Proof *)proof;
        memcpy(out32, which == 0 ? p->trace_root : which == 1 ? p->constraint_root : p->pow_seed, 32);
    });
}
int dg_proof_pow_nonce(const dg_proof_t *proof, uint64_t *nonce) {
    return guarded([&] { DG_REQUIRE(proof && nonce, "null argument"); *nonce = ((const Proof *)proof)->pow_nonce; });
}
void dg_proof_free(dg_proof_t *proof) { delete (Proof *)proof; }

// ---- multi-GPU ---------------------------------------------------------------------------------------------------------------------
int dg_comm_unique_id(uint8_t id128[128]) { return guarded([&] { comm_unique_id(id128); }); }
int dg_comm_init(int rank, int world, const uint8_t id128[128]) {
    return guarded([&] {
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DG_REQUIRE(world == 1 || c.mem_limit == 0, "a memory limit applies to one GPU: clear it (dg_set_memory_limit(0)) before spanning several");
        comm_init(c, rank, world, id128);
    });
}
int dg_comm_finalize(void) { return guarded([&] { Context &c = ctx(); std::lock_guard<std::mutex> lk(c.mu); comm_finalize(c); }); }
int dg_host_shard_locate(uint64_t n, int log_blk, int log_g, int is_node, uint64_t index, int64_t out[3]) {
    return guarded([&] {
        ShardGeom geo; geo.n = n; geo.log_blk = log_blk; geo.log_g = log_g;
        ShardLocation l = is_node ? geo.node(index) : geo.item(index);
        out[0] = l.owner; out[1] = l.kind; out[2] = (int64_t)l.index;
    });
}

static void host_group_traces(uint32_t count, const uint64_t *lengths, const uint32_t *extension_factors, const uint32_t *widths,
                              const uint32_t *ctx_depths, const uint32_t *loop_depths, const uint64_t *footprints, uint64_t budget, uint32_t cap,
                              uint32_t *order_out, uint32_t *group_sizes_out, uint32_t *n_groups) {
    DG_REQUIRE(lengths && widths && ctx_depths && loop_depths && footprints && order_out && group_sizes_out && n_groups, "null argument");
    DG_REQUIRE(cap >= 1, "a group holds at least one trace");
    const std::vector<uint32_t> factors = extension_factors ? std::vector<uint32_t>(extension_factors, extension_factors + count)
                                                            : std::vector<uint32_t>(count, 0);
    uint32_t at = 0, groups = 0;
    for (const std::vector<uint32_t> &idx : partition_traces(std::vector<uint64_t>(lengths, lengths + count), factors)) {
        std::vector<uint32_t> w;
        std::vector<size_t> foot;
        for (uint32_t i : idx) { w.push_back(widths[i]); foot.push_back(footprints[i]); }
        size_t first = 0;
        for (uint32_t k : cut_groups(w, foot, budget, cap)) {
            std::vector<RegisterShape> keys;
            for (size_t m = first; m < first + k; m++) keys.push_back(RegisterShape{widths[idx[m]], ctx_depths[idx[m]], loop_depths[idx[m]]});
            for (uint32_t m : shape_order(keys)) order_out[at++] = idx[first + m];
            group_sizes_out[groups++] = k;
            first += k;
        }
    }
    *n_groups = groups;
}
int dg_host_group_traces(uint32_t count, const uint64_t *lengths, const uint32_t *widths, const uint32_t *ctx_depths, const uint32_t *loop_depths,
                         const uint64_t *footprints, uint64_t budget, uint32_t cap, uint32_t *order_out, uint32_t *group_sizes_out,
                         uint32_t *n_groups) {
    return guarded([&] {
        host_group_traces(count, lengths, nullptr, widths, ctx_depths, loop_depths, footprints, budget, cap, order_out, group_sizes_out, n_groups);
    });
}
int dg_host_group_traces_with_options(uint32_t count, const uint64_t *lengths, const uint32_t *extension_factors, const uint32_t *widths,
                                      const uint32_t *ctx_depths, const uint32_t *loop_depths, const uint64_t *footprints, uint64_t budget,
                                      uint32_t cap, uint32_t *order_out, uint32_t *group_sizes_out, uint32_t *n_groups) {
    return guarded([&] {
        DG_REQUIRE(extension_factors, "null argument");
        host_group_traces(count, lengths, extension_factors, widths, ctx_depths, loop_depths, footprints, budget, cap, order_out, group_sizes_out,
                     n_groups);
    });
}

// ---- host-only helpers (no device access) ---------------------------------------------------------------------------------------------
int dg_host_prng_vector(const uint8_t seed[32], uint64_t count, uint8_t *out16) {
    return guarded([&] { DG_REQUIRE(seed && (out16 || count == 0), "null argument"); std::vector<fe> v = fs::prng_vector(seed, count); memcpy(out16, v.data(), count * 16); });
}
int dg_host_query_positions(const uint8_t seed[32], uint64_t domain_size, uint32_t extension_factor, uint32_t num_queries, uint64_t *out) {
    return guarded([&] {
        try {
            std::vector<uint64_t> p = fs::query_positions(seed, domain_size, extension_factor, num_queries);
            memcpy(out, p.data(), p.size() * 8);
        } catch (const std::exception &e) { throw Error(DG_ERR_EXHAUSTED, e.what()); }
    });
}
int dg_host_blake3(const uint8_t *data, size_t len, uint8_t out32[32]) { return guarded([&] { fs::blake3_short(data, len, out32); }); }
int dg_host_plan_batch(const uint64_t *indexes, uint32_t n_indexes, uint64_t n_leaves, uint64_t *out, size_t cap, size_t *written) {
    return guarded([&] {
        DG_REQUIRE(indexes && out && written, "null argument");
        DG_REQUIRE(n_leaves >= 2 && (n_leaves & (n_leaves - 1)) == 0, "number of leaves must be a power of 2 and >= 2");
        for (uint32_t i = 0; i < n_indexes; i++) DG_REQUIRE(indexes[i] < n_leaves, "invalid index (merkle.rs:296-303 asserts index <= max_valid)");
        fs::BatchPlan plan = fs::plan_batch_proof(std::vector<uint64_t>(indexes, indexes + n_indexes), n_leaves);
        std::vector<uint64_t> flat = {(uint64_t)plan.nodes.size(), (uint64_t)plan.depth};
        for (auto &slot : plan.nodes) {
            flat.push_back(slot.size());
            for (auto &r : slot) { flat.push_back(r.leaf ? 1 : 0); flat.push_back(r.index); }
        }
        DG_REQUIRE(flat.size() <= cap, "buffer too small");
        memcpy(out, flat.data(), flat.size() * 8);
        *written = flat.size();
    });
}
int dg_host_tree_plan(const uint64_t *indexes, uint32_t count, uint64_t n_leaves, uint64_t *out, size_t cap, size_t *written) {
    return guarded([&] {
        DG_REQUIRE((indexes || count == 0) && out && written, "null argument");
        DG_REQUIRE(n_leaves >= 2 && (n_leaves & (n_leaves - 1)) == 0, "number of leaves must be a power of 2 and >= 2");
        Tree t;
        t.L = n_leaves;
        require_tree_indexes(t, indexes, count);
        const TreePlan p = plan_tree_update(indexes, count, n_leaves);
        std::vector<uint64_t> flat = {(uint64_t)p.leaves.size(), (uint64_t)p.level_size.size(), (uint64_t)p.ids.size()};
        flat.insert(flat.end(), p.leaves.begin(), p.leaves.end());
        flat.insert(flat.end(), p.source.begin(), p.source.end());
        size_t at = 0;
        for (uint32_t n : p.level_size) {
            flat.push_back(n);
            flat.insert(flat.end(), p.ids.begin() + at, p.ids.begin() + at + n);
            flat.insert(flat.end(), p.first.begin() + at, p.first.begin() + at + n);
            at += n;
        }
        DG_REQUIRE(flat.size() <= cap, "buffer too small");
        memcpy(out, flat.data(), flat.size() * 8);
        *written = flat.size();
    });
}
int dg_host_merkle_verify_plan(const uint64_t *indexes, uint32_t n_indexes, uint32_t depth, uint32_t n_values, const uint32_t *node_counts,
                               uint32_t n_slots, uint32_t *ops, size_t ops_cap, uint32_t *n_ops, uint32_t *level_start, size_t levels_cap,
                               uint32_t *n_levels, uint32_t *root_slot) {
    return guarded([&] {
        DG_REQUIRE(indexes && node_counts && ops && n_ops && level_start && n_levels && root_slot, "null argument");
        std::vector<uint32_t> o, ls;
        uint32_t root = 0;
        if (!host_plan_verify_batch(std::vector<uint64_t>(indexes, indexes + n_indexes), (int)depth, n_values,
                                    std::vector<uint32_t>(node_counts, node_counts + n_slots), o, ls, root))
            throw Error(DG_ERR_REJECTED, "batch proof structure rejected (merkle.rs:154-263 returns false)");
        DG_REQUIRE(o.size() <= ops_cap && ls.size() <= levels_cap, "buffer too small");
        memcpy(ops, o.data(), o.size() * 4);
        memcpy(level_start, ls.data(), ls.size() * 4);
        *n_ops = (uint32_t)(o.size() / 3);
        *n_levels = (uint32_t)ls.size() - 1;
        *root_slot = root;
    });
}
int dg_host_periodic_tables(uint8_t *out16) {
    return guarded([&] { std::vector<fe> t = fs::periodic_tables(); memcpy(out16, t.data(), t.size() * 16); });
}
int dg_host_constraint_name(uint32_t ctx_depth, uint32_t loop_depth, uint32_t stack_depth, uint32_t index, char *name, size_t cap) {
    return guarded([&] {
        DG_REQUIRE(name && cap, "null argument");
        const std::string s = constraint_name(ctx_depth, loop_depth, stack_depth, index);
        strncpy(name, s.c_str(), cap - 1);
        name[cap - 1] = 0;
    });
}

// ---- test hooks: the coefficient-domain stage kernels of the prover, one call each, on host buffers ---------------------------------------
// Each hook checks every argument before it touches the device and then calls the host function prover.cu calls, with the parameters
// prover.cu gives it.  Output buffers are zero-filled on the device first, so that a test also sees what a kernel writes outside its range.
static bool is_pow2(uint64_t v) { return v && !(v & (v - 1)); }
static std::vector<fe> host_fes(const uint8_t *p, uint64_t n) {
    std::vector<fe> v(n);
    memcpy(v.data(), p, n * 16);
    return v;
}
static void upload(Context &c, DevBuf &d, const uint8_t *p, size_t n) {
    d.alloc(n * 16);
    DG_CUDA(cudaMemcpyAsync(d.p, p, n * 16, cudaMemcpyHostToDevice, c.stream));
}
static void zeroed(Context &c, DevBuf &d, size_t n) {
    d.alloc(n * 16);
    DG_CUDA(cudaMemsetAsync(d.p, 0, n * 16, c.stream));
}
static void download(Context &c, uint8_t *p, const DevBuf &d, size_t bytes) {
    DG_CUDA(cudaMemcpyAsync(p, d.p, bytes, cudaMemcpyDeviceToHost, c.stream));
    DG_CUDA(cudaStreamSynchronize(c.stream));
}
static void require_batch(uint32_t batch) { DG_REQUIRE(batch >= 1 && batch <= 65535, "batch must be in 1..65535"); }
// a vector of len elements per batch entry, `stride` elements apart: the elements the buffer spans
static uint64_t strided_span(uint32_t batch, uint64_t stride, uint64_t len, const char *what) {
    DG_REQUIRE(stride >= len && stride <= (1ULL << 32), std::string(what) + " must be at least the vector length and at most 2^32");
    return (uint64_t)(batch - 1) * stride + len;
}

int dg_test_syn_div(const uint8_t *in16, uint8_t *out16, uint32_t batch, uint64_t len, uint64_t in_stride, uint64_t out_stride, int in_place,
                    const uint8_t *b16, int shared, const uint8_t *sub0_16) {
    return guarded([&] {
        DG_REQUIRE(in16 && out16 && b16 && sub0_16, "null buffer");
        require_batch(batch);
        DG_REQUIRE(is_pow2(len) && len >= 2 && len <= (1ULL << 28), "len must be a power of 2 in 2..2^28");
        DG_REQUIRE((len + 1023) / 1024 * batch < (1ULL << 31), "division batch too large for one launch");
        const uint64_t in_n = strided_span(batch, in_stride, len, "in_stride"), out_n = strided_span(batch, out_stride, len, "out_stride");
        DG_REQUIRE(!in_place || in_stride == out_stride, "an in-place division has one stride");
        const uint32_t tables = shared ? 1 : batch;
        require_canonical(in16, in_n, 1, "input element");
        require_canonical(b16, tables, 1, "point");
        require_canonical(sub0_16, batch, 1, "sub0");
        // the (base, step) pairs of the tables of b, then of 1 / b
        const std::vector<fe> b = host_fes(b16, tables);
        std::vector<fe> pack(4 * (size_t)tables);
        for (uint32_t q = 0; q < tables; q++) {
            DG_REQUIRE(b[q].lo || b[q].hi, "point " + std::to_string(q) + " is zero");
            PowTables::pack_point(&pack[2 * q], 2 * (size_t)tables, b[q], len + 1);
        }
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_in, d_out, d_pack, d_sub0;
        upload(c, d_in, in16, in_n);
        upload(c, d_pack, (const uint8_t *)pack.data(), pack.size());
        upload(c, d_sub0, sub0_16, batch);
        if (!in_place) zeroed(c, d_out, out_n);
        fe *out = in_place ? d_in.as<fe>() : d_out.as<fe>();
        if (shared) {                       // one table for all vectors (stage 4: 1 and x_last)
            PowTables pows(c, d_pack.as<fe>(), 2, len + 1);
            syn_div(c, (int)batch, d_in.as<fe>(), in_stride, out, out_stride, len, pows.ref(0), 0, 0, pows.ref(1), 0, 0, d_sub0.as<fe>());
        } else {                            // a table per vector (stage 6: z and z g of every proof)
            PowTables t(c, d_pack.as<fe>(), (int)batch, len + 1), ti(c, d_pack.as<fe>() + 2 * batch, (int)batch, len + 1);
            syn_div(c, (int)batch, d_in.as<fe>(), in_stride, out, out_stride, len, t.ref(0), t.lo_n, t.hi_n, ti.ref(0), ti.lo_n, ti.hi_n,
                    d_sub0.as<fe>());
        }
        download(c, out16, in_place ? d_in : d_out, out_n * 16);
    });
}

int dg_test_syn_div_expanded_sum(const uint8_t *a16, const uint8_t *add0_16, const uint8_t *add1_16, uint8_t *out16, uint32_t batch, uint64_t n,
                                 uint64_t in_stride, uint64_t out_stride, const uint8_t *e16) {
    return guarded([&] {
        DG_REQUIRE(a16 && out16 && e16, "null buffer");
        require_batch(batch);
        DG_REQUIRE(is_pow2(n) && n <= (1ULL << 26), "n must be a power of 2 up to 2^26");
        const uint64_t len = 8 * n;
        const uint64_t in_n = strided_span(batch, in_stride, len, "in_stride"), out_n = strided_span(batch, out_stride, len, "out_stride");
        require_canonical(a16, in_n, 1, "a element");
        if (add0_16) require_canonical(add0_16, in_n, 1, "add0 element");
        if (add1_16) require_canonical(add1_16, in_n, 1, "add1 element");
        require_canonical(e16, 1, 1, "point");
        const fe e = host_fes(e16, 1)[0];
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_a, d_add0, d_add1, d_scratch((size_t)batch * len * 16), d_out;
        upload(c, d_a, a16, in_n);
        if (add0_16) upload(c, d_add0, add0_16, in_n);
        if (add1_16) upload(c, d_add1, add1_16, in_n);
        zeroed(c, d_out, out_n);
        syn_div_expanded_sum(c, d_a.as<fe>(), d_scratch.as<fe>(), add0_16 ? d_add0.as<fe>() : nullptr, add1_16 ? d_add1.as<fe>() : nullptr,
                             d_out.as<fe>(), n, len, e, (int)batch, in_stride, out_stride);
        download(c, out16, d_out, out_n * 16);
    });
}

int dg_test_eval_polys_at(const uint8_t *polys16, uint32_t cols, uint32_t log_n, const uint8_t *z16, uint32_t n_z, const uint32_t *col_proof,
                          uint8_t *out16) {
    return guarded([&] {
        DG_REQUIRE(polys16 && z16 && out16, "null buffer");
        DG_REQUIRE(cols >= 1 && cols <= 65535 && n_z >= 1 && n_z <= 65535, "cols and n_z must be in 1..65535");
        DG_REQUIRE(log_n >= 1 && log_n <= 26, "log_n must be in 1..26");
        const uint64_t n = 1ULL << log_n, E = 8 * n, len = col_proof ? n : E;
        if (col_proof) {
            for (uint32_t j = 0; j < cols; j++) DG_REQUIRE(col_proof[j] < n_z, "column " + std::to_string(j) + " names no point");
        } else {
            DG_REQUIRE(cols == n_z, "the one-point form evaluates column q at point q");
        }
        require_canonical(polys16, cols * len, 1, "coefficient");
        require_canonical(z16, n_z, 1, "point");
        const std::vector<fe> z = host_fes(z16, n_z);
        std::vector<fe> pack(2 * (size_t)n_z);
        for (uint32_t q = 0; q < n_z; q++) { pack[2 * q] = z[q]; pack[2 * q + 1] = PowTables::step(z[q], E + 1); }
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_polys, d_pack, d_cp, d_out;
        upload(c, d_polys, polys16, cols * len);
        upload(c, d_pack, (const uint8_t *)pack.data(), pack.size());
        zeroed(c, d_out, 2 * (size_t)cols);
        PowTables z_t(c, d_pack.as<fe>(), (int)n_z, E + 1);
        if (col_proof) {                    // stage 6: trace polynomials at z and z w_n, proofs of several widths
            d_cp.alloc((size_t)cols * 4);
            DG_CUDA(cudaMemcpyAsync(d_cp.p, col_proof, (size_t)cols * 4, cudaMemcpyHostToDevice, c.stream));
            eval_polys_at(c, d_polys.as<fe>(), n, (int)cols, z_t.ref(0), c.twiddle((int)log_n, false), true, d_out.as<fe>(), 1 << 30, z_t.lo_n,
                          z_t.hi_n, d_cp.as<unsigned>());
        } else {                            // stage 6: the constraint polynomial of every proof at its z
            eval_polys_at(c, d_polys.as<fe>(), E, (int)cols, z_t.ref(0), c.twiddle((int)log_n, false), false, d_out.as<fe>(), 1, z_t.lo_n,
                          z_t.hi_n);
        }
        download(c, out16, d_out, 2 * (size_t)cols * 16);
    });
}

int dg_test_eval_trace_rows(const uint8_t *polys16, uint32_t cols, uint32_t log_n, uint32_t log_N, const uint64_t *pos, const uint32_t *col,
                            const uint32_t *width, uint32_t count, uint8_t *out16) {
    return guarded([&] {
        DG_REQUIRE(polys16 && pos && col && width && out16, "null buffer");
        DG_REQUIRE(cols >= 1 && count >= 1, "cols and count must be at least 1");
        DG_REQUIRE(log_n >= 1 && log_N >= log_n && log_N <= log_n + 8 && log_N <= 30, "log_n and log_N out of range");
        const uint64_t n = 1ULL << log_n;
        std::vector<TraceRow> points(count);
        for (uint32_t m = 0; m < count; m++) {
            DG_REQUIRE(pos[m] < (1ULL << log_N), "position " + std::to_string(m) + " is outside the domain");
            DG_REQUIRE(width[m] >= 1 && width[m] <= 128 && col[m] <= cols && width[m] <= cols - col[m],
                       "row " + std::to_string(m) + ": columns out of range (width 1..128)");
            points[m] = TraceRow{pos[m], 0, col[m], width[m]};
        }
        require_canonical(polys16, cols * n, 1, "coefficient");
        uint64_t values = 0;
        for (uint32_t m = 0; m < count; m++) values += width[m];
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_polys, d_out;
        upload(c, d_polys, polys16, cols * n);
        zeroed(c, d_out, values);
        eval_trace_rows(c, d_polys.as<fe>(), n, points, (int)log_N, d_out.as<fe>());
        download(c, out16, d_out, values * 16);
    });
}

int dg_test_lde_fold8(const uint8_t *coeffs16, uint8_t *out16, uint32_t log_n, uint32_t log_b, uint32_t coset0, uint32_t ncosets, uint32_t batch,
                      uint64_t dst_stride) {
    return guarded([&] {
        DG_REQUIRE(coeffs16 && out16, "null buffer");
        require_batch(batch);
        DG_REQUIRE(log_n >= 1 && log_n <= 22 && log_b >= 3 && log_b <= 8, "log_n must be in 1..22 and log_b in 3..8");
        const uint64_t n = 1ULL << log_n, E = 8 * n, b = 1ULL << log_b;
        DG_REQUIRE(ncosets >= 1 && coset0 < b && ncosets <= b - coset0, "coset range out of bounds");
        const uint64_t out_n = strided_span(batch, dst_stride, ncosets * n, "dst_stride");
        require_canonical(coeffs16, batch * E, 1, "coefficient");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_in, d_out;
        upload(c, d_in, coeffs16, batch * E);
        zeroed(c, d_out, out_n);
        // stages 5 and 6: the constraint / composition polynomials of the batch, E apart
        lde_batch(c, d_in.as<fe>(), d_out.as<fe>(), (int)log_n, (int)log_b, 8, (int)batch, E, dst_stride, coset0, ncosets);
        download(c, out16, d_out, out_n * 16);
    });
}

int dg_test_coset_interp(const uint8_t *evals16, uint8_t *out16, uint32_t log_n, uint32_t batch, uint64_t out_stride) {
    return guarded([&] {
        DG_REQUIRE(evals16 && out16, "null buffer");
        require_batch(batch);
        DG_REQUIRE(log_n >= 1 && log_n <= 24, "log_n must be in 1..24");
        const uint64_t n = 1ULL << log_n, E = 8 * n;
        const uint64_t out_n = strided_span(batch, out_stride, E, "out_stride");
        require_canonical(evals16, batch * E, 1, "evaluation");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_evals, d_out;
        upload(c, d_evals, evals16, batch * E);
        zeroed(c, d_out, out_n);
        // stage 3: size-n inverse transforms of the 8 cosets of every vector, then the 8-point inverse DFT across them
        ntt_batch(c, d_evals.as<fe>(), d_evals.as<fe>(), (int)log_n, (int)batch * 8, n, n, true);
        coset_interp_finish(c, d_evals.as<fe>(), d_out.as<fe>(), (int)log_n, (int)batch, E, out_stride);
        download(c, out16, d_out, out_n * 16);
    });
}

int dg_test_fri_layer(const uint8_t *values16, uint32_t batch, uint64_t values_stride, uint32_t log_d, int32_t log_b, uint32_t log_N,
                      const uint8_t *roots32, uint64_t root_stride, uint8_t *leaves32, uint8_t *alphas16, uint8_t *root_copies32, uint8_t *next16) {
    return guarded([&] {
        DG_REQUIRE(values16 && roots32 && leaves32 && alphas16 && root_copies32 && next16, "null buffer");
        require_batch(batch);
        DG_REQUIRE(log_N <= 30 && log_d >= 4 && log_d <= log_N && (log_N - log_d) % 2 == 0,
                   "log_d must be in 4..log_N <= 30, an even number of folds below log_N");
        DG_REQUIRE(log_b >= -1 && log_b <= (int32_t)log_d, "log_b must be -1 (natural layout) or in 0..log_d");
        DG_REQUIRE(root_stride >= 32 && root_stride % 4 == 0 && root_stride <= (1ULL << 32), "root_stride must be a multiple of 4 in 32..2^32");
        const uint64_t D = 1ULL << log_d, R = D / 4;
        const uint64_t in_n = strided_span(batch, values_stride, D, "values_stride");
        require_canonical(values16, in_n, 1, "value");
        const Layout in{(int)log_d, log_b}, rows = fri_next_layout(in);
        const FoldConstants fold = fri_fold_constants();
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_vals, d_roots((batch - 1) * root_stride + 32), d_leaves, d_alpha, d_copies, d_next;
        upload(c, d_vals, values16, in_n);
        DG_CUDA(cudaMemsetAsync(d_roots.p, 0, d_roots.bytes, c.stream));
        DG_CUDA(cudaMemcpy2DAsync(d_roots.p, root_stride, roots32, 32, 32, batch, cudaMemcpyHostToDevice, c.stream));
        zeroed(c, d_leaves, batch * R * 2);
        zeroed(c, d_alpha, batch);
        zeroed(c, d_copies, batch * 2);
        zeroed(c, d_next, batch * R);
        fri_hash_rows(c, d_vals.as<fe>(), in, rows, d_leaves.p, (int)batch, values_stride);
        fri_alpha(c, d_roots.p, d_alpha.as<fe>(), d_copies.p, (int)batch, root_stride);
        fri_fold(c, d_vals.as<fe>(), in, d_next.as<fe>(), rows, d_alpha.as<fe>(), c.twiddle((int)log_N, true), (int)log_N, fold.tau_inv, fold.inv4,
                 (int)batch, values_stride);
        DG_CUDA(cudaMemcpyAsync(leaves32, d_leaves.p, batch * R * 32, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaMemcpyAsync(alphas16, d_alpha.p, (size_t)batch * 16, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaMemcpyAsync(root_copies32, d_copies.p, (size_t)batch * 32, cudaMemcpyDeviceToHost, c.stream));
        download(c, next16, d_next, batch * R * 16);
    });
}

// ---- test hooks: the evaluation-domain stage kernels (stage 1 trace extension, stage 2 trace commitment, stage 5 constraint items) -------
int dg_test_trace_lde(const uint8_t *regs16, uint32_t cols, uint32_t log_n, uint32_t log_b, uint32_t coset0, uint32_t ncosets, uint64_t col_stride,
                      int copy_coset0, uint8_t *polys16, uint8_t *ext16) {
    return guarded([&] {
        DG_REQUIRE(regs16 && polys16 && ext16, "null buffer");
        DG_REQUIRE(cols >= 1 && cols <= 65535, "cols must be in 1..65535");
        DG_REQUIRE(log_b >= 1 && log_b <= 16 && log_n >= 1 && log_n + log_b <= 30, "log_b must be in 1..16 and log_n in 1..30 - log_b");
        const uint64_t n = 1ULL << log_n, b = 1ULL << log_b;
        DG_REQUIRE(ncosets >= 1 && coset0 < b && ncosets <= b - coset0, "coset range out of bounds");
        const uint64_t out_n = strided_span(cols, col_stride, ncosets * n, "col_stride");
        require_canonical(regs16, cols * n, 1, "register element");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_regs, d_polys, d_ext;
        upload(c, d_regs, regs16, cols * n);
        zeroed(c, d_polys, cols * n);
        zeroed(c, d_ext, out_n);
        // stage 1: interpolate the register columns, then extend them onto the coset range (coset 0 copied from the registers when given)
        ntt_batch(c, d_regs.as<fe>(), d_polys.as<fe>(), (int)log_n, (int)cols, n, n, true);
        extend_trace_columns(c, d_polys.as<fe>(), copy_coset0 ? d_regs.as<fe>() : nullptr, d_ext.as<fe>(), (int)cols, (int)log_n, (int)log_b,
                             col_stride, coset0, ncosets);
        DG_CUDA(cudaMemcpyAsync(polys16, d_polys.p, cols * n * 16, cudaMemcpyDeviceToHost, c.stream));
        download(c, ext16, d_ext, out_n * 16);
    });
}

int dg_test_hash_trace_rows(const uint8_t *ext16, uint32_t total_cols, uint32_t log_n, uint32_t log_blowup, uint32_t c0, uint32_t nc, uint32_t batch,
                            const uint32_t *col_table, uint64_t leaf_stride, uint8_t *leaves32) {
    return guarded([&] {
        DG_REQUIRE(ext16 && leaves32, "null buffer");
        require_batch(batch);
        DG_REQUIRE(log_blowup <= 16 && log_n >= 1 && log_n + log_blowup <= 30, "log_blowup must be in 0..16 and log_n in 1..30 - log_blowup");
        const uint64_t n = 1ULL << log_n, all = n << log_blowup, rows = (uint64_t)nc * n;
        DG_REQUIRE(nc >= 1 && c0 < (1ULL << log_blowup) && nc <= (1ULL << log_blowup) - c0, "coset range out of bounds");
        DG_REQUIRE(total_cols >= 1 && total_cols <= 65535, "total_cols must be in 1..65535");
        uint32_t w = 0;
        if (col_table) {
            for (uint32_t q = 0; q < batch; q++)
                DG_REQUIRE(col_table[2 * q + 1] >= 1 && col_table[2 * q + 1] <= 127 && col_table[2 * q] < total_cols &&
                               col_table[2 * q + 1] <= total_cols - col_table[2 * q],
                           "matrix " + std::to_string(q) + ": columns out of range (width 1..127)");
        } else {
            DG_REQUIRE(total_cols % batch == 0, "without a column table the batch's matrices share total_cols evenly");
            w = total_cols / batch;
            DG_REQUIRE(w >= 1 && w <= 127, "width must be in 1..127");
        }
        DG_REQUIRE(leaf_stride == 0 || (leaf_stride >= all && leaf_stride <= (1ULL << 32)), "leaf_stride must be 0 or in 2^(log_n + log_blowup)..2^32");
        const uint64_t stride = leaf_stride ? leaf_stride : all, leaves = (batch - 1) * stride + all;
        require_canonical(ext16, total_cols * rows, 1, "extension element");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_ext, d_table, d_leaves;
        upload(c, d_ext, ext16, total_cols * rows);
        if (col_table) {
            d_table.alloc((size_t)batch * 8);
            DG_CUDA(cudaMemcpyAsync(d_table.p, col_table, (size_t)batch * 8, cudaMemcpyHostToDevice, c.stream));
        }
        zeroed(c, d_leaves, 2 * leaves);
        // stage 2 (the prover's Group::hash_chunk): the rows of the cosets [c0, c0 + nc) of every matrix, column stride nc n
        hash_trace_rows(c, d_ext.as<fe>(), d_leaves.p, (int)w, (int)log_n, (int)log_blowup, (int)batch, (unsigned long long)w * rows, c0, nc,
                        leaf_stride, col_table ? d_table.as<uint2>() : nullptr);
        download(c, leaves32, d_leaves, leaves * 32);
    });
}

int dg_test_merkle_batch(const uint8_t *leaves32, uint64_t L, uint32_t batch, uint8_t *nodes32) {
    return guarded([&] {
        DG_REQUIRE(leaves32 && nodes32, "null buffer");
        require_batch(batch);
        DG_REQUIRE(is_pow2(L) && L >= 2 && L <= (1ULL << 30), "L must be a power of 2 in 2..2^30");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_leaves, d_nodes;
        upload(c, d_leaves, leaves32, 2 * batch * L);
        zeroed(c, d_nodes, 2 * batch * L);
        // stages 2 and 5: the K trees of a batch, one launch per level for all of them
        merkle_build(c, d_leaves.p, d_nodes.p, L, (int)batch);
        download(c, nodes32, d_nodes, batch * L * 32);
    });
}

int dg_test_constraint_items(const uint8_t *evals16, uint32_t log_n, uint32_t log_nc, uint32_t batch, uint8_t *items32) {
    return guarded([&] {
        DG_REQUIRE(evals16 && items32, "null buffer");
        require_batch(batch);
        DG_REQUIRE(log_nc >= 2 && log_nc <= 16 && log_n >= 1 && log_n + log_nc <= 30, "log_nc must be in 2..16 and log_n in 1..30 - log_nc");
        const uint64_t slab = 1ULL << (log_n + log_nc), items = slab / 4;
        require_canonical(evals16, batch * slab, 1, "evaluation");
        Context &c = ctx();
        std::lock_guard<std::mutex> lk(c.mu);
        DevBuf d_evals, d_items;
        upload(c, d_evals, evals16, batch * slab);
        zeroed(c, d_items, 2 * batch * items);
        // stage 5: the first level of the constraint tree of every slab
        constraint_items_local(c, d_evals.as<fe>(), (int)log_n, (int)log_nc, d_items.p, (int)batch);
        download(c, items32, d_items, batch * items * 32);
    });
}

}  // extern "C"
