// Host orchestration of the CUDA prove pipeline: the body that replaces /root/reference/src/stark/prover.rs:17-169.
// Stage numbering and names follow the reference's nine debug!() sections (prover.rs:19-167) so that per-stage timings of
// the CPU prover and of this backend line up.  Only 32-byte roots, a handful of challenges and the final openings cross
// the PCIe bus after the register traces have been uploaded.
#include "prover.h"
#include "air.h"
#include "host_fs.h"
#include "poly.h"
#include "shard.h"
#include <algorithm>
#include <array>
#include <atomic>
#include <memory>
#include <thread>

namespace dg {

namespace {

struct StageClock {
    cudaStream_t s;
    cudaEvent_t ev[10];
    explicit StageClock(cudaStream_t stream) : s(stream) { for (auto &e : ev) DG_CUDA(cudaEventCreate(&e)); }
    ~StageClock() { for (auto &e : ev) cudaEventDestroy(e); }
    void mark(int i) { DG_CUDA(cudaEventRecord(ev[i], s)); }
    float between(int a, int b) { float ms = 0; cudaEventElapsedTime(&ms, ev[a], ev[b]); return ms; }
};

// optional fine-grained device timeline (DG_SUBSTAGE=1): named event marks inside the nine stages, printed by rank 0 after the proof
struct SubClock {
    bool on;
    cudaStream_t s;
    std::vector<std::pair<std::string, cudaEvent_t>> marks;
    explicit SubClock(cudaStream_t stream) : on(getenv("DG_SUBSTAGE") != nullptr), s(stream) {}
    void mark(const char *name) {
        if (!on) return;
        cudaEvent_t e;
        cudaEventCreate(&e);
        cudaEventRecord(e, s);
        marks.emplace_back(name, e);
    }
    void report(int rank) {
        if (!on) return;
        cudaStreamSynchronize(s);
        std::string line = "SUBSTAGE rank " + std::to_string(rank) + ":";
        for (size_t i = 1; i < marks.size(); i++) {
            float ms = 0;
            cudaEventElapsedTime(&ms, marks[i - 1].second, marks[i].second);
            char buf[96];
            snprintf(buf, sizeof buf, " %s=%.3f", marks[i].first.c_str(), ms);
            line += buf;
        }
        if (rank == 0 || atoi(getenv("DG_SUBSTAGE")) >= 2) fprintf(stderr, "%s\n", line.c_str());
        for (auto &m : marks) cudaEventDestroy(m.second);
        marks.clear();
    }
};

void d2h(Context &c, void *dst, const void *src, size_t bytes) {
    DG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c.stream));
    DG_CUDA(cudaStreamSynchronize(c.stream));
}
void h2d(Context &c, void *dst, const void *src, size_t bytes) {
    DG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c.stream));
}

// optional dump of intermediate device buffers (differential debugging against the oracle): DG_DEBUG_DUMP=<dir>
void debug_dump(Context &c, const char *name, const void *dev, size_t bytes) {
    const char *dir = getenv("DG_DEBUG_DUMP");
    if (!dir) return;
    std::vector<uint8_t> host(bytes);
    d2h(c, host.data(), dev, bytes);
    std::string path = std::string(dir) + "/" + name + ".bin";
    FILE *f = fopen(path.c_str(), "wb");
    if (!f) return;
    fwrite(host.data(), 1, bytes, f);
    fclose(f);
}

void debug_dump_host(const char *name, const void *host, size_t bytes) {
    const char *dir = getenv("DG_DEBUG_DUMP");
    if (!dir) return;
    std::string path = std::string(dir) + "/" + name + ".bin";
    FILE *f = fopen(path.c_str(), "wb");
    if (!f) return;
    fwrite(host, 1, bytes, f);
    fclose(f);
}

void require_extension_factor(uint64_t b) {
    DG_REQUIRE(b >= 16 && b <= 256 && (b & (b - 1)) == 0, "extension_factor must be a power of 2 between 16 and 256");
}

struct FriLayerDev {
    DevBuf leaves, nodes, folded;     // sharded layer: row hashes, tree and folded values of this rank
    const void *leaves_p = nullptr, *nodes_p = nullptr;     // replicated layer: row hashes and tree (buffers shared by the batch's proofs)
    const fe *vals;                   // replicated layer: the whole vector; sharded layer: this rank's cosets [c - c0][k]
    Layout layout;                    // layout of the (whole) layer (domain size 2^layout.log_d)
    bool sharded = false;             // multi-GPU: rows hashed / folded per coset range, tree = ShardedTree over [k'][c - c0] items
    ShardedTree tree;
};

}  // namespace

void check_options(const dg_options_t &o) {
    DG_REQUIRE(o.hash_id == 0, "unsupported hash function (only blake3 is serialisable, options.rs:107)");
    require_extension_factor(o.extension_factor);
    DG_REQUIRE(o.num_queries > 0 && o.num_queries <= 128, "num_queries must be in 1..128");
    DG_REQUIRE(o.grinding_factor <= 32, "grinding factor cannot be greater than 32");
}

// prover.h; dg_test_trace_lde calls it as stage 1 does
void extend_trace_columns(Context &c, const fe *polys, const fe *regs, fe *ext, int cols, int log_n, int log_b, uint64_t N_loc, unsigned c0,
                          unsigned nc) {
    const size_t n = (size_t)1 << log_n;
    if (c0 != 0 || !regs) {
        lde_batch(c, polys, ext, log_n, log_b, 1, cols, n, N_loc, c0, nc);
        return;
    }
    if (nc > 1) lde_batch(c, polys, ext + n, log_n, log_b, 1, cols, n, N_loc, 1, nc - 1);
    DG_CUDA(cudaMemcpy2DAsync(ext, N_loc * sizeof(fe), regs, n * sizeof(fe), n * sizeof(fe), cols, cudaMemcpyDeviceToDevice, c.stream));
}

// Upload of a host trace, overlapped with stage 1: column chunk i is extended as soon as its copy has landed.
//   * pinned (page-locked / registered) columns: cudaMemcpyAsync straight from the caller's memory on the copy stream;
//   * pageable columns (what a Rust Vec<u128> is): cudaMemcpyAsync would stage them through the driver's bounce buffer at ~8 GB/s and
//     block the calling thread.  Instead a few worker threads memcpy columns into the
//     library's own pinned slots and enqueue the DMA from there, so staging, DMA and the LDE of earlier columns run concurrently.
// The destructor joins the workers and drains the copy streams: on an error path no DMA from the caller's buffers is left in flight
// (the caller may free them as soon as dg_prove returns).
class TraceUploader {
public:
    static const int WORKERS = 4, SLOTS = 2;
    // chunk i = columns [bounds[i], bounds[i + 1])
    TraceUploader(Context &c, fe *d_regs, const uint8_t *const *host_cols, int w, uint64_t n, const std::vector<int> &bounds)
        : c_(c), w_(w), bounds_(bounds), nchunks_((int)bounds.size() - 1), col_bytes_(n * 16), done_(nchunks_, nullptr), recorded_(nchunks_) {
        for (auto &r : recorded_) r.store(0);
        for (auto &e : done_) DG_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        // the destination comes from the stream-ordered pool / arena of the compute stream: order the copies after it
        cudaEvent_t ready;
        DG_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
        DG_CUDA(cudaEventRecord(ready, c.stream));
        cudaPointerAttributes attr;
        const bool pinned = cudaPointerGetAttributes(&attr, host_cols[0]) == cudaSuccess && attr.type != cudaMemoryTypeUnregistered;
        cudaGetLastError();
        if (pinned) {
            DG_CUDA(cudaStreamWaitEvent(c.copy_stream, ready, 0));
            for (int i = 0; i < nchunks_; i++) {           // enqueue every upload first: the copy engine runs ahead of the compute stream
                for (int j = bounds_[i]; j < bounds_[i + 1]; j++)
                    DG_CUDA(cudaMemcpyAsync(d_regs + (size_t)j * n, host_cols[j], col_bytes_, cudaMemcpyHostToDevice, c.copy_stream));
                DG_CUDA(cudaEventRecord(done_[i], c.copy_stream));
                recorded_[i].store(1);
            }
        } else {
            c.staging.ensure((size_t)WORKERS * SLOTS * col_bytes_);
            for (int t = 0; t < WORKERS; t++) {
                if (!c.staging_streams[t]) DG_CUDA(cudaStreamCreateWithFlags(&c.staging_streams[t], cudaStreamNonBlocking));
                DG_CUDA(cudaStreamWaitEvent(c.staging_streams[t], ready, 0));
            }
            const int dev = c.device;
            for (int t = 0; t < WORKERS; t++)
                workers_.emplace_back([this, t, dev, d_regs, host_cols, n]() {
                    cudaSetDevice(dev);
                    cudaStream_t st = c_.staging_streams[t];
                    cudaEvent_t slot_free[SLOTS] = {nullptr, nullptr};
                    int use = 0;
                    // worker t owns the chunks i = t, t + WORKERS, ... ; chunks complete in order per worker, the consumer waits per chunk
                    for (int i = t; i < nchunks_ && !failed_.load(); i += WORKERS) {
                        for (int j = bounds_[i]; j < bounds_[i + 1]; j++, use++) {
                            const int s = use % SLOTS;
                            uint8_t *slot = (uint8_t *)c_.staging.p + ((size_t)t * SLOTS + s) * col_bytes_;
                            if (slot_free[s]) cudaEventSynchronize(slot_free[s]);
                            else cudaEventCreateWithFlags(&slot_free[s], cudaEventDisableTiming);
                            memcpy(slot, host_cols[j], col_bytes_);
                            if (cudaMemcpyAsync(d_regs + (size_t)j * n, slot, col_bytes_, cudaMemcpyHostToDevice, st) != cudaSuccess) failed_.store(true);
                            cudaEventRecord(slot_free[s], st);
                        }
                        if (cudaEventRecord(done_[i], st) != cudaSuccess) failed_.store(true);
                        recorded_[i].store(1);
                    }
                    for (int i = t; i < nchunks_; i += WORKERS) recorded_[i].store(1);      // after a failure: release the consumer
                    cudaStreamSynchronize(st);
                    for (auto &e : slot_free) if (e) cudaEventDestroy(e);
                });
        }
        cudaEventDestroy(ready);
    }
    // makes the compute stream wait for chunk i (blocks the host only until the copy of that chunk has been enqueued)
    void wait_chunk(int i) {
        while (!recorded_[i].load()) std::this_thread::yield();
        if (failed_.load()) throw Error(DG_ERR_CUDA, "host trace upload failed");
        DG_CUDA(cudaStreamWaitEvent(c_.stream, done_[i], 0));
    }
    int chunks() const { return nchunks_; }
    ~TraceUploader() {
        failed_.store(true);                               // stops workers that have not started their next chunk (normal exit: all done)
        for (auto &t : workers_) t.join();
        cudaStreamSynchronize(c_.copy_stream);
        for (auto &e : done_) if (e) cudaEventDestroy(e);
    }
private:
    Context &c_;
    int w_;
    std::vector<int> bounds_;
    int nchunks_;
    size_t col_bytes_;
    std::vector<cudaEvent_t> done_;
    std::vector<std::atomic<int>> recorded_;
    std::atomic<bool> failed_{false};
    std::vector<std::thread> workers_;
};

void upload_trace_columns(Context &c, fe *d_regs, const uint8_t *const *host_cols, int cols, uint64_t n) {
    const int chunk = (int)std::max<uint64_t>(1, std::min<uint64_t>(cols, ((uint64_t)1 << 26) / (n * 16)));     // ~64 MB per chunk
    std::vector<int> bounds = {0};
    while (bounds.back() < cols) bounds.push_back(std::min(cols, bounds.back() + chunk));
    TraceUploader up(c, d_regs, host_cols, cols, n, bounds);
    for (int i = 0; i < up.chunks(); i++) up.wait_chunk(i);
}

namespace {

typedef std::vector<std::vector<size_t>> Offsets;

// Per-proof host state of a batch.  A proof that fails (unsatisfied constraints, exhausted query positions) is marked dead and
// takes part in no later host-side work; its device lanes in the batched transforms keep computing on meaningless values.
struct ProofState {
    bool live = true;
    int status = DG_OK;
    std::string message;
    std::unique_ptr<Proof> proof{new Proof()};
    StarkProof stark;                     // filled by the stages that produce each field, written out in stage 9
    std::vector<fe> inputs, outputs;
    fs::ConstraintCoefficients cc;
    fs::CompositionCoefficients dc;
    ShardedTree t_tree, c_tree;
    std::vector<FriLayerDev> layers;
    std::vector<uint64_t> positions;
    void fail(int code, const std::string &m) { live = false; status = code; message = m; }
};

bool any_live(const std::vector<ProofState> &ps) {
    for (auto &s : ps) if (s.live) return true;
    return false;
}

// the 32-byte roots at `roots_dev` on the host: one copy for one tree, one FetchBatch for many
std::vector<Digest> fetch_roots(Context &c, const std::vector<const void *> &roots_dev) {
    std::vector<Digest> out(roots_dev.size());
    if (roots_dev.size() == 1) {
        d2h(c, out[0].data(), roots_dev[0], 32);
        return out;
    }
    FetchBatch fb(c);
    std::vector<size_t> off;
    for (const void *r : roots_dev) off.push_back(fb.add32(FetchRef{r, 0, -1}));
    fb.run();
    for (size_t i = 0; i < off.size(); i++) out[i] = fb.digest(off[i]);
    return out;
}

// the fine-grained device timeline (DG_SUBSTAGE): prove_core routes c.mark to its SubClock while the marks are on
void substage(Context &c, const char *name) {
    if (c.mark) c.mark(name);
}

// everything a proof opens, as offsets into the batch's FetchBatch (stage 9)
struct LayerOpen { std::vector<size_t> val_off; Offsets node_off; uint8_t depth; };
struct OpenPlan {
    std::vector<size_t> row_off;
    fs::BatchPlan tplan, cplan;
    Offsets t_off, c_off;
    std::vector<size_t> cval_off, rem_off;
    std::vector<LayerOpen> fri_open;
};

// The group of K proofs prove_core proves: what the call fixes (the constructor checks it and derives the geometry) and the device
// buffers that one stage writes and a later stage reads.  Each buffer is allocated by the stage that first writes it and lives until the
// group ends; a buffer only one stage uses is a local of that stage's function.
struct Group {
    // ---- the batch (trace_table.rs:23-58, options.rs:29-50, lib.rs:33-34) ----
    fe *d_regs;                                // [W][n] on the device; with host_cols not there yet (stage 1 uploads them)
    const uint8_t *const *host_cols;
    const std::vector<int> &order;             // Fiat-Shamir order of the proofs
    int K = 0;
    size_t W = 0;                              // columns of the whole batch
    std::vector<TraceShape> shapes;
    std::vector<uint32_t> col0;                // the column table: proof p's registers are the columns [col0[p], col0[p] + w_p) of the batch
    std::vector<int> shape_first = {0};        // runs of proofs of one shape: [shape_first[s], shape_first[s + 1])
    int wmax = 0, Tmax = 0;
    uint64_t n = 0, b = 0, N = 0, E = 0;
    int log_n = 0, log_b = 0, log_N = 0;
    fe root_n;                                 // w_n, generator of the trace domain
    // ---- sharding: rank g owns the LDE cosets [c0, c0 + nc) of every column (world == 1: all of them) ----
    int G = 1, g = 0, log_g = 0, log_nc = 0;
    uint64_t nc = 0, N_loc = 0;
    unsigned c0 = 0;
    // G > 1: the interpolation is sharded by columns -- rank r interpolates the columns [col_start(r), col_start(r) + col_count(r)), an even
    // split (the first w mod G ranks own one more), and the polynomials are all-gathered in equal slots of cpr columns per rank
    int w = 0, cpr = 0;                        // the width of the one proof; slot size of the gather = largest share
    // ---- layout of the extension.  ext holds `chunk` cosets of every column at a time ([W][chunk][n]).  The retained slab holds the
    // cosets stage 3 reads: in the full layout the whole extension (slab = ext), in the evaluation-coset layout the 8 cosets
    // c = 0 (mod b / 8), [W][8][n].  An opened row outside the retained cosets is computed from the trace polynomials in stage 9. ----
    unsigned chunk = 0;
    bool full = true;
    int log_ret = 0;                           // retained cosets: all of this rank's, or the 8 evaluation cosets
    uint64_t slab_col = 0, rstep = 0;          // slab column stride; retained cosets are c = 0 (mod rstep)
    uint64_t ext_col = 0;                      // column stride of ext (N_loc in the full layout)
    // the column table on the device: [K] (first column, width) of every proof, then [W] the proof of every column
    DevBuf d_table;
    const uint2 *d_cols = nullptr;
    const unsigned *d_col_proof = nullptr;
    // ---- buffers that cross stages (and those a stage keeps to the end of the group) ----
    DevBuf polys, ext, slab_own, t_leaves, t_nodes;      // 1-2: trace polynomials, extension, retained slab, trace trees
    DevBuf d_violation, d_coef, evals;                   // 3: violation flags, coefficients, [K][3][E] boundary / transition coefficients
    DevBuf combined, scratch, scratch2;                  // 4: the constraint polynomial, division scratch (scratch2: stage 6)
    DevBuf c_ext, c_items, c_nodes;                      // 5: constraint extension and trees
    DevBuf comp, comp_ext;                               // 6: composition polynomial and its extension
    DevBuf fri_gathered;                                 // 7, multi-GPU: the first replicated layer, gathered from the ranks' slabs
    std::vector<DevBuf> layer_bufs;                      // 7: replicated layers: row hashes, trees and folded values of all K proofs
    DevBuf d_rows;                                       // 9: opened trace rows computed from the polynomials

    Group(Context &c, fe *d_regs, const uint8_t *const *host_cols, const std::vector<RegisterShape> &regs_shape, uint64_t length,
          const std::vector<int> &order, std::vector<ProofState> &ps, const std::vector<dg_options_t> &opts, unsigned chunk);
    int col_count(int r) const { return w / G + (r < w % G ? 1 : 0); }
    int col_start(int r) const { return r * (w / G) + std::min(r, w % G); }
    const fe *slab_of(int p) const { return (full ? ext.as<fe>() : slab_own.as<fe>()) + (size_t)col0[p] * slab_col; }
    const fe *c_ext_of(int p) const { return c_ext.as<fe>() + (size_t)p * N_loc; }
    bool retained(uint64_t pos) const { return ((pos & (b - 1)) & (rstep - 1)) == 0; }
    void alloc_extension();
    void hash_chunk(Context &c, unsigned cc);
};

Group::Group(Context &c, fe *d_regs_, const uint8_t *const *host_cols_, const std::vector<RegisterShape> &regs_shape, uint64_t length,
             const std::vector<int> &order_, std::vector<ProofState> &ps, const std::vector<dg_options_t> &opts, unsigned chunk_)
    : d_regs(d_regs_), host_cols(host_cols_), order(order_) {
    K = (int)ps.size();
    DG_REQUIRE(K >= 1 && regs_shape.size() == ps.size() && order.size() == ps.size() && opts.size() == ps.size(), "batch must hold at least one trace");
    n = length;
    b = opts[0].extension_factor;
    for (const RegisterShape &r : regs_shape) W += r.width;
    DG_REQUIRE(W <= 65535, "batch too large for one launch (batched calls split larger batches into groups)");
    for (const dg_options_t &o : opts) {
        check_options(o);
        DG_REQUIRE(o.extension_factor == b, "the proofs of a group share one extension factor");
    }
    DG_REQUIRE(n >= 16 && (n & (n - 1)) == 0, "execution trace length must be a power of 2 and at least 16");
    for (const RegisterShape &r : regs_shape) shapes.push_back(TraceShape::of_trace(r.width, r.ctx_depth, r.loop_depth));
    col0.assign(K + 1, 0);
    for (int p = 0; p < K; p++) {
        col0[p + 1] = col0[p] + shapes[p].w;
        wmax = std::max(wmax, shapes[p].w);
        Tmax = std::max(Tmax, shapes[p].T);
    }
    log_n = ceil_log2(n);
    log_b = ceil_log2(b);
    log_N = log_n + log_b;
    DG_REQUIRE(log_N <= 30, "LDE domain too large");
    N = n * b;
    E = n * 8;
    for (int p = 0; p < K; p++) {             // what the call fixes in every proof: the register shape and its options (blake3)
        TraceInfo &t = ps[p].stark.trace_info;
        t.ctx_depth = (uint8_t)shapes[p].ctx_depth; t.loop_depth = (uint8_t)shapes[p].loop_depth; t.stack_depth = (uint8_t)shapes[p].stack_depth;
        ps[p].stark.options = ProofOptions{(uint8_t)log_b, (uint8_t)opts[p].num_queries, (uint8_t)opts[p].grinding_factor, 0};
    }
    for (int p = 1; p < K; p++)
        if (!(regs_shape[p] == regs_shape[p - 1])) shape_first.push_back(p);
    shape_first.push_back(K);
    root_n = host_root_of_unity(log_n);

    G = c.world;
    g = c.rank;
    DG_REQUIRE(G == 1 || K == 1, "a batch of proofs runs on one GPU (the context spans several)");
    log_g = ceil_log2(G);
    DG_REQUIRE((b >> log_g) >= 4 && G <= 8, "extension factor too small for this many GPUs (need >= 4 cosets per rank)");
    log_nc = log_b - log_g;
    nc = 1ULL << log_nc;
    N_loc = n * nc;
    c0 = (unsigned)(g * nc);
    w = shapes[0].w;
    cpr = (w + G - 1) / G;

    chunk = chunk_;
    if (G > 1 || chunk == 0 || chunk > nc) chunk = (unsigned)nc;
    DG_REQUIRE((chunk & (chunk - 1)) == 0, "coset chunk must be a power of 2");
    full = chunk == nc;
    log_ret = full ? log_nc : 3;
    slab_col = n << log_ret;
    rstep = nc >> log_ret;
    ext_col = n * chunk;

    d_table.alloc((2 * K + W) * 4);
    std::vector<uint32_t> table(2 * K + W);
    for (int p = 0; p < K; p++) {
        table[2 * p] = col0[p];
        table[2 * p + 1] = (uint32_t)shapes[p].w;
        for (uint32_t j = col0[p]; j < col0[p + 1]; j++) table[2 * K + j] = (uint32_t)p;
    }
    h2d(c, d_table.p, table.data(), table.size() * 4);
    d_cols = d_table.as<uint2>();
    d_col_proof = d_table.as<unsigned>() + 2 * K;
}

// ---- 1: extend execution trace ------------------------------------------------------------------------------------------------------------
void Group::alloc_extension() {
    polys.alloc(W * n * 16);
    ext.alloc(W * ext_col * 16);
    if (!full) slab_own.alloc(W * slab_col * 16);
    t_leaves.alloc((size_t)K * N_loc * 32);
}

// rows of the chunk at cc: leaves (k << log_b) + c of every proof; then its retained cosets into the slab
void Group::hash_chunk(Context &c, unsigned cc) {
    hash_trace_rows(c, ext.as<fe>(), t_leaves.p, w, log_n, log_nc, K, 0, cc, chunk, N_loc, d_cols);   // local rows, [k][c - c0], per proof
    if (full) return;
    for (unsigned cs = cc; cs < cc + chunk; cs++)
        if (cs % rstep == 0)
            DG_CUDA(cudaMemcpy2DAsync(slab_own.as<fe>() + (cs / rstep) * n, slab_col * 16, ext.as<fe>() + (size_t)(cs - cc) * n, ext_col * 16, n * 16, W,
                                      cudaMemcpyDeviceToDevice, c.stream));
}

// One GPU: the K proofs' registers are the W columns of one batch, interpolated in column chunks: a host trace is uploaded in chunks of
// ~64 MB, but a short ramp first (1, 2 columns), so that the first transform starts after one column's worth of copying; every column
// chunk is extended on the first coset chunk as soon as it has been interpolated.  Every coset chunk but the last is hashed here.
void extend_trace(Context &c, Group &grp) {
    grp.alloc_extension();
    const uint64_t n = grp.n;
    const int W = (int)grp.W;
    fe *regs = grp.d_regs, *polys = grp.polys.as<fe>(), *ext = grp.ext.as<fe>();
    std::vector<int> bounds = {0};
    std::unique_ptr<TraceUploader> up;
    if (grp.host_cols) {
        const int step_max = (int)std::max<uint64_t>(1, std::min<uint64_t>(W, ((uint64_t)1 << 26) / (n * 16)));
        for (int step = 1; bounds.back() < W; step = std::min(step_max, step * 2)) bounds.push_back(std::min(W, bounds.back() + step));
        up.reset(new TraceUploader(c, regs, grp.host_cols, W, n, bounds));
    } else {
        bounds.push_back(W);
    }
    for (unsigned cc = 0; cc < grp.nc; cc += grp.chunk) {
        if (cc > 0) grp.hash_chunk(c, cc - grp.chunk);          // the last chunk is hashed in stage 2
        for (size_t i = 0; i + 1 < bounds.size(); i++) {
            const int j0 = bounds[i], cols = bounds[i + 1] - j0;
            if (cc == 0) {
                if (up) up->wait_chunk((int)i);
                ntt_batch(c, regs + (size_t)j0 * n, polys + (size_t)j0 * n, grp.log_n, cols, n, n, true);
            }
            extend_trace_columns(c, polys + (size_t)j0 * n, regs + (size_t)j0 * n, ext + (size_t)j0 * grp.ext_col, cols, grp.log_n, grp.log_b,
                                 grp.ext_col, cc, grp.chunk);
        }
    }
}

// Several GPUs (one proof): rank g interpolates its share of the columns and only needs (from a host trace: only uploads) those
// registers; the polynomials are all-gathered (and compacted into natural column order) while the rank extends its own columns, then
// every rank extends all columns on its cosets.
void extend_trace_sharded(Context &c, Group &grp) {
    grp.alloc_extension();
    const uint64_t n = grp.n, N_loc = grp.N_loc;
    const int G = grp.G, cpr = grp.cpr, w = grp.w, log_n = grp.log_n, log_b = grp.log_b;
    const unsigned c0 = grp.c0, nc = (unsigned)grp.nc;
    fe *regs = grp.d_regs, *polys = grp.polys.as<fe>(), *ext = grp.ext.as<fe>();
    const uint8_t *const *host_cols = grp.host_cols;
    const int j0 = grp.col_start(grp.g), mine = grp.col_count(grp.g);
    DevBuf own((size_t)cpr * n * 16), slots((size_t)cpr * G * n * 16);
    if (mine > 0) {
        if (host_cols) {
            std::vector<int> bounds(mine + 1);
            for (int i = 0; i <= mine; i++) bounds[i] = i;
            TraceUploader up(c, regs + (size_t)j0 * n, host_cols + j0, mine, n, bounds);      // one column per chunk: all staging workers busy
            for (int i = 0; i < up.chunks(); i++) {              // interpolate every column as soon as it has landed
                up.wait_chunk(i);
                ntt_batch(c, regs + (size_t)(j0 + i) * n, own.as<fe>() + (size_t)i * n, log_n, 1, n, n, true);
            }
        } else {
            ntt_batch(c, regs + (size_t)j0 * n, own.as<fe>(), log_n, mine, n, n, true);
        }
    }
    substage(c, "1.intt");
    // the all-gather of the polynomials (and their compaction into column order) runs on the communication stream while this rank
    // already extends its own columns
    cudaEvent_t ev_own, ev_all;
    DG_CUDA(cudaEventCreateWithFlags(&ev_own, cudaEventDisableTiming));
    DG_CUDA(cudaEventCreateWithFlags(&ev_all, cudaEventDisableTiming));
    DG_CUDA(cudaEventRecord(ev_own, c.stream));
    DG_CUDA(cudaStreamWaitEvent(c.comm_stream, ev_own, 0));
    comm_all_gather(c, own.p, slots.p, (size_t)cpr * n * 16, c.comm_stream);
    for (int r = 0; r < G; r++)
        if (grp.col_count(r) > 0)
            DG_CUDA(cudaMemcpyAsync(polys + (size_t)grp.col_start(r) * n, slots.as<fe>() + (size_t)r * cpr * n, (size_t)grp.col_count(r) * n * 16,
                                    cudaMemcpyDeviceToDevice, c.comm_stream));
    DG_CUDA(cudaEventRecord(ev_all, c.comm_stream));
    if (mine > 0) extend_trace_columns(c, own.as<fe>(), regs + (size_t)j0 * n, ext + (size_t)j0 * N_loc, mine, log_n, log_b, N_loc, c0, nc);
    substage(c, "1.lde_own");
    DG_CUDA(cudaStreamWaitEvent(c.stream, ev_all, 0));
    // the other ranks' registers are on this device only when the trace was given in device memory (a host trace uploads own columns only)
    if (j0 > 0) extend_trace_columns(c, polys, host_cols ? nullptr : regs, ext, j0, log_n, log_b, N_loc, c0, nc);
    if (j0 + mine < w)
        extend_trace_columns(c, polys + (size_t)(j0 + mine) * n, host_cols ? nullptr : regs + (size_t)(j0 + mine) * n, ext + (size_t)(j0 + mine) * N_loc,
                             w - j0 - mine, log_n, log_b, N_loc, c0, nc);
    cudaEventDestroy(ev_own);
    cudaEventDestroy(ev_all);
}

// ---- 2: trace Merkle tree -------------------------------------------------------------------------------------------------------------------
// one GPU: the K trees level by level in one launch per level; several GPUs (K == 1): the sharded tree
void commit_trace(Context &c, Group &grp, std::vector<ProofState> &ps) {
    const int K = grp.K;
    const uint64_t N_loc = grp.N_loc;
    grp.hash_chunk(c, (unsigned)(grp.nc - grp.chunk));
    substage(c, "2.hash_rows");
    if (grp.G == 1) {
        grp.t_nodes.alloc((size_t)K * N_loc * 32);
        merkle_build(c, grp.t_leaves.p, grp.t_nodes.p, N_loc, K);
    }
    std::vector<const void *> roots;
    for (int p = 0; p < K; p++) {
        const uint8_t *leaves = (const uint8_t *)grp.t_leaves.p + (size_t)p * N_loc * 32;
        if (grp.G == 1) ps[p].t_tree.attach(c, leaves, (const uint8_t *)grp.t_nodes.p + (size_t)p * N_loc * 32, grp.n, grp.log_nc);
        else ps[p].t_tree.build(c, leaves, grp.n, grp.log_nc, false);
        roots.push_back(ps[p].t_tree.root_dev());
    }
    std::vector<Digest> r = fetch_roots(c, roots);
    for (int p = 0; p < K; p++) ps[p].stark.trace_root = r[p];
}

// ---- 3: evaluate constraints --------------------------------------------------------------------------------------------------------------
// false when every proof failed its transition constraints: the group ends there
bool evaluate_constraints(Context &c, Group &grp, std::vector<ProofState> &ps) {
    const int K = grp.K, G = grp.G, log_n = grp.log_n;
    const uint64_t n = grp.n, E = grp.E;
    const std::vector<TraceShape> &shapes = grp.shapes;
    std::vector<fe> last_rows((size_t)3 * K);      // op_counter and program hash of the last trace step of every proof (evaluator.rs:73-74)
    if (grp.host_cols) {
        for (int p = 0; p < K; p++)
            for (int j = 0; j < 3; j++) memcpy(&last_rows[3 * p + j], grp.host_cols[grp.col0[p] + j] + (n - 1) * 16, 16);
    } else {
        DevBuf d_last((size_t)48 * K);
        for (size_t s = 0; s + 1 < grp.shape_first.size(); s++) {          // the proofs of one shape are w n elements apart
            const int p0 = grp.shape_first[s], k = grp.shape_first[s + 1] - p0;
            for (int j = 0; j < 3; j++)
                DG_CUDA(cudaMemcpy2DAsync((uint8_t *)d_last.p + 48 * p0 + 16 * j, 48, grp.d_regs + (size_t)(grp.col0[p0] + j) * n + (n - 1),
                                          (size_t)shapes[p0].w * n * 16, 16, k, cudaMemcpyDeviceToDevice, c.stream));
        }
        d2h(c, last_rows.data(), d_last.p, (size_t)48 * K);
    }
    grp.d_violation.alloc((size_t)4 * K);
    // per proof [coefA | coefB | bAi | bBi | bAf | bBf], coef_stride elements apart, then the boundary constants [K][KiA, KiB, KfA, KfB].
    // The transition coefficients of a proof are T of its shape: coefA and coefB are padded to the batch's largest count Tmax.  The
    // boundary vectors have one entry per register that carries a boundary constraint, which depends on the shape and on the number of
    // public inputs / outputs: they are padded with zero coefficients to the largest count nbm (a zero coefficient adds nothing to the
    // boundary numerators).
    const size_t T = grp.Tmax;
    size_t nbm = 0;
    for (int p : grp.order) {
        ProofState &s = ps[p];
        s.stark.trace_info.op_count = (uint32_t)last_rows[3 * p].lo;       // op_count as u32 (proof.rs:62)
        const fe program_hash[2] = {last_rows[3 * p + 1], last_rows[3 * p + 2]};
        s.cc = fs::draw_constraint_coefficients(s.stark.trace_root.data(), shapes[p], s.inputs, s.outputs, last_rows[3 * p], program_hash);
        DG_REQUIRE(s.cc.bAi.size() <= (size_t)shapes[p].w, "more boundary registers than registers");
        nbm = std::max(nbm, s.cc.bAi.size());
    }
    const size_t coef_stride = 2 * T + 4 * nbm;
    {
        std::vector<fe> pack(coef_stride * K + 4 * K, fe_make(0, 0));
        for (int p = 0; p < K; p++) {
            ProofState &s = ps[p];
            auto at = pack.begin() + (size_t)p * coef_stride;
            std::copy(s.cc.coefA.begin(), s.cc.coefA.end(), at);
            std::copy(s.cc.coefB.begin(), s.cc.coefB.end(), at + T);
            int slot = 0;
            for (const auto *v : {&s.cc.bAi, &s.cc.bBi, &s.cc.bAf, &s.cc.bBf}) std::copy(v->begin(), v->end(), at + 2 * T + (slot++) * nbm);
            const fe consts[4] = {s.cc.KiA, s.cc.KiB, s.cc.KfA, s.cc.KfB};
            std::copy(consts, consts + 4, pack.begin() + coef_stride * K + 4 * p);
        }
        grp.d_coef.alloc(pack.size() * 16);
        h2d(c, grp.d_coef.p, pack.data(), pack.size() * 16);
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }
    const fe *coef = grp.d_coef.as<fe>();
    DG_CUDA(cudaMemsetAsync(grp.d_violation.p, 0, (size_t)4 * K, c.stream));
    // per proof: [boundary numerator, first step | boundary numerator, last step | transition combination]
    grp.evals.alloc((size_t)K * 3 * E * 16);
    fe *evals = grp.evals.as<fe>();
    const int num_c8 = 8 >> grp.log_g;
    const uint64_t E_loc = n * num_c8;
    DevBuf evals_loc((size_t)K * E_loc * 16), gathered;
    if (G > 1) gathered.alloc(E * 16);
    // one launch per register shape, over that shape's proofs (adjacent, so at uniform strides)
    for (size_t s = 0; s + 1 < grp.shape_first.size(); s++) {
        const int p0 = grp.shape_first[s], k = grp.shape_first[s + 1] - p0;
        AirParams P = shapes[p0].air_params(n);
        // the retained slab: all cosets (log_blowup = log_b, powers of w_N), or the 8 evaluation cosets as an extension by 8 (powers of
        // w_8n = w_N^(b/8): lde_index * inc selects the same power of the root)
        P.log_blowup = grp.full ? grp.log_b : 3;
        P.ext = grp.slab_of(p0); P.col_stride = grp.slab_col;
        P.c8_base = grp.g * num_c8; P.num_c8 = num_c8;
        P.t_ev = evals_loc.as<fe>() + (size_t)p0 * E_loc;
        P.periodic = periodic_table(c);
        const fe *base = coef + (size_t)p0 * coef_stride;
        P.coefA = base; P.coefB = base + T;
        P.twN = c.twiddle(grp.full ? grp.log_N : log_n + 3, false);
        P.violation = grp.d_violation.as<unsigned>() + p0;
        P.ext_stride = (size_t)shapes[p0].w * grp.slab_col; P.t_ev_stride = E_loc; P.coef_stride = coef_stride;
        if (s == 0) substage(c, "3.setup");
        launch_constraint_eval(c, P, k);
    }
    substage(c, "3.eval");
    comm_all_reduce_max_u32(c, grp.d_violation.as<unsigned>(), 1);
    std::vector<unsigned> violation(K);
    d2h(c, violation.data(), grp.d_violation.p, (size_t)4 * K);
    for (int p = 0; p < K; p++)
        if (violation[p])
            ps[p].fail(DG_ERR_UNSATISFIED, "transition constraints at step " + std::to_string(violation_step(violation[p])) + " were not satisfied");
    if (!any_live(ps)) return false;
    // interpolation of the transition combination (constraint_table.rs:54-63), coset by coset: size-n inverse transforms of the own
    // cosets (sharded), all-gather, then the 8-point inverse DFT across cosets (poly.cu: coset_interp_finish) -> the 8n coefficients
    // in natural order; no transposition and no replicated 8n-point transform
    substage(c, "3.violation_sync");
    ntt_batch(c, evals_loc.as<fe>(), evals_loc.as<fe>(), log_n, K * num_c8, n, n, true);
    if (G > 1) comm_all_gather(c, evals_loc.as<fe>(), gathered.as<fe>(), E_loc * 16);
    substage(c, "3.intt+gather");
    coset_interp_finish(c, G > 1 ? gathered.as<fe>() : evals_loc.as<fe>(), evals + 2 * E, log_n, K, E_loc, 3 * E);
    // boundary constraints (evaluator.rs:181-326), directly as the 8n coefficients the reference obtains by interpolation
    boundary_coeffs(c, K, grp.polys.as<fe>(), 0, n, (int)nbm, coef + 2 * T, coef_stride, coef + coef_stride * K, evals, evals + E, 3 * E, grp.d_cols);
    if (K == 1) debug_dump(c, "t_coeffs", evals + 2 * E, E * 16);
    return true;
}

// ---- 4: convert constraint evaluations into a polynomial -----------------------------------------------------------------------------------
void constraint_polynomial(Context &c, Group &grp) {
    const int K = grp.K;
    const uint64_t E = grp.E;
    grp.combined.alloc((size_t)K * E * 16);
    grp.scratch.alloc((size_t)K * E * 16);
    grp.scratch2.alloc((size_t)K * E * 16);
    const fe x_last = host_inv(grp.root_n);                    // w_n^(n-1)   (evaluator.rs:128-131)
    fe *ic = grp.evals.as<fe>(), *fc = ic + E, *tc = ic + 2 * E;          // of proof 0; proof p at + 3 E p
    if (K == 1) {
        debug_dump(c, "i_coeffs", ic, E * 16);
        debug_dump(c, "f_coeffs", fc, E * 16);
    }
    // one upload: the (base, step) pairs of the power tables of 1, x_last and 1 / x_last (shared by the K proofs), then K zeros (sub0)
    std::vector<fe> pack(6 + K, fe_make(0, 0));
    pack[0] = fe_make(1, 0);
    pack[1] = PowTables::step(pack[0], E + 1);
    PowTables::pack_point(pack.data() + 2, 2, x_last, E + 1);
    DevBuf d_pack(pack.size() * 16);
    h2d(c, d_pack.p, pack.data(), pack.size() * 16);
    PowTables pows(c, d_pack.as<fe>(), 3, E + 1);
    const fe *zeros = d_pack.as<fe>() + 6;
    syn_div(c, K, ic, 3 * E, ic, 3 * E, E, pows.ref(0), 0, 0, pows.ref(0), 0, 0, zeros);   // / (x - 1)
    syn_div(c, K, fc, 3 * E, fc, 3 * E, E, pows.ref(1), 0, 0, pows.ref(2), 0, 0, zeros);   // / (x - x_last)
    syn_div_expanded_sum(c, tc, grp.scratch.as<fe>(), ic, fc, grp.combined.as<fe>(), grp.n, E, x_last, K, 3 * E, E);   // / ((x^n - 1)/(x - x_last)), summed
    if (K == 1) debug_dump(c, "constraint_poly", grp.combined.p, E * 16);
}

// ---- 5: constraint evaluations over the LDE domain + their Merkle tree ---------------------------------------------------------------------
void commit_constraints(Context &c, Group &grp, std::vector<ProofState> &ps) {
    const int K = grp.K, log_nc = grp.log_nc;
    const uint64_t N_loc = grp.N_loc;
    grp.c_ext.alloc((size_t)K * N_loc * 16);
    grp.c_items.alloc((size_t)K * (N_loc / 4) * 32);
    lde_batch(c, grp.combined.as<fe>(), grp.c_ext.as<fe>(), grp.log_n, grp.log_b, 8, K, grp.E, N_loc, grp.c0, (unsigned)grp.nc);
    substage(c, "5.lde");
    constraint_items_local(c, grp.c_ext.as<fe>(), grp.log_n, log_nc, grp.c_items.p, K);      // first tree level: H(4 evaluations), [k][c4 local], per proof
    substage(c, "5.items");
    if (grp.G == 1) {
        grp.c_nodes.alloc((size_t)K * (N_loc / 4) * 32);
        merkle_build(c, grp.c_items.p, grp.c_nodes.p, N_loc / 4, K);
    }
    std::vector<const void *> roots;
    std::vector<int> who;
    for (int p = 0; p < K; p++) {
        if (!ps[p].live) continue;
        const uint8_t *items = (const uint8_t *)grp.c_items.p + (size_t)p * (N_loc / 4) * 32;
        if (grp.G == 1) ps[p].c_tree.attach(c, items, (const uint8_t *)grp.c_nodes.p + (size_t)p * (N_loc / 4) * 32, grp.n, log_nc - 2);
        else ps[p].c_tree.build(c, items, grp.n, log_nc - 2, false);
        roots.push_back(ps[p].c_tree.root_dev());
        who.push_back(p);
    }
    std::vector<Digest> r = fetch_roots(c, roots);
    for (size_t i = 0; i < who.size(); i++) ps[who[i]].stark.constraint_root = r[i];
}

// ---- 6: DEEP composition polynomial --------------------------------------------------------------------------------------------------------
void deep_composition(Context &c, Group &grp, std::vector<ProofState> &ps) {
    const int K = grp.K, G = grp.G, cpr = grp.cpr, wmax = grp.wmax;
    const uint64_t n = grp.n, E = grp.E;
    fe *polys = grp.polys.as<fe>(), *combined = grp.combined.as<fe>();
    grp.comp.alloc((size_t)K * E * 16);
    grp.comp_ext.alloc((size_t)K * grp.N_loc * 16);
    TwiddleRef g_t = c.twiddle(grp.log_n, false);
    // trace polynomials at z and z*g: every rank evaluates its own columns (the split of stage 1); slots of 2 cpr values are gathered.
    // d_deep = 2 trace values per column (one GPU: proof p's from column col0[p] on; several: G slots of cpr columns), then [K][2]
    // values of the constraint polynomial at z
    const size_t deep_cols = G == 1 ? grp.W : (size_t)cpr * G;
    DevBuf d_deep((2 * deep_cols + 2 * K) * 16);
    fe *deep_c = d_deep.as<fe>() + 2 * deep_cols;
    DG_CUDA(cudaMemsetAsync(d_deep.p, 0, d_deep.bytes, c.stream));
    // powers of z, 1/z, z g, 1/(z g) of every proof: four batched tables from one upload of the (base, step) pairs, [table][proof][2]
    std::vector<fe> base_step((size_t)8 * K, fe_make(0, 0));
    for (int p : grp.order) {
        ProofState &s = ps[p];
        if (!s.live) continue;
        s.dc = fs::draw_composition_coefficients(s.stark.constraint_root.data(), grp.shapes[p].w);
        PowTables::pack_point(&base_step[(size_t)2 * p], (size_t)2 * K, s.dc.z, E + 1);
        PowTables::pack_point(&base_step[(size_t)2 * (2 * K + p)], (size_t)2 * K, fe_mul(s.dc.z, grp.root_n), n + 1);
    }
    DevBuf d_base_step(base_step.size() * 16);
    h2d(c, d_base_step.p, base_step.data(), base_step.size() * 16);
    const fe *bs = d_base_step.as<fe>();
    PowTables z_t(c, bs, K, E + 1), zi_t(c, bs + 2 * K, K, E + 1), zg_t(c, bs + 4 * K, K, n + 1), zgi_t(c, bs + 6 * K, K, n + 1);
    if (G == 1) {
        eval_polys_at(c, polys, n, (int)grp.W, z_t.ref(0), g_t, true, d_deep.as<fe>(), 1 << 30, z_t.lo_n, z_t.hi_n, grp.d_col_proof);
    } else {
        const int j0 = grp.col_start(grp.g), mine = grp.col_count(grp.g);
        if (mine > 0) eval_polys_at(c, polys + (size_t)j0 * n, n, mine, z_t.ref(0), g_t, true, d_deep.as<fe>() + (size_t)2 * grp.g * cpr);
        comm_all_gather(c, d_deep.as<fe>() + (size_t)2 * grp.g * cpr, d_deep.p, (size_t)2 * cpr * 16);
    }
    eval_polys_at(c, combined, E, K, z_t.ref(0), g_t, false, deep_c, 1, z_t.lo_n, z_t.hi_n);
    std::vector<fe> deep_slots(2 * deep_cols + 2 * K);
    d2h(c, deep_slots.data(), d_deep.p, deep_slots.size() * 16);
    substage(c, "6.deep_values");
    // one upload: [K][2 wmax] coefficients of the trace combinations (proof p's trace1 | trace2 at p 2 wmax, p 2 wmax + wmax) | sub0
    // of the three divisions [3][K] | compose's k1, k2, kc [K][3]
    std::vector<fe> pack((size_t)K * (2 * wmax + 6), fe_make(0, 0));
    fe *ccs = pack.data(), *subs = ccs + (size_t)K * 2 * wmax, *ks = subs + (size_t)3 * K;
    for (int p = 0; p < K; p++) {
        ProofState &s = ps[p];
        if (!s.live) continue;
        const int wq = grp.shapes[p].w;
        const fe *slots = deep_slots.data() + 2 * (size_t)grp.col0[p];           // several GPUs: K == 1, col0[0] == 0
        std::vector<fe> deep(2 * wq);
        for (int r = 0; r < G; r++)
            for (int o = 0; o < (G == 1 ? wq : grp.col_count(r)); o++) {
                const int from = G == 1 ? o : r * cpr + o, to = G == 1 ? o : grp.col_start(r) + o;
                deep[2 * to] = slots[2 * from];
                deep[2 * to + 1] = slots[2 * from + 1];
            }
        std::vector<fe> &z1 = s.stark.trace_at_z1, &z2 = s.stark.trace_at_z2;
        z1.resize(wq); z2.resize(wq);
        fe sub1 = fe_make(0, 0), sub2 = fe_make(0, 0);
        for (int i = 0; i < wq; i++) {
            z1[i] = deep[2 * i]; z2[i] = deep[2 * i + 1];
            sub1 = fe_add(sub1, fe_mul(z1[i], s.dc.trace1[i]));
            sub2 = fe_add(sub2, fe_mul(z2[i], s.dc.trace2[i]));
        }
        subs[p] = sub1; subs[K + p] = sub2; subs[2 * K + p] = deep_slots[2 * deep_cols + 2 * p];
        std::copy(s.dc.trace1.begin(), s.dc.trace1.begin() + wq, ccs + (size_t)p * 2 * wmax);
        std::copy(s.dc.trace2.begin(), s.dc.trace2.begin() + wq, ccs + (size_t)p * 2 * wmax + wmax);
        ks[3 * p] = s.dc.t1_degree; ks[3 * p + 1] = s.dc.t2_degree; ks[3 * p + 2] = s.dc.constraints;
    }
    DevBuf d_pack(pack.size() * 16), t12((size_t)K * 2 * n * 16);
    h2d(c, d_pack.p, pack.data(), pack.size() * 16);
    const fe *d_cc = d_pack.as<fe>(), *d_subs = d_cc + (size_t)K * 2 * wmax, *d_ks = d_subs + (size_t)3 * K;
    fe *t1 = t12.as<fe>(), *t2 = t12.as<fe>() + n;                      // of proof 0; proof p at + 2 n p
    fe *scratch2 = grp.scratch2.as<fe>();
    lincomb2(c, polys, n, wmax, d_cc, d_cc + wmax, t1, t2, K, 2 * wmax, 2 * n, grp.d_cols);
    syn_div(c, K, t1, 2 * n, t1, 2 * n, n, z_t.ref(0), z_t.lo_n, z_t.hi_n, zi_t.ref(0), zi_t.lo_n, zi_t.hi_n, d_subs);
    //                                                                                                   (T1(x) - T1(z)) / (x - z)
    syn_div(c, K, t2, 2 * n, t2, 2 * n, n, zg_t.ref(0), zg_t.lo_n, zg_t.hi_n, zgi_t.ref(0), zgi_t.lo_n, zgi_t.hi_n, d_subs + K);
    //                                                                                                   (T2(x) - T2(zg)) / (x - zg)
    syn_div(c, K, combined, E, scratch2, E, E, z_t.ref(0), z_t.lo_n, z_t.hi_n, zi_t.ref(0), zi_t.lo_n, zi_t.hi_n, d_subs + 2 * K);
    //                                                                                                   (C(x) - C(z)) / (x - z)
    substage(c, "6.lincomb+syndiv");
    compose(c, K, t1, t2, 2 * n, scratch2, grp.comp.as<fe>(), n, E, 6 * n + 1, d_ks);
    if (K == 1) debug_dump(c, "composition_poly", grp.comp.p, E * 16);
    // every rank extends its own cosets; the first FRI layers work on these slabs directly (no all-gather of the N evaluations)
    lde_batch(c, grp.comp.as<fe>(), grp.comp_ext.as<fe>(), grp.log_n, grp.log_b, 8, K, E, grp.N_loc, grp.c0, (unsigned)grp.nc);
}

// ---- 7: FRI layers -------------------------------------------------------------------------------------------------------------------------
// The layer roots and folding points of a group stay on the device, [layer][proof] (special_x = prng(root) is derived by fri_alpha): the
// host sees the roots in one copy after the last layer.  With host RNG callbacks registered each layer asks the host instead: one copy
// of the layer's K roots, the callbacks of the live proofs in proof order, one upload of the K folding points.
struct FriRun {
    static const int MAX_LAYERS = 20;
    Context &c;
    const std::vector<ProofState> &ps;
    const std::vector<int> &order;
    const int K;
    DevBuf d_alpha, d_roots;
    const bool host_rng = fs::rng_hooks_active();
    FriRun(Context &c_, const Group &grp, const std::vector<ProofState> &ps_)
        : c(c_), ps(ps_), order(grp.order), K(grp.K), d_alpha((size_t)MAX_LAYERS * K * 16), d_roots((size_t)MAX_LAYERS * K * 32) {}
    fe *alpha(size_t layer) { return d_alpha.as<fe>() + layer * K; }
    uint8_t *root_slots(size_t layer) { return (uint8_t *)d_roots.p + 32 * layer * K; }
    // the K roots of layer `li`, root_stride bytes apart from root0, into their slots
    void copy_roots(const void *root0, size_t root_stride, size_t li) {
        DG_REQUIRE(li < (size_t)MAX_LAYERS, "too many FRI layers");
        DG_CUDA(cudaMemcpy2DAsync(root_slots(li), 32, root0, std::max<size_t>(root_stride, 32), 32, K, cudaMemcpyDeviceToDevice, c.stream));
    }
    void folding_points(const void *root0, size_t root_stride, size_t li) {
        DG_REQUIRE(li < (size_t)MAX_LAYERS, "too many FRI layers");
        if (!host_rng) { fri_alpha(c, root0, alpha(li), root_slots(li), K, root_stride); return; }
        copy_roots(root0, root_stride, li);
        std::vector<uint8_t> r((size_t)32 * K);
        d2h(c, r.data(), root_slots(li), r.size());
        std::vector<fe> alphas(K, fe_make(0, 0));
        for (int p : order)
            if (ps[p].live) alphas[p] = fs::prng_vector(r.data() + 32 * p, 1)[0];   // field::prng(seed) = first draw of the generator (field.rs:264-269)
        DG_CUDA(cudaMemcpyAsync(alpha(li), alphas.data(), (size_t)16 * K, cudaMemcpyHostToDevice, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }
};

void fri_layers(Context &c, Group &grp, std::vector<ProofState> &ps) {
    const int K = grp.K, log_b = grp.log_b, log_N = grp.log_N;
    TwiddleRef inv_root = c.twiddle(log_N, true);
    const FoldConstants fold = fri_fold_constants();
    // the K proofs' layers are one buffer each: layer d of proof p = cur + p * cur_stride
    const fe *cur = grp.comp_ext.as<fe>();
    uint64_t cur_stride = grp.N_loc;
    Layout lay{log_N, log_b};
    bool local = grp.G > 1;                                // `cur` is this rank's coset slab of the layer (K == 1)
    FriRun run(c, grp, ps);
    size_t n_layers = 0;
    for (;;) {
        const int log_r = lay.log_d - 2;
        const uint64_t R = 1ULL << log_r;
        // layers below 2^22 values are latency-bound (two collectives per sharded tree cost more than hashing them whole): gather the
        // first such layer once (<= 32 MB) and finish redundantly on every rank
        if (local && (lay.log_d < 22 || log_r - log_b < 6)) {
            grp.fri_gathered.alloc((size_t)16 << lay.log_d);
            comm_all_gather(c, cur, grp.fri_gathered.p, ((size_t)16 << lay.log_d) >> grp.log_g);     // rank-major == coset-major
            cur = grp.fri_gathered.as<fe>();
            local = false;
        }
        const size_t li = n_layers++;
        if (local) {
            FriLayerDev &L = ps[0].layers.emplace_back();
            L.vals = cur; L.layout = lay; L.sharded = true;
            // rows r = b k' + c of the own cosets: hashes in ShardedTree order, n' = R / b subtrees of nc leaves per rank
            L.leaves.alloc((R >> grp.log_g) * 32);
            fri_hash_rows_local(c, cur, lay.log_d, log_b, grp.log_nc, L.leaves.p);
            L.tree.build(c, L.leaves.p, R >> log_b, grp.log_nc, false);
            run.folding_points(L.tree.root_dev(), 0, li);
            L.folded.alloc((R >> grp.log_g) * 16);
            fri_fold_local(c, cur, lay.log_d, log_b, grp.log_nc, grp.c0, L.folded.as<fe>(), run.alpha(li), inv_root, log_N, fold.tau_inv, fold.inv4);
            cur = L.folded.as<fe>();
            lay = Layout{log_r, log_b};
            continue;
        }
        const Layout rows = fri_next_layout(lay);
        grp.layer_bufs.emplace_back((size_t)K * R * 32);
        const uint8_t *leaves = grp.layer_bufs.back().as<uint8_t>();
        grp.layer_bufs.emplace_back((size_t)K * R * 32);
        const uint8_t *nodes = grp.layer_bufs.back().as<uint8_t>();
        fri_hash_rows(c, cur, lay, rows, (void *)leaves, K, cur_stride);
        merkle_build(c, leaves, (void *)nodes, R, K);
        for (int p = 0; p < K; p++) {
            if (!ps[p].live) continue;
            FriLayerDev &L = ps[p].layers.emplace_back();
            L.vals = cur + (size_t)p * cur_stride; L.layout = lay; L.sharded = false;
            L.leaves_p = leaves + (size_t)p * R * 32; L.nodes_p = nodes + (size_t)p * R * 32;
        }
        if (R * 4 <= 256) {                                    // MAX_REMAINDER_LENGTH (fri/mod.rs:13): the remainder's root only
            run.copy_roots(nodes + 32, R * 32, li);
            break;
        }
        run.folding_points(nodes + 32, R * 32, li);            // special_x = prng(root)  (fri/prover.rs:29)
        grp.layer_bufs.emplace_back((size_t)K * R * 16);       // values of the next layer
        fe *folded = grp.layer_bufs.back().as<fe>();
        fri_fold(c, cur, lay, folded, rows, run.alpha(li), inv_root, log_N, fold.tau_inv, fold.inv4, K, cur_stride);
        cur = folded;
        cur_stride = R;
        lay = rows;
    }
    std::vector<uint8_t> roots(32 * n_layers * K);
    d2h(c, roots.data(), run.d_roots.p, roots.size());
    // the last layer is the remainder: its root is the FRI proof's rem_root
    for (int p = 0; p < K; p++) {
        if (!ps[p].live) continue;
        FriProof &f = ps[p].stark.degree_proof;
        auto root = [&](size_t i) { return roots.data() + 32 * (i * K + p); };
        f.layers.resize(n_layers - 1);
        for (size_t i = 0; i + 1 < n_layers; i++) memcpy(f.layers[i].root.data(), root(i), 32);
        memcpy(f.rem_root.data(), root(n_layers - 1), 32);
    }
}

// ---- 8: query positions --------------------------------------------------------------------------------------------------------------------
void query_positions(Context &c, const Group &grp, std::vector<ProofState> &ps) {
    std::vector<std::array<uint8_t, 32>> seeds;
    std::vector<unsigned> grinding;
    std::vector<int> who;
    for (int p : grp.order) {
        if (!ps[p].live) continue;
        const FriProof &f = ps[p].stark.degree_proof;
        std::vector<uint8_t> roots;
        for (auto &l : f.layers) roots.insert(roots.end(), l.root.begin(), l.root.end());
        roots.insert(roots.end(), f.rem_root.begin(), f.rem_root.end());
        if (grp.K == 1) debug_dump_host("fri_roots", roots.data(), roots.size());
        seeds.emplace_back();
        fs::blake3_short(roots.data(), roots.size(), seeds.back().data());
        grinding.push_back(ps[p].stark.options.grinding_factor);
        who.push_back(p);
    }
    std::vector<unsigned long long> nonces = pow_search_batch(c, seeds, grinding);
    for (size_t i = 0; i < who.size(); i++) {
        ProofState &s = ps[who[i]];
        s.stark.pow_nonce = nonces[i];
        pow_hash(seeds[i].data(), s.stark.pow_nonce, s.proof->pow_seed);
        try {
            s.positions = fs::query_positions(s.proof->pow_seed, grp.N, grp.b, s.stark.options.num_queries);
        } catch (const std::exception &e) { s.fail(DG_ERR_EXHAUSTED, e.what()); continue; }
        if (grp.K == 1) debug_dump_host("positions", s.positions.data(), s.positions.size() * 8);
    }
}

// ---- 9: build proof objects ----------------------------------------------------------------------------------------------------------------
// Every opening of every proof is planned on the host, all opened values / digests are fetched in one batched pass (FetchBatch), then
// each proof is written.

// registers the nodes of a batch-proof plan; leaf_ref / node_ref map leaf indices / heap indices to fetch references
template <class LeafRef, class NodeRef>
Offsets plan_offsets(FetchBatch &fb, const fs::BatchPlan &plan, LeafRef leaf_ref, NodeRef node_ref) {
    Offsets o(plan.nodes.size());
    for (size_t sidx = 0; sidx < plan.nodes.size(); sidx++)
        for (auto &r : plan.nodes[sidx]) o[sidx].push_back(fb.add32(r.leaf ? leaf_ref(r.index) : node_ref(r.index)));
    return o;
}

std::vector<std::vector<Digest>> digests_at(const FetchBatch &fb, const Offsets &o) {
    std::vector<std::vector<Digest>> v(o.size());
    for (size_t i = 0; i < o.size(); i++)
        for (size_t off : o[i]) v[i].push_back(fb.digest(off));
    return v;
}

// what proof p opens; its trace rows outside the retained cosets are in grp.d_rows from value row0 on
OpenPlan plan_openings(const Group &grp, FetchBatch &fb, ProofState &s, int p, size_t row0) {
    const uint64_t n = grp.n, b = grp.b, N = grp.N, nc = grp.nc;
    const int log_n = grp.log_n, log_b = grp.log_b, log_nc = grp.log_nc, w = grp.shapes[p].w;
    const fe *slab_p = grp.slab_of(p), *c_ext_p = grp.c_ext_of(p);
    OpenPlan O;
    const std::vector<uint64_t> &positions = s.positions;
    const int nq = (int)positions.size();
    // trace rows at the queried positions (trace_table.rs:127-134): the rank owning the position's coset reads the row from the retained
    // slab, or it was computed into d_rows
    O.row_off.resize(nq);
    for (int q = 0; q < nq; q++) {
        const uint64_t cpos = positions[q] & (b - 1), k = positions[q] >> log_b;
        if (!grp.retained(positions[q])) {
            O.row_off[q] = fb.add16(FetchRef{grp.d_rows.p, row0, -1});
            for (int j = 1; j < w; j++) fb.add16(FetchRef{grp.d_rows.p, row0 + j, -1});
            row0 += w;
            continue;
        }
        const int owner = (int)(cpos >> log_nc);
        const uint64_t phys = (((cpos - (uint64_t)owner * nc) / grp.rstep) << log_n) + k;
        for (int j = 0; j < w; j++) {
            const size_t off = fb.add16(FetchRef{slab_p + (size_t)j * grp.slab_col, phys, owner});
            if (j == 0) O.row_off[q] = off;
        }
    }
    // trace tree openings: leaves are the row hashes
    O.tplan = fs::plan_batch_proof(positions, N);
    O.t_off = plan_offsets(fb, O.tplan, [&](uint64_t i) { return s.t_tree.item_ref(i); }, [&](uint64_t h) { return s.t_tree.node_ref(h); });

    // constraint tree openings: leaf j = evaluations (2j, 2j+1), unhashed (prover.rs:180-187); evaluation 2j+1 lives in the next
    // coset at the same k, i.e. n elements further in the owner's slab: two 16-byte units registered back to back = one 32-byte item
    auto constraint_leaf = [&](uint64_t j) {
        const uint64_t i = 2 * j, cpos = i & (b - 1), k = i >> log_b;
        const int owner = (int)(cpos >> log_nc);
        const uint64_t p0 = ((cpos - (uint64_t)owner * nc) << log_n) + k;
        const size_t off = fb.add16(FetchRef{c_ext_p, p0, owner});
        fb.add16(FetchRef{c_ext_p, p0 + n, owner});
        return off;
    };
    std::vector<uint64_t> c_positions = fs::constraint_positions(positions);
    O.cplan = fs::plan_batch_proof(c_positions, N / 2);
    for (uint64_t j : O.cplan.value_leaves) O.cval_off.push_back(constraint_leaf(j));
    O.c_off.resize(O.cplan.nodes.size());
    for (size_t sidx = 0; sidx < O.cplan.nodes.size(); sidx++)
        for (auto &r : O.cplan.nodes[sidx]) {
            // heap indices of the tree over N/2 leaves: [N/4, N/2) is the first hashed level (= level-0 items of c_tree)
            if (r.leaf) O.c_off[sidx].push_back(constraint_leaf(r.index));
            else if (r.index >= N / 4) O.c_off[sidx].push_back(fb.add32(s.c_tree.item_ref(r.index - N / 4)));
            else O.c_off[sidx].push_back(fb.add32(s.c_tree.node_ref(r.index)));
        }

    // FRI layers (fri/prover.rs:55-95)
    O.fri_open.resize(s.layers.size() - 1);
    std::vector<uint64_t> fpos = positions;
    for (size_t d = 0; d + 1 < s.layers.size(); d++) {
        FriLayerDev &L = s.layers[d];
        LayerOpen &lo = O.fri_open[d];
        const uint64_t D = 1ULL << L.layout.log_d, R = D / 4;
        fpos = fs::augmented_positions(fpos, D);
        fs::BatchPlan plan = fs::plan_batch_proof(fpos, R);
        lo.depth = plan.depth;
        for (uint64_t p : fpos)
            for (int j = 0; j < 4; j++) {
                size_t off;
                if (L.sharded) {
                    const uint64_t cpos = p & (b - 1), k = (p >> log_b) + (uint64_t)j * (R >> log_b);
                    const int owner = (int)(cpos >> log_nc);
                    off = fb.add16(FetchRef{L.vals, ((cpos - (uint64_t)owner * nc) << (L.layout.log_d - log_b)) + k, owner});
                } else {
                    off = fb.add16(FetchRef{L.vals, L.layout.phys(p + j * R), -1});
                }
                if (j == 0) lo.val_off.push_back(off);
            }
        if (L.sharded) lo.node_off = plan_offsets(fb, plan, [&](uint64_t i) { return L.tree.item_ref(i); }, [&](uint64_t h) { return L.tree.node_ref(h); });
        else lo.node_off = plan_offsets(fb, plan, [&](uint64_t i) { return FetchRef{L.leaves_p, i, -1}; }, [&](uint64_t h) { return FetchRef{L.nodes_p, h, -1}; });
    }
    {
        FriLayerDev &L = s.layers.back();
        const uint64_t D = 1ULL << L.layout.log_d;
        for (uint64_t i = 0; i < D; i++) O.rem_off.push_back(fb.add16(FetchRef{L.vals, L.layout.phys(i), -1}));   // remainder, natural order
    }
    return O;
}

// the opened values and digests into the proof, which is then written out
void fill_openings(const FetchBatch &fb, ProofState &s, const OpenPlan &O, int w) {
    StarkProof &P = s.stark;
    P.trace_info.domain_depth = O.tplan.depth;
    P.trace_nodes = digests_at(fb, O.t_off);
    P.trace_evaluations.assign(O.row_off.size(), std::vector<fe>(w));
    for (size_t q = 0; q < O.row_off.size(); q++)
        for (int j = 0; j < w; j++) P.trace_evaluations[q][j] = fb.value(O.row_off[q] + j);
    for (size_t off : O.cval_off) P.constraint_proof.values.push_back(fb.digest(off));
    P.constraint_proof.nodes = digests_at(fb, O.c_off);
    P.constraint_proof.depth = O.cplan.depth;
    for (size_t d = 0; d < O.fri_open.size(); d++) {
        const LayerOpen &lo = O.fri_open[d];
        FriLayer &l = P.degree_proof.layers[d];
        for (size_t off : lo.val_off) l.values.push_back({fb.value(off), fb.value(off + 1), fb.value(off + 2), fb.value(off + 3)});
        l.nodes = digests_at(fb, lo.node_off);
        l.depth = lo.depth;
    }
    for (size_t off : O.rem_off) P.degree_proof.rem_values.push_back(fb.value(off));
    Proof &h = *s.proof;
    h.bytes = write_proof(P);
    memcpy(h.trace_root, P.trace_root.data(), 32);
    memcpy(h.constraint_root, P.constraint_root.data(), 32);
    h.pow_nonce = P.pow_nonce;
}

void build_proofs(Context &c, Group &grp, std::vector<ProofState> &ps) {
    const int K = grp.K;
    FetchBatch fb(c);
    // opened trace rows outside the retained cosets (evaluation-coset layout): the trace polynomials at w_N^pos, all proofs in one launch,
    // into d_rows (the w_p values of each computed row of the batch, rows in proof and query order)
    std::vector<size_t> first_row(K, 0);                       // proof p's first value in d_rows
    std::vector<TraceRow> points;
    size_t values = 0;
    for (int p = 0; p < K; p++) {
        first_row[p] = values;
        if (ps[p].live)
            for (uint64_t pos : ps[p].positions)
                if (!grp.retained(pos)) {
                    points.push_back(TraceRow{pos, 0, grp.col0[p], (unsigned)grp.shapes[p].w});
                    values += grp.shapes[p].w;
                }
    }
    if (!points.empty()) {
        grp.d_rows.alloc(values * 16);
        eval_trace_rows(c, grp.polys.as<fe>(), grp.n, points, grp.log_N, grp.d_rows.as<fe>());
    }
    std::vector<OpenPlan> plans(K);
    for (int p = 0; p < K; p++)
        if (ps[p].live) plans[p] = plan_openings(grp, fb, ps[p], p, first_row[p]);
    fb.run();
    for (int p = 0; p < K; p++)
        if (ps[p].live) fill_openings(fb, ps[p], plans[p], grp.shapes[p].w);
}

}  // namespace

// Proves K traces of one length and extension factor (K == 1: dg_prove / dg_prove_device); opts[p] are proof p's options, which may
// differ in num_queries and grinding_factor.  Every device buffer is proof-major: the registers, polynomials and
// trace extension are sum(w_p) columns, proof p's w_p columns from column col0[p] on, and every per-proof vector ([K][...]) has the
// single-proof layout inside.  So the transforms run once over all the proofs' columns, and each host round trip (violation flags, roots,
// DEEP values, FRI roots, PoW, openings) moves the values of all K proofs at once.  shapes[p] is proof p's register shape; proofs of one
// shape are adjacent, so that the constraint kernel runs once per shape over proofs at a uniform stride (a one-shape batch: one launch).
// order: the proofs in the order their Fiat-Shamir draws are made (the RNG callbacks see them in that order, stage by stage).
// d_regs: register traces in device memory, [sum w_p][n]; when `host_cols` (sum w_p column pointers) is given they are not there yet:
// column chunks are uploaded on the copy stream while the previous chunk is being interpolated and extended (the upload hides behind the
// LDE).  chunk (one GPU): cosets of the trace extension held at a time (ProvePlan).  The full layout (chunk = b) keeps the whole extension;
// the evaluation-coset layout (chunk < b) extends and hashes chunk cosets at a time and keeps only the 8 cosets stage 3 reads.
// The stages are the reference's nine debug!() sections, one function each, in order.
static void prove_core(Context &c, fe *d_regs, const uint8_t *const *host_cols, const std::vector<RegisterShape> &regs_shape, uint64_t length,
                       const std::vector<int> &order, std::vector<ProofState> &ps, const std::vector<dg_options_t> &opts,
                       dg_prove_stats_t *stats, unsigned chunk) {
    ArenaScope arena_scope;                   // all DevBufs below come from the per-proof arena (no driver allocation inside a proof)
    StageClock clk(c.stream);
    SubClock sub(c.stream);
    if (sub.on) c.mark = [&sub](const char *name) { sub.mark(name); }; else c.mark = nullptr;
    struct MarkReset { Context &c; ~MarkReset() { c.mark = nullptr; } } mark_reset{c};
    // the proofs' trees and FRI layers come from the arena too: release them before the arena scope closes
    struct DeviceStateReset {
        std::vector<ProofState> &ps;
        ~DeviceStateReset() { for (auto &s : ps) { s.t_tree = ShardedTree(); s.c_tree = ShardedTree(); s.layers.clear(); } }
    } state_reset{ps};
    const unsigned long long launches0 = c.launches;
    Group grp(c, d_regs, host_cols, regs_shape, length, order, ps, opts, chunk);

    clk.mark(0);
    sub.mark("start");
    if (grp.G == 1) extend_trace(c, grp);
    else extend_trace_sharded(c, grp);
    clk.mark(1);
    sub.mark("1.lde");
    commit_trace(c, grp, ps);
    clk.mark(2);
    sub.mark("2.tree");
    if (!evaluate_constraints(c, grp, ps)) return;
    clk.mark(3);
    sub.mark("3.finish+boundary");
    constraint_polynomial(c, grp);
    clk.mark(4);
    sub.mark("4.combine");
    commit_constraints(c, grp, ps);
    clk.mark(5);
    sub.mark("5.tree");
    deep_composition(c, grp, ps);
    clk.mark(6);
    sub.mark("6.compose+lde");
    fri_layers(c, grp, ps);
    clk.mark(7);
    sub.mark("7.fri");
    query_positions(c, grp, ps);
    if (!any_live(ps)) return;
    clk.mark(8);
    sub.mark("8.pow");
    build_proofs(c, grp, ps);
    clk.mark(9);
    sub.mark("9.openings");
    sub.report(c.rank);
    DG_CUDA(cudaStreamSynchronize(c.stream));
    if (stats) {
        for (int i = 0; i < 9; i++) stats->stage_ms[i] = clk.between(i, i + 1);
        stats->h2d_ms = 0.0f;                        // host variant: uploads overlap stage 1 and are part of stage_ms[0]
        stats->total_ms = clk.between(0, 9);
        stats->kernel_launches = c.launches - launches0;
    }
}

namespace {

std::vector<ProofState> make_states(uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs, const uint8_t *const *outputs16,
                                    const uint32_t *n_outputs) {
    std::vector<ProofState> ps(count);
    for (uint32_t i = 0; i < count; i++) {
        const uint32_t ni = n_inputs ? n_inputs[i] : 0, no = n_outputs ? n_outputs[i] : 0;
        ps[i].inputs.resize(ni);
        ps[i].outputs.resize(no);
        if (ni) memcpy(ps[i].inputs.data(), inputs16[i], ni * 16);
        if (no) memcpy(ps[i].outputs.data(), outputs16[i], no * 16);
    }
    return ps;
}

}  // namespace

// Device bytes one proof of this shape takes in a batch on one GPU: the buffers prove_core allocates per proof, stage by stage (every
// one stays in the bump arena until the group ends), plus its register columns (the upload buffer of a host batch).  chunk: cosets of
// the trace extension held at a time; b is the full layout, fewer the evaluation-coset layout (a chunk and the 8 retained cosets).
size_t proof_footprint(uint32_t w, uint64_t n, uint32_t b, uint32_t chunk) {
    const size_t N = (size_t)n * b, E = (size_t)n * 8, fe16 = 16, dg32 = 32;
    size_t f = 0;
    f += (size_t)w * n * fe16;                // registers (host batch: upload buffer)
    f += (size_t)w * n * fe16;                // 1: polynomials
    if (chunk >= b) {
        f += (size_t)w * N * fe16;            // 1: trace LDE
    } else {
        f += (size_t)w * n * (chunk + 8) * fe16;      // 1: a coset chunk of the trace LDE + the 8 retained cosets
        const size_t tiles = std::min<size_t>(64, (n + 2047) / 2048);
        f += (size_t)128 * (w * (tiles + 1) + 1) * fe16;   // 9: computed opened rows (<= 128 queries), their tile sums and points
    }
    f += 2 * N * dg32;                        // 2: row hashes + tree
    f += 3 * E * fe16 + E * fe16;             // 3: i / f / t coefficients, coset-local transition evaluations
    f += 3 * E * fe16;                        // 4: combined polynomial + the two division scratch vectors
    f += N * fe16 + 2 * (N / 4) * dg32;       // 5: constraint LDE, first hashed level + tree
    f += 2 * N * fe16;                        // 5, 6: prefolded input of the two fold-8 extensions (both live until the group ends)
    f += E * fe16 + N * fe16;                 // 6: composition polynomial + its LDE
    f += 2 * n * fe16;                        // 6: the two trace quotients
    size_t pow_n = 0;                         // 6: the four power tables of z, 1/z (E + 1 entries), z g, 1/(z g) (n + 1 entries)
    for (uint64_t len : {E + 1, E + 1, (uint64_t)n + 1, (uint64_t)n + 1}) pow_n += PowTables::entries(len);
    f += pow_n * fe16;
    f += (N / 4) * (2 * dg32 + fe16) * 4 / 3; // 7: FRI layers (R = D / 4 row hashes, tree and folded values per layer, D = N, N / 4, ...)
    f += (size_t)1 << 20;                     // coefficients, DEEP values, scan descriptors, evaluation partials, PoW, openings (< 1 MB)
    return f + f / 16;                        // + 256-byte alignment of every arena allocation
}

// Largest group of one launch: the batched kernels put the proof (and the DEEP evaluation every column of every proof) on the grid's y
// dimension, which holds at most 65535 blocks.
int max_group_for_grid(uint32_t w) { return (int)(65535 / std::max<uint32_t>(w, 1)); }

long long batch_group_cap(long long k) {
    if (const char *e = getenv("DG_BATCH_GROUP")) {
        const long long cap = atoll(e);
        DG_REQUIRE(cap >= 1, "DG_BATCH_GROUP must be a positive integer");
        k = std::min(k, cap);
    }
    return k;
}

// Transform scratch and tables a prove call adds outside the arena (persistent, from the pool): the multi-pass LDE of a coset chunk
// (<= 4 GiB), the other multi-pass transforms (<= 1 GiB) and the first-pass tables of the trace LDE (lde_tables_to_add), less what the
// library holds already
static size_t prove_scratch(Context &c, uint32_t w, uint64_t n, uint32_t b, uint32_t chunk, long long k) {
    const size_t four = (size_t)4 << 30, one = (size_t)1 << 30;
    const size_t ntt = std::max(std::min(four, (size_t)(16 * n * chunk * w * k)), std::min(one, (size_t)(16 * n * b * k)));
    size_t add = ntt > c.ntt_tmp.bytes ? ntt - c.ntt_tmp.bytes : 0;
    return add + lde_tables_to_add(c, ceil_log2(n), ceil_log2(b));
}

ProvePlan plan_prove(Context &c, uint32_t w, uint64_t n, uint32_t b, uint32_t count) {
    DG_REQUIRE(count >= 1, "batch must hold at least one trace");
    require_extension_factor(b);
    DG_REQUIRE(n >= 16 && (n & (n - 1)) == 0 && n <= (1ULL << 30), "execution trace length must be a power of 2 and at least 16");
    DG_REQUIRE(w >= 1 && w < 128, "execution trace cannot have more than 128 registers");
    const long long k_max = std::min<long long>(count, max_group_for_grid(w));
    // the largest group of the layout that keeps `ch` cosets at a time (0 if not even one proof fits); the scratch grows with the group
    auto group_of = [&](uint32_t ch, size_t &avail) {
        const size_t per = proof_footprint(w, n, b, ch);
        avail = memory_budget(c, Budget::ARENA, (size_t)k_max * per, prove_scratch(c, w, n, b, ch, 1));
        long long g = std::min<long long>(k_max, (long long)(avail / per));
        while (g > 1 && (size_t)g * per > memory_budget(c, Budget::ARENA, (size_t)g * per, prove_scratch(c, w, n, b, ch, g))) g = g * 3 / 4;
        return g;
    };
    // the full layout when a group of one proof fits; else the evaluation-coset layout with the largest coset chunk that fits
    for (uint32_t ch = b; ch >= 1; ch = ch == b ? b / 2 : ch / 2) {
        size_t avail = 0;
        const long long g = group_of(ch, avail);
        if (g < 1) continue;
        ProvePlan P;
        P.full = ch == b;
        P.chunk = ch;
        P.per_proof = proof_footprint(w, n, b, ch);
        P.fixed = memory_held_outside_arena(c) + prove_scratch(c, w, n, b, ch, g);
        P.group = (int)batch_group_cap(g);
        P.available = avail;
        return P;
    }
    const size_t need = proof_footprint(w, n, b, 1) + memory_held_outside_arena(c) + prove_scratch(c, w, n, b, 1, 1);
    throw Error(DG_ERR_INVALID, "a proof of " + std::to_string(w) + " x " + std::to_string(n) + " at extension factor " + std::to_string(b) + " needs " +
                                    std::to_string(need) + " bytes of device memory; the memory limit is " + std::to_string(c.mem_limit) + " bytes");
}

namespace {

// before a group runs under a memory limit: an arena too small for it is released, so that the group runs on the pool alone and what the
// library holds stays within the limit (the arena is sized again, within the limit, after the group)
void prepare_arena(Context &c, const ProvePlan &P) {
    if (c.mem_limit && c.arena.base && (size_t)P.group * P.per_proof > c.arena.cap) arena_release(c);
}

}  // namespace

void add_stats(dg_prove_stats_t *sum, const dg_prove_stats_t &s) {
    for (int i = 0; i < 9; i++) sum->stage_ms[i] += s.stage_ms[i];
    sum->h2d_ms += s.h2d_ms;
    sum->total_ms += s.total_ms;
    sum->kernel_launches += s.kernel_launches;
}

std::vector<std::vector<uint32_t>> partition_traces(const std::vector<uint64_t> &length, const std::vector<uint32_t> &extension_factor) {
    std::vector<std::vector<uint32_t>> parts;
    std::vector<std::pair<uint64_t, uint32_t>> seen;
    for (uint32_t i = 0; i < length.size(); i++) {
        const std::pair<uint64_t, uint32_t> key{length[i], extension_factor[i]};
        const size_t at = std::find(seen.begin(), seen.end(), key) - seen.begin();
        if (at == seen.size()) { seen.push_back(key); parts.emplace_back(); }
        parts[at].push_back(i);
    }
    return parts;
}

std::vector<uint32_t> cut_groups(const std::vector<uint32_t> &width, const std::vector<size_t> &footprint, size_t budget, uint32_t cap) {
    std::vector<uint32_t> sizes;
    uint32_t k = 0;
    size_t bytes = 0, cols = 0;
    for (size_t i = 0; i < width.size(); i++) {
        if (k > 0 && (k == cap || bytes + footprint[i] > budget || cols + width[i] > 65535)) {
            sizes.push_back(k);
            k = 0; bytes = 0; cols = 0;
        }
        k++; bytes += footprint[i]; cols += width[i];
    }
    if (k > 0) sizes.push_back(k);
    return sizes;
}

std::vector<uint32_t> shape_order(const std::vector<RegisterShape> &shape) {
    std::vector<uint32_t> out;
    std::vector<bool> done(shape.size(), false);
    for (size_t i = 0; i < shape.size(); i++) {
        if (done[i]) continue;
        for (size_t j = i; j < shape.size(); j++)
            if (!done[j] && shape[j] == shape[i]) { out.push_back((uint32_t)j); done[j] = true; }
    }
    return out;
}

void prove_traces(Context &c, const std::vector<TraceRef> &traces, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                  const uint8_t *const *outputs16, const uint32_t *n_outputs, const std::vector<dg_options_t> &opts, bool batch,
                  Proof **proofs_out, int *status, std::vector<std::string> &messages, dg_prove_stats_t *stats, uint32_t *groups) {
    const uint32_t count = (uint32_t)traces.size();
    DG_REQUIRE(count >= 1, "batch must hold at least one trace");
    DG_REQUIRE(opts.size() == count, "one set of options per trace");
    const bool host = traces[0].host_cols != nullptr;
    std::vector<ProofState> all = make_states(count, inputs16, n_inputs, outputs16, n_outputs);
    if (batch)
        DG_REQUIRE(c.world == 1 && ctx_device_count() == 1, "batched proving runs on one GPU: the library was initialised for several (dg_init_devices / dg_comm_init)");
    // every partition's plan and groups before any proof runs: a partition that fits in no way fails the call before the device computes
    std::vector<uint64_t> lengths;
    std::vector<uint32_t> factors;
    for (uint32_t i = 0; i < count; i++) { lengths.push_back(traces[i].length); factors.push_back(opts[i].extension_factor); }
    struct PartitionRun { std::vector<uint32_t> idx; ProvePlan plan; std::vector<uint32_t> sizes; };
    std::vector<PartitionRun> runs;
    for (std::vector<uint32_t> &idx : partition_traces(lengths, factors)) {
        PartitionRun r;
        r.idx = std::move(idx);
        r.sizes.assign(r.idx.size(), 1);           // several GPUs (one trace): one group, and prove_core shards the full layout
        if (c.world == 1) {
            // planned for the widest shape of the partition: its group's bytes are the budget the groups of mixed widths are cut to
            uint32_t wmax = 0;
            for (uint32_t i : r.idx) wmax = std::max(wmax, traces[i].width);
            const uint64_t n = traces[r.idx[0]].length;
            const uint32_t b = opts[r.idx[0]].extension_factor;
            r.plan = plan_prove(c, wmax, n, b, (uint32_t)r.idx.size());
            std::vector<uint32_t> width;
            std::vector<size_t> foot;
            for (uint32_t i : r.idx) {
                width.push_back(traces[i].width);
                foot.push_back(proof_footprint(traces[i].width, n, b, r.plan.chunk));
            }
            r.sizes = cut_groups(width, foot, (size_t)r.plan.group * r.plan.per_proof, (uint32_t)r.plan.group);
        }
        runs.push_back(std::move(r));
    }
    if (stats) memset(stats, 0, sizeof *stats);
    if (groups) *groups = 0;
    for (uint32_t i = 0; i < count; i++) { proofs_out[i] = nullptr; status[i] = DG_OK; }
    messages.assign(count, std::string());
    // a group that fails as a whole fails the call: the proofs of the earlier groups are freed, nothing is returned
    struct ReleaseOnError {
        Proof **out; uint32_t count; bool done = false;
        ~ReleaseOnError() { if (!done) for (uint32_t i = 0; i < count; i++) { delete out[i]; out[i] = nullptr; } }
    } release{proofs_out, count};
    for (const PartitionRun &r : runs) {
        const uint64_t n = traces[r.idx[0]].length;
        size_t first = 0;
        for (uint32_t k : r.sizes) {
            // the group's traces in input order, and on the device grouped by shape (shapes in order of first appearance)
            const std::vector<uint32_t> members(r.idx.begin() + first, r.idx.begin() + first + k);
            first += k;
            std::vector<RegisterShape> keys;
            for (uint32_t i : members) keys.push_back(traces[i].shape());
            std::vector<uint32_t> dev;                                   // trace of device slot p
            for (uint32_t m : shape_order(keys)) dev.push_back(members[m]);
            std::vector<int> order(k);                                   // device slot of the group's m-th trace in input order
            for (uint32_t p = 0; p < k; p++) order[std::find(members.begin(), members.end(), dev[p]) - members.begin()] = (int)p;
            std::vector<ProofState> ps;
            std::vector<RegisterShape> shapes;
            std::vector<dg_options_t> group_opts;
            std::vector<const uint8_t *> cols;
            size_t W = 0;
            for (uint32_t i : dev) {
                const TraceRef &t = traces[i];
                ps.push_back(std::move(all[i]));
                shapes.push_back(t.shape());
                group_opts.push_back(opts[i]);
                if (host) cols.insert(cols.end(), t.host_cols, t.host_cols + t.width);
                W += t.width;
            }
            dg_prove_stats_t st;
            memset(&st, 0, sizeof st);
            prepare_arena(c, r.plan);
            // the group's registers as W columns: host traces are uploaded into the upload buffer by prove_core; device traces are read in
            // place when they are adjacent in one allocation (a one-shape batch), else copied there.  Separate allocations that happen to
            // be adjacent are copied: a copy may not span two allocations.
            fe *regs = const_cast<fe *>(traces[dev[0]].d_regs);
            bool adjacent = !host;
            for (uint32_t p = 1; p < k && adjacent; p++)
                adjacent = traces[dev[p]].slab && traces[dev[p]].slab == traces[dev[p - 1]].slab &&
                           traces[dev[p]].d_regs == traces[dev[p - 1]].d_regs + (size_t)traces[dev[p - 1]].width * n;
            if (!adjacent) {
                c.upload_buf.ensure((size_t)n * 16 * W, true);
                regs = c.upload_buf.as<fe>();
                if (!host) {
                    size_t col = 0;
                    for (uint32_t i : dev) {
                        DG_CUDA(cudaMemcpyAsync(regs + col * n, traces[i].d_regs, (size_t)traces[i].width * n * 16, cudaMemcpyDeviceToDevice, c.stream));
                        col += traces[i].width;
                    }
                }
            }
            prove_core(c, regs, host ? cols.data() : nullptr, shapes, n, order, ps, group_opts, &st, r.plan.chunk);
            if (stats) add_stats(stats, st);
            if (groups) ++*groups;
            for (uint32_t p = 0; p < k; p++) {
                const uint32_t i = dev[p];
                status[i] = ps[p].status;
                messages[i] = ps[p].message;
                if (ps[p].status == DG_OK) proofs_out[i] = ps[p].proof.release();
            }
        }
    }
    release.done = true;
}

std::vector<TraceRef> one_shape_traces(const fe *d_regs, uint32_t count, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth) {
    std::vector<TraceRef> traces(count);
    for (uint32_t i = 0; i < count; i++) {
        TraceRef &t = traces[i];
        t.width = width; t.length = length; t.ctx_depth = ctx_depth; t.loop_depth = loop_depth;
        t.d_regs = d_regs + (size_t)i * width * length;
        t.slab = d_regs;
    }
    return traces;
}

}  // namespace dg
