// Host orchestration of the CUDA prove pipeline: the body that replaces /root/reference/src/stark/prover.rs:17-169.
// Stage numbering and names follow the reference's nine debug!() sections (prover.rs:19-167) so that per-stage timings of
// the CPU prover and of this backend line up.  Only 32-byte roots, a handful of challenges and the final openings cross
// the PCIe bus after the register traces have been uploaded.
#include "prover.h"
#include "air.h"
#include "host_fs.h"
#include "poly.h"
#include "shard.h"
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


void write_digest_vec(fs::ByteWriter &w, const std::vector<Digest> &v) {
    w.u64(v.size());
    for (auto &d : v) w.raw(d.data(), 32);
}
void write_digest_vv(fs::ByteWriter &w, const std::vector<std::vector<Digest>> &v) {
    w.u64(v.size());
    for (auto &x : v) write_digest_vec(w, x);
}
void write_felt_vec(fs::ByteWriter &w, const std::vector<fe> &v) {
    w.u64(v.size());
    for (auto &x : v) w.felt(x);
}

int ilog2(uint64_t v) { int l = 0; while ((1ULL << l) < v) l++; return l; }

// Trace LDE of `cols` columns (polynomials `polys`, stride n) onto the cosets [c0, c0 + nc), written to ext (column stride N_loc).
// Coset 0 is P(w_n^k), which is register row k itself (polys = iNTT(regs) exactly): when the range starts at coset 0 and the registers
// are on the device (`regs`, stride n; null if not), slab 0 is copied from them and only the other cosets are transformed.
void extend_trace_columns(Context &c, const fe *polys, const fe *regs, fe *ext, int cols, int log_n, int log_b, uint64_t N_loc, unsigned c0,
                          unsigned nc) {
    const size_t n = (size_t)1 << log_n;
    if (c0 != 0 || !regs) {
        lde_batch(c, polys, ext, log_n, log_b, 1, cols, n, N_loc, c0, nc);
        return;
    }
    DG_REQUIRE(nc >= 2, "coset range too small");
    lde_batch(c, polys, ext + n, log_n, log_b, 1, cols, n, N_loc, 1, nc - 1);
    DG_CUDA(cudaMemcpy2DAsync(ext, N_loc * sizeof(fe), regs, n * sizeof(fe), n * sizeof(fe), cols, cudaMemcpyDeviceToDevice, c.stream));
}

struct FriLayerDev {
    DevBuf leaves, nodes, folded;     // sharded layer: row hashes, tree and folded values of this rank
    const void *leaves_p = nullptr, *nodes_p = nullptr;     // replicated layer: row hashes and tree (buffers shared by the batch's proofs)
    const fe *vals;                   // replicated layer: the whole vector; sharded layer: this rank's cosets [c - c0][k]
    Layout layout;                    // layout of the (whole) layer (domain size 2^layout.log_d)
    bool sharded = false;             // multi-GPU: rows hashed / folded per coset range, tree = ShardedTree over [k'][c - c0] items
    ShardedTree tree;
    Digest root;
};

}  // namespace

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

namespace {

typedef std::vector<std::vector<size_t>> Offsets;

// Per-proof host state of a batch.  A proof that fails (unsatisfied constraints, exhausted query positions) is marked dead and
// takes part in no later host-side work; its device lanes in the batched transforms keep computing on meaningless values.
struct ProofState {
    bool live = true;
    int status = DG_OK;
    std::string message;
    std::unique_ptr<Proof> proof{new Proof()};
    std::vector<fe> inputs, outputs;
    fe op_count;
    fs::ConstraintCoefficients cc;
    fs::CompositionCoefficients dc;
    std::vector<fe> state1, state2;
    ShardedTree t_tree, c_tree;
    std::vector<FriLayerDev> layers;
    std::vector<uint64_t> positions;
    void fail(int code, const std::string &m) { live = false; status = code; message = m; }
};

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

// everything a proof opens, as offsets into the batch's FetchBatch (stage 9)
struct LayerOpen { std::vector<uint64_t> pos; std::vector<size_t> val_off; Offsets node_off; uint8_t depth; };
struct OpenPlan {
    std::vector<size_t> row_off;
    fs::BatchPlan tplan, cplan;
    Offsets t_off, c_off;
    std::vector<size_t> cval_off, rem_off;
    std::vector<LayerOpen> fri_open;
};

}  // namespace

// Proves K traces of one shape (K == 1: dg_prove / dg_prove_device).  Every device buffer is proof-major ([K][...] with the single-proof
// layout inside), so the transforms run once over the K proofs' columns, and each host round trip (violation flags, roots, DEEP values,
// FRI roots, PoW, openings) moves the values of all K proofs at once.
// d_regs: register traces in device memory, [K][w][n]; when `host_cols` (K * w column pointers) is given they are not there yet: column
// chunks are uploaded on the copy stream while the previous chunk is being interpolated and extended (the upload hides behind the LDE).
static void prove_core(Context &c, fe *d_regs, const uint8_t *const *host_cols, int K, uint32_t width, uint64_t length, uint32_t ctx_depth,
                       uint32_t loop_depth, std::vector<ProofState> &ps, const dg_options_t &opt, dg_prove_stats_t *stats) {
    // ---- argument checks (trace_table.rs:23-58, options.rs:29-50, lib.rs:33-34) -----------------------------------------------
    const uint64_t n = length, b = opt.extension_factor;
    DG_REQUIRE(K >= 1 && (int)ps.size() == K, "batch must hold at least one trace");
    DG_REQUIRE((uint64_t)K * width <= 65535, "batch too large for one launch (batched calls split larger batches into groups)");
    DG_REQUIRE(opt.hash_id == 0, "unsupported hash function (only blake3 is serialisable, options.rs:107)");
    DG_REQUIRE(b >= 16 && b <= 256 && (b & (b - 1)) == 0, "extension_factor must be a power of 2 between 16 and 256");
    DG_REQUIRE(opt.num_queries > 0 && opt.num_queries <= 128, "num_queries must be in 1..128");
    DG_REQUIRE(opt.grinding_factor <= 32, "grinding factor cannot be greater than 32");
    DG_REQUIRE(n >= 16 && (n & (n - 1)) == 0, "execution trace length must be a power of 2 and at least 16");
    DG_REQUIRE(ctx_depth <= 16, "context depth cannot be greater than 16");
    DG_REQUIRE(loop_depth <= 8, "loop depth cannot be greater than 8");
    DG_REQUIRE(width < 128, "execution trace cannot have more than 128 registers");
    DG_REQUIRE(width > 15 + ctx_depth + loop_depth, "user stack must consist of at least one register");
    for (auto &s : ps) DG_REQUIRE(s.inputs.size() <= 8 && s.outputs.size() <= 8, "cannot have more than 8 public inputs / outputs");
    const int w = (int)width, log_n = ilog2(n), log_b = ilog2(b), log_N = log_n + log_b;
    DG_REQUIRE(log_N <= 30, "LDE domain too large");
    const uint64_t N = n * b, E = n * 8;
    const int stack_depth = w - 15 - (int)ctx_depth - (int)loop_depth;
    DG_REQUIRE(stack_depth <= 32, "stack depth cannot be greater than 32");
    auto any_live = [&] { for (auto &s : ps) if (s.live) return true; return false; };

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

    // ---- sharding: rank g owns the LDE cosets [c0, c0 + nc) of every column (world == 1: all of them) ------------------------------
    const int G = c.world, g = c.rank;
    DG_REQUIRE(G == 1 || K == 1, "a batch of proofs runs on one GPU (the context spans several)");
    int log_g = 0;
    while ((1 << log_g) < G) log_g++;
    DG_REQUIRE((b >> log_g) >= 4 && G <= 8, "extension factor too small for this many GPUs (need >= 4 cosets per rank)");
    const int log_nc = log_b - log_g;
    const uint64_t nc = 1ULL << log_nc, N_loc = n * nc;
    const unsigned c0 = (unsigned)(g * nc);
    const size_t W = (size_t)K * w;                            // columns of the whole batch

    // ---- 1: extend execution trace ---------------------------------------------------------------------------------------------------
    clk.mark(0);
    sub.mark("start");
    // G > 1: the interpolation is sharded by columns -- rank r interpolates the columns [col_start(r), col_start(r) + col_count(r)), an
    // even split (the first w mod G ranks own one more), and only needs (from a host trace: only uploads) those registers -- the
    // polynomials are all-gathered (equal slots of cpr columns per rank, then compacted into natural column order) and every rank
    // extends all columns on its cosets
    const int cpr = (w + G - 1) / G;                           // slot size of the gather = largest share
    auto col_count = [&](int r) { return w / G + (r < w % G ? 1 : 0); };
    auto col_start = [&](int r) { return r * (w / G) + std::min(r, w % G); };
    DevBuf polys(W * n * 16), ext(W * N_loc * 16);
    if (G == 1) {
        // the K proofs' registers are K * w columns of one batch
        if (!host_cols) {
            ntt_batch(c, d_regs, polys.as<fe>(), log_n, (int)W, n, n, true);
            extend_trace_columns(c, polys.as<fe>(), d_regs, ext.as<fe>(), (int)W, log_n, log_b, N_loc, c0, (unsigned)nc);
        } else {
            // chunks of ~64 MB, but a short ramp first (1, 2 columns): the first transform starts after one column's worth of copying
            const int chunk = (int)std::max<uint64_t>(1, std::min<uint64_t>(W, ((uint64_t)1 << 26) / (n * 16)));
            std::vector<int> bounds = {0};
            for (int step = 1; bounds.back() < (int)W; step = std::min(chunk, step * 2)) bounds.push_back(std::min((int)W, bounds.back() + step));
            TraceUploader up(c, d_regs, host_cols, (int)W, n, bounds);
            for (int i = 0; i < up.chunks(); i++) {
                const int j0 = bounds[i], cols = bounds[i + 1] - j0;
                up.wait_chunk(i);
                ntt_batch(c, d_regs + (size_t)j0 * n, polys.as<fe>() + (size_t)j0 * n, log_n, cols, n, n, true);
                extend_trace_columns(c, polys.as<fe>() + (size_t)j0 * n, d_regs + (size_t)j0 * n, ext.as<fe>() + (size_t)j0 * N_loc, cols, log_n, log_b, N_loc,
                                     c0, (unsigned)nc);
            }
        }
    } else {
        const int j0 = col_start(g), mine = col_count(g);
        DevBuf own((size_t)cpr * n * 16), slots((size_t)cpr * G * n * 16);
        if (mine > 0) {
            if (host_cols) {
                std::vector<int> bounds(mine + 1);
                for (int i = 0; i <= mine; i++) bounds[i] = i;
                TraceUploader up(c, d_regs + (size_t)j0 * n, host_cols + j0, mine, n, bounds);      // one column per chunk: all staging workers busy
                for (int i = 0; i < up.chunks(); i++) {              // interpolate every column as soon as it has landed
                    up.wait_chunk(i);
                    ntt_batch(c, d_regs + (size_t)(j0 + i) * n, own.as<fe>() + (size_t)i * n, log_n, 1, n, n, true);
                }
            } else {
                ntt_batch(c, d_regs + (size_t)j0 * n, own.as<fe>(), log_n, mine, n, n, true);
            }
        }
    sub.mark("1.intt");
        // the all-gather of the polynomials (and their compaction into column order) runs on the communication stream while this rank
        // already extends its own columns
        cudaEvent_t ev_own, ev_all;
        DG_CUDA(cudaEventCreateWithFlags(&ev_own, cudaEventDisableTiming));
        DG_CUDA(cudaEventCreateWithFlags(&ev_all, cudaEventDisableTiming));
        DG_CUDA(cudaEventRecord(ev_own, c.stream));
        DG_CUDA(cudaStreamWaitEvent(c.comm_stream, ev_own, 0));
        comm_all_gather(c, own.p, slots.p, (size_t)cpr * n * 16, c.comm_stream);
        for (int r = 0; r < G; r++)
            if (col_count(r) > 0)
                DG_CUDA(cudaMemcpyAsync(polys.as<fe>() + (size_t)col_start(r) * n, slots.as<fe>() + (size_t)r * cpr * n, (size_t)col_count(r) * n * 16,
                                        cudaMemcpyDeviceToDevice, c.comm_stream));
        DG_CUDA(cudaEventRecord(ev_all, c.comm_stream));
        if (mine > 0)
            extend_trace_columns(c, own.as<fe>(), d_regs + (size_t)j0 * n, ext.as<fe>() + (size_t)j0 * N_loc, mine, log_n, log_b, N_loc, c0, (unsigned)nc);
    sub.mark("1.lde_own");
        DG_CUDA(cudaStreamWaitEvent(c.stream, ev_all, 0));
        // the other ranks' registers are on this device only when the trace was given in device memory (a host trace uploads own columns only)
        if (j0 > 0) extend_trace_columns(c, polys.as<fe>(), host_cols ? nullptr : d_regs, ext.as<fe>(), j0, log_n, log_b, N_loc, c0, (unsigned)nc);
        if (j0 + mine < w)
            extend_trace_columns(c, polys.as<fe>() + (size_t)(j0 + mine) * n, host_cols ? nullptr : d_regs + (size_t)(j0 + mine) * n,
                                 ext.as<fe>() + (size_t)(j0 + mine) * N_loc, w - j0 - mine, log_n, log_b, N_loc, c0, (unsigned)nc);
        cudaEventDestroy(ev_own);
        cudaEventDestroy(ev_all);
    }
    auto ext_of = [&](int p) { return ext.as<fe>() + (size_t)p * w * N_loc; };

    // ---- 2: trace Merkle tree ----------------------------------------------------------------------------------------------------------
    clk.mark(1);
    sub.mark("1.lde");
    DevBuf t_leaves((size_t)K * N_loc * 32), t_nodes;
    hash_trace_rows(c, ext.as<fe>(), t_leaves.p, w, log_n, log_nc, K, (size_t)w * N_loc);      // local rows, [k][c - c0], per proof
    sub.mark("2.hash_rows");
    {
        // one GPU: the K trees level by level in one launch per level; several GPUs (K == 1): the sharded tree
        if (G == 1) {
            t_nodes.alloc((size_t)K * N_loc * 32);
            merkle_build(c, t_leaves.p, t_nodes.p, N_loc, K);
        }
        std::vector<const void *> roots;
        for (int p = 0; p < K; p++) {
            const uint8_t *leaves = (const uint8_t *)t_leaves.p + (size_t)p * N_loc * 32;
            if (G == 1) ps[p].t_tree.attach(c, leaves, (const uint8_t *)t_nodes.p + (size_t)p * N_loc * 32, n, log_nc);
            else ps[p].t_tree.build(c, leaves, n, log_nc, false);
            roots.push_back(ps[p].t_tree.root_dev());
        }
        std::vector<Digest> r = fetch_roots(c, roots);
        for (int p = 0; p < K; p++) memcpy(ps[p].proof->trace_root, r[p].data(), 32);
    }

    // ---- 3: evaluate constraints --------------------------------------------------------------------------------------------------------
    clk.mark(2);
    sub.mark("2.tree");
    std::vector<fe> last_rows((size_t)3 * K);      // op_counter and program hash of the last trace step of every proof (evaluator.rs:73-74)
    if (host_cols) {
        for (int p = 0; p < K; p++)
            for (int j = 0; j < 3; j++) memcpy(&last_rows[3 * p + j], host_cols[(size_t)p * w + j] + (n - 1) * 16, 16);
    } else {
        DevBuf d_last((size_t)48 * K);
        for (int j = 0; j < 3; j++)
            DG_CUDA(cudaMemcpy2DAsync((uint8_t *)d_last.p + 16 * j, 48, d_regs + (size_t)j * n + (n - 1), (size_t)w * n * 16, 16, K,
                                      cudaMemcpyDeviceToDevice, c.stream));
        d2h(c, last_rows.data(), d_last.p, (size_t)48 * K);
    }
    DevBuf &d_periodic = c.d_periodic;
    if (!d_periodic.p) {
        std::vector<fe> per = fs::periodic_tables();
        d_periodic.alloc(per.size() * 16, true);
        h2d(c, d_periodic.p, per.data(), per.size() * 16);
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }
    DevBuf d_coef, d_violation((size_t)4 * K);
    // per proof [coefA | coefB | bAi | bBi | bAf | bBf], coef_stride elements apart, then the boundary constants [K][KiA, KiB, KfA, KfB].
    // The transition coefficients have the same count for every proof of a shape; the boundary vectors have one entry per register that
    // carries a boundary constraint, which depends on the number of public inputs / outputs: they are padded with zero coefficients to
    // the largest count nbm (a zero coefficient adds nothing to the boundary numerators).
    size_t coef_stride = 0, T = 0, nbm = 0;
    {
        for (int p = 0; p < K; p++) {
            ProofState &s = ps[p];
            s.op_count = last_rows[3 * p];
            const fe program_hash[2] = {last_rows[3 * p + 1], last_rows[3 * p + 2]};
            s.cc = fs::draw_constraint_coefficients(s.proof->trace_root, ctx_depth, loop_depth, stack_depth, s.inputs, s.outputs, s.op_count,
                                                    program_hash);
            DG_REQUIRE(s.cc.coefA.size() == ps[0].cc.coefA.size(), "transition constraint counts differ inside a batch");
            T = s.cc.coefA.size();
            nbm = std::max(nbm, s.cc.bAi.size());
        }
        DG_REQUIRE(nbm <= (size_t)w, "more boundary registers than registers");
        coef_stride = 2 * T + 4 * nbm;
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
        d_coef.alloc(pack.size() * 16);
        h2d(c, d_coef.p, pack.data(), pack.size() * 16);
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }
    DG_CUDA(cudaMemsetAsync(d_violation.p, 0, (size_t)4 * K, c.stream));
    // per proof: [boundary numerator, first step | boundary numerator, last step | transition combination]
    DevBuf evals((size_t)K * 3 * E * 16);
    {
        const int num_c8 = 8 >> log_g;
        const uint64_t E_loc = n * num_c8;
        DevBuf evals_loc((size_t)K * E_loc * 16), gathered;
        if (G > 1) gathered.alloc(E * 16);
        AirParams P;
        memset(&P, 0, sizeof P);
        P.w = w; P.ctx_depth = ctx_depth; P.loop_depth = loop_depth; P.stack_depth = stack_depth;
        P.cl = std::max<int>(ctx_depth, 1); P.ll = std::max<int>(loop_depth, 1); P.sl = std::max(stack_depth, 8);
        P.log_n = log_n; P.log_blowup = log_b;
        P.ext = ext.as<fe>(); P.col_stride = N_loc;
        P.c8_base = g * num_c8; P.num_c8 = num_c8;
        P.t_ev = evals_loc.as<fe>();
        P.periodic = d_periodic.as<fe>();
        const fe *base = d_coef.as<fe>();
        P.coefA = base; P.coefB = base + T;
        P.twN = c.twiddle(log_N, false);
        static const int GROUP_DEG[6] = {2, 3, 4, 6, 7, 8};
        for (int gi = 0; gi < 6; gi++) P.inc[gi] = (8 * n - 1) - (n - 1) * GROUP_DEG[gi];
        P.violation = d_violation.as<unsigned>();
        P.ext_stride = (size_t)w * N_loc; P.t_ev_stride = E_loc; P.coef_stride = coef_stride;
    sub.mark("3.setup");
        launch_constraint_eval(c, P, K);
    sub.mark("3.eval");
        comm_all_reduce_max_u32(c, d_violation.as<unsigned>(), 1);
        std::vector<unsigned> violation(K);
        d2h(c, violation.data(), d_violation.p, (size_t)4 * K);
        for (int p = 0; p < K; p++)
            if (violation[p])
                ps[p].fail(DG_ERR_UNSATISFIED, "transition constraints at step " + std::to_string(violation[p] - 1) + " were not satisfied");
        if (!any_live()) return;
        // interpolation of the transition combination (constraint_table.rs:54-63), coset by coset: size-n inverse transforms of the own
        // cosets (sharded), all-gather, then the 8-point inverse DFT across cosets (poly.cu: coset_interp_finish) -> the 8n coefficients
        // in natural order; no transposition and no replicated 8n-point transform
    sub.mark("3.violation_sync");
        ntt_batch(c, evals_loc.as<fe>(), evals_loc.as<fe>(), log_n, K * num_c8, n, n, true);
        if (G > 1) comm_all_gather(c, evals_loc.as<fe>(), gathered.as<fe>(), E_loc * 16);
    sub.mark("3.intt+gather");
        coset_interp_finish(c, G > 1 ? gathered.as<fe>() : evals_loc.as<fe>(), evals.as<fe>() + 2 * E, log_n, K, E_loc, 3 * E);
        // boundary constraints (evaluator.rs:181-326), directly as the 8n coefficients the reference obtains by interpolation
        boundary_coeffs(c, K, polys.as<fe>(), (size_t)w * n, n, (int)nbm, d_coef.as<fe>() + 2 * T, coef_stride, d_coef.as<fe>() + coef_stride * K,
                        evals.as<fe>(), evals.as<fe>() + E, 3 * E);
    }
    if (K == 1) debug_dump(c, "t_coeffs", evals.as<fe>() + 2 * E, E * 16);

    // ---- 4: convert constraint evaluations into a polynomial -----------------------------------------------------------------------------
    clk.mark(3);
    sub.mark("3.finish+boundary");
    DevBuf combined((size_t)K * E * 16), scratch((size_t)K * E * 16), scratch2((size_t)K * E * 16);
    const fe root_n = host_root_of_unity(log_n);
    const fe x_last = host_inv(root_n);                        // w_n^(n-1)   (evaluator.rs:128-131)
    {
        if (K == 1) {
            debug_dump(c, "i_coeffs", evals.as<fe>(), E * 16);
            debug_dump(c, "f_coeffs", evals.as<fe>() + E, E * 16);
        }
        // one upload: the (base, step) pairs of the power tables of 1, x_last and 1 / x_last (shared by the K proofs), then K zeros (sub0)
        std::vector<fe> pack(6 + K, fe_make(0, 0));
        const fe bases[3] = {fe_make(1, 0), x_last, root_n};
        for (int t = 0; t < 3; t++) { pack[2 * t] = bases[t]; pack[2 * t + 1] = PowTables::step(bases[t], E + 1); }
        DevBuf d_pack(pack.size() * 16);
        h2d(c, d_pack.p, pack.data(), pack.size() * 16);
        PowTables pows(c, d_pack.as<fe>(), 3, E + 1);
        const fe *zeros = d_pack.as<fe>() + 6;
        fe *ic = evals.as<fe>(), *fc = evals.as<fe>() + E, *tc = evals.as<fe>() + 2 * E;          // of proof 0; proof p at + 3 E p
        syn_div(c, K, ic, 3 * E, ic, 3 * E, E, pows.ref(0), 0, 0, pows.ref(0), 0, 0, zeros);   // / (x - 1)
        syn_div(c, K, fc, 3 * E, fc, 3 * E, E, pows.ref(1), 0, 0, pows.ref(2), 0, 0, zeros);   // / (x - x_last)
        syn_div_expanded_sum(c, tc, scratch.as<fe>(), ic, fc, combined.as<fe>(), n, E, x_last, K, 3 * E, E);   // / ((x^n - 1)/(x - x_last)), summed
    }
    if (K == 1) debug_dump(c, "constraint_poly", combined.p, E * 16);

    // ---- 5: constraint evaluations over the LDE domain + their Merkle tree -----------------------------------------------------------------
    clk.mark(4);
    sub.mark("4.combine");
    DevBuf c_ext((size_t)K * N_loc * 16), c_items((size_t)K * (N_loc / 4) * 32), c_nodes;
    auto c_ext_of = [&](int p) { return c_ext.as<fe>() + (size_t)p * N_loc; };
    lde_batch(c, combined.as<fe>(), c_ext.as<fe>(), log_n, log_b, 8, K, E, N_loc, c0, (unsigned)nc);
    sub.mark("5.lde");
    constraint_items_local(c, c_ext.as<fe>(), log_n, log_nc, c_items.p, K);      // first tree level: H(4 evaluations), [k][c4 local], per proof
    sub.mark("5.items");
    {
        if (G == 1) {
            c_nodes.alloc((size_t)K * (N_loc / 4) * 32);
            merkle_build(c, c_items.p, c_nodes.p, N_loc / 4, K);
        }
        std::vector<const void *> roots;
        std::vector<int> who;
        for (int p = 0; p < K; p++) {
            if (!ps[p].live) continue;
            const uint8_t *items = (const uint8_t *)c_items.p + (size_t)p * (N_loc / 4) * 32;
            if (G == 1) ps[p].c_tree.attach(c, items, (const uint8_t *)c_nodes.p + (size_t)p * (N_loc / 4) * 32, n, log_nc - 2);
            else ps[p].c_tree.build(c, items, n, log_nc - 2, false);
            roots.push_back(ps[p].c_tree.root_dev());
            who.push_back(p);
        }
        std::vector<Digest> r = fetch_roots(c, roots);
        for (size_t i = 0; i < who.size(); i++) memcpy(ps[who[i]].proof->constraint_root, r[i].data(), 32);
    }

    // ---- 6: DEEP composition polynomial ---------------------------------------------------------------------------------------------------------
    clk.mark(5);
    sub.mark("5.tree");
    DevBuf comp((size_t)K * E * 16), comp_ext((size_t)K * N_loc * 16);
    {
        TwiddleRef g_t = c.twiddle(log_n, false);
        // trace polynomials at z and z*g: every rank evaluates its own columns (the split of stage 1); slots of 2 cpr values are gathered.
        // d_deep = [K][2 wp] trace values, then [K][2] values of the constraint polynomial at z
        const int wp = cpr * G;
        DevBuf d_deep((size_t)K * (2 * wp + 2) * 16);
        fe *deep_c = d_deep.as<fe>() + (size_t)K * 2 * wp;
        DG_CUDA(cudaMemsetAsync(d_deep.p, 0, d_deep.bytes, c.stream));
        // powers of z, 1/z, z g, 1/(z g) of every proof: four batched tables from one upload of the (base, step) pairs, [table][proof][2]
        std::vector<fe> base_step((size_t)8 * K, fe_make(0, 0));
        for (int p = 0; p < K; p++) {
            ProofState &s = ps[p];
            if (!s.live) continue;
            s.dc = fs::draw_composition_coefficients(s.proof->constraint_root, w);
            const fe z = s.dc.z, zg = fe_mul(z, root_n);
            const fe bases[4] = {z, host_inv(z), zg, host_inv(zg)};
            for (int t = 0; t < 4; t++) {
                base_step[(size_t)2 * (t * K + p)] = bases[t];
                base_step[(size_t)2 * (t * K + p) + 1] = PowTables::step(bases[t], t < 2 ? E + 1 : n + 1);
            }
        }
        DevBuf d_base_step(base_step.size() * 16);
        h2d(c, d_base_step.p, base_step.data(), base_step.size() * 16);
        const fe *bs = d_base_step.as<fe>();
        PowTables z_t(c, bs, K, E + 1), zi_t(c, bs + 2 * K, K, E + 1), zg_t(c, bs + 4 * K, K, n + 1), zgi_t(c, bs + 6 * K, K, n + 1);
        if (G == 1) {
            eval_polys_at(c, polys.as<fe>(), n, K * w, z_t.ref(0), g_t, true, d_deep.as<fe>(), w, z_t.lo_n, z_t.hi_n);
        } else {
            const int j0 = col_start(g), mine = col_count(g);
            if (mine > 0) eval_polys_at(c, polys.as<fe>() + (size_t)j0 * n, n, mine, z_t.ref(0), g_t, true, d_deep.as<fe>() + (size_t)2 * g * cpr);
            comm_all_gather(c, d_deep.as<fe>() + (size_t)2 * g * cpr, d_deep.p, (size_t)2 * cpr * 16);
        }
        eval_polys_at(c, combined.as<fe>(), E, K, z_t.ref(0), g_t, false, deep_c, 1, z_t.lo_n, z_t.hi_n);
        std::vector<fe> deep_slots((size_t)K * (2 * wp + 2));
        d2h(c, deep_slots.data(), d_deep.p, deep_slots.size() * 16);
    sub.mark("6.deep_values");
        // one upload: [K][2w] coefficients of the trace combinations | sub0 of the three divisions [3][K] | compose's k1, k2, kc [K][3]
        std::vector<fe> pack((size_t)K * (2 * w + 6), fe_make(0, 0));
        fe *ccs = pack.data(), *subs = ccs + (size_t)K * 2 * w, *ks = subs + (size_t)3 * K;
        for (int p = 0; p < K; p++) {
            ProofState &s = ps[p];
            if (!s.live) continue;
            const fe *slots = deep_slots.data() + (size_t)p * 2 * wp;
            std::vector<fe> deep(2 * w);
            for (int r = 0; r < G; r++)
                for (int o = 0; o < col_count(r); o++) {
                    deep[2 * (col_start(r) + o)] = slots[2 * (r * cpr + o)];
                    deep[2 * (col_start(r) + o) + 1] = slots[2 * (r * cpr + o) + 1];
                }
            s.state1.resize(w); s.state2.resize(w);
            fe sub1 = fe_make(0, 0), sub2 = fe_make(0, 0);
            for (int i = 0; i < w; i++) {
                s.state1[i] = deep[2 * i]; s.state2[i] = deep[2 * i + 1];
                sub1 = fe_add(sub1, fe_mul(s.state1[i], s.dc.trace1[i]));
                sub2 = fe_add(sub2, fe_mul(s.state2[i], s.dc.trace2[i]));
            }
            subs[p] = sub1; subs[K + p] = sub2; subs[2 * K + p] = deep_slots[(size_t)K * 2 * wp + 2 * p];
            std::copy(s.dc.trace1.begin(), s.dc.trace1.begin() + w, ccs + (size_t)p * 2 * w);
            std::copy(s.dc.trace2.begin(), s.dc.trace2.begin() + w, ccs + (size_t)p * 2 * w + w);
            ks[3 * p] = s.dc.t1_degree; ks[3 * p + 1] = s.dc.t2_degree; ks[3 * p + 2] = s.dc.constraints;
        }
        DevBuf d_pack(pack.size() * 16), t12((size_t)K * 2 * n * 16);
        h2d(c, d_pack.p, pack.data(), pack.size() * 16);
        const fe *d_cc = d_pack.as<fe>(), *d_subs = d_cc + (size_t)K * 2 * w, *d_ks = d_subs + (size_t)3 * K;
        fe *t1 = t12.as<fe>(), *t2 = t12.as<fe>() + n;                      // of proof 0; proof p at + 2 n p
        lincomb2(c, polys.as<fe>(), n, w, d_cc, d_cc + w, t1, t2, K, 2 * w, 2 * n);
        syn_div(c, K, t1, 2 * n, t1, 2 * n, n, z_t.ref(0), z_t.lo_n, z_t.hi_n, zi_t.ref(0), zi_t.lo_n, zi_t.hi_n, d_subs);
        //                                                                                                   (T1(x) - T1(z)) / (x - z)
        syn_div(c, K, t2, 2 * n, t2, 2 * n, n, zg_t.ref(0), zg_t.lo_n, zg_t.hi_n, zgi_t.ref(0), zgi_t.lo_n, zgi_t.hi_n, d_subs + K);
        //                                                                                                   (T2(x) - T2(zg)) / (x - zg)
        syn_div(c, K, combined.as<fe>(), E, scratch2.as<fe>(), E, E, z_t.ref(0), z_t.lo_n, z_t.hi_n, zi_t.ref(0), zi_t.lo_n, zi_t.hi_n,
                d_subs + 2 * K);                                                                           // (C(x) - C(z)) / (x - z)
    sub.mark("6.lincomb+syndiv");
        compose(c, K, t1, t2, 2 * n, scratch2.as<fe>(), comp.as<fe>(), n, E, 6 * n + 1, d_ks);
        if (K == 1) debug_dump(c, "composition_poly", comp.p, E * 16);
        // every rank extends its own cosets; the first FRI layers work on these slabs directly (no all-gather of the N evaluations)
        lde_batch(c, comp.as<fe>(), comp_ext.as<fe>(), log_n, log_b, 8, K, E, N_loc, c0, (unsigned)nc);
    }

    // ---- 7: FRI layers ---------------------------------------------------------------------------------------------------------------------------
    clk.mark(6);
    sub.mark("6.compose+lde");
    DevBuf fri_gathered;                                       // multi-GPU: the first replicated layer, gathered from the ranks' slabs
    std::vector<DevBuf> layer_bufs;                            // replicated layers: row hashes, trees and folded values of all K proofs
    size_t n_layers = 0;
    {
        TwiddleRef inv_root = c.twiddle(log_N, true);
        const fe tau_inv = host_inv(host_root_of_unity(2));
        const fe inv4 = host_inv(fe_make(4, 0));
        // the K proofs' layers are one buffer each: layer d of proof p = cur + p * cur_stride
        const fe *cur = comp_ext.as<fe>();
        uint64_t cur_stride = N_loc;
        Layout lay{log_N, log_b};
        bool local = G > 1;                                    // `cur` is this rank's coset slab of the layer (K == 1)
        // layer roots and folding points stay on the device, [layer][proof] (special_x = prng(root) is derived by fri_alpha): the host
        // sees the roots in one copy after the last layer.  With host RNG callbacks registered each layer asks the host instead: one
        // copy of the layer's K roots, the callbacks of the live proofs in proof order, one upload of the K folding points.
        const int MAX_LAYERS = 20;
        DevBuf d_alpha((size_t)MAX_LAYERS * K * 16), d_roots((size_t)MAX_LAYERS * K * 32);
        const bool host_rng = fs::rng_hooks_active();
        auto alpha_dev = [&](size_t layer) { return d_alpha.as<fe>() + layer * K; };
        auto root_slots = [&](size_t layer) { return (uint8_t *)d_roots.p + 32 * layer * K; };
        // the K roots of layer `li`, root_stride bytes apart from root0, into their slots
        auto copy_roots = [&](const void *root0, size_t root_stride, size_t li) {
            DG_REQUIRE(li < (size_t)MAX_LAYERS, "too many FRI layers");
            DG_CUDA(cudaMemcpy2DAsync(root_slots(li), 32, root0, std::max<size_t>(root_stride, 32), 32, K, cudaMemcpyDeviceToDevice, c.stream));
        };
        auto folding_points = [&](const void *root0, size_t root_stride, size_t li) {
            DG_REQUIRE(li < (size_t)MAX_LAYERS, "too many FRI layers");
            if (!host_rng) { fri_alpha(c, root0, alpha_dev(li), root_slots(li), K, root_stride); return; }
            copy_roots(root0, root_stride, li);
            std::vector<uint8_t> r((size_t)32 * K);
            d2h(c, r.data(), root_slots(li), r.size());
            std::vector<fe> alphas(K, fe_make(0, 0));
            for (int p = 0; p < K; p++)
                if (ps[p].live) alphas[p] = fs::prng_vector(r.data() + 32 * p, 1)[0];   // field::prng(seed) = first draw of the generator (field.rs:264-269)
            DG_CUDA(cudaMemcpyAsync(alpha_dev(li), alphas.data(), (size_t)16 * K, cudaMemcpyHostToDevice, c.stream));
            DG_CUDA(cudaStreamSynchronize(c.stream));
        };
        for (;;) {
            const int log_r = lay.log_d - 2;
            const uint64_t R = 1ULL << log_r;
            // layers below 2^22 values are latency-bound (two collectives per sharded tree cost more than hashing them whole): gather the
            // first such layer once (<= 32 MB) and finish redundantly on every rank
            if (local && (lay.log_d < 22 || log_r - log_b < 6)) {
                fri_gathered.alloc((size_t)16 << lay.log_d);
                comm_all_gather(c, cur, fri_gathered.p, ((size_t)16 << lay.log_d) >> log_g);     // rank-major == coset-major
                cur = fri_gathered.as<fe>();
                local = false;
            }
            const size_t li = n_layers++;
            if (local) {
                FriLayerDev &L = ps[0].layers.emplace_back();
                L.vals = cur; L.layout = lay; L.sharded = true;
                // rows r = b k' + c of the own cosets: hashes in ShardedTree order, n' = R / b subtrees of nc leaves per rank
                L.leaves.alloc((R >> log_g) * 32);
                fri_hash_rows_local(c, cur, lay.log_d, log_b, log_nc, L.leaves.p);
                L.tree.build(c, L.leaves.p, R >> log_b, log_nc, false);
                folding_points(L.tree.root_dev(), 0, li);
                L.folded.alloc((R >> log_g) * 16);
                fri_fold_local(c, cur, lay.log_d, log_b, log_nc, c0, L.folded.as<fe>(), alpha_dev(li), inv_root, log_N, tau_inv, inv4);
                cur = L.folded.as<fe>();
                lay = Layout{log_r, log_b};
                continue;
            }
            const Layout rows{log_r, (lay.log_b >= 0 && log_r >= lay.log_b) ? lay.log_b : -1};
            layer_bufs.emplace_back((size_t)K * R * 32);
            const uint8_t *leaves = layer_bufs.back().as<uint8_t>();
            layer_bufs.emplace_back((size_t)K * R * 32);
            const uint8_t *nodes = layer_bufs.back().as<uint8_t>();
            fri_hash_rows(c, cur, lay, rows, (void *)leaves, K, cur_stride);
            merkle_build(c, leaves, (void *)nodes, R, K);
            for (int p = 0; p < K; p++) {
                if (!ps[p].live) continue;
                FriLayerDev &L = ps[p].layers.emplace_back();
                L.vals = cur + (size_t)p * cur_stride; L.layout = lay; L.sharded = false;
                L.leaves_p = leaves + (size_t)p * R * 32; L.nodes_p = nodes + (size_t)p * R * 32;
            }
            if (R * 4 <= 256) {                                    // MAX_REMAINDER_LENGTH (fri/mod.rs:13): the remainder's root only
                copy_roots(nodes + 32, R * 32, li);
                break;
            }
            folding_points(nodes + 32, R * 32, li);                // special_x = prng(root)  (fri/prover.rs:29)
            layer_bufs.emplace_back((size_t)K * R * 16);           // values of the next layer
            fe *folded = layer_bufs.back().as<fe>();
            fri_fold(c, cur, lay, folded, rows, alpha_dev(li), inv_root, log_N, tau_inv, inv4, K, cur_stride);
            cur = folded;
            cur_stride = R;
            lay = rows;
        }
        std::vector<uint8_t> roots(32 * n_layers * K);
        d2h(c, roots.data(), d_roots.p, roots.size());
        for (int p = 0; p < K; p++)
            if (ps[p].live)
                for (size_t i = 0; i < n_layers; i++) memcpy(ps[p].layers[i].root.data(), roots.data() + 32 * (i * K + p), 32);
    }

    // ---- 8: query positions ------------------------------------------------------------------------------------------------------------------------
    clk.mark(7);
    sub.mark("7.fri");
    {
        std::vector<std::array<uint8_t, 32>> seeds;
        std::vector<int> who;
        for (int p = 0; p < K; p++) {
            if (!ps[p].live) continue;
            std::vector<uint8_t> roots;
            for (auto &L : ps[p].layers) roots.insert(roots.end(), L.root.begin(), L.root.end());
            if (K == 1) debug_dump_host("fri_roots", roots.data(), roots.size());
            seeds.emplace_back();
            fs::blake3_short(roots.data(), roots.size(), seeds.back().data());
            who.push_back(p);
        }
        std::vector<unsigned long long> nonces = pow_search_batch(c, seeds, opt.grinding_factor);
        for (size_t i = 0; i < who.size(); i++) {
            ProofState &s = ps[who[i]];
            s.proof->pow_nonce = nonces[i];
            pow_hash(seeds[i].data(), s.proof->pow_nonce, s.proof->pow_seed);
            try {
                s.positions = fs::query_positions(s.proof->pow_seed, N, b, opt.num_queries);
            } catch (const std::exception &e) { s.fail(DG_ERR_EXHAUSTED, e.what()); continue; }
            if (K == 1) debug_dump_host("positions", s.positions.data(), s.positions.size() * 8);
        }
        if (!any_live()) return;
    }

    // ---- 9: build proof objects --------------------------------------------------------------------------------------------------------------------------
    clk.mark(8);
    sub.mark("8.pow");
    // Plan every opening of every proof on the host, fetch all opened values / digests in one batched pass (FetchBatch), then serialise.
    FetchBatch fb(c);
    // registers the nodes of a batch-proof plan; leaf_ref / node_ref map leaf indices / heap indices to fetch references
    auto plan_offsets = [&](const fs::BatchPlan &plan, auto leaf_ref, auto node_ref) {
        Offsets o(plan.nodes.size());
        for (size_t sidx = 0; sidx < plan.nodes.size(); sidx++)
            for (auto &r : plan.nodes[sidx]) o[sidx].push_back(fb.add32(r.leaf ? leaf_ref(r.index) : node_ref(r.index)));
        return o;
    };
    auto digests_at = [&](const Offsets &o) {
        std::vector<std::vector<Digest>> v(o.size());
        for (size_t i = 0; i < o.size(); i++)
            for (size_t off : o[i]) v[i].push_back(fb.digest(off));
        return v;
    };
    auto plan_openings = [&](ProofState &s, const fe *ext_p, const fe *c_ext_p) {
        OpenPlan O;
        const std::vector<uint64_t> &positions = s.positions;
        const int nq = (int)positions.size();
        // trace rows at the queried positions (trace_table.rs:127-134): the rank owning the position's coset reads the row
        O.row_off.resize(nq);
        for (int q = 0; q < nq; q++) {
            const uint64_t cpos = positions[q] & (b - 1), k = positions[q] >> log_b;
            const int owner = (int)(cpos >> log_nc);
            const uint64_t phys = ((cpos - (uint64_t)owner * nc) << log_n) + k;
            for (int j = 0; j < w; j++) {
                const size_t off = fb.add16(FetchRef{ext_p + (size_t)j * N_loc, phys, owner});
                if (j == 0) O.row_off[q] = off;
            }
        }
        // trace tree openings: leaves are the row hashes
        O.tplan = fs::plan_batch_proof(positions, N);
        O.t_off = plan_offsets(O.tplan, [&](uint64_t i) { return s.t_tree.item_ref(i); }, [&](uint64_t h) { return s.t_tree.node_ref(h); });

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
            lo.pos = fpos;
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
            if (L.sharded) lo.node_off = plan_offsets(plan, [&](uint64_t i) { return L.tree.item_ref(i); }, [&](uint64_t h) { return L.tree.node_ref(h); });
            else lo.node_off = plan_offsets(plan, [&](uint64_t i) { return FetchRef{L.leaves_p, i, -1}; }, [&](uint64_t h) { return FetchRef{L.nodes_p, h, -1}; });
        }
        {
            FriLayerDev &L = s.layers.back();
            const uint64_t D = 1ULL << L.layout.log_d;
            for (uint64_t i = 0; i < D; i++) O.rem_off.push_back(fb.add16(FetchRef{L.vals, L.layout.phys(i), -1}));   // remainder, natural order
        }
        return O;
    };
    // serialise (proof.rs:10-37; bincode: u64 length prefixes, arrays raw, little endian)
    auto serialise = [&](ProofState &s, const OpenPlan &O) {
        fs::ByteWriter out;
        Proof *proof = s.proof.get();
        const int nq = (int)s.positions.size();
        out.raw(proof->trace_root, 32);
        out.u8(O.tplan.depth); out.u8((uint8_t)ctx_depth); out.u8((uint8_t)loop_depth); out.u8((uint8_t)stack_depth);
        out.u32((uint32_t)s.op_count.lo);                                             // op_count as u32 (proof.rs:62)
        write_digest_vv(out, digests_at(O.t_off));
        out.u64(nq);
        for (int q = 0; q < nq; q++) {
            out.u64(w);
            for (int j = 0; j < w; j++) out.felt(fb.value(O.row_off[q] + j));
        }
        out.raw(proof->constraint_root, 32);
        out.u64(O.cval_off.size());
        for (size_t off : O.cval_off) { Digest dgt = fb.digest(off); out.raw(dgt.data(), 32); }
        write_digest_vv(out, digests_at(O.c_off));
        out.u8(O.cplan.depth);
        write_felt_vec(out, s.state1);
        write_felt_vec(out, s.state2);

        out.u64(s.layers.size() - 1);
        for (size_t d = 0; d + 1 < s.layers.size(); d++) {
            const LayerOpen &lo = O.fri_open[d];
            out.raw(s.layers[d].root.data(), 32);
            out.u64(lo.pos.size());
            for (size_t off : lo.val_off)
                for (int j = 0; j < 4; j++) out.felt(fb.value(off + j));
            write_digest_vv(out, digests_at(lo.node_off));
            out.u8(lo.depth);
        }
        out.raw(s.layers.back().root.data(), 32);
        out.u64(O.rem_off.size());
        for (size_t off : O.rem_off) out.felt(fb.value(off));
        out.u64(proof->pow_nonce);
        out.u8((uint8_t)log_b); out.u8((uint8_t)opt.num_queries); out.u8((uint8_t)opt.grinding_factor); out.u8(0);
        proof->bytes = std::move(out.b);
    };
    {
        std::vector<OpenPlan> plans(K);
        for (int p = 0; p < K; p++)
            if (ps[p].live) plans[p] = plan_openings(ps[p], ext_of(p), c_ext_of(p));
        fb.run();
        for (int p = 0; p < K; p++)
            if (ps[p].live) serialise(ps[p], plans[p]);
    }
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
        DG_REQUIRE(ni <= 8 && no <= 8, "cannot have more than 8 public inputs / outputs");
        DG_REQUIRE((ni == 0 || (inputs16 && inputs16[i])) && (no == 0 || (outputs16 && outputs16[i])), "null public inputs / outputs");
        ps[i].inputs.resize(ni);
        ps[i].outputs.resize(no);
        if (ni) memcpy(ps[i].inputs.data(), inputs16[i], ni * 16);
        if (no) memcpy(ps[i].outputs.data(), outputs16[i], no * 16);
    }
    return ps;
}

// the single-trace entry points: a batch of one whose failure is the call's error
Proof *prove_one(Context &c, fe *d_regs, const uint8_t *const *host_cols, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                 const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16, uint32_t n_outputs, const dg_options_t &opt,
                 dg_prove_stats_t *stats) {
    std::vector<ProofState> ps = make_states(1, &inputs16, &n_inputs, &outputs16, &n_outputs);
    prove_core(c, d_regs, host_cols, 1, width, length, ctx_depth, loop_depth, ps, opt, stats);
    if (ps[0].status != DG_OK) throw Error(ps[0].status, ps[0].message);
    return ps[0].proof.release();
}

// Device bytes one proof of this shape takes in a batch on one GPU: the buffers prove_core allocates per proof, stage by stage (every
// one stays in the bump arena until the group ends), plus its register columns (the upload buffer of a host batch).
size_t proof_footprint(uint32_t w, uint64_t n, uint32_t b) {
    const size_t N = (size_t)n * b, E = (size_t)n * 8, fe16 = 16, dg32 = 32;
    size_t f = 0;
    f += (size_t)w * n * fe16;                // registers (host batch: upload buffer)
    f += (size_t)w * n * fe16;                // 1: polynomials
    f += (size_t)w * N * fe16;                // 1: trace LDE
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

int batch_group_size(Context &c, uint32_t w, uint64_t n, uint32_t b, uint32_t count) {
    const size_t per = proof_footprint(w, n, b);
    long long k = std::min<long long>(count, max_group_for_grid(w));
    if ((size_t)count * per > c.arena.cap) {                 // does not fit in the arena the library already holds: ask the driver
        size_t free_b = 0, total_b = 0;
        DG_CUDA(cudaMemGetInfo(&free_b, &total_b));
        const size_t avail = (free_b + c.arena.cap) / 10 * 8;
        k = std::min<long long>(k, (long long)std::max<size_t>(1, avail / per));
    }
    if (const char *e = getenv("DG_BATCH_GROUP")) {
        const long long cap = atoll(e);
        DG_REQUIRE(cap >= 1, "DG_BATCH_GROUP must be a positive integer");
        k = std::min(k, cap);
    }
    return (int)k;
}

void add_stats(dg_prove_stats_t *sum, const dg_prove_stats_t &s) {
    for (int i = 0; i < 9; i++) sum->stage_ms[i] += s.stage_ms[i];
    sum->h2d_ms += s.h2d_ms;
    sum->total_ms += s.total_ms;
    sum->kernel_launches += s.kernel_launches;
}

// runs the batch group by group; run_group(first, k, states, stats) proves traces [first, first + k)
template <typename F>
void prove_groups(Context &c, uint32_t count, uint32_t w, uint64_t n, const dg_options_t &opt, std::vector<ProofState> &all, Proof **proofs_out,
                  int *status, std::vector<std::string> &messages, dg_prove_stats_t *stats, F &&run_group) {
    DG_REQUIRE(c.world == 1 && ctx_device_count() == 1, "batched proving runs on one GPU: the library was initialised for several (dg_init_devices / dg_comm_init)");
    const int group = batch_group_size(c, w, n, opt.extension_factor, count);
    if (stats) memset(stats, 0, sizeof *stats);
    for (uint32_t i = 0; i < count; i++) { proofs_out[i] = nullptr; status[i] = DG_OK; }
    messages.assign(count, std::string());
    // a group that fails as a whole fails the call: the proofs of the earlier groups are freed, nothing is returned
    struct ReleaseOnError {
        Proof **out; uint32_t count; bool done = false;
        ~ReleaseOnError() { if (!done) for (uint32_t i = 0; i < count; i++) { delete out[i]; out[i] = nullptr; } }
    } release{proofs_out, count};
    for (uint32_t first = 0; first < count; first += group) {
        const int k = (int)std::min<uint32_t>(group, count - first);
        std::vector<ProofState> ps;
        for (int i = 0; i < k; i++) ps.push_back(std::move(all[first + i]));
        dg_prove_stats_t st;
        memset(&st, 0, sizeof st);
        run_group(first, k, ps, &st);
        if (stats) add_stats(stats, st);
        for (int i = 0; i < k; i++) {
            status[first + i] = ps[i].status;
            messages[first + i] = ps[i].message;
            if (ps[i].status == DG_OK) proofs_out[first + i] = ps[i].proof.release();
        }
    }
    release.done = true;
}

}  // namespace

Proof *prove_device(Context &c, const fe *d_regs, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                    const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16, uint32_t n_outputs, const dg_options_t &opt,
                    dg_prove_stats_t *stats, float) {
    return prove_one(c, const_cast<fe *>(d_regs), nullptr, width, length, ctx_depth, loop_depth, inputs16, n_inputs, outputs16, n_outputs, opt, stats);
}

Proof *prove_host(Context &c, const dg_trace_t &trace, const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16,
                  uint32_t n_outputs, const dg_options_t &opt, dg_prove_stats_t *stats) {
    DG_REQUIRE(trace.columns && trace.width >= 16 && trace.width < 128, "invalid trace");
    DG_REQUIRE(trace.length >= 16 && (trace.length & (trace.length - 1)) == 0, "execution trace length must be a power of 2 and at least 16");
    for (uint32_t j = 0; j < trace.width; j++) DG_REQUIRE(trace.columns[j] != nullptr, "null register column");
    c.upload_buf.ensure((size_t)trace.length * 16 * trace.width, true);
    return prove_one(c, c.upload_buf.as<fe>(), trace.columns, trace.width, trace.length, trace.ctx_depth, trace.loop_depth, inputs16, n_inputs,
                     outputs16, n_outputs, opt, stats);
}

void prove_batch_host(Context &c, const dg_trace_t *traces, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                      const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t &opt, Proof **proofs_out, int *status,
                      std::vector<std::string> &messages, dg_prove_stats_t *stats) {
    DG_REQUIRE(count >= 1, "batch must hold at least one trace");
    const dg_trace_t &t0 = traces[0];
    for (uint32_t i = 0; i < count; i++) {
        const dg_trace_t &t = traces[i];
        DG_REQUIRE(t.width == t0.width && t.length == t0.length && t.ctx_depth == t0.ctx_depth && t.loop_depth == t0.loop_depth,
                   "all traces of a batch must have the same width, length, context depth and loop depth");
        DG_REQUIRE(t.columns && t.width >= 16 && t.width < 128, "invalid trace");
        for (uint32_t j = 0; j < t.width; j++) DG_REQUIRE(t.columns[j] != nullptr, "null register column");
    }
    DG_REQUIRE(t0.length >= 16 && (t0.length & (t0.length - 1)) == 0, "execution trace length must be a power of 2 and at least 16");
    std::vector<ProofState> all = make_states(count, inputs16, n_inputs, outputs16, n_outputs);
    prove_groups(c, count, t0.width, t0.length, opt, all, proofs_out, status, messages, stats, [&](uint32_t first, int k, std::vector<ProofState> &ps, dg_prove_stats_t *st) {
        std::vector<const uint8_t *> cols;
        for (int i = 0; i < k; i++) cols.insert(cols.end(), traces[first + i].columns, traces[first + i].columns + t0.width);
        c.upload_buf.ensure((size_t)t0.length * 16 * t0.width * k, true);
        prove_core(c, c.upload_buf.as<fe>(), cols.data(), k, t0.width, t0.length, t0.ctx_depth, t0.loop_depth, ps, opt, st);
    });
}

void prove_batch_device(Context &c, const fe *d_regs, uint32_t count, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                        const uint8_t *const *inputs16, const uint32_t *n_inputs, const uint8_t *const *outputs16, const uint32_t *n_outputs,
                        const dg_options_t &opt, Proof **proofs_out, int *status, std::vector<std::string> &messages, dg_prove_stats_t *stats) {
    DG_REQUIRE(count >= 1, "batch must hold at least one trace");
    std::vector<ProofState> all = make_states(count, inputs16, n_inputs, outputs16, n_outputs);
    prove_groups(c, count, width, length, opt, all, proofs_out, status, messages, stats, [&](uint32_t first, int k, std::vector<ProofState> &ps, dg_prove_stats_t *st) {
        prove_core(c, const_cast<fe *>(d_regs) + (size_t)first * width * length, nullptr, k, width, length, ctx_depth, loop_depth, ps, opt, st);
    });
}

}  // namespace dg
