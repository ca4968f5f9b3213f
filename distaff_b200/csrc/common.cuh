// Shared host-side plumbing for the CUDA prover: error handling, device buffers, the per-process context.
#pragma once
#include <cuda_runtime.h>
#include <array>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>
#include "fp128.cuh"

namespace dg {

typedef std::array<uint8_t, 32> Digest;

struct Error : public std::runtime_error {
    int code;
    Error(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};

#define DG_CUDA(expr)                                                                                         \
    do {                                                                                                      \
        cudaError_t _e = (expr);                                                                              \
        if (_e != cudaSuccess)                                                                                \
            throw dg::Error(-2, std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " + __FILE__ + ":" + std::to_string(__LINE__)); \
    } while (0)

#define DG_REQUIRE(cond, msg)                                      \
    do {                                                           \
        if (!(cond)) throw dg::Error(-1, std::string(msg));        \
    } while (0)

// stream on which DevBuf allocations are ordered: the stream of the calling thread's current context
cudaStream_t &alloc_stream();

// Per-proof arena: a proof's buffers (tens of GB at 2^20 steps) are carved out of one device allocation with a bump pointer, so a
// proof performs no driver allocation at all.  The first proof of a given size runs on the stream-ordered pool and records how
// much it needed; the arena is then (re)sized for the following proofs.  Persistent objects (twiddle tables, NTT scratch) never
// come from the arena.
struct Arena {
    void *base = nullptr;
    size_t cap = 0, off = 0, counted = 0;
    bool active = false, counting = false;
    void *take(size_t n) {
        const size_t a = (n + 255) & ~(size_t)255;
        if (off + a > cap) return nullptr;
        void *p = (uint8_t *)base + off;
        off += a;
        return p;
    }
};
Arena &arena();

// RAII device buffer: arena (inside a proof), else stream-ordered allocator (cudaMallocAsync with a retained pool)
struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    bool from_arena = false;
    DevBuf() {}
    explicit DevBuf(size_t n) { alloc(n); }
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    DevBuf(DevBuf &&o) noexcept : p(o.p), bytes(o.bytes), from_arena(o.from_arena) { o.p = nullptr; o.bytes = 0; }
    DevBuf &operator=(DevBuf &&o) noexcept {
        if (this != &o) { release(); p = o.p; bytes = o.bytes; from_arena = o.from_arena; o.p = nullptr; o.bytes = 0; }
        return *this;
    }
    ~DevBuf() { release(); }
    void alloc(size_t n, bool persistent = false) {
        release();
        if (n == 0) return;
        Arena &a = arena();
        if (!persistent) {
            if (a.counting) a.counted += (n + 255) & ~(size_t)255;
            if (a.active) {
                p = a.take(n);
                if (p) { bytes = n; from_arena = true; return; }
            }
        }
        DG_CUDA(cudaMallocAsync(&p, n, alloc_stream()));
        bytes = n;
        from_arena = false;
    }
    void ensure(size_t n, bool persistent = false) { if (bytes < n) alloc(n, persistent); }
    void release() {
        if (p && !from_arena) cudaFreeAsync(p, alloc_stream());
        p = nullptr; bytes = 0; from_arena = false;
    }
    template <typename T> T *as() const { return (T *)p; }
};

// brackets one proof: activates the arena when it is large enough, otherwise measures the proof so that the next one fits
struct ArenaScope {
    ArenaScope();
    ~ArenaScope();
};

// two-level table of powers of a root of unity of order 2^log_order:
//   w^e = hi[e >> lo_bits] * lo[e & (2^lo_bits - 1)]
struct TwiddleTable {
    DevBuf lo, hi;
    int log_order = 0, lo_bits = 0;
};
struct TwiddleRef {
    const fe *lo, *hi;
    int lo_bits;
    unsigned mask;    // order - 1
};

struct Context {
    int device = 0;
    Arena arena;                            // per-proof bump arena of this device
    void *nccl_comm = nullptr;              // this rank's NCCL communicator (comm.cu), one per context
    DevBuf d_periodic;                      // periodic AIR tables on this device (prover.cu stage 3)
    bool air_consts = false, alghash_consts = false, vm_consts = false;     // __constant__ tables uploaded to this device
    std::map<const void *, size_t> func_smem;            // per-device cudaFuncSetAttribute(MaxDynamicSharedMemorySize) already applied
    DevBuf l2_scratch;
    int num_sms = 132;                      // H100 SXM; set from the device properties
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;     // host->device uploads that overlap compute (prover.cu stage 1)
    std::function<void(const char *)> mark;     // optional sub-stage marker of the running proof (DG_SUBSTAGE), else empty
    cudaStream_t comm_stream = nullptr;     // collectives that overlap compute (the all-gather of the trace polynomials)
    std::mutex mu;
    // small root tables for the in-shared-memory transforms: per size 2^l (l = 1..MAX_LOG_L) the per-stage roots, then their fe_mul_tw
    // companions (context.cu)
    DevBuf small_roots[2];
    size_t small_root_offset[16];
    std::map<int, TwiddleTable> twiddles;   // key = log_order * 2 + inverse
    DevBuf ntt_tmp;
    struct PinnedBuf {                       // page-locked host memory owned by the library (staging of pageable traces)
        void *p = nullptr; size_t bytes = 0;
        void ensure(size_t n) {
            if (bytes >= n) return;
            if (p) cudaFreeHost(p);
            p = nullptr; bytes = 0;
            DG_CUDA(cudaHostAlloc(&p, n, cudaHostAllocDefault));
            bytes = n;
        }
    } staging;
    cudaStream_t staging_streams[4] = {nullptr, nullptr, nullptr, nullptr};
    DevBuf upload_buf;                       // device copy of a host trace (dg_prove), kept between proofs                         // scratch of the multi-pass transforms
    std::string last_error;
    unsigned long long launches = 0;        // kernels launched by this library (bench.py's gpu_launches)
    int rank = 0, world = 1;                // multi-GPU sharding (comm.cu); world == 1: no communication
    size_t mem_limit = 0;                   // most device bytes the library may hold (arena + pool), 0 = no limit (dg_set_memory_limit)
    size_t mem_peak = 0;                    // most held since the limit was set, up to the last change of the arena (memory_usage)
    size_t pool_floor = 0;                  // under a limit: pool memory the trim at dg_set_memory_limit could not hand back beside what
                                            // was in use (chunks that persistent buffers keep partly used); Budget::FREE counts it as held

    TwiddleRef twiddle(int log_order, bool inverse);
    std::map<int, DevBuf> single_tables;    // full power tables w^e, e < 2^log_order (small orders only)
    const fe *single_table(int log_order);
    std::map<long long, DevBuf> lde_twiddles;   // per (log_n, log_blowup, first pass size): merged lane/coset twiddles of the LDE's first pass (ntt.cu)
    std::map<long long, DevBuf> coset_roots;    // per (first pass size, log_blowup): butterfly factors of the fold-1 LDE's first pass (ntt.cu)
    const fe *roots(int log_l, bool inverse) const { return small_roots[inverse ? 1 : 0].as<fe>() + small_root_offset[log_l]; }
};

// The calling thread's current context.  A process normally has one (device 0 or $DG_DEVICE / dg_init), created lazily; after
// dg_init_devices(n) there is one context per device and dg_prove drives them from n host threads, each bound to its own.
Context &ctx();
void ctx_init(int device);
void ctx_init_devices(int n);               // contexts for devices 0 .. n-1 + one NCCL communicator per device (single-process multi-GPU)
int ctx_device_count();                     // number of contexts (1 unless ctx_init_devices was called)
Context &ctx_of(int index);
// throws DG_ERR_INVALID ("<what> is not device memory of the library's device") unless p is device or managed memory of c's device
void require_device_memory(const Context &c, const void *p, const std::string &what);
void ctx_bind(Context *c);                  // makes c the calling thread's current context (and its device current)
// raises the dynamic shared-memory limit of a kernel on c's device once
void set_func_smem(Context &c, const void *func, size_t bytes);

// ---- device-memory budget (context.cu) -------------------------------------------------------------------------------------
// The one budget of every grouped call (prover, trace check, batched verification).  ARENA (prover): the arena when `need` fits in it,
// else 80 % of the free memory plus the arena, which the group replaces; FREE: 80 % of the free memory; FIXED: `need` itself.  With a
// memory limit the result is capped by the limit less what the library holds outside the arena and the `scratch` bytes the call adds.
enum class Budget { ARENA, FREE, FIXED };
size_t memory_budget(Context &c, Budget kind, size_t need, size_t scratch = 0);
size_t memory_held_outside_arena(Context &c);      // pool memory in use: persistent tables, transform scratch, upload buffer
void arena_release(Context &c);                   // frees the arena (the next proofs run on the pool until it is sized again)
void memory_set_limit(Context &c, size_t bytes);  // 0 = no limit; resets the peak
void memory_usage(Context &c, size_t *held, size_t *peak);

// host-side field helpers (portable path of fp128.cuh)
fe host_root_of_unity(int log_order);            // w of order 2^log_order  (field::get_root_of_unity)
fe host_pow(fe b, unsigned long long e);
fe host_inv(fe a);

// the least l with 2^l >= v
inline int ceil_log2(uint64_t v) { int l = 0; while ((1ULL << l) < v) l++; return l; }

static const int MAX_LOG_L = 10;                 // largest in-shared-memory transform: 1024 points

// device time between construction and stop() on a stream, in ms; does nothing when ms is null
struct EventTimer {
    cudaEvent_t a = nullptr, b = nullptr;
    cudaStream_t s;
    float *out;
    EventTimer(cudaStream_t stream, float *ms) : s(stream), out(ms) {
        if (!out) return;
        DG_CUDA(cudaEventCreate(&a));
        DG_CUDA(cudaEventCreate(&b));
        DG_CUDA(cudaEventRecord(a, s));
    }
    void stop() {
        if (!out) return;
        DG_CUDA(cudaEventRecord(b, s));
        DG_CUDA(cudaEventSynchronize(b));
        DG_CUDA(cudaEventElapsedTime(out, a, b));
    }
    ~EventTimer() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
};

// ---- NTT engine (ntt.cu) ------------------------------------------------------------------------------------------
// natural-order DFT over the subgroup of order n = 2^log_n for `batch` vectors laid out with `stride` elements apart;
// dst may equal src.  inverse: multiplies by n^-1 (polynom::interpolate_fft semantics).
void ntt_batch(Context &c, const fe *src, fe *dst, int log_n, int batch, size_t src_stride, size_t dst_stride, bool inverse);
// coset low-degree extension: coefficient vectors (batch of them, `coeff_len` = fold * n coefficients each, stride
// `src_stride`) are evaluated over the 2^log_blowup cosets of the order-n subgroup; output per vector is
// [coset c][k] = P(w_N^c * w_n^k), N = n << log_blowup, i.e. LDE index i = (k << log_blowup) + c lives at c*n + k.
void lde_batch(Context &c, const fe *src, fe *dst, int log_n, int log_blowup, int fold, int batch, size_t src_stride, size_t dst_stride,
               unsigned coset0 = 0, unsigned ncosets = 0 /* 0 = all 2^log_blowup */);
// bytes of the per-shape tables a fold-1 LDE of this shape would build that the context does not hold yet
size_t lde_tables_to_add(Context &c, int log_n, int log_blowup);

// ---- multi-GPU plumbing (comm.cu) -----------------------------------------------------------------------------------------
void comm_unique_id(uint8_t out[128]);
void comm_init(Context &c, int rank, int world, const uint8_t id_bytes[128]);
void comm_init_all(std::vector<Context *> &ctxs);     // single process: ncclCommInitAll over the contexts' devices
void comm_finalize(Context &c);
void comm_all_gather(Context &c, const void *send, void *recv, size_t bytes_per_rank, cudaStream_t stream = nullptr);   // default: the compute stream
void comm_all_to_all(Context &c, const void *send, void *recv, size_t bytes_per_peer);
void comm_all_reduce_max_u32(Context &c, unsigned *buf, size_t count);
void comm_all_reduce_sum_u32(Context &c, const unsigned *send, unsigned *recv, size_t count);

}  // namespace dg
