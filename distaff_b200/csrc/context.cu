// Per-process device context: stream, root-of-unity tables, scratch.  No CPU fallback exists: every entry point needs a
// CUDA device and fails loudly (dg::Error -> negative return code + dg_last_error()) when there is none.
#include "common.cuh"

namespace dg {

// 2^40-th root of unity G (/root/reference/src/math/field.rs:14)
static const fe G40 = {0x86b8723e1920f4aaULL, 0x120532e7b364080aULL};

fe host_pow(fe b, unsigned long long e) { return fe_pow_u64(b, e); }
fe host_inv(fe a) { return fe_inv(a); }
fe host_root_of_unity(int log_order) {
    DG_REQUIRE(log_order >= 0 && log_order <= 40, "order cannot exceed 2^40");
    fe r = G40;
    for (int i = 0; i < 40 - log_order; i++) r = fe_sqr(r);
    return r;
}

// out[i] = base^(i * step_pow)   where step = base^(2^shift) is passed precomputed
__global__ void power_table_kernel(fe *out, fe step, unsigned count) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) out[i] = fe_pow_u64(step, i);
}
// companions of fixed twiddles for fe_mul_tw: out[i] = in[i] * 2^64
__global__ void companion_table_kernel(fe *out, const fe *in, unsigned count) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) out[i] = fe_tw_companion(in[i]);
}

static thread_local Context *tl_ctx = nullptr;
cudaStream_t &alloc_stream() { return ctx().stream; }
Arena &arena() { return ctx().arena; }

ArenaScope::ArenaScope() {
    Arena &a = arena();
    a.off = 0;
    a.counted = 0;
    a.counting = true;
    a.active = a.base != nullptr && !getenv("DG_NO_ARENA");
}
static cudaMemPool_t device_pool(const Context &c) {
    cudaMemPool_t pool = nullptr;
    if (cudaDeviceGetDefaultMemPool(&pool, c.device) != cudaSuccess) cudaGetLastError();
    return pool;
}
static size_t pool_attr(const Context &c, cudaMemPoolAttr attr) {
    unsigned long long v = 0;
    if (cudaMemPoolGetAttribute(device_pool(c), attr, &v) != cudaSuccess) cudaGetLastError();
    return (size_t)v;
}
// folds what was held since the last fold (the arena + the pool's high-water mark) into the peak, and restarts the pool's mark; called
// whenever the arena changes size (no error is raised: it runs in destructors)
static void reset_pool_high(Context &c) {
    unsigned long long zero = 0;       // restarts the mark at the current reservation
    if (cudaMemPoolSetAttribute(device_pool(c), cudaMemPoolAttrReservedMemHigh, &zero) != cudaSuccess) cudaGetLastError();
}
static void fold_peak(Context &c) {
    c.mem_peak = std::max(c.mem_peak, c.arena.cap + pool_attr(c, cudaMemPoolAttrReservedMemHigh));
    reset_pool_high(c);
}

// the pool keeps what it frees up to what the limit leaves beside the arena (everything without a limit)
static void apply_release_threshold(Context &c) {
    unsigned long long threshold = ~(unsigned long long)0;
    if (c.mem_limit) threshold = c.mem_limit > c.arena.cap ? c.mem_limit - c.arena.cap : 0;
    if (cudaMemPoolSetAttribute(device_pool(c), cudaMemPoolAttrReleaseThreshold, &threshold) != cudaSuccess) cudaGetLastError();
}

ArenaScope::~ArenaScope() {
    Arena &a = arena();
    a.counting = false;
    const bool overflowed = a.counted > a.cap;
    a.active = false;
    if (overflowed && !getenv("DG_NO_ARENA")) {          // grow for the next proof of this size (driver call, outside the timed path)
        Context &c = ctx();
        cudaStreamSynchronize(alloc_stream());
        fold_peak(c);
        if (a.base) cudaFree(a.base);
        a.base = nullptr;
        a.cap = 0;
        const size_t want = a.counted + (a.counted >> 4) + (64 << 20);
        // hand the measuring proof's pool memory back before taking the arena
        cudaMemPoolTrimTo(device_pool(c), 0);
        reset_pool_high(c);
        // under a memory limit an arena that does not fit beside what the pool holds is not taken: the proofs keep running on the pool
        const bool fits = !c.mem_limit || want + pool_attr(c, cudaMemPoolAttrReservedMemCurrent) <= c.mem_limit;
        if (fits && cudaMalloc(&a.base, want) == cudaSuccess) a.cap = want;
        else { a.base = nullptr; cudaGetLastError(); }
        apply_release_threshold(c);
        fold_peak(c);
    }
}

void arena_release(Context &c) {
    DG_CUDA(cudaStreamSynchronize(c.stream));
    fold_peak(c);
    if (c.arena.base) cudaFree(c.arena.base);
    c.arena.base = nullptr;
    c.arena.cap = 0;
    apply_release_threshold(c);
}

size_t memory_held_outside_arena(Context &c) { return pool_attr(c, cudaMemPoolAttrUsedMemCurrent); }

size_t memory_budget(Context &c, Budget kind, size_t need, size_t scratch) {
    size_t avail = need;
    if (kind == Budget::ARENA && need <= c.arena.cap) {
        avail = c.arena.cap;
    } else if (kind != Budget::FIXED) {                  // does not fit in the arena the library already holds: ask the driver
        size_t free_b = 0, total_b = 0;
        DG_CUDA(cudaMemGetInfo(&free_b, &total_b));
        avail = (free_b + (kind == Budget::ARENA ? c.arena.cap : 0)) / 10 * 8;
    }
    if (c.mem_limit) {
        // free-memory budgets (execution buffers, trace checks) come on top of the pool's floor as well: memory the pool could not hand
        // back when the limit was set, because persistent buffers of earlier calls keep its chunks partly used
        const size_t held = memory_held_outside_arena(c) + scratch + (kind == Budget::FREE ? c.pool_floor : 0);
        avail = std::min(avail, c.mem_limit > held ? c.mem_limit - held : 0);
    }
    return avail;
}

void memory_set_limit(Context &c, size_t bytes) {
    DG_CUDA(cudaStreamSynchronize(c.stream));
    c.mem_limit = bytes;
    c.pool_floor = 0;
    apply_release_threshold(c);
    if (bytes) {
        if (c.arena.cap + memory_held_outside_arena(c) > bytes) arena_release(c);
        // hand back everything the pool holds unused; what stays reserved beyond the memory in use is the floor
        DG_CUDA(cudaMemPoolTrimTo(device_pool(c), 0));
        const size_t reserved = pool_attr(c, cudaMemPoolAttrReservedMemCurrent), used = pool_attr(c, cudaMemPoolAttrUsedMemCurrent);
        c.pool_floor = reserved > used ? reserved - used : 0;
    }
    fold_peak(c);
    c.mem_peak = c.arena.cap + pool_attr(c, cudaMemPoolAttrReservedMemCurrent);
}

void memory_usage(Context &c, size_t *held, size_t *peak) {
    const size_t now = c.arena.cap + pool_attr(c, cudaMemPoolAttrReservedMemCurrent);
    if (held) *held = now;
    if (peak) *peak = std::max(c.mem_peak, c.arena.cap + pool_attr(c, cudaMemPoolAttrReservedMemHigh));
}

static std::mutex g_ctx_mu;
static std::vector<Context *> g_ctxs;            // [0] = primary context; more after ctx_init_devices

static Context *build_context(int device) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        throw Error(-3, "no CUDA device available: distaff_b200 has no CPU path (cudaGetDeviceCount: " + std::string(cudaGetErrorString(e)) + ")");
    DG_REQUIRE(device < count, "requested CUDA device does not exist");
    DG_CUDA(cudaSetDevice(device));
    Context *c = new Context();
    c->device = device;
    Context *prev = tl_ctx;
    tl_ctx = c;                                          // the allocations below are ordered on this context's stream
    cudaDeviceProp prop;
    DG_CUDA(cudaGetDeviceProperties(&prop, device));
    c->num_sms = prop.multiProcessorCount;
    DG_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    DG_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    DG_CUDA(cudaStreamCreateWithFlags(&c->comm_stream, cudaStreamNonBlocking));
    {   // keep freed blocks in the pool instead of returning them to the driver between proofs
        cudaMemPool_t pool;
        DG_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
        unsigned long long threshold = ~0ULL;
        DG_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold));
    }
    // small root tables
    // per-stage tables of every sub-transform size L = 2^l: stage st occupies [L - (L >> st), L - (L >> (st+1))) with
    // W_st[j] = w_L^(j << st), j < L >> (st+1); L entries reserved per size (the last one is unused), followed by the L companions
    // W_st[j] * 2^64 of fe_mul_tw at the same positions + L
    size_t total = 0;
    for (int l = 1; l <= MAX_LOG_L; l++) { c->small_root_offset[l] = total; total += (size_t)2 << l; }
    c->small_root_offset[0] = 0;
    for (int inv = 0; inv < 2; inv++) {
        c->small_roots[inv].alloc(total * sizeof(fe), true);
        DG_CUDA(cudaMemsetAsync(c->small_roots[inv].p, 0, total * sizeof(fe), c->stream));
        for (int l = 1; l <= MAX_LOG_L; l++) {
            fe w = host_root_of_unity(l);
            if (inv) w = host_inv(w);
            const unsigned L = 1u << l;
            for (int st = 0; st < l; st++) {
                unsigned cnt = L >> (st + 1);
                fe *out = c->small_roots[inv].as<fe>() + c->small_root_offset[l] + (L - (L >> st));
                power_table_kernel<<<(cnt + 127) / 128, 128, 0, c->stream>>>(out, w, cnt);
                DG_CUDA(cudaGetLastError());
                w = fe_sqr(w);
            }
            fe *roots = c->small_roots[inv].as<fe>() + c->small_root_offset[l];
            companion_table_kernel<<<(L + 127) / 128, 128, 0, c->stream>>>(roots + L, roots, L);
            DG_CUDA(cudaGetLastError());
        }
    }
    DG_CUDA(cudaStreamSynchronize(c->stream));
    tl_ctx = prev;
    return c;
}

void ctx_init(int device) {
    {
        std::lock_guard<std::mutex> lk(g_ctx_mu);
        if (g_ctxs.empty()) {
            if (device < 0) {
                const char *env = getenv("DG_DEVICE");
                device = env ? atoi(env) : 0;
            }
            g_ctxs.push_back(build_context(device));
        } else if (device >= 0 && device != g_ctxs[0]->device) {
            // a late dg_init(other device) must not silently keep the old device (every rank of a multi-GPU host would share one GPU)
            throw Error(-1, "the library is already initialised on device " + std::to_string(g_ctxs[0]->device) + "; cannot switch to device " +
                                std::to_string(device));
        }
    }
    if (!tl_ctx) tl_ctx = g_ctxs[0];
    DG_CUDA(cudaSetDevice(tl_ctx->device));
}

Context &ctx() {
    if (!tl_ctx) ctx_init(-1);
    else cudaSetDevice(tl_ctx->device);                  // the host may have switched the thread's device (e.g. another library)
    return *tl_ctx;
}

void ctx_bind(Context *c) {
    tl_ctx = c;
    if (c) DG_CUDA(cudaSetDevice(c->device));
}
int ctx_device_count() { std::lock_guard<std::mutex> lk(g_ctx_mu); return (int)std::max<size_t>(1, g_ctxs.size()); }
Context &ctx_of(int index) { std::lock_guard<std::mutex> lk(g_ctx_mu); DG_REQUIRE(index >= 0 && index < (int)g_ctxs.size(), "no such device context"); return *g_ctxs[index]; }

void ctx_init_devices(int n) {
    DG_REQUIRE(n == 1 || n == 2 || n == 4 || n == 8, "device count must be 1, 2, 4 or 8");
    ctx_init(-1);
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    DG_REQUIRE(g_ctxs[0]->device == 0, "single-process multi-GPU mode uses devices 0 .. n-1: the primary context must be on device 0");
    DG_REQUIRE(g_ctxs[0]->world == 1 || (int)g_ctxs.size() == g_ctxs[0]->world, "a multi-process communicator is already active (dg_comm_init)");
    if ((int)g_ctxs.size() == n) return;
    DG_REQUIRE(g_ctxs.size() == 1, "the device set cannot be changed once it has been initialised");
    int count = 0;
    DG_CUDA(cudaGetDeviceCount(&count));
    DG_REQUIRE(n <= count, "not enough CUDA devices");
    Context *me = tl_ctx;
    for (int d = 1; d < n; d++) g_ctxs.push_back(build_context(d));
    for (int a = 0; a < n; a++)                          // device-resident inputs on one device are read by the others over NVLink
        for (int b2 = 0; b2 < n; b2++) {
            if (a == b2) continue;
            DG_CUDA(cudaSetDevice(a));
            cudaError_t e = cudaDeviceEnablePeerAccess(b2, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) DG_CUDA(e);
            cudaGetLastError();
        }
    if (n > 1) comm_init_all(g_ctxs);
    ctx_bind(me);
}

void set_func_smem(Context &c, const void *func, size_t bytes) {
    size_t &have = c.func_smem[func];
    if (have >= bytes) return;
    DG_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    have = bytes;
}

const fe *Context::single_table(int log_order) {
    DG_REQUIRE(log_order <= 20, "single-level table too large");
    auto it = single_tables.find(log_order);
    if (it == single_tables.end()) {
        DevBuf t;
        t.alloc(((size_t)1 << log_order) * sizeof(fe), true);
        const unsigned cnt = 1u << log_order;
        power_table_kernel<<<(cnt + 127) / 128, 128, 0, stream>>>(t.as<fe>(), host_root_of_unity(log_order), cnt); launches++;
        DG_CUDA(cudaGetLastError());
        it = single_tables.emplace(log_order, std::move(t)).first;
    }
    return it->second.as<fe>();
}

TwiddleRef Context::twiddle(int log_order, bool inverse) {
    int key = log_order * 2 + (inverse ? 1 : 0);
    auto it = twiddles.find(key);
    if (it == twiddles.end()) {
        TwiddleTable t;
        t.log_order = log_order;
        t.lo_bits = (log_order + 1) / 2;
        unsigned lo_n = 1u << t.lo_bits, hi_n = 1u << (log_order - t.lo_bits);
        fe w = host_root_of_unity(log_order);
        if (inverse) w = host_inv(w);
        fe whi = host_pow(w, lo_n);
        t.lo.alloc(lo_n * sizeof(fe), true);
        t.hi.alloc(hi_n * sizeof(fe), true);
        power_table_kernel<<<(lo_n + 127) / 128, 128, 0, stream>>>(t.lo.as<fe>(), w, lo_n); launches++;
        power_table_kernel<<<(hi_n + 127) / 128, 128, 0, stream>>>(t.hi.as<fe>(), whi, hi_n); launches++;
        DG_CUDA(cudaGetLastError());
        it = twiddles.emplace(key, std::move(t)).first;
    }
    TwiddleRef r;
    r.lo = it->second.lo.as<fe>();
    r.hi = it->second.hi.as<fe>();
    r.lo_bits = it->second.lo_bits;
    r.mask = log_order >= 32 ? 0xffffffffu : ((1u << log_order) - 1u);
    return r;
}

}  // namespace dg
