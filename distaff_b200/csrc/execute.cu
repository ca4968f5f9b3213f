// Host orchestration of dg_trace_programs / dg_execute_programs (distaff::execute, lib.rs:30-65, for many programs and inputs; dg_trace_batch
// and dg_execute_batch are the one-program case): validate each program's encoding, put every program into one set of tables and upload
// them and the inputs once, run the shape pass for every execution, and write the successful executions in waves -- one write launch
// (vm.cu) per wave for every shape in it -- into one slab per shape, which is copied to the caller's buffers (dg_trace_programs) or
// proven in place (dg_execute_programs, through prove_traces).  dg_trace_many / dg_execute_many (and dg_trace_one / dg_execute_one, their
// one-execution case) run the executions from the sponge tables: every program's table level by level, one sequential pass for every
// execution, and the segment pass (vm.cu) in the same waves, with the batch path for the programs whose hashes are inconsistent.
#include "vm.h"
#include "air.h"
#include "prover.h"
#include <algorithm>
#include <deque>
#include <functional>
#include <map>
#include <numeric>
#include <set>
#include <tuple>

namespace dg {

// One execution's inputs for pack_inputs_kernel: its values go to data[dst ..), the public inputs (n[0]) from src[src[0] ..) in order, tape
// A (n[1]) and tape B (n[2]) from src[src[1] ..) and src[src[2] ..) reversed.  The items of a launch have values and follow each other in
// data, so dst grows with the item.
struct PackItem { unsigned long long dst, src[3], n[3]; };

// Thread t writes data[t]: it finds its item (the last whose dst <= t) and the region r and reading position j of the value there, copies
// it, and for the public inputs also to pubs[8 q + j].  A value at or above M lowers bad[3 q + r] to j, so that each region keeps the first
// bad position.
__global__ void __launch_bounds__(256) pack_inputs_kernel(const PackItem *__restrict__ items, unsigned n_items, unsigned long long total,
                                                          const fe *__restrict__ src, fe *__restrict__ data, fe *__restrict__ pubs,
                                                          unsigned long long *__restrict__ bad) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    unsigned q = 0, hi = n_items;
    while (hi - q > 1) {
        const unsigned mid = (q + hi) / 2;
        if (items[mid].dst <= t) q = mid; else hi = mid;
    }
    const PackItem &it = items[q];
    unsigned long long k = t - it.dst;
    int r = 0;
    while (r < 2 && k >= it.n[r]) k -= it.n[r++];
    const unsigned long long j = r == 0 ? k : it.n[r] - 1 - k;
    const fe v = src[it.src[r] + j];
    if (v.hi == DG_M_HI && v.lo >= DG_M_LO) atomicMin(bad + 3ULL * q + r, j);
    data[t] = v;
    if (r == 0) pubs[8ULL * q + j] = v;
}

namespace {

// ---- validation of the encoding (Span::new, validate_block_list, the ctx / loop limits) ---------------------------------------------
struct Validator {
    const dg_program_t &p;
    // lists may be shared between blocks (the encoding is a DAG): each (list, depth, loops, prefix) is checked once, so validation stays
    // polynomial in the size of the encoding however often a block is referred to
    std::set<std::tuple<uint32_t, uint32_t, int, int, uint32_t>> done;
    [[noreturn]] void bad(const std::string &m) { throw Error(DG_ERR_INVALID, "invalid program encoding: " + m); }
    static fe value_of(const uint8_t v[16]) { fe x; memcpy(&x, v, 16); return x; }

    void span(uint32_t bi, const dg_block_t &b) {
        const std::string at = "span block " + std::to_string(bi) + ": ";
        if ((uint64_t)b.first + b.count > p.n_ops) bad(at + "op range out of range");
        if (b.count % 16 != 15) bad(at + "span length must be one less than a multiple of 16");
        for (uint32_t i = 0; i < b.count; i++) {
            const dg_op_hint_t &h = p.hints[b.first + i];
            if (h.kind > DG_HINT_PMPATH_START) bad(at + "unknown hint kind at op " + std::to_string(i));
            if ((h.kind == DG_HINT_RC_START || h.kind == DG_HINT_CMP_START) && (h.n < 1 || h.n > 128))
                bad(at + "RcStart / CmpStart parameter must be in 1..128 at op " + std::to_string(i));
            if (h.kind == DG_HINT_PMPATH_START && (h.n < 2 || h.n > 256)) bad(at + "PmpathStart parameter must be in 2..256 at op " + std::to_string(i));
            if (h.kind == DG_HINT_PUSH) {
                const fe v = value_of(h.value16);
                if (v.hi == DG_M_HI && v.lo >= DG_M_LO) bad(at + "push value must be smaller than the field modulus at op " + std::to_string(i));
            }
            if (p.ops[b.first + i] == 0x1f) {            // PUSH
                if (i % 8 != 0) bad(at + "PUSH must be on a step which is a multiple of 8");
                if (h.kind != DG_HINT_PUSH) bad(at + "PUSH value missing");
            }
        }
    }
    // a block list at nesting depth `depth` (the root body is 0) inside `loops` loops; `starts` the ops its first span must begin with
    void list(uint32_t first, uint32_t count, int depth, int loops, std::initializer_list<uint8_t> starts, const std::string &what) {
        uint32_t prefix = (uint32_t)starts.size();
        for (uint8_t op : starts) prefix = prefix << 8 | op;
        if (!done.insert(std::make_tuple(first, count, depth, loops, prefix)).second) return;
        if (count == 0) bad(what + ": a sequence of blocks must contain at least one block");
        if ((uint64_t)first + count > p.n_children) bad(what + ": child list out of range");
        bool was_span = false;
        for (uint32_t k = 0; k < count; k++) {
            const uint32_t bi = p.children[first + k];
            if (bi >= p.n_blocks) bad(what + ": block index " + std::to_string(bi) + " out of range");
            const dg_block_t &b = p.blocks[bi];
            if (b.kind > DG_BLOCK_LOOP) bad("block " + std::to_string(bi) + ": unknown block kind");
            const bool is_span = b.kind == DG_BLOCK_SPAN;
            if (k == 0 && !is_span) bad(what + ": a sequence of blocks must start with a Span block");
            if (k > 0 && is_span && was_span) bad(what + ": a Span block cannot be followed by another Span block");
            was_span = is_span;
            if (is_span) {
                span(bi, b);
                if (k == 0) {
                    uint32_t i = 0;
                    for (uint8_t op : starts) if (i >= b.count || p.ops[b.first + i++] != op) bad(what + ": invalid first instructions of a branch");
                }
                continue;
            }
            if (depth + 1 > 15) bad("block " + std::to_string(bi) + ": blocks nested more than 15 deep (the context stack holds 16)");
            const std::string in = "block " + std::to_string(bi);
            if (b.kind == DG_BLOCK_GROUP) list(b.first, b.count, depth + 1, loops, {}, in + " body");
            else if (b.kind == DG_BLOCK_SWITCH) {
                list(b.first, b.count, depth + 1, loops, {0x60}, in + " true branch");           // ASSERT
                list(b.alt_first, b.alt_count, depth + 1, loops, {0x6e, 0x60}, in + " false branch");   // NOT ASSERT
            } else {
                if (loops + 1 > 8) bad(in + ": loops nested more than 8 deep");
                list(b.first, b.count, depth + 1, loops + 1, {0x60}, in + " loop body");
                list(b.alt_first, b.alt_count, depth + 1, loops, {}, in + " loop skip");
            }
        }
    }
};

void validate(const dg_program_t *p) {
    DG_REQUIRE(p, "null program");
    DG_REQUIRE((p->n_ops == 0 || (p->ops && p->hints)) && p->blocks && p->n_blocks && p->children && p->n_children, "invalid program encoding: null or empty arrays");
    DG_REQUIRE(p->n_ops < (1ULL << 32), "invalid program encoding: too many ops");
    Validator{*p, {}}.list(p->root_first, p->root_count, 0, 0, {0x00}, "root body");       // a program starts with BEGIN
}

// ---- one call: the programs and inputs on the device, the shape pass, the waves ----------------------------------------------------------
using ShapeKey = std::tuple<uint32_t, uint64_t, uint32_t, uint32_t>;      // width, length, ctx depth, loop depth

// one shape's executions of a wave, in input order: [k][width][length] at regs
struct Slab {
    dg_execution_info_t shape;
    std::vector<unsigned> ids;
    fe *regs;
};

struct Executions {
    Context &c;
    const ExecutionCall &x;
    DevBuf d_ops, d_hints, d_blocks, d_children, d_programs, d_in, d_data, d_res, d_tapes, d_off, d_cap, d_ids, d_outs, d_pad_ids;
    VmLaunch L;
    std::vector<VmInput> in;                      // what setup() packed; zero but the program for an execution the inputs failed
    std::vector<fe> pub;                          // 8 per execution: its public inputs (in[i].n_pub of them), for the prover
    std::vector<VmResult> res;
    std::vector<int> status;
    std::vector<std::string> messages;
    std::vector<unsigned long long> off, cap;
    dg_execution_stats_t stats;
    cudaEvent_t ev[2] = {nullptr, nullptr};

    Executions(Context &ctx_, const ExecutionCall &call)
        : c(ctx_), x(call), in(call.count), pub(8 * (size_t)call.count), res(call.count), status(call.count, DG_OK), messages(call.count),
          off(call.count, 0), cap(2 * (size_t)call.count, 0) {
        memset(&stats, 0, sizeof stats);
        DG_CUDA(cudaEventCreate(&ev[0]));
        DG_CUDA(cudaEventCreate(&ev[1]));
    }
    ~Executions() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }

    void fail(uint32_t i, int code, const std::string &m) { status[i] = code; messages[i] = m; }

    template <typename T> void upload(DevBuf &d, const std::vector<T> &v) {
        d.alloc(std::max<size_t>(v.size(), 1) * sizeof(T));
        if (!v.empty()) DG_CUDA(cudaMemcpyAsync(d.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }
    // device milliseconds of the launches f enqueues
    template <typename F> float timed(F &&f) {
        DG_CUDA(cudaEventRecord(ev[0], c.stream));
        f();
        DG_CUDA(cudaEventRecord(ev[1], c.stream));
        DG_CUDA(cudaEventSynchronize(ev[1]));
        float ms = 0;
        DG_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
        return ms;
    }

    void setup() {
        memset(&L, 0, sizeof L);
        // every program's ops, hints, blocks and child lists appended to one table each; a span's range is rebased by the ops before it,
        // the child-list ranges by the child entries before it, and the block indices of the child lists by the blocks before it
        std::vector<uint8_t> ops;
        std::vector<VmHint> hints;
        std::vector<VmBlock> blocks;
        std::vector<unsigned> children;
        std::vector<VmProgram> programs(x.n_programs);
        for (uint32_t p = 0; p < x.n_programs; p++) {
            const dg_program_t &g = x.programs[p];
            const unsigned op0 = (unsigned)ops.size(), b0 = (unsigned)blocks.size(), c0 = (unsigned)children.size();
            ops.insert(ops.end(), g.ops, g.ops + g.n_ops);
            for (uint64_t i = 0; i < g.n_ops; i++) {
                VmHint h;
                h.kind = g.hints[i].kind;
                h.n = g.hints[i].n;
                memcpy(&h.value, g.hints[i].value16, 16);
                hints.push_back(h);
            }
            for (uint32_t i = 0; i < g.n_blocks; i++) {
                const dg_block_t &b = g.blocks[i];
                VmBlock v;
                memset(&v, 0, sizeof v);
                const bool span = b.kind == DG_BLOCK_SPAN;
                v.kind = b.kind; v.count = b.count; v.alt_count = b.alt_count;
                v.first = b.first + (span ? op0 : c0);
                v.alt_first = span ? b.alt_first : b.alt_first + c0;
                memcpy(&v.hash[0], b.hash0, 16); memcpy(&v.hash[1], b.hash1, 16); memcpy(&v.hash[2], b.hash2, 16);
                blocks.push_back(v);
            }
            for (uint32_t i = 0; i < g.n_children; i++) children.push_back(g.children[i] + b0);
            programs[p].root_first = g.root_first + c0;
            programs[p].root_count = g.root_count;
            memcpy(&programs[p].hash[0], g.hash32, 16); memcpy(&programs[p].hash[1], g.hash32 + 16, 16);
        }
        upload(d_ops, ops); upload(d_hints, hints); upload(d_blocks, blocks); upload(d_children, children); upload(d_programs, programs);
        pack_inputs();
        d_res.alloc((size_t)x.count * sizeof(VmResult));
        DG_CUDA(cudaMemsetAsync(d_res.p, 0, (size_t)x.count * sizeof(VmResult), c.stream));
        L.ops = d_ops.as<uint8_t>(); L.hints = d_hints.as<VmHint>(); L.blocks = d_blocks.as<VmBlock>(); L.children = d_children.as<unsigned>();
        L.programs = d_programs.as<VmProgram>();
        L.in = d_in.as<VmInput>(); L.data = d_data.as<fe>();
        L.res = d_res.as<VmResult>();
        L.max_steps = x.max_steps;
        for (uint32_t i = 0; i < x.count; i++) { cap[2 * i] = in[i].n_a; cap[2 * i + 1] = in[i].n_b; }
    }

    // The inputs, packed for the VM into d_data: per execution its public inputs, then both tapes reversed (the next value to read is the
    // last one, as in the host VM), executions one after the other; d_in describes them.  The counts are checked here; the values by one
    // pack_inputs_kernel launch over every value of the call, from one source buffer: the caller's device buffer (device inputs), or the
    // host inputs gathered into one upload.  Only the first bad index of each region and the public inputs come back.
    void pack_inputs() {
        const dg_device_inputs_t *dv = x.device_inputs;
        std::vector<PackItem> items;
        std::vector<unsigned> item_of;            // the execution of each item
        std::vector<fe> staged;                   // host inputs: the values of every item, in reading order
        unsigned long long total = 0;
        for (uint32_t i = 0; i < x.count; i++) {
            memset(&in[i], 0, sizeof(VmInput));
            in[i].program = x.program_of[i];
            const uint64_t n[3] = {dv ? dv->n_public[i] : x.inputs[i].n_public, dv ? dv->n_secret_a[i] : x.inputs[i].n_secret_a,
                                   dv ? dv->n_secret_b[i] : x.inputs[i].n_secret_b};
            if (n[0] > 8) { fail(i, DG_ERR_EXECUTION, "expected no more than 8 public inputs"); continue; }      // lib.rs:32
            if (n[1] < n[2]) { fail(i, DG_ERR_EXECUTION, "tape A cannot be shorter than tape B"); continue; }   // inputs.rs:17
            in[i].n_pub = (unsigned)n[0]; in[i].pub = total;
            in[i].n_a = n[1]; in[i].a = total + n[0];
            in[i].n_b = n[2]; in[i].b = total + n[0] + n[1];
            if (n[0] + n[1] + n[2] == 0) continue;
            PackItem it{total, {0, 0, 0}, {n[0], n[1], n[2]}};
            if (dv) {
                it.src[0] = dv->public_first[i]; it.src[1] = dv->secret_a_first[i]; it.src[2] = dv->secret_b_first[i];
            } else {
                const uint8_t *p[3] = {x.inputs[i].public16, x.inputs[i].secret_a16, x.inputs[i].secret_b16};
                for (int r = 0; r < 3; r++) {
                    it.src[r] = staged.size();
                    staged.resize(staged.size() + n[r]);
                    if (n[r]) memcpy(&staged[it.src[r]], p[r], 16 * n[r]);
                }
            }
            items.push_back(it);
            item_of.push_back(i);
            total += n[0] + n[1] + n[2];
        }
        d_data.alloc(std::max<unsigned long long>(total, 1) * sizeof(fe));
        if (!items.empty()) {
            const fe *src = (const fe *)(dv ? dv->d_values : nullptr);
            DevBuf d_staged, d_items, d_checks(items.size() * (8 * sizeof(fe) + 3 * sizeof(unsigned long long)));
            if (dv) {
                require_device_memory(c, src, "device inputs: d_values");
            } else {
                upload(d_staged, staged);
                src = d_staged.as<fe>();
            }
            upload(d_items, items);
            fe *pubs = d_checks.as<fe>();         // 8 per item, then 3 first bad indexes per item (all ones: none)
            unsigned long long *bad = (unsigned long long *)(pubs + 8 * items.size());
            DG_CUDA(cudaMemsetAsync(bad, 0xff, items.size() * 3 * sizeof(unsigned long long), c.stream));
            pack_inputs_kernel<<<(unsigned)((total + 255) / 256), 256, 0, c.stream>>>(d_items.as<PackItem>(), (unsigned)items.size(), total, src,
                                                                                         d_data.as<fe>(), pubs, bad);
            c.launches++;
            DG_CUDA(cudaGetLastError());
            std::vector<uint8_t> checks(d_checks.bytes);
            DG_CUDA(cudaMemcpyAsync(checks.data(), d_checks.p, checks.size(), cudaMemcpyDeviceToHost, c.stream));
            DG_CUDA(cudaStreamSynchronize(c.stream));
            const fe *got_pub = (const fe *)checks.data();
            const unsigned long long *got_bad = (const unsigned long long *)(got_pub + 8 * items.size());
            // the VM's arithmetic assumes canonical operands: a value in [M, 2^128) fails its execution (the reference does not check)
            static const char *what[3] = {"public input", "tape A value", "tape B value"};
            for (size_t q = 0; q < items.size(); q++) {
                const unsigned i = item_of[q];
                for (int r = 0; r < 3; r++)
                    if (got_bad[3 * q + r] != ~0ULL) {
                        fail(i, DG_ERR_EXECUTION, std::string(what[r]) + " " + std::to_string(got_bad[3 * q + r]) + " is not a field element");
                        memset(&in[i], 0, sizeof(VmInput));
                        in[i].program = x.program_of[i];
                        break;
                    }
                if (status[i] == DG_OK) std::copy(got_pub + 8 * q, got_pub + 8 * q + in[i].n_pub, pub.begin() + 8 * (size_t)i);
            }
        }
        upload(d_in, in);
    }

    // tape scratch for `ids`: capacity cap[2e], cap[2e + 1] each
    void place_tapes(const std::vector<unsigned> &ids) {
        unsigned long long total = 0;
        for (unsigned e : ids) { off[e] = total; total += cap[2 * e] + cap[2 * e + 1]; }
        d_tapes.alloc(std::max<unsigned long long>(total, 1) * 16);
        upload(d_off, off); upload(d_cap, cap);
        L.tapes = d_tapes.as<fe>(); L.tape_off = d_off.as<unsigned long long>(); L.cap = d_cap.as<unsigned long long>();
    }
    // the launch order of `ids`: by program, each program's executions from a multiple of 32 on and in input order, so that no warp
    // mixes two programs' instruction streams; the lanes after a program's last execution are idle.  Returns the lanes.
    unsigned launch_ids(std::vector<unsigned> ids) {
        std::stable_sort(ids.begin(), ids.end(), [&](unsigned a, unsigned b) { return x.program_of[a] < x.program_of[b]; });
        std::vector<unsigned> lanes;
        for (size_t i = 0; i < ids.size(); i++) {
            if (i > 0 && x.program_of[ids[i]] != x.program_of[ids[i - 1]]) lanes.resize((lanes.size() + 31) / 32 * 32, VM_NO_EXECUTION);
            lanes.push_back(ids[i]);
        }
        lanes.resize((lanes.size() + 31) / 32 * 32, VM_NO_EXECUTION);
        upload(d_ids, lanes);
        L.ids = d_ids.as<unsigned>();
        L.count = (unsigned)lanes.size();
        return L.count;
    }
    void download_results() {
        DG_CUDA(cudaMemcpyAsync(res.data(), d_res.p, (size_t)x.count * sizeof(VmResult), cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }

    // the shape pass of the executions `ids` (those the inputs did not fail); an execution whose hints outgrow its tape scratch (256
    // elements beyond its inputs at first; what the assembler's macros need) runs again with 16 times more
    void shapes(const std::vector<unsigned> &ids) {
        std::vector<unsigned> pending;
        for (unsigned i : ids) if (status[i] == DG_OK) pending.push_back(i);
        for (unsigned long long extra = 256; !pending.empty(); extra *= 16) {
            for (unsigned e : pending) { cap[2 * e] = in[e].n_a + extra; cap[2 * e + 1] = in[e].n_b + extra; }
            place_tapes(pending);
            launch_ids(pending);
            stats.shape_ms += timed([&] { vm_shape_pass(c, L); });
            stats.shape_launches++;
            download_results();
            std::vector<unsigned> again;
            for (unsigned e : pending) if (res[e].code == VM_TAPE_SCRATCH) again.push_back(e);
            pending.swap(again);
        }
        for (unsigned i : ids)
            if (status[i] == DG_OK && res[i].code != VM_OK) fail(i, DG_ERR_EXECUTION, vm_message(res[i].code, res[i].fail_step, x.max_steps));
        // the write pass runs with the tape scratch each execution needed
        std::vector<unsigned> ok;
        for (unsigned i : ids)
            if (status[i] == DG_OK) { ok.push_back(i); cap[2 * i] = res[i].peak_a; cap[2 * i + 1] = res[i].peak_b; }
        place_tapes(ok);
    }

    dg_execution_info_t info(uint32_t i) const {
        dg_execution_info_t v;
        memset(&v, 0, sizeof v);
        const VmResult &r = res[i];
        v.ctx_depth = r.ctx_cols - 1; v.loop_depth = r.loop_cols; v.stack_depth = r.max_depth;
        v.width = TraceShape(v.ctx_depth, v.loop_depth, v.stack_depth).w;
        v.steps = r.steps;
        v.length = 16;
        while (v.length <= r.steps) v.length *= 2;
        return v;
    }
    static ShapeKey key(const dg_execution_info_t &v) { return std::make_tuple(v.width, v.length, v.ctx_depth, v.loop_depth); }
    // the successful executions of `ids` by shape, shapes in order and input order inside a shape
    std::vector<unsigned> shape_order(const std::vector<unsigned> &ids) const {
        std::map<ShapeKey, std::vector<unsigned>> g;
        for (unsigned i : ids) if (status[i] == DG_OK) g[key(info(i))].push_back(i);
        std::vector<unsigned> order;
        for (auto &kv : g) order.insert(order.end(), kv.second.begin(), kv.second.end());
        return order;
    }

    // The executions `order` (in shape order) in waves: a wave is a run of them, given one slab per shape in a fresh register buffer and
    // handed to write(wave, slabs, last) while its traces are on the device; waves follow each other, so the executions reach write in
    // shape order, input order inside a shape.  A wave's traces take at most half of the device memory the library may use, and with
    // `opts` (the options of every execution) they leave room beside them for one proof of the wave's largest shape and extension factor.
    // $DG_BATCH_GROUP caps its executions.  L.out / L.outs and d_pad_ids (the wave, in slab order) are set for the wave.
    template <typename F> void cut_waves(const std::vector<unsigned> &order, const dg_options_t *opts, uint8_t *const *registers_out, F &&write) {
        const size_t most = (size_t)batch_group_cap(65535);         // one padding launch holds 65535 executions
        std::map<std::pair<ShapeKey, uint32_t>, size_t> room;      // bytes one proof of a shape and extension factor needs beside the traces
        std::vector<VmOut> outs(x.count);
        for (size_t first = 0; first < order.size();) {
            size_t avail = memory_budget(c, Budget::FREE, 0);
            if (c.mem_limit) avail = avail > c.arena.cap ? avail - c.arena.cap : 0;      // proofs may keep the arena beside the traces
            size_t end = first, bytes = 0, need = 0;
            while (end < order.size() && end - first < most) {
                const dg_execution_info_t s = info(order[end]);
                const size_t per = (size_t)s.width * s.length * 16;
                size_t r = 0;
                if (opts) {
                    const uint32_t b = opts[order[end]].extension_factor;
                    auto it = room.find({key(s), b});
                    if (it == room.end()) {
                        const ProvePlan P = plan_prove(c, s.width, s.length, b, 1);
                        it = room.emplace(std::make_pair(key(s), b), P.per_proof + P.fixed - memory_held_outside_arena(c)).first;
                    }
                    r = it->second;
                }
                if (end > first && (bytes + per > avail / 2 || bytes + per + std::max(need, r) > avail)) break;
                if (registers_out) DG_REQUIRE(registers_out[order[end]], "null register buffer of execution " + std::to_string(order[end]));
                if (!opts && c.mem_limit && per > avail)
                    throw Error(DG_ERR_INVALID, "a trace of " + std::to_string(s.width) + " x " + std::to_string(s.length) + " needs " +
                                                    std::to_string(per) + " bytes of device memory beyond what the memory limit leaves");
                bytes += per;
                need = std::max(need, r);
                end++;
            }
            const std::vector<unsigned> wave(order.begin() + first, order.begin() + end);
            DevBuf regs(bytes);
            std::vector<Slab> slabs;
            size_t at = 0;
            for (unsigned e : wave) {
                const dg_execution_info_t s = info(e);
                if (slabs.empty() || key(slabs.back().shape) != key(s)) slabs.push_back(Slab{s, {}, regs.as<fe>() + at});
                slabs.back().ids.push_back(e);
                outs[e] = VmOut{at, s.length, s.width, s.ctx_depth, s.loop_depth, s.stack_depth};
                at += (size_t)s.width * s.length;
            }
            upload(d_outs, outs);
            upload(d_pad_ids, wave);
            L.out = regs.as<fe>();
            L.outs = d_outs.as<VmOut>();
            write(wave, slabs, end == order.size());
            first = end;
        }
    }
    // the padding rows of a wave's slabs (after its rows are written)
    void pad(const std::vector<Slab> &slabs) {
        size_t q = 0;
        for (const Slab &s : slabs) {
            vm_pad_rows(c, s.regs, L.res, d_pad_ids.as<unsigned>() + q, (unsigned)s.ids.size(), s.shape.width, s.shape.length);
            q += s.ids.size();
        }
    }

    // The write pass of the successful executions of `ids`, in waves (cut_waves): one launch per wave for every shape in it, then
    // done(slabs).
    template <typename F> void write_waves(const std::vector<unsigned> &ids, const dg_options_t *opts, uint8_t *const *registers_out, F &&done) {
        cut_waves(shape_order(ids), opts, registers_out, [&](const std::vector<unsigned> &wave, const std::vector<Slab> &slabs, bool) {
            stats.lanes += launch_ids(wave);
            stats.write_ms += timed([&] {
                vm_write_pass(c, L);
                pad(slabs);
            });
            stats.write_launches++;
            stats.waves++;
            download_results();
            for (unsigned e : wave)
                if (res[e].code != VM_OK) fail(e, DG_ERR_EXECUTION, vm_message(res[e].code, res[e].fail_step, x.max_steps));
            done(slabs);
        });
    }
};

void check_one_gpu(Context &c) {
    DG_REQUIRE(c.world == 1 && ctx_device_count() == 1, "batched execution runs on one GPU: the library was initialised for several (dg_init_devices / dg_comm_init)");
}

// the registers of a wave's successful executions to the caller's buffers
void copy_slabs(Context &c, const Executions &X, const std::vector<Slab> &slabs, uint8_t *const *registers_out) {
    for (const Slab &s : slabs) {
        const size_t per = (size_t)s.shape.width * s.shape.length * 16;
        for (size_t q = 0; q < s.ids.size(); q++)
            if (X.status[s.ids[q]] == DG_OK) {
                DG_REQUIRE(registers_out[s.ids[q]], "null register buffer of execution " + std::to_string(s.ids[q]));
                DG_CUDA(cudaMemcpyAsync(registers_out[s.ids[q]], (const uint8_t *)s.regs + q * per, per, cudaMemcpyDeviceToHost, c.stream));
            }
    }
    DG_CUDA(cudaStreamSynchronize(c.stream));
}

// Each shape's successful traces of a wave proven together where they were written (prove_traces), each with its execution's options
// (opts[i]): RNG callbacks shape by shape, inside a shape extension factor by extension factor (in order of first appearance) and in
// input order inside those.  Executions the rows failed are left out: the traces after them move down over them, and their outputs (8 per
// execution in outs) are zeroed, as those of executions the VM failed earlier.  Adds the prove groups to `groups`.
void prove_slabs(Context &c, Executions &X, const std::vector<Slab> &slabs, const uint32_t *num_outputs, const dg_options_t *opts,
                 std::vector<fe> &outs, Proof **proofs_out, dg_prove_stats_t *stats, uint32_t &groups) {
    const ExecutionCall &x = X.x;
    for (const Slab &s : slabs) {
        const size_t per = (size_t)s.shape.width * s.shape.length;
        std::vector<unsigned> ok;
        for (size_t q = 0; q < s.ids.size(); q++) {
            if (X.status[s.ids[q]] != DG_OK) {
                std::fill(outs.begin() + (size_t)s.ids[q] * 8, outs.begin() + (size_t)s.ids[q] * 8 + 8, fe_make(0, 0));
                continue;
            }
            if (ok.size() != q)
                DG_CUDA(cudaMemcpyAsync(s.regs + ok.size() * per, s.regs + q * per, per * 16, cudaMemcpyDeviceToDevice, c.stream));
            ok.push_back(s.ids[q]);
        }
        if (ok.empty()) continue;
        const uint32_t k = (uint32_t)ok.size();
        std::vector<const uint8_t *> in16(k), out16(k);
        std::vector<uint32_t> n_in(k), n_out(k);
        std::vector<dg_options_t> opt(k);
        for (uint32_t q = 0; q < k; q++) {
            in16[q] = (const uint8_t *)&X.pub[(size_t)ok[q] * 8]; n_in[q] = X.in[ok[q]].n_pub;
            out16[q] = (const uint8_t *)&outs[(size_t)ok[q] * 8]; n_out[q] = num_outputs[ok[q]];
            opt[q] = opts[ok[q]];
        }
        std::vector<Proof *> proofs(k, nullptr);
        std::vector<int> st(k, DG_OK);
        std::vector<std::string> msg;
        dg_prove_stats_t gs;
        memset(&gs, 0, sizeof gs);
        uint32_t g = 0;
        prove_traces(c, one_shape_traces(s.regs, k, s.shape.width, s.shape.length, s.shape.ctx_depth, s.shape.loop_depth), in16.data(),
                     n_in.data(), out16.data(), n_out.data(), opt, true, proofs.data(), st.data(), msg, &gs, &g);
        for (uint32_t q = 0; q < k; q++) {
            proofs_out[ok[q]] = proofs[q];
            if (st[q] != DG_OK) X.fail(ok[q], st[q], msg[q]);
        }
        groups += g;
        if (stats) add_stats(stats, gs);
    }
}

// The batch path for the executions `ids`: the shape pass, then (with `write`) the write pass in waves, the registers copied to
// registers_out when it is given.  Without `write` the failures that need the sponge (program hash, loop image) go unreported.  With
// `precheck` every buffer of an execution the shape pass let through must be there before the write pass; without, only those of the
// executions the write pass lets through (a caller that learned of a write-pass failure from an earlier call may pass NULL for it).
void batch_trace(Context &c, Executions &X, const std::vector<unsigned> &ids, uint8_t *const *registers_out, bool write, bool precheck) {
    X.shapes(ids);
    if (write)
        X.write_waves(ids, nullptr, precheck ? registers_out : nullptr, [&](const std::vector<Slab> &slabs) {
            if (registers_out) copy_slabs(c, X, slabs, registers_out);
        });
}

// The batch path for the executions `ids`, proven: the shape pass, outputs from the final stacks, the write pass in waves and each wave
// proven in place
void batch_execute(Context &c, Executions &X, const std::vector<unsigned> &ids, const uint32_t *num_outputs, const dg_options_t *opts,
                   std::vector<fe> &outs, Proof **proofs_out, dg_prove_stats_t *stats) {
    X.shapes(ids);
    for (unsigned i : ids)
        if (X.status[i] == DG_OK) for (uint32_t j = 0; j < num_outputs[i]; j++) outs[(size_t)i * 8 + j] = X.res[i].top[j];
    X.write_waves(ids, opts, nullptr, [&](const std::vector<Slab> &slabs) {
        prove_slabs(c, X, slabs, num_outputs, opts, outs, proofs_out, stats, X.stats.prove_groups);
    });
}

// the per-execution results of a call: info (may be null; zero for a failed execution), status, messages and the VM passes' stats
void finish(const Executions &X, dg_execution_info_t *info, int *status, std::vector<std::string> &messages, dg_execution_stats_t *vm_stats) {
    for (uint32_t i = 0; i < X.x.count; i++) {
        if (info) {
            if (X.status[i] == DG_OK) info[i] = X.info(i);
            else memset(&info[i], 0, sizeof info[i]);
        }
        status[i] = X.status[i];
    }
    messages = X.messages;
    if (vm_stats) *vm_stats = X.stats;
}

// The frame of an execute call around run(outs): proofs_out and stats start null / zero, the proofs of the waves done so far are freed
// when a later wave fails the call, and the 8 output elements per execution that run leaves in outs go to outputs16 (when given).
template <typename F> void proven(uint32_t count, Proof **proofs_out, uint8_t *outputs16, dg_prove_stats_t *stats, F &&run) {
    for (uint32_t i = 0; i < count; i++) proofs_out[i] = nullptr;
    if (stats) memset(stats, 0, sizeof *stats);
    try {
        std::vector<fe> outs((size_t)count * 8, fe_make(0, 0));
        run(outs);
        if (outputs16) memcpy(outputs16, outs.data(), outs.size() * 16);
    } catch (...) {
        for (uint32_t i = 0; i < count; i++) { delete proofs_out[i]; proofs_out[i] = nullptr; }
        throw;
    }
}

// ---- executions from the sponge tables --------------------------------------------------------------------------------------------------
// The chains of a program (vm.h): every block list reachable from the root once (lists may be shared: a list is its child range) and, per
// loop, the chain after BREAK.  A chain's level is one above every chain it reads -- a list reads its group, switch and loop children's
// closing states, the break chains of its loops and its loops' skips; a break chain reads the body's last state -- so one launch per
// level computes them in order.  Nothing is hashed here: the host only counts each chain's entries and lays the table out by level.
struct ChainPlan {
    std::vector<VmChainRef> refs;                 // per block
    std::vector<VmChainItem> items;               // level by level
    std::vector<size_t> level_start;              // the items of level l (from 1) are [level_start[l - 1], level_start[l])
    unsigned long long root = 0, entries = 0, rounds = 0;
};

ChainPlan plan_chains(const dg_program_t &p) {
    struct List { uint32_t first, count; unsigned level; unsigned long long len, ends; };      // ends: child end_block entries
    std::map<std::pair<uint32_t, uint32_t>, unsigned> ids;
    std::vector<List> lists;
    std::vector<unsigned> brk_level(p.n_blocks, 0);
    std::function<unsigned(uint32_t, uint32_t)> list = [&](uint32_t first, uint32_t count) -> unsigned {
        const auto it = ids.find({first, count});
        if (it != ids.end()) return it->second;
        unsigned level = 0;
        unsigned long long len = 1, ends = 0;                                  // the closing NOOP
        for (uint32_t k = 0; k < count; k++) {
            const uint32_t bi = p.children[first + k];
            const dg_block_t &b = p.blocks[bi];
            if (b.kind == DG_BLOCK_SPAN) { len += b.count + (k > 0); continue; }
            len += 15;                                                         // end_block and 14 NOOPs
            ends++;
            const unsigned main = lists[list(b.first, b.count)].level;
            unsigned m = main;
            if (b.kind != DG_BLOCK_GROUP) m = std::max(m, lists[list(b.alt_first, b.alt_count)].level);
            if (b.kind == DG_BLOCK_LOOP) { brk_level[bi] = main + 1; m = std::max(m, main + 1); }
            level = std::max(level, m);
        }
        lists.push_back(List{first, count, level + 1, len, ends});
        return ids[{first, count}] = (unsigned)lists.size() - 1;
    };
    const unsigned root = list(p.root_first, p.root_count);
    unsigned levels = 0;
    for (const List &l : lists) levels = std::max(levels, l.level);
    ChainPlan P;
    P.refs.assign(p.n_blocks, VmChainRef{0, 0, 0, 0, 0, 0});
    std::vector<unsigned long long> out(lists.size());
    P.level_start.push_back(0);
    for (unsigned level = 1; level <= levels; level++) {
        for (size_t i = 0; i < lists.size(); i++) {
            const List &l = lists[i];
            if (l.level != level) continue;
            out[i] = P.entries;
            const bool tail = i == root;
            P.items.push_back(VmChainItem{VM_CHAIN_LIST, l.first, l.count, 0, tail ? 1u : 0u, 0, P.entries});
            P.entries += l.len + (tail ? 15 : 0);
            P.rounds += l.len - l.ends + (tail ? 14 : 0);
        }
        for (uint32_t bi = 0; bi < p.n_blocks; bi++) {
            if (brk_level[bi] != level) continue;
            const dg_block_t &b = p.blocks[bi];
            const unsigned long long len = p.blocks[p.children[b.alt_first]].count + 1;    // the skip's first span and a NOOP
            P.refs[bi].brk = P.entries;
            P.refs[bi].brk_close = P.entries + len - 1;
            P.items.push_back(VmChainItem{VM_CHAIN_BREAK, 0, 0, bi, 0, 0, P.entries});
            P.entries += len;
            P.rounds += len;
        }
        P.level_start.push_back(P.items.size());
    }
    for (uint32_t bi = 0; bi < p.n_blocks; bi++) {
        const dg_block_t &b = p.blocks[bi];
        if (b.kind == DG_BLOCK_SPAN) continue;
        const auto at = [&](uint32_t first, uint32_t count, unsigned long long &start, unsigned long long &close) {
            const auto it = ids.find({first, count});
            if (it == ids.end()) return;                                     // a block the root does not reach
            start = out[it->second];
            close = start + lists[it->second].len - 1;
        };
        at(b.first, b.count, P.refs[bi].main, P.refs[bi].main_close);
        if (b.kind != DG_BLOCK_GROUP) at(b.alt_first, b.alt_count, P.refs[bi].alt, P.refs[bi].alt_close);
    }
    P.root = out[root];
    return P;
}

// S when the caller leaves it to the library: at most 4096 segments for an execution of max_steps steps (DESIGN.md section 7i measures it
// against the executions a call holds)
uint64_t default_segment_steps(uint64_t max_steps) {
    uint64_t s = 16;
    while (s < (1ULL << 40) && s * 4096 < max_steps) s *= 2;
    return s;
}

// The executions of a call from the sponge tables.  tables() computes every program's chains in one table (one launch per level for all
// programs) and sorts the executions the inputs did not fail into `run` (their program's hashes are consistent) and `fallback` (they are
// not: the batch path runs them, in X, so results are identical either way).  sequential() runs every execution of `run` in one launch,
// one warp each (again, for the executions that outgrew their tape scratch, read log or checkpoint buffer, with the room they reported),
// and waves() writes the rows of its successful executions in waves, one segment launch per wave for all their checkpoints.  The stats
// reach `out` (may be null) in the destructor, so also when a pass throws: dg_trace_one reports a failed call's.
struct TabledExecutions {
    Context &c;
    Executions X;
    uint64_t S;
    dg_many_stats_t st;
    dg_many_stats_t *out;
    std::vector<char> tabled;                     // per program
    std::vector<unsigned> run, fallback;          // in input order
    std::vector<VmTabled> T;                      // per execution
    std::vector<VmSequential> seq;                // per execution
    std::deque<DevBuf> logs;                      // the read logs and checkpoints of each sequential launch
    DevBuf d_refs, d_tab, d_T, d_seq, d_codes, d_execs, d_first;
    VmTables G;

    TabledExecutions(Context &ctx_, const ExecutionCall &x, uint64_t segment_steps, dg_many_stats_t *stats)
        : c(ctx_), X(ctx_, x), S(segment_steps ? segment_steps : default_segment_steps(x.max_steps)), out(stats), tabled(x.n_programs, 0),
          T(x.count), seq(x.count) {
        memset(&st, 0, sizeof st);
        memset(T.data(), 0, T.size() * sizeof(VmTabled));
        memset(seq.data(), 0, seq.size() * sizeof(VmSequential));
        st.segment_steps = S;
        G = VmTables{nullptr, nullptr, S};
        X.setup();
    }
    ~TabledExecutions() { if (out) *out = st; }

    // the chains of every program with an execution to run, rebased as X.setup() rebased the programs: child ranges by the child entries
    // before the program, block indices by the blocks before it, table indices by the entries before it
    void tables() {
        const ExecutionCall &x = X.x;
        std::vector<char> used(x.n_programs, 0);
        for (uint32_t i = 0; i < x.count; i++) if (X.status[i] == DG_OK) used[x.program_of[i]] = 1;
        std::vector<VmChainRef> refs;
        std::vector<std::vector<VmChainItem>> levels;
        std::vector<unsigned long long> root(x.n_programs, 0);
        unsigned long long entries = 0;
        unsigned b0 = 0, c0 = 0;
        for (uint32_t p = 0; p < x.n_programs; p++) {
            const dg_program_t &g = x.programs[p];
            refs.resize(b0 + g.n_blocks, VmChainRef{0, 0, 0, 0, 0, 0});
            if (used[p]) {
                const ChainPlan P = plan_chains(g);
                for (uint32_t bi = 0; bi < g.n_blocks; bi++) {
                    const VmChainRef &r = P.refs[bi];
                    refs[b0 + bi] = VmChainRef{r.main + entries, r.alt + entries, r.brk + entries, r.main_close + entries,
                                               r.alt_close + entries, r.brk_close + entries};
                }
                if (levels.size() + 1 < P.level_start.size()) levels.resize(P.level_start.size() - 1);
                for (size_t l = 0; l + 1 < P.level_start.size(); l++)
                    for (size_t k = P.level_start[l]; k < P.level_start[l + 1]; k++) {
                        VmChainItem it = P.items[k];
                        if (it.kind == VM_CHAIN_LIST) it.first += c0; else it.block += b0;
                        it.program = p;
                        it.out += entries;
                        levels[l].push_back(it);
                    }
                root[p] = P.root + entries;
                entries += P.entries;
                st.table_rounds += P.rounds;
            }
            b0 += g.n_blocks;
            c0 += g.n_children;
        }
        std::vector<VmChainItem> items;
        std::vector<size_t> level_start{0};
        for (const auto &l : levels) { items.insert(items.end(), l.begin(), l.end()); level_start.push_back(items.size()); }
        DevBuf d_items, d_bad;
        X.upload(d_refs, refs);
        X.upload(d_items, items);
        d_tab.alloc(std::max<unsigned long long>(entries, 1) * sizeof(VmSponge));
        std::vector<unsigned> bad(x.n_programs, 0);
        X.upload(d_bad, bad);
        st.table_ms = X.timed([&] {
            for (size_t l = 0; l + 1 < level_start.size(); l++)
                vm_table_level(c, X.L, d_items.as<VmChainItem>() + level_start[l], (unsigned)(level_start[l + 1] - level_start[l]),
                               d_refs.as<VmChainRef>(), d_tab.as<VmSponge>(), d_bad.as<unsigned>());
        });
        st.table_levels = (uint32_t)levels.size();
        st.table_entries = entries;
        DG_CUDA(cudaMemcpy(bad.data(), d_bad.p, bad.size() * sizeof(unsigned), cudaMemcpyDeviceToHost));
        for (uint32_t p = 0; p < x.n_programs; p++) {
            tabled[p] = used[p] && !bad[p];
            st.tabled_programs += tabled[p];
            st.fallback_programs += used[p] && bad[p];
        }
        G.tab = d_tab.as<VmSponge>();
        G.chains = d_refs.as<VmChainRef>();
        for (uint32_t i = 0; i < x.count; i++) {
            if (X.status[i] != DG_OK) continue;
            (tabled[x.program_of[i]] ? run : fallback).push_back(i);
            T[i].root = root[x.program_of[i]];
        }
    }

    void sequential() {
        if (run.empty()) return;
        const ExecutionCall &x = X.x;
        const size_t cpb = vm_checkpoint_bytes();
        // the first logs and checkpoint buffers take at most a quarter of the memory the library may use, shared equally
        const size_t share = memory_budget(c, Budget::FREE, 0) / 4 / run.size();
        const unsigned long long cp0 = std::max<unsigned long long>(2, std::min<unsigned long long>(std::min<uint64_t>(x.max_steps / S + 2, 4096), share / 2 / cpb));
        const unsigned long long log0 = std::max<unsigned long long>(1, std::min<unsigned long long>(std::min<uint64_t>(2 * x.max_steps, 1ULL << 21), share / 2 / 16));
        std::vector<unsigned long long> extra(x.count, 256), log_cap(x.count, log0), cp_cap(x.count, cp0);
        X.upload(d_seq, seq);
        std::vector<unsigned> pending = run;
        while (!pending.empty()) {
            for (unsigned e : pending) { X.cap[2 * e] = X.in[e].n_a + extra[e]; X.cap[2 * e + 1] = X.in[e].n_b + extra[e]; }
            X.place_tapes(pending);
            // one warp per execution: the executions of a warp would take different paths through the interpreter (DESIGN.md section 7i)
            std::vector<unsigned> lanes;
            for (unsigned e : pending) { lanes.push_back(e); lanes.resize(lanes.size() + 31, VM_NO_EXECUTION); }
            X.upload(X.d_ids, lanes);
            X.L.ids = X.d_ids.as<unsigned>();
            X.L.count = (unsigned)lanes.size();
            size_t log_n = 0, cp_n = 0;
            for (unsigned e : pending) { log_n += log_cap[e]; cp_n += cp_cap[e]; }
            logs.emplace_back(std::max<size_t>(log_n, 1) * sizeof(fe));
            fe *log = logs.back().as<fe>();
            logs.emplace_back(cp_n * cpb);
            uint8_t *cp = (uint8_t *)logs.back().p;
            for (unsigned e : pending) {
                T[e].log = log; T[e].log_cap = log_cap[e]; log += log_cap[e];
                T[e].checkpoints = cp; T[e].cp_cap = cp_cap[e]; cp += cp_cap[e] * cpb;
            }
            X.upload(d_T, T);
            st.sequential_ms += X.timed([&] { vm_sequential_pass(c, X.L, G, d_T.as<VmTabled>(), d_seq.as<VmSequential>()); });
            st.sequential_launches++;
            X.download_results();
            DG_CUDA(cudaMemcpy(seq.data(), d_seq.p, seq.size() * sizeof(VmSequential), cudaMemcpyDeviceToHost));
            std::vector<unsigned> again;
            for (unsigned e : pending) {
                const VmResult &r = X.res[e];
                if (r.code == VM_TAPE_SCRATCH) { extra[e] *= 16; again.push_back(e); continue; }
                if (r.code != VM_OK) { X.fail(e, DG_ERR_EXECUTION, vm_message(r.code, r.fail_step, x.max_steps)); continue; }
                if (seq[e].checkpoints + 1 <= cp_cap[e] && seq[e].logged <= log_cap[e]) continue;
                cp_cap[e] = std::max(cp_cap[e], seq[e].checkpoints + 1);                   // the sizes this execution needs
                log_cap[e] = std::max(log_cap[e], seq[e].logged);
                again.push_back(e);
            }
            pending.swap(again);
        }
        X.d_tapes.release();                      // the segments read the logs
        for (unsigned e : run)
            if (X.status[e] == DG_OK) { st.checkpoints += seq[e].checkpoints + 1; st.segments += seq[e].checkpoints; st.logged += seq[e].logged; }
    }

    // The rows of the successful executions of `run`, in waves as the batch path cuts them: per wave one segment launch for every
    // checkpoint of its executions and one padding launch per shape, then done(slabs).  A segment that fails is an internal error of its
    // execution.  The tables, logs and checkpoints are freed before the last wave's done.
    template <typename F> void waves(const dg_options_t *opts, uint8_t *const *registers_out, F &&done) {
        X.cut_waves(X.shape_order(run), opts, registers_out, [&](const std::vector<unsigned> &wave, const std::vector<Slab> &slabs, bool last) {
            std::vector<unsigned long long> first{0};
            for (unsigned e : wave) first.push_back(first.back() + seq[e].checkpoints);
            const unsigned long long segments = first.back();
            X.upload(d_execs, wave);
            X.upload(d_first, first);
            d_codes.alloc(std::max<unsigned long long>(2 * segments, 1) * sizeof(unsigned long long));
            st.segment_ms += X.timed([&] {
                vm_segment_pass(c, X.L, G, d_T.as<VmTabled>(), d_execs.as<unsigned>(), d_first.as<unsigned long long>(), (unsigned)wave.size(),
                                segments, d_codes.as<unsigned long long>());
                X.pad(slabs);
            });
            st.waves++;
            std::vector<unsigned long long> codes(2 * segments);
            DG_CUDA(cudaMemcpy(codes.data(), d_codes.p, codes.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
            for (size_t j = 0; j < wave.size(); j++)
                for (unsigned long long g = first[j]; g < first[j + 1]; g++) {
                    const unsigned code = (unsigned)codes[2 * g];
                    if (code == VM_OK) continue;
                    const std::string m = vm_message(code, codes[2 * g + 1], X.x.max_steps);
                    X.fail(wave[j], DG_ERR_EXECUTION, code == VM_SEGMENT ? m : "internal error: trace segment " + std::to_string(g - first[j]) +
                                                                             " failed where the sequential pass did not: " + m);
                    break;
                }
            if (last) release();
            done(slabs);
        });
    }
    // the buffers the rows no longer need, before a proof
    void release() {
        for (DevBuf *d : {&d_refs, &d_tab, &d_T, &d_seq, &d_codes, &d_execs, &d_first, &X.d_tapes}) d->release();
        logs.clear();
    }

    // dg_trace_many: the fallback executions on the batch path (with the write pass even without registers_out, so that a shapes-only
    // call reports what a full one reports), then the tabled ones
    void trace(uint8_t *const *registers_out) {
        tables();
        if (run.empty()) release();
        batch_trace(c, X, fallback, registers_out, true, false);
        sequential();
        if (registers_out) waves(nullptr, registers_out, [&](const std::vector<Slab> &slabs) { copy_slabs(c, X, slabs, registers_out); });
        st.fallback = X.stats;
    }
    // dg_execute_many: the same, every trace proven where it was written; outs holds 8 elements per execution
    void execute(const uint32_t *num_outputs, const dg_options_t *opts, std::vector<fe> &outs, Proof **proofs_out, dg_prove_stats_t *stats) {
        tables();
        if (run.empty()) release();
        batch_execute(c, X, fallback, num_outputs, opts, outs, proofs_out, stats);
        sequential();
        for (unsigned e : run)
            if (X.status[e] == DG_OK) for (uint32_t j = 0; j < num_outputs[e]; j++) outs[(size_t)e * 8 + j] = X.res[e].top[j];
        waves(opts, nullptr, [&](const std::vector<Slab> &slabs) { prove_slabs(c, X, slabs, num_outputs, opts, outs, proofs_out, stats, st.prove_groups); });
        st.fallback = X.stats;
    }
};

}  // namespace

// the whole-call checks of device inputs: every array there, and every non-empty range inside d_values, which is there and aligned when
// some range is not empty
static void check_device_inputs(const dg_device_inputs_t &d, uint32_t count) {
    DG_REQUIRE(d.public_first && d.n_public && d.secret_a_first && d.n_secret_a && d.secret_b_first && d.n_secret_b,
               "device inputs: null offset or count array");
    bool any = false;
    static const char *what[3] = {"public inputs", "tape A", "tape B"};
    for (uint32_t i = 0; i < count; i++) {
        const uint64_t first[3] = {d.public_first[i], d.secret_a_first[i], d.secret_b_first[i]};
        const uint64_t n[3] = {d.n_public[i], d.n_secret_a[i], d.n_secret_b[i]};
        for (int r = 0; r < 3; r++) {
            if (n[r] == 0) continue;
            any = true;
            const std::string at = "device inputs of execution " + std::to_string(i) + ": " + what[r] + " [" + std::to_string(first[r]) + ", + " +
                                   std::to_string(n[r]) + ")";
            DG_REQUIRE(first[r] + n[r] >= first[r], at + " overflows");
            DG_REQUIRE(first[r] + n[r] <= d.n_values, at + " ends past n_values = " + std::to_string(d.n_values));
        }
    }
    if (!any) return;
    DG_REQUIRE(d.d_values, "device inputs: d_values is null");
    DG_REQUIRE(((uintptr_t)d.d_values & 15) == 0, "device inputs: d_values is not 16-byte aligned");
}

void check_execution_call(const ExecutionCall &x, const std::optional<OutputCounts> &outputs, std::optional<uint64_t> segment_steps) {
    DG_REQUIRE(x.count >= 1, "at least one execution is needed");
    DG_REQUIRE(x.n_programs >= 1, "at least one program is needed");
    DG_REQUIRE(x.programs && x.program_of, "null program table");
    DG_REQUIRE(x.inputs || x.device_inputs, "null inputs");
    DG_REQUIRE(x.max_steps >= 16, "max_steps must be at least 16");
    uint64_t ops = 0, blocks = 0, children = 0;
    for (uint32_t p = 0; p < x.n_programs; p++) {
        try {
            validate(&x.programs[p]);
        } catch (const Error &e) {
            if (x.n_programs == 1) throw;
            throw Error(e.code, "program " + std::to_string(p) + ": " + e.what());
        }
        ops += x.programs[p].n_ops; blocks += x.programs[p].n_blocks; children += x.programs[p].n_children;
    }
    // the programs share one table of each, indexed by 32-bit offsets
    DG_REQUIRE(ops <= (1ULL << 32), "the programs of a call hold more than 2^32 ops");
    DG_REQUIRE(blocks <= (1ULL << 32) && children <= (1ULL << 32), "the programs of a call hold more than 2^32 blocks or child entries");
    for (uint32_t i = 0; i < x.count; i++) {
        DG_REQUIRE(x.program_of[i] < x.n_programs, "program_of[" + std::to_string(i) + "] = " + std::to_string(x.program_of[i]) +
                                                       " is out of range: the call has " + std::to_string(x.n_programs) + " programs");
        if (x.device_inputs) continue;
        const dg_program_inputs_t &v = x.inputs[i];
        DG_REQUIRE((v.n_public == 0 || v.public16) && (v.n_secret_a == 0 || v.secret_a16) && (v.n_secret_b == 0 || v.secret_b16),
                   "null inputs of execution " + std::to_string(i));
    }
    if (x.device_inputs) check_device_inputs(*x.device_inputs, x.count);
    if (outputs) {
        DG_REQUIRE(outputs->num_outputs, "null num_outputs");
        bool any = false;
        for (uint32_t i = 0; i < x.count; i++) {
            DG_REQUIRE(outputs->num_outputs[i] <= 8, "cannot have more than 8 outputs");
            any |= outputs->num_outputs[i] > 0;
        }
        DG_REQUIRE(!any || outputs->outputs16, "null outputs");
    }
    if (segment_steps) {
        const uint64_t s = *segment_steps;
        DG_REQUIRE(s == 0 || (s >= 16 && (s & (s - 1)) == 0), "segment_steps must be 0 or a power of two of at least 16");
    }
}

void trace_programs(Context &c, const ExecutionCall &x, dg_execution_info_t *info, uint8_t *const *registers_out, int *status,
                    std::vector<std::string> &messages, dg_execution_stats_t *vm_stats) {
    check_one_gpu(c);
    Executions X(c, x);
    X.setup();
    std::vector<unsigned> all(x.count);
    std::iota(all.begin(), all.end(), 0u);
    batch_trace(c, X, all, registers_out, registers_out != nullptr, true);
    finish(X, info, status, messages, vm_stats);
}

void execute_programs(Context &c, const ExecutionCall &x, const uint32_t *num_outputs, const dg_options_t *opts, Proof **proofs_out,
                      uint8_t *outputs16, int *status, std::vector<std::string> &messages, dg_prove_stats_t *stats, dg_execution_stats_t *vm_stats) {
    check_one_gpu(c);
    proven(x.count, proofs_out, outputs16, stats, [&](std::vector<fe> &outs) {
        Executions X(c, x);
        X.setup();
        std::vector<unsigned> all(x.count);
        std::iota(all.begin(), all.end(), 0u);
        batch_execute(c, X, all, num_outputs, opts, outs, proofs_out, stats);
        finish(X, nullptr, status, messages, vm_stats);
    });
}

void trace_many(Context &c, const ExecutionCall &x, uint64_t segment_steps, dg_execution_info_t *info, uint8_t *const *registers_out, int *status,
                std::vector<std::string> &messages, dg_many_stats_t *stats) {
    check_one_gpu(c);
    TabledExecutions E(c, x, segment_steps, stats);
    E.trace(registers_out);
    finish(E.X, info, status, messages, nullptr);
}

void execute_many(Context &c, const ExecutionCall &x, const uint32_t *num_outputs, uint64_t segment_steps, const dg_options_t *opts,
                  Proof **proofs_out, uint8_t *outputs16, dg_execution_info_t *info, int *status, std::vector<std::string> &messages,
                  dg_prove_stats_t *prove_stats, dg_many_stats_t *stats) {
    check_one_gpu(c);
    proven(x.count, proofs_out, outputs16, prove_stats, [&](std::vector<fe> &outs) {
        TabledExecutions E(c, x, segment_steps, stats);
        E.execute(num_outputs, opts, outs, proofs_out, prove_stats);
        finish(E.X, info, status, messages, nullptr);
    });
}

}  // namespace dg
