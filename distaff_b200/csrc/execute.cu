// Host orchestration of dg_trace_programs / dg_execute_programs (distaff::execute, lib.rs:30-65, for many programs and inputs; dg_trace_batch
// and dg_execute_batch are the one-program case): validate each program's encoding, put every program into one set of tables and upload
// them and the inputs once, run the shape pass for every execution, and write the successful executions in waves -- one write launch
// (vm.cu) per wave for every shape in it -- into one slab per shape, which is copied to the caller's buffers (dg_trace_programs) or
// proven in place (dg_execute_programs, through prove_traces).
#include "vm.h"
#include "air.h"
#include "prover.h"
#include <algorithm>
#include <map>
#include <set>
#include <tuple>

namespace dg {
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
    std::vector<VmResult> res;
    std::vector<int> status;
    std::vector<std::string> messages;
    std::vector<unsigned long long> off, cap;
    dg_execution_stats_t stats;
    cudaEvent_t ev[2] = {nullptr, nullptr};

    Executions(Context &ctx_, const ExecutionCall &call)
        : c(ctx_), x(call), res(call.count), status(call.count, DG_OK), messages(call.count), off(call.count, 0), cap(2 * (size_t)call.count, 0) {
        memset(&stats, 0, sizeof stats);
        DG_CUDA(cudaEventCreate(&ev[0]));
        DG_CUDA(cudaEventCreate(&ev[1]));
    }
    ~Executions() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }

    void fail(uint32_t i, int code, const std::string &m) { status[i] = code; messages[i] = m; }
    // "<what> <j> is not a field element" for the first of n values at or above M, else ""
    static std::string first_non_element(const uint8_t *p, uint64_t n, const char *what) {
        for (uint64_t j = 0; j < n; j++) {
            fe e;
            memcpy(&e, p + 16 * j, 16);
            if (e.hi == DG_M_HI && e.lo >= DG_M_LO) return std::string(what) + " " + std::to_string(j) + " is not a field element";
        }
        return "";
    }

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
        // inputs, packed: public inputs, then both tapes reversed (the next value to read is the last one, as in the host VM)
        std::vector<VmInput> in(x.count);
        std::vector<fe> data;
        for (uint32_t i = 0; i < x.count; i++) {
            const dg_program_inputs_t &v = x.inputs[i];
            memset(&in[i], 0, sizeof(VmInput));
            in[i].program = x.program_of[i];
            if (v.n_public > 8) { fail(i, DG_ERR_EXECUTION, "expected no more than 8 public inputs"); continue; }      // lib.rs:32
            if (v.n_secret_a < v.n_secret_b) { fail(i, DG_ERR_EXECUTION, "tape A cannot be shorter than tape B"); continue; }   // inputs.rs:17
            // the VM's arithmetic assumes canonical operands: a value in [M, 2^128) fails its execution (the reference does not check)
            std::string bad = first_non_element(v.public16, v.n_public, "public input");
            if (bad.empty()) bad = first_non_element(v.secret_a16, v.n_secret_a, "tape A value");
            if (bad.empty()) bad = first_non_element(v.secret_b16, v.n_secret_b, "tape B value");
            if (!bad.empty()) { fail(i, DG_ERR_EXECUTION, bad); continue; }
            auto put = [&](const uint8_t *p, uint64_t n, bool reverse) {
                const size_t at = data.size();
                for (uint64_t j = 0; j < n; j++) { fe e; memcpy(&e, p + 16 * (reverse ? n - 1 - j : j), 16); data.push_back(e); }
                return (unsigned long long)at;
            };
            in[i].n_pub = v.n_public; in[i].pub = put(v.public16, v.n_public, false);
            in[i].n_a = v.n_secret_a; in[i].a = put(v.secret_a16, v.n_secret_a, true);
            in[i].n_b = v.n_secret_b; in[i].b = put(v.secret_b16, v.n_secret_b, true);
        }
        upload(d_in, in); upload(d_data, data);
        d_res.alloc((size_t)x.count * sizeof(VmResult));
        DG_CUDA(cudaMemsetAsync(d_res.p, 0, (size_t)x.count * sizeof(VmResult), c.stream));
        L.ops = d_ops.as<uint8_t>(); L.hints = d_hints.as<VmHint>(); L.blocks = d_blocks.as<VmBlock>(); L.children = d_children.as<unsigned>();
        L.programs = d_programs.as<VmProgram>();
        L.in = d_in.as<VmInput>(); L.data = d_data.as<fe>();
        L.res = d_res.as<VmResult>();
        L.max_steps = x.max_steps;
        for (uint32_t i = 0; i < x.count; i++) { cap[2 * i] = in[i].n_a; cap[2 * i + 1] = in[i].n_b; }
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

    // the shape pass; an execution whose hints outgrow its tape scratch (256 elements beyond its inputs at first; what the assembler's
    // macros need) runs again with 16 times more
    void shapes() {
        std::vector<unsigned> pending;
        for (uint32_t i = 0; i < x.count; i++) if (status[i] == DG_OK) pending.push_back(i);
        for (unsigned long long extra = 256; !pending.empty(); extra *= 16) {
            for (unsigned e : pending) { cap[2 * e] = x.inputs[e].n_secret_a + extra; cap[2 * e + 1] = x.inputs[e].n_secret_b + extra; }
            place_tapes(pending);
            launch_ids(pending);
            stats.shape_ms += timed([&] { vm_shape_pass(c, L); });
            stats.shape_launches++;
            download_results();
            std::vector<unsigned> again;
            for (unsigned e : pending) if (res[e].code == VM_TAPE_SCRATCH) again.push_back(e);
            pending.swap(again);
        }
        for (uint32_t i = 0; i < x.count; i++)
            if (status[i] == DG_OK && res[i].code != VM_OK) fail(i, DG_ERR_EXECUTION, vm_message(res[i].code, res[i].fail_step, x.max_steps));
        // the write pass runs with the tape scratch each execution needed
        std::vector<unsigned> ok;
        for (uint32_t i = 0; i < x.count; i++)
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
    // the successful executions by shape, shapes in order and input order inside a shape
    std::vector<unsigned> shape_order() const {
        std::map<ShapeKey, std::vector<unsigned>> g;
        for (uint32_t i = 0; i < x.count; i++) if (status[i] == DG_OK) g[key(info(i))].push_back(i);
        std::vector<unsigned> order;
        for (auto &kv : g) order.insert(order.end(), kv.second.begin(), kv.second.end());
        return order;
    }

    // The write pass of every successful execution, in waves.  A wave is a run of the executions in shape order, written by one launch
    // into one slab per shape and handed to done(slabs) while its traces are on the device; waves follow each other, so the executions
    // reach done in shape order, input order inside a shape.  A wave's traces take at most half of the device memory the library may
    // use, and with `opt` they leave room beside them for one proof of the wave's largest shape.  $DG_BATCH_GROUP caps its executions.
    template <typename F> void write_waves(const dg_options_t *opt, uint8_t *const *registers_out, F &&done) {
        const std::vector<unsigned> order = shape_order();
        const size_t most = (size_t)batch_group_cap(65535);         // one padding launch holds 65535 executions
        std::map<ShapeKey, size_t> room;                           // bytes one proof of a shape needs beside the traces
        std::vector<VmOut> outs(x.count);
        for (size_t first = 0; first < order.size();) {
            size_t avail = memory_budget(c, Budget::FREE, 0);
            if (c.mem_limit) avail = avail > c.arena.cap ? avail - c.arena.cap : 0;      // proofs may keep the arena beside the traces
            size_t end = first, bytes = 0, need = 0;
            while (end < order.size() && end - first < most) {
                const dg_execution_info_t s = info(order[end]);
                const size_t per = (size_t)s.width * s.length * 16;
                size_t r = 0;
                if (opt) {
                    auto it = room.find(key(s));
                    if (it == room.end()) {
                        const ProvePlan P = plan_prove(c, s.width, s.length, opt->extension_factor, 1);
                        it = room.emplace(key(s), P.per_proof + P.fixed - memory_held_outside_arena(c)).first;
                    }
                    r = it->second;
                }
                if (end > first && (bytes + per > avail / 2 || bytes + per + std::max(need, r) > avail)) break;
                if (registers_out) DG_REQUIRE(registers_out[order[end]], "null register buffer of execution " + std::to_string(order[end]));
                if (!opt && c.mem_limit && per > avail)
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
            upload(d_pad_ids, wave);                               // the wave is in slab order
            L.out = regs.as<fe>();
            L.outs = d_outs.as<VmOut>();
            stats.lanes += launch_ids(wave);
            stats.write_ms += timed([&] {
                vm_write_pass(c, L);
                size_t q = 0;
                for (const Slab &s : slabs) {
                    vm_pad_rows(c, s.regs, L.res, d_pad_ids.as<unsigned>() + q, (unsigned)s.ids.size(), s.shape.width, s.shape.length);
                    q += s.ids.size();
                }
            });
            stats.write_launches++;
            stats.waves++;
            download_results();
            for (unsigned e : wave)
                if (res[e].code != VM_OK) fail(e, DG_ERR_EXECUTION, vm_message(res[e].code, res[e].fail_step, x.max_steps));
            done(slabs);
            first = end;
        }
    }
};

void check_one_gpu(Context &c) {
    DG_REQUIRE(c.world == 1 && ctx_device_count() == 1, "batched execution runs on one GPU: the library was initialised for several (dg_init_devices / dg_comm_init)");
}

void finish(const Executions &X, int *status, std::vector<std::string> &messages, dg_execution_stats_t *vm_stats) {
    for (uint32_t i = 0; i < X.x.count; i++) status[i] = X.status[i];
    messages = X.messages;
    if (vm_stats) *vm_stats = X.stats;
}

}  // namespace

void check_execution_call(const ExecutionCall &x) {
    DG_REQUIRE(x.count >= 1, "at least one execution is needed");
    DG_REQUIRE(x.n_programs >= 1, "at least one program is needed");
    DG_REQUIRE(x.programs && x.program_of, "null program table");
    DG_REQUIRE(x.inputs, "null inputs");
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
        const dg_program_inputs_t &v = x.inputs[i];
        DG_REQUIRE((v.n_public == 0 || v.public16) && (v.n_secret_a == 0 || v.secret_a16) && (v.n_secret_b == 0 || v.secret_b16),
                   "null inputs of execution " + std::to_string(i));
    }
}

void check_output_counts(uint32_t count, const uint32_t *num_outputs, const uint8_t *outputs16) {
    DG_REQUIRE(num_outputs, "null num_outputs");
    bool any = false;
    for (uint32_t i = 0; i < count; i++) {
        DG_REQUIRE(num_outputs[i] <= 8, "cannot have more than 8 outputs");
        any |= num_outputs[i] > 0;
    }
    DG_REQUIRE(!any || outputs16, "null outputs");
}

void trace_programs(Context &c, const ExecutionCall &x, dg_execution_info_t *info, uint8_t *const *registers_out, int *status,
                    std::vector<std::string> &messages, dg_execution_stats_t *vm_stats) {
    check_execution_call(x);
    check_one_gpu(c);
    Executions X(c, x);
    X.setup();
    X.shapes();
    if (registers_out) {
        X.write_waves(nullptr, registers_out, [&](const std::vector<Slab> &slabs) {
            for (const Slab &s : slabs) {
                const size_t per = (size_t)s.shape.width * s.shape.length * 16;
                for (size_t q = 0; q < s.ids.size(); q++)
                    if (X.status[s.ids[q]] == DG_OK)
                        DG_CUDA(cudaMemcpyAsync(registers_out[s.ids[q]], (const uint8_t *)s.regs + q * per, per, cudaMemcpyDeviceToHost, c.stream));
            }
            DG_CUDA(cudaStreamSynchronize(c.stream));
        });
    }
    if (info)
        for (uint32_t i = 0; i < x.count; i++) {
            if (X.status[i] == DG_OK) info[i] = X.info(i);
            else memset(&info[i], 0, sizeof info[i]);
        }
    finish(X, status, messages, vm_stats);
}

void execute_programs(Context &c, const ExecutionCall &x, const uint32_t *num_outputs, const dg_options_t &opt, Proof **proofs_out,
                      uint8_t *outputs16, int *status, std::vector<std::string> &messages, dg_prove_stats_t *stats, dg_execution_stats_t *vm_stats) {
    check_execution_call(x);
    check_output_counts(x.count, num_outputs, outputs16);
    check_one_gpu(c);
    for (uint32_t i = 0; i < x.count; i++) proofs_out[i] = nullptr;
    if (stats) memset(stats, 0, sizeof *stats);
    Executions X(c, x);
    X.setup();
    X.shapes();
    // the proofs of the waves done so far are freed when a later wave fails the call
    struct ReleaseOnError {
        Proof **out; uint32_t count; bool done = false;
        ~ReleaseOnError() { if (!done) for (uint32_t i = 0; i < count; i++) { delete out[i]; out[i] = nullptr; } }
    } release{proofs_out, x.count};
    std::vector<fe> outs((size_t)x.count * 8, fe_make(0, 0));
    for (uint32_t i = 0; i < x.count; i++)
        if (X.status[i] == DG_OK) for (uint32_t j = 0; j < num_outputs[i]; j++) outs[(size_t)i * 8 + j] = X.res[i].top[j];
    X.write_waves(&opt, nullptr, [&](const std::vector<Slab> &slabs) {
        for (const Slab &s : slabs) {
            // executions the write pass failed are left out: the traces after them move down over them, and their outputs are zero, as
            // those of executions the shape pass failed
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
            for (uint32_t q = 0; q < k; q++) {
                in16[q] = x.inputs[ok[q]].public16; n_in[q] = x.inputs[ok[q]].n_public;
                out16[q] = (const uint8_t *)&outs[(size_t)ok[q] * 8]; n_out[q] = num_outputs[ok[q]];
            }
            std::vector<Proof *> proofs(k, nullptr);
            std::vector<int> st(k, DG_OK);
            std::vector<std::string> msg;
            dg_prove_stats_t gs;
            memset(&gs, 0, sizeof gs);
            uint32_t groups = 0;
            prove_traces(c, s.regs, nullptr, k, s.shape.width, s.shape.length, s.shape.ctx_depth, s.shape.loop_depth, in16.data(), n_in.data(),
                         out16.data(), n_out.data(), opt, true, proofs.data(), st.data(), msg, &gs, &groups);
            for (uint32_t q = 0; q < k; q++) {
                proofs_out[ok[q]] = proofs[q];
                if (st[q] != DG_OK) X.fail(ok[q], st[q], msg[q]);
            }
            X.stats.prove_groups += groups;
            if (stats) {
                for (int i = 0; i < 9; i++) stats->stage_ms[i] += gs.stage_ms[i];
                stats->h2d_ms += gs.h2d_ms; stats->total_ms += gs.total_ms; stats->kernel_launches += gs.kernel_launches;
            }
        }
    });
    release.done = true;
    if (outputs16) memcpy(outputs16, outs.data(), outs.size() * 16);
    finish(X, status, messages, vm_stats);
}

}  // namespace dg