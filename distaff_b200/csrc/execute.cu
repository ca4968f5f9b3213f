// Host orchestration of dg_trace_batch / dg_execute_batch (distaff::execute, lib.rs:30-65, for many inputs): validate the program
// encoding, upload it and the inputs once, run the shape pass for every execution, group the successful executions by trace shape, and
// per group run the write pass (vm.cu) into the caller's buffers (dg_trace_batch) or into the buffer the prover reads (dg_execute_batch,
// through prove_batch_generated: the prove_core path of dg_prove_batch_device).
#include "vm.h"
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

// ---- one call: the program and inputs on the device, the shape pass, the groups ---------------------------------------------------------
struct Executions {
    Context &c;
    const dg_program_t &prog;
    uint32_t count;
    const dg_program_inputs_t *inputs;
    unsigned long long max_steps;
    DevBuf d_ops, d_hints, d_blocks, d_children, d_in, d_data, d_res, d_tapes, d_off, d_cap, d_ids;
    VmLaunch L;
    std::vector<VmResult> res;
    std::vector<int> status;
    std::vector<std::string> messages;
    std::vector<unsigned long long> off, cap;

    Executions(Context &ctx_, const dg_program_t &p, uint32_t n, const dg_program_inputs_t *in, unsigned long long ms)
        : c(ctx_), prog(p), count(n), inputs(in), max_steps(ms), res(n), status(n, DG_OK), messages(n), off(n, 0), cap(2 * (size_t)n, 0) {}

    void fail(uint32_t i, int code, const std::string &m) { status[i] = code; messages[i] = m; }

    template <typename T> void upload(DevBuf &d, const std::vector<T> &v) {
        d.alloc(std::max<size_t>(v.size(), 1) * sizeof(T));
        if (!v.empty()) DG_CUDA(cudaMemcpyAsync(d.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }

    void setup() {
        memset(&L, 0, sizeof L);
        std::vector<uint8_t> ops(prog.ops, prog.ops + prog.n_ops);
        std::vector<VmHint> hints(prog.n_ops);
        for (uint64_t i = 0; i < prog.n_ops; i++) {
            hints[i].kind = prog.hints[i].kind;
            hints[i].n = prog.hints[i].n;
            memcpy(&hints[i].value, prog.hints[i].value16, 16);
        }
        std::vector<VmBlock> blocks(prog.n_blocks);
        for (uint32_t i = 0; i < prog.n_blocks; i++) {
            const dg_block_t &b = prog.blocks[i];
            memset(&blocks[i], 0, sizeof(VmBlock));
            blocks[i].kind = b.kind; blocks[i].first = b.first; blocks[i].count = b.count; blocks[i].alt_first = b.alt_first; blocks[i].alt_count = b.alt_count;
            memcpy(&blocks[i].hash[0], b.hash0, 16); memcpy(&blocks[i].hash[1], b.hash1, 16); memcpy(&blocks[i].hash[2], b.hash2, 16);
        }
        upload(d_ops, ops); upload(d_hints, hints); upload(d_blocks, blocks);
        upload(d_children, std::vector<unsigned>(prog.children, prog.children + prog.n_children));
        // inputs, packed: public inputs, then both tapes reversed (the next value to read is the last one, as in the host VM)
        std::vector<VmInput> in(count);
        std::vector<fe> data;
        for (uint32_t i = 0; i < count; i++) {
            const dg_program_inputs_t &x = inputs[i];
            memset(&in[i], 0, sizeof(VmInput));
            if (x.n_public > 8) { fail(i, DG_ERR_EXECUTION, "expected no more than 8 public inputs"); continue; }      // lib.rs:32
            if (x.n_secret_a < x.n_secret_b) { fail(i, DG_ERR_EXECUTION, "tape A cannot be shorter than tape B"); continue; }   // inputs.rs:17
            auto put = [&](const uint8_t *v, uint64_t n, bool reverse) {
                const size_t at = data.size();
                for (uint64_t j = 0; j < n; j++) { fe e; memcpy(&e, v + 16 * (reverse ? n - 1 - j : j), 16); data.push_back(e); }
                return (unsigned long long)at;
            };
            in[i].n_pub = x.n_public; in[i].pub = put(x.public16, x.n_public, false);
            in[i].n_a = x.n_secret_a; in[i].a = put(x.secret_a16, x.n_secret_a, true);
            in[i].n_b = x.n_secret_b; in[i].b = put(x.secret_b16, x.n_secret_b, true);
        }
        upload(d_in, in); upload(d_data, data);
        d_res.alloc((size_t)count * sizeof(VmResult));
        DG_CUDA(cudaMemsetAsync(d_res.p, 0, (size_t)count * sizeof(VmResult), c.stream));
        L.ops = d_ops.as<uint8_t>(); L.hints = d_hints.as<VmHint>(); L.blocks = d_blocks.as<VmBlock>(); L.children = d_children.as<unsigned>();
        L.root_first = prog.root_first; L.root_count = prog.root_count;
        memcpy(&L.hash[0], prog.hash32, 16); memcpy(&L.hash[1], prog.hash32 + 16, 16);
        L.in = d_in.as<VmInput>(); L.data = d_data.as<fe>();
        L.res = d_res.as<VmResult>();
        L.max_steps = max_steps;
        for (uint32_t i = 0; i < count; i++) { cap[2 * i] = in[i].n_a; cap[2 * i + 1] = in[i].n_b; }
    }

    // tape scratch for `ids`: capacity cap[2e], cap[2e + 1] each
    void place_tapes(const std::vector<unsigned> &ids) {
        unsigned long long total = 0;
        for (unsigned e : ids) { off[e] = total; total += cap[2 * e] + cap[2 * e + 1]; }
        d_tapes.alloc(std::max<unsigned long long>(total, 1) * 16);
        upload(d_off, off); upload(d_cap, cap);
        L.tapes = d_tapes.as<fe>(); L.tape_off = d_off.as<unsigned long long>(); L.cap = d_cap.as<unsigned long long>();
    }
    void launch_ids(const std::vector<unsigned> &ids) {
        upload(d_ids, ids);
        L.ids = d_ids.as<unsigned>();
        L.count = (unsigned)ids.size();
    }
    void download_results() {
        DG_CUDA(cudaMemcpyAsync(res.data(), d_res.p, (size_t)count * sizeof(VmResult), cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }

    // the shape pass; an execution whose hints outgrow its tape scratch (256 elements beyond its inputs at first; what the assembler's
    // macros need) runs again with 16 times more
    void shapes() {
        std::vector<unsigned> pending;
        for (uint32_t i = 0; i < count; i++) if (status[i] == DG_OK) pending.push_back(i);
        for (unsigned long long extra = 256; !pending.empty(); extra *= 16) {
            for (unsigned e : pending) { cap[2 * e] = inputs[e].n_secret_a + extra; cap[2 * e + 1] = inputs[e].n_secret_b + extra; }
            place_tapes(pending);
            launch_ids(pending);
            vm_shape_pass(c, L);
            download_results();
            std::vector<unsigned> again;
            for (unsigned e : pending) if (res[e].code == VM_TAPE_SCRATCH) again.push_back(e);
            pending.swap(again);
        }
        for (uint32_t i = 0; i < count; i++)
            if (status[i] == DG_OK && res[i].code != VM_OK) fail(i, DG_ERR_EXECUTION, vm_message(res[i].code, res[i].fail_step, max_steps));
        // the write pass runs with the tape scratch each execution needed
        std::vector<unsigned> ok;
        for (uint32_t i = 0; i < count; i++)
            if (status[i] == DG_OK) { ok.push_back(i); cap[2 * i] = res[i].peak_a; cap[2 * i + 1] = res[i].peak_b; }
        place_tapes(ok);
    }

    dg_execution_info_t info(uint32_t i) const {
        dg_execution_info_t x;
        memset(&x, 0, sizeof x);
        const VmResult &r = res[i];
        x.ctx_depth = r.ctx_cols - 1; x.loop_depth = r.loop_cols; x.stack_depth = r.max_depth;
        x.width = 15 + x.ctx_depth + x.loop_depth + x.stack_depth;
        x.steps = r.steps;
        x.length = 16;
        while (x.length <= r.steps) x.length *= 2;
        return x;
    }
    // successful executions by shape (width, length, ctx depth, loop depth), in input order inside a group
    std::map<std::tuple<uint32_t, uint64_t, uint32_t, uint32_t>, std::vector<unsigned>> groups() const {
        std::map<std::tuple<uint32_t, uint64_t, uint32_t, uint32_t>, std::vector<unsigned>> g;
        for (uint32_t i = 0; i < count; i++) {
            if (status[i] != DG_OK) continue;
            const dg_execution_info_t x = info(i);
            g[std::make_tuple(x.width, x.length, x.ctx_depth, x.loop_depth)].push_back(i);
        }
        return g;
    }
    // the write pass of executions ids (one shape) into d_out; returns per id DG_OK or the failure only the sponge reveals
    void write(const std::vector<unsigned> &ids, fe *d_out, std::vector<std::pair<int, std::string>> &failed) {
        const dg_execution_info_t x = info(ids[0]);
        L.out = d_out; L.length = x.length; L.width = x.width;
        L.ctx_out = x.ctx_depth; L.loop_out = x.loop_depth; L.stack_out = x.stack_depth;
        launch_ids(ids);
        vm_write_pass(c, L);
        download_results();
        failed.assign(ids.size(), {DG_OK, std::string()});
        for (size_t q = 0; q < ids.size(); q++) {
            const VmResult &r = res[ids[q]];
            if (r.code != VM_OK) failed[q] = {DG_ERR_EXECUTION, vm_message(r.code, r.fail_step, max_steps)};
        }
    }
};

void check_one_gpu(Context &c) {
    DG_REQUIRE(c.world == 1 && ctx_device_count() == 1, "batched execution runs on one GPU: the library was initialised for several (dg_init_devices / dg_comm_init)");
}

}  // namespace

void check_execution_call(const dg_program_t *program, uint32_t count, const dg_program_inputs_t *inputs, uint64_t max_steps) {
    DG_REQUIRE(count >= 1, "at least one execution is needed");
    DG_REQUIRE(inputs, "null inputs");
    DG_REQUIRE(max_steps >= 16, "max_steps must be at least 16");
    validate(program);
    for (uint32_t i = 0; i < count; i++) {
        const dg_program_inputs_t &x = inputs[i];
        DG_REQUIRE((x.n_public == 0 || x.public16) && (x.n_secret_a == 0 || x.secret_a16) && (x.n_secret_b == 0 || x.secret_b16),
                   "null inputs of execution " + std::to_string(i));
    }
}

void trace_batch(Context &c, const dg_program_t *program, uint32_t count, const dg_program_inputs_t *inputs, uint64_t max_steps,
                 dg_execution_info_t *info, uint8_t *const *registers_out, int *status, std::vector<std::string> &messages) {
    check_execution_call(program, count, inputs, max_steps);
    check_one_gpu(c);
    Executions X(c, *program, count, inputs, max_steps);
    X.setup();
    X.shapes();
    if (registers_out) {
        for (auto &kv : X.groups()) {
            const std::vector<unsigned> &ids = kv.second;
            const dg_execution_info_t x = X.info(ids[0]);
            const size_t per = (size_t)x.width * x.length * 16;
            for (unsigned e : ids) DG_REQUIRE(registers_out[e], "null register buffer of execution " + std::to_string(e));
            const size_t avail = memory_budget(c, Budget::FREE, per * ids.size());
            DG_REQUIRE(!c.mem_limit || per <= avail, "a trace of " + std::to_string(x.width) + " x " + std::to_string(x.length) + " needs " +
                                                         std::to_string(per) + " bytes of device memory beyond what the memory limit leaves");
            const size_t group = (size_t)batch_group_cap((long long)std::min<size_t>({ids.size(), 65535, std::max<size_t>(1, avail / per)}));
            for (size_t first = 0; first < ids.size(); first += group) {
                const std::vector<unsigned> part(ids.begin() + first, ids.begin() + std::min(ids.size(), first + group));
                DevBuf out(per * part.size());
                std::vector<std::pair<int, std::string>> failed;
                X.write(part, out.as<fe>(), failed);
                for (size_t q = 0; q < part.size(); q++) {
                    if (failed[q].first != DG_OK) { X.fail(part[q], failed[q].first, failed[q].second); continue; }
                    DG_CUDA(cudaMemcpyAsync(registers_out[part[q]], out.as<uint8_t>() + q * per, per, cudaMemcpyDeviceToHost, c.stream));
                }
                DG_CUDA(cudaStreamSynchronize(c.stream));
            }
        }
    }
    for (uint32_t i = 0; i < count; i++) {
        status[i] = X.status[i];
        if (info) {
            if (X.status[i] == DG_OK) info[i] = X.info(i);
            else memset(&info[i], 0, sizeof info[i]);
        }
    }
    messages = std::move(X.messages);
}

void execute_batch(Context &c, const dg_program_t *program, uint32_t count, const dg_program_inputs_t *inputs, uint32_t num_outputs,
                   uint64_t max_steps, const dg_options_t &opt, Proof **proofs_out, uint8_t *outputs16, int *status,
                   std::vector<std::string> &messages, dg_prove_stats_t *stats) {
    DG_REQUIRE(num_outputs <= 8, "cannot have more than 8 outputs");
    DG_REQUIRE(num_outputs == 0 || outputs16, "null outputs");
    check_execution_call(program, count, inputs, max_steps);
    check_one_gpu(c);
    for (uint32_t i = 0; i < count; i++) proofs_out[i] = nullptr;
    if (stats) memset(stats, 0, sizeof *stats);
    Executions X(c, *program, count, inputs, max_steps);
    X.setup();
    X.shapes();
    // the proofs of the groups done so far are freed when a later group fails the call
    struct ReleaseOnError {
        Proof **out; uint32_t count; bool done = false;
        ~ReleaseOnError() { if (!done) for (uint32_t i = 0; i < count; i++) { delete out[i]; out[i] = nullptr; } }
    } release{proofs_out, count};
    std::vector<fe> outs((size_t)count * std::max(num_outputs, 1u), fe_make(0, 0));
    for (uint32_t i = 0; i < count; i++)
        if (X.status[i] == DG_OK) for (uint32_t j = 0; j < num_outputs; j++) outs[(size_t)i * num_outputs + j] = X.res[i].top[j];
    for (auto &kv : X.groups()) {
        const std::vector<unsigned> &ids = kv.second;
        const dg_execution_info_t x = X.info(ids[0]);
        const uint32_t k = (uint32_t)ids.size();
        std::vector<const uint8_t *> in16(k), out16(k);
        std::vector<uint32_t> n_in(k), n_out(k, num_outputs);
        for (uint32_t q = 0; q < k; q++) {
            in16[q] = inputs[ids[q]].public16; n_in[q] = inputs[ids[q]].n_public;
            out16[q] = (const uint8_t *)&outs[(size_t)ids[q] * num_outputs];
        }
        std::vector<Proof *> proofs(k, nullptr);
        std::vector<int> st(k, DG_OK);
        std::vector<std::string> msg;
        dg_prove_stats_t gs;
        memset(&gs, 0, sizeof gs);
        prove_batch_generated(c, k, x.width, x.length, x.ctx_depth, x.loop_depth, in16.data(), n_in.data(), out16.data(), n_out.data(), opt,
                              proofs.data(), st.data(), msg, &gs, [&](uint32_t first, int kk, fe *d_regs, std::vector<std::pair<int, std::string>> &failed) {
                                  X.write(std::vector<unsigned>(ids.begin() + first, ids.begin() + first + kk), d_regs, failed);
                              });
        for (uint32_t q = 0; q < k; q++) {
            proofs_out[ids[q]] = proofs[q];
            if (st[q] != DG_OK) X.fail(ids[q], st[q], msg[q]);
        }
        if (stats) {
            for (int s = 0; s < 9; s++) stats->stage_ms[s] += gs.stage_ms[s];
            stats->h2d_ms += gs.h2d_ms; stats->total_ms += gs.total_ms; stats->kernel_launches += gs.kernel_launches;
        }
    }
    release.done = true;
    for (uint32_t i = 0; i < count; i++) {
        status[i] = X.status[i];
        if (num_outputs) memcpy(outputs16 + (size_t)16 * num_outputs * i, &outs[(size_t)i * num_outputs], (size_t)16 * num_outputs);
    }
    messages = std::move(X.messages);
}

}  // namespace dg
