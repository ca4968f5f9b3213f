// The trace check (dg_check_traces / dg_check_traces_device): which transition constraints a trace breaks at which steps, and which
// registers of its first and last rows break a boundary assertion, without proving it.
//
// Coset 0 of the prover's coset-major extension is the register trace itself, so the constraint kernel runs on the registers unchanged
// (num_c8 = 1, col_stride = n, log_blowup = 3: stride 1, periodic row 8k mod 128) in its CHECK instantiation, which writes a 3-word mask
// of nonzero constraints per step; check_reduce_kernel turns the masks into per-constraint counts and lowest steps.  The boundary
// assertions (evaluator.rs:181-326) are compared on the host with the first and last rows, 2 w elements per trace.
#include "prover.h"
#include "air.h"

namespace dg {

namespace {

const char *const DECODER_NAMES[20] = {
    "op bit 0 binary", "op bit 1 binary", "op bit 2 binary", "op bit 3 binary", "op bit 4 binary", "op bit 5 binary", "op bit 6 binary",
    "op bit 7 binary", "op bit 8 binary", "op bit 9 binary", "op counter", "op combination (ld, hd)", "op combination (cf)", "void sequence",
    "op alignment", "sponge 0", "sponge 1", "sponge 2", "sponge 3", "loop image"};

bool fe_equal(const fe &a, const fe &b) { return a.lo == b.lo && a.hi == b.hi; }

// Device bytes one trace takes in a group: its upload (host traces), its step masks (unless the caller's), statistics and rows.
size_t check_footprint(uint32_t w, uint64_t n, bool upload, bool own_masks) {
    return (upload ? (size_t)w * n * 16 : 0) + (own_masks ? (size_t)n * 12 : 0) + CHECK_STATS * 8 + 512;
}

int check_group_size(uint32_t w, uint64_t n, bool upload, bool own_masks, uint32_t count) {
    long long k = std::min<long long>(count, 65535);
    const size_t per = check_footprint(w, n, upload, own_masks), avail = memory_budget(ctx(), Budget::FREE, per);
    DG_REQUIRE(!ctx().mem_limit || per <= avail, "a trace check of " + std::to_string(w) + " x " + std::to_string(n) + " needs " + std::to_string(per) +
                                                     " bytes of device memory beyond what the memory limit leaves");
    k = std::min<long long>(k, (long long)std::max<size_t>(1, avail / per));
    return (int)batch_group_cap(k);
}

}  // namespace

std::string constraint_name(uint32_t ctx_depth, uint32_t loop_depth, uint32_t stack_depth, uint32_t index) {
    DG_REQUIRE(TraceShape::in_range(ctx_depth, loop_depth, stack_depth), "register shape out of range");
    const TraceShape shape(ctx_depth, loop_depth, stack_depth);
    DG_REQUIRE(index < (uint32_t)shape.T, "constraint index out of range");
    if (index < 20) return DECODER_NAMES[index];
    index -= 20;
    if (index < (uint32_t)shape.cl) return "ctx stack " + std::to_string(index);
    index -= shape.cl;
    if (index < (uint32_t)shape.ll) return "loop stack " + std::to_string(index);
    index -= shape.ll;
    if (index < 2) return "stack aux " + std::to_string(index);
    return "stack slot " + std::to_string(index - 2);
}

void check_traces(Context &c, const std::vector<TraceRef> &traces, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                  const uint8_t *const *outputs16, const uint32_t *n_outputs, const uint8_t *program_hashes32, dg_trace_report_t *reports,
                  uint32_t *step_masks, uint32_t *d_step_masks) {
    const uint32_t count = (uint32_t)traces.size();
    const uint64_t n = traces[0].length;
    const bool host = traces[0].host_cols != nullptr;
    const TraceShape shape = TraceShape::of_trace(traces[0].width, traces[0].ctx_depth, traces[0].loop_depth);
    const int w = shape.w, stack_depth = shape.stack_depth, T = shape.T, stk = shape.stack_reg;
    DG_REQUIRE(c.world == 1 && ctx_device_count() == 1,
               "the trace check runs on one GPU: the library was initialised for several (dg_init_devices / dg_comm_init)");
    const fe *periodic = periodic_table(c);
    const int group = check_group_size(w, n, host, d_step_masks == nullptr, count);
    DevBuf d_masks, d_stats;
    std::vector<unsigned long long> stats;
    std::vector<fe> rows_first, rows_last;
    for (uint32_t first = 0; first < count; first += group) {
        const int k = (int)std::min<uint32_t>(group, count - first);
        const fe *regs = traces[first].d_regs;
        if (host) {
            std::vector<const uint8_t *> cols;
            for (int q = 0; q < k; q++) cols.insert(cols.end(), traces[first + q].host_cols, traces[first + q].host_cols + w);
            c.upload_buf.ensure((size_t)k * w * n * 16, true);
            upload_trace_columns(c, c.upload_buf.as<fe>(), cols.data(), k * w, n);
            regs = c.upload_buf.as<fe>();
        }
        unsigned *masks = d_step_masks;
        if (masks) masks += (size_t)first * n * 3;
        else { d_masks.ensure((size_t)k * n * 12); masks = d_masks.as<unsigned>(); }
        d_stats.ensure((size_t)k * CHECK_STATS * 8);

        AirParams P = shape.air_params(n);
        P.log_blowup = 3;
        P.ext = regs; P.col_stride = n; P.ext_stride = (size_t)w * n;
        P.c8_base = 0; P.num_c8 = 1;
        P.periodic = periodic;
        P.masks = masks;
        launch_constraint_check(c, P, k);
        launch_check_reduce(c, masks, n, T, k, d_stats.as<unsigned long long>());

        // the first and last rows: element 0 and n - 1 of every column of the group
        rows_first.resize((size_t)k * w);
        rows_last.resize((size_t)k * w);
        DG_CUDA(cudaMemcpy2DAsync(rows_first.data(), 16, regs, n * 16, 16, (size_t)k * w, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaMemcpy2DAsync(rows_last.data(), 16, regs + (n - 1), n * 16, 16, (size_t)k * w, cudaMemcpyDeviceToHost, c.stream));
        stats.resize((size_t)k * CHECK_STATS);
        DG_CUDA(cudaMemcpyAsync(stats.data(), d_stats.p, stats.size() * 8, cudaMemcpyDeviceToHost, c.stream));
        if (step_masks)
            DG_CUDA(cudaMemcpyAsync(step_masks + (size_t)first * n * 3, masks, (size_t)k * n * 12, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));

        for (int q = 0; q < k; q++) {
            const uint32_t t = first + q;
            dg_trace_report_t &r = reports[t];
            memset(&r, 0, sizeof r);
            const unsigned long long *s = stats.data() + (size_t)q * CHECK_STATS;
            r.n_constraints = (uint32_t)T;
            r.violating_steps = s[CHECK_SLOTS - 1];
            r.first_step = s[2 * CHECK_SLOTS - 1];
            for (int j = 0; j < 128; j++) {
                r.constraint_steps[j] = j < T ? s[j] : 0;
                r.constraint_first[j] = j < T ? s[CHECK_SLOTS + j] : ~0ULL;
            }
            // boundary assertions (evaluator.rs:181-326)
            const fe *f = rows_first.data() + (size_t)q * w, *l = rows_last.data() + (size_t)q * w;
            const fe zero = fe_make(0, 0), one = fe_make(1, 0);
            auto mark = [](uint64_t *bits, int reg) { bits[reg >> 6] |= 1ULL << (reg & 63); };
            for (int j = 0; j < stk; j++) {
                if (!fe_equal(f[j], zero)) mark(r.first_row_registers, j);    // op counter, sponge, op bits, context and loop stacks: 0
                const bool op_bit = j >= 5 && j < 15;
                if (j >= 5 && !fe_equal(l[j], op_bit ? one : zero)) mark(r.last_row_registers, j);   // op bits 1, stacks 0
            }
            const uint32_t ni = n_inputs ? n_inputs[t] : 0, no = n_outputs ? n_outputs[t] : 0;
            for (uint32_t i = 0; i < ni && (int)i < stack_depth; i++) {
                fe v;
                memcpy(&v, inputs16[t] + 16 * (size_t)i, 16);
                if (!fe_equal(f[stk + i], v)) mark(r.first_row_registers, stk + (int)i);
            }
            for (uint32_t i = 0; i < no && (int)i < stack_depth; i++) {
                fe v;
                memcpy(&v, outputs16[t] + 16 * (size_t)i, 16);
                if (!fe_equal(l[stk + i], v)) mark(r.last_row_registers, stk + (int)i);
            }
            // what execute asserts before proving (lib.rs:48-60): at least 16 operations, and the program hash in sponge[0..2]
            r.op_count = l[0].hi ? ~0ULL : l[0].lo;
            r.op_count_ok = (l[0].hi || l[0].lo >= 16) ? 1 : 0;
            r.program_hash_matches = program_hashes32 ? (memcmp(&l[1], program_hashes32 + 32 * (size_t)t, 32) == 0 ? 1 : 0) : -1;
        }
    }
}

}  // namespace dg
