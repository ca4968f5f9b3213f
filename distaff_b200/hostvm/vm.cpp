// Host-side stand-in for the part of Distaff that STAYS on the host: the assembly compiler and the VM
// (`distaff::execute` up to the point where it calls `stark::prove`, /root/reference/src/lib.rs:30-62).
// The Rust host keeps this in production; this container has no Rust toolchain, so tests, smoke() and bench.py
// need a way to produce genuine execution traces (register columns) to feed the prover.  This file mirrors:
//   programs::assembly::compile      /root/reference/src/programs/assembly/{mod.rs:19-317, parsers.rs}
//   programs::blocks / hashing       /root/reference/src/programs/blocks/mod.rs, hashing.rs:16-74, mod.rs:32-52
//   processor::execute               /root/reference/src/processor/{mod.rs:23-182, decoder/mod.rs, stack/mod.rs}
// It is an INPUT GENERATOR: it is neither part of the prove hot path nor of the oracle.
// C-ABI at the bottom (vm_execute / vm_free ...), consumed from Python through ctypes.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include <map>
#include <sstream>
#include <stdexcept>
#include <algorithm>
#include "../csrc/air_constants.h"
#include "../../include/distaff_gpu.h"

namespace vm {

typedef unsigned __int128 u128;
typedef uint64_t u64;
static inline u128 mk(u64 lo, u64 hi) { return ((u128)hi << 64) | lo; }
static const u128 M = mk(0xffffd30000000001ULL, 0xffffffffffffffffULL);
static const u128 C = ((u128)45 << 40) - 1;   // 2^128 = C (mod M)

static inline u128 fadd(u128 a, u128 b) { u128 s = a + b; if (s < a || s >= M) s -= M; return s; }
static inline u128 fsub(u128 a, u128 b) { return a >= b ? a - b : a + (M - b); }
// (a*b) mod M through the identity 2^128 = 45*2^40 - 1 (mod M)
static inline u128 fmul(u128 a, u128 b) {
    u64 a0 = (u64)a, a1 = (u64)(a >> 64), b0 = (u64)b, b1 = (u64)(b >> 64);
    u128 p00 = (u128)a0 * b0, p01 = (u128)a0 * b1, p10 = (u128)a1 * b0, p11 = (u128)a1 * b1;
    u128 mid = (p00 >> 64) + (u64)p01 + (u64)p10;
    u128 lo = ((u128)(u64)mid << 64) | (u64)p00;
    u128 hi = p11 + (p01 >> 64) + (p10 >> 64) + (mid >> 64);
    // fold: value = lo + hi * C ;  hi*C < 2^174
    while (hi != 0) {
        u64 h0 = (u64)hi, h1 = (u64)(hi >> 64);
        u128 q0 = (u128)h0 * (u64)C;                 // C < 2^46 fits one limb
        u128 q1 = (u128)h1 * (u64)C;
        u128 add_lo = q0 + (q1 << 64);
        u128 carry = (q1 >> 64) + ((add_lo < q0) ? 1 : 0);
        u128 nlo = lo + add_lo;
        if (nlo < lo) carry += 1;
        lo = nlo; hi = carry;
    }
    if (lo >= M) lo -= M;
    return lo;
}
static inline u128 fexp(u128 b, u128 p) {
    u128 r = 1;
    while (p) { if (p & 1) r = fmul(r, b); b = fmul(b, b); p >>= 1; }
    return r;
}
static inline u128 finv(u128 x) { return x == 0 ? 0 : fexp(x, M - 2); }
static inline u128 cst(const unsigned long long c[2]) { return mk(c[0], c[1]); }
static const u128 INV_ALPHA = mk(DG_INV_ALPHA[0], DG_INV_ALPHA[1]);

// x^(1/3) = x^INV_ALPHA.  INV_ALPHA = 0xaaaa...8caaaaaaaaab: plain square-and-multiply
static inline u128 cube_root(u128 x) { return x == 0 ? 0 : fexp(x, INV_ALPHA); }
static inline u128 cube(u128 x) { return fmul(fmul(x, x), x); }

template <int W>
static inline void matmul(u128 *s, const unsigned long long (*m)[2]) {
    u128 r[W];
    for (int i = 0; i < W; i++) { r[i] = 0; for (int j = 0; j < W; j++) r[i] = fadd(r[i], fmul(cst(m[i * W + j]), s[j])); }
    for (int i = 0; i < W; i++) s[i] = r[i];
}
// utils/sponge.rs:13-30
static inline void sponge_round(u128 *s, u128 op_code, u128 op_value, size_t step) {
    size_t idx = step % 16;
    for (int i = 0; i < 4; i++) s[i] = cube(fadd(s[i], cst(DG_SPONGE_ARK[i * 16 + idx])));
    matmul<4>(s, DG_SPONGE_MDS);
    s[0] = fadd(s[0], op_code); s[1] = fadd(s[1], op_value);
    for (int i = 0; i < 4; i++) s[i] = cube_root(fadd(s[i], cst(DG_SPONGE_ARK[(4 + i) * 16 + idx])));
    matmul<4>(s, DG_SPONGE_MDS);
}
// utils/hasher.rs:28-40
static inline void hasher_round(u128 *s, size_t step) {
    size_t idx = step % 16;
    for (int i = 0; i < 6; i++) s[i] = cube(fadd(s[i], cst(DG_HASHER_ARK[i * 16 + idx])));
    matmul<6>(s, DG_HASHER_MDS);
    for (int i = 0; i < 6; i++) s[i] = cube_root(fadd(s[i], cst(DG_HASHER_ARK[(6 + i) * 16 + idx])));
    matmul<6>(s, DG_HASHER_MDS);
}

// ---- opcodes (processor/opcodes.rs) ------------------------------------------------------------------------
enum Op : uint8_t {
    ASSERT = 0x60, ASSERTEQ = 0x61, EQ = 0x62, DROP = 0x63, DROP4 = 0x64, CHOOSE = 0x65, CHOOSE2 = 0x66, CSWAP2 = 0x67,
    ADD = 0x68, MUL = 0x69, AND = 0x6a, OR = 0x6b, INV = 0x6c, NEG = 0x6d, NOT = 0x6e,
    READ = 0x70, READ2 = 0x71, DUP = 0x72, DUP2 = 0x73, DUP4 = 0x74, PAD2 = 0x75,
    SWAP = 0x78, SWAP2 = 0x79, SWAP4 = 0x7a, ROLL4 = 0x7b, ROLL8 = 0x7c, BINACC = 0x7d,
    PUSH = 0x1f, CMP = 0x3f, RESCR = 0x5f, BEGIN = 0x00, NOOP = 0x7f,
};
enum FlowOp : uint8_t { HACC = 0, F_BEGIN = 1, TEND = 2, FEND = 3, LOOP = 4, WRAP = 5, BREAK = 6, VOID = 7 };
enum HintKind { H_NONE = 0, H_PUSH, H_EQSTART, H_CMPSTART, H_RCSTART, H_PMPATH };
struct Hint { HintKind kind = H_NONE; u128 value = 0; uint32_t n = 0; };

// ---- program blocks (programs/blocks/mod.rs) ------------------------------------------------------------------
struct Span {
    std::vector<uint8_t> ops;
    std::map<size_t, Hint> hints;
    Hint hint(size_t i) const { auto it = hints.find(i); return it == hints.end() ? Hint() : it->second; }
};
enum BlockKind { B_SPAN, B_GROUP, B_SWITCH, B_LOOP };
struct Block {
    BlockKind kind;
    Span span;
    std::vector<Block> body;      // group body / switch true branch / loop body
    std::vector<Block> alt;       // switch false branch / loop skip
    // hashes carried by a decoded program encoding (dg_block_t): switch true / false branch, loop image / body / skip; when absent the
    // VM hashes the blocks itself
    bool has_hashes = false;
    u128 hashes[3] = {0, 0, 0};
};

static void check_span(const Span &s) {
    if (s.ops.size() % 16 != 15) throw std::runtime_error("span length must be one less than a multiple of 16");
    for (size_t i = 0; i < s.ops.size(); i++)
        if (s.ops[i] == PUSH) {
            if (i % 8 != 0) throw std::runtime_error("PUSH must be on a step which is a multiple of 8");
            if (s.hint(i).kind != H_PUSH) throw std::runtime_error("PUSH value missing");
        }
}
static Block span_block(std::vector<uint8_t> ops, std::map<size_t, Hint> hints = {}) {
    Block b; b.kind = B_SPAN; b.span.ops = std::move(ops); b.span.hints = std::move(hints);
    check_span(b.span);
    return b;
}
static void validate_block_list(const std::vector<Block> &blocks, const std::vector<uint8_t> &starts_with) {
    if (blocks.empty()) throw std::runtime_error("a sequence of blocks must contain at least one block");
    if (blocks[0].kind != B_SPAN) throw std::runtime_error("a sequence of blocks must start with a Span block");
    for (size_t i = 0; i < starts_with.size(); i++)
        if (blocks[0].span.ops.size() <= i || blocks[0].span.ops[i] != starts_with[i]) throw std::runtime_error("invalid first instructions of a branch");
    bool was_span = true;
    for (size_t i = 1; i < blocks.size(); i++) {
        if (blocks[i].kind == B_SPAN) { if (was_span) throw std::runtime_error("a Span block cannot be followed by another Span block"); was_span = true; }
        else was_span = false;
    }
}
static std::vector<uint8_t> loop_skip_ops() { std::vector<uint8_t> v(15, NOOP); v[0] = NOT; v[1] = ASSERT; return v; }

// ---- program hashing (programs/hashing.rs) ----------------------------------------------------------------------
static void block_hash(const Block &b, u128 &v0, u128 &v1);
static void span_hash(const Span &s, u128 st[4]) {
    for (size_t i = 0; i < s.ops.size(); i++) {
        u128 val = s.ops[i] == PUSH ? s.hint(i).value : 0;
        sponge_round(st, s.ops[i], val, i);
    }
}
static void hash_acc(u128 parent, u128 v0, u128 v1, u128 st[4]) {
    st[0] = parent; st[1] = v0; st[2] = v1; st[3] = 0;
    for (size_t i = 1; i < 1 + 14; i++) sponge_round(st, NOOP, 0, i);
}
static u128 hash_seq(const std::vector<Block> &blocks, const std::vector<uint8_t> &suffix, size_t suffix_offset) {
    u128 st[4] = {0, 0, 0, 0};
    span_hash(blocks[0].span, st);
    for (size_t k = 1; k < blocks.size(); k++) {
        const Block &b = blocks[k];
        if (b.kind == B_SPAN) {
            sponge_round(st, NOOP, 0, 15);
            span_hash(b.span, st);
        } else {
            u128 v0, v1;
            block_hash(b, v0, v1);
            u128 ns[4];
            hash_acc(st[0], v0, v1, ns);
            memcpy(st, ns, sizeof ns);
        }
    }
    for (size_t i = 0; i < suffix.size(); i++) sponge_round(st, suffix[i], 0, suffix_offset + i);
    return st[0];
}
static const std::vector<uint8_t> BLOCK_SUFFIX = { NOOP };
static std::vector<uint8_t> loop_suffix() { std::vector<uint8_t> v(16, NOOP); v[0] = NOT; v[1] = ASSERT; return v; }
static void block_hash(const Block &b, u128 &v0, u128 &v1) {
    switch (b.kind) {
        case B_GROUP:  v0 = hash_seq(b.body, BLOCK_SUFFIX, 15); v1 = 0; break;
        case B_SWITCH: v0 = hash_seq(b.body, BLOCK_SUFFIX, 15); v1 = hash_seq(b.alt, BLOCK_SUFFIX, 15); break;
        case B_LOOP:   v0 = hash_seq(b.body, loop_suffix(), 0); v1 = hash_seq(b.alt, BLOCK_SUFFIX, 15); break;
        default: throw std::runtime_error("span has no block hash");
    }
}

// ---- assembler (programs/assembly) ---------------------------------------------------------------------------------
struct Asm {
    std::vector<std::string> tokens;

    static std::vector<std::string> split(const std::string &s, char c) {
        std::vector<std::string> r; std::string cur;
        for (char ch : s) { if (ch == c) { r.push_back(cur); cur.clear(); } else cur.push_back(ch); }
        r.push_back(cur);
        return r;
    }
    static uint32_t param(const std::vector<std::string> &op, bool dflt1 = true) {
        if (op.size() == 1) { if (dflt1) return 1; throw std::runtime_error("missing parameter: " + op[0]); }
        if (op.size() > 2) throw std::runtime_error("extra parameter: " + op[0]);
        size_t pos; unsigned long v = std::stoul(op[1], &pos, 10);
        if (pos != op[1].size() || v == 0) throw std::runtime_error("invalid parameter: " + op[0] + "." + op[1]);
        return (uint32_t)v;
    }
    static u128 value(const std::vector<std::string> &op) {
        if (op.size() != 2) throw std::runtime_error("push needs exactly one parameter");
        const std::string &s = op[1];
        u128 r = 0;
        if (s.rfind("0x", 0) == 0) {
            if (s.size() > 34) throw std::runtime_error("push value too large");
            for (size_t i = 2; i < s.size(); i++) {
                char c = s[i]; int d = c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1;
                if (d < 0) throw std::runtime_error("invalid hex value");
                r = (r << 4) | (u128)d;
            }
        } else {
            for (char c : s) {
                if (c < '0' || c > '9') throw std::runtime_error("invalid decimal value");
                u128 nr = r * 10 + (u128)(c - '0');
                if (nr / 10 != r) throw std::runtime_error("push value too large");
                r = nr;
            }
        }
        if (r >= M) throw std::runtime_error("push value must be smaller than the field modulus");
        return r;
    }
    static void push_op(std::vector<uint8_t> &p, std::map<size_t, Hint> &h, u128 v) {
        size_t pad = (8 - p.size() % 8) % 8;
        p.resize(p.size() + pad, NOOP);
        Hint hh; hh.kind = H_PUSH; hh.value = v;
        h[p.size()] = hh;
        p.push_back(PUSH);
    }
    static void ext(std::vector<uint8_t> &p, std::initializer_list<uint8_t> l) { p.insert(p.end(), l); }
    static void align16(std::vector<uint8_t> &p) { p.resize(p.size() + (16 - p.size() % 16) % 16, NOOP); }

    // parsers.rs
    void parse_op(const std::vector<std::string> &op, std::vector<uint8_t> &p, std::map<size_t, Hint> &h) {
        const std::string &o = op[0];
        auto noparam = [&]() { if (op.size() > 1) throw std::runtime_error("extra parameter: " + o); };
        Hint hint;
        if (o == "noop") { noparam(); p.push_back(NOOP); }
        else if (o == "assert") {
            if (op.size() == 1) p.push_back(ASSERT);
            else if (op.size() == 2 && op[1] == "eq") p.push_back(ASSERTEQ);
            else throw std::runtime_error("invalid assert parameter");
        }
        else if (o == "push") push_op(p, h, value(op));
        else if (o == "read") {
            if (op.size() == 1 || (op.size() == 2 && op[1] == "a")) p.push_back(READ);
            else if (op.size() == 2 && op[1] == "ab") p.push_back(READ2);
            else throw std::runtime_error("invalid read parameter");
        }
        else if (o == "dup") { switch (param(op)) { case 1: p.push_back(DUP); break; case 2: p.push_back(DUP2); break;
            case 3: ext(p, {DUP4, ROLL4, DROP}); break; case 4: p.push_back(DUP4); break; default: throw std::runtime_error("invalid dup parameter"); } }
        else if (o == "pad") { switch (param(op)) {
            case 1: ext(p, {PAD2, DROP}); break; case 2: ext(p, {PAD2}); break; case 3: ext(p, {PAD2, PAD2, DROP}); break;
            case 4: ext(p, {PAD2, PAD2}); break; case 5: ext(p, {PAD2, PAD2, PAD2, DROP}); break; case 6: ext(p, {PAD2, PAD2, PAD2}); break;
            case 7: ext(p, {PAD2, PAD2, DUP4, DROP}); break; case 8: ext(p, {PAD2, PAD2, DUP4}); break; default: throw std::runtime_error("invalid pad parameter"); } }
        else if (o == "pick") { switch (param(op)) {
            case 1: ext(p, {DUP2, DROP}); break; case 2: ext(p, {DUP4, ROLL4, DROP, DROP, DROP}); break; case 3: ext(p, {DUP4, DROP, DROP, DROP}); break;
            default: throw std::runtime_error("invalid pick parameter"); } }
        else if (o == "drop") { switch (param(op)) {
            case 1: ext(p, {DROP}); break; case 2: ext(p, {DROP, DROP}); break; case 3: ext(p, {DUP, DROP4}); break; case 4: ext(p, {DROP4}); break;
            case 5: ext(p, {DROP, DROP4}); break; case 6: ext(p, {DROP, DROP, DROP4}); break; case 7: ext(p, {DUP, DROP4, DROP4}); break;
            case 8: ext(p, {DROP4, DROP4}); break; default: throw std::runtime_error("invalid drop parameter"); } }
        else if (o == "swap") { switch (param(op)) { case 1: p.push_back(SWAP); break; case 2: p.push_back(SWAP2); break; case 4: p.push_back(SWAP4); break;
            default: throw std::runtime_error("invalid swap parameter"); } }
        else if (o == "roll") { switch (param(op)) { case 4: p.push_back(ROLL4); break; case 8: p.push_back(ROLL8); break; default: throw std::runtime_error("invalid roll parameter"); } }
        else if (o == "add") { noparam(); p.push_back(ADD); }
        else if (o == "sub") { noparam(); ext(p, {NEG, ADD}); }
        else if (o == "mul") { noparam(); p.push_back(MUL); }
        else if (o == "div") { noparam(); ext(p, {INV, MUL}); }
        else if (o == "neg") { noparam(); p.push_back(NEG); }
        else if (o == "inv") { noparam(); p.push_back(INV); }
        else if (o == "not") { noparam(); p.push_back(NOT); }
        else if (o == "and") { noparam(); p.push_back(AND); }
        else if (o == "or") { noparam(); p.push_back(OR); }
        else if (o == "eq") { noparam(); hint.kind = H_EQSTART; h[p.size()] = hint; ext(p, {READ, EQ}); }
        else if (o == "ne") { noparam(); hint.kind = H_EQSTART; h[p.size()] = hint; ext(p, {READ, EQ, NOT}); }
        else if (o == "gt" || o == "lt") {
            uint32_t n = param(op);
            if (n < 4 || n > 128) throw std::runtime_error("gt/lt parameter must be between 4 and 128");
            ext(p, {PAD2, PAD2, PAD2, DUP});
            push_op(p, h, (u128)1 << (n - 1));
            hint.kind = H_CMPSTART; hint.n = n; h[p.size()] = hint;
            p.resize(p.size() + n, CMP);
            if (o == "gt") ext(p, {DROP4, PAD2, SWAP4, ROLL4, ASSERTEQ, ASSERTEQ, ROLL4, DUP, DROP4});
            else ext(p, {DROP4, PAD2, SWAP4, ROLL4, ASSERTEQ, ASSERTEQ, DUP, DROP4});
        }
        else if (o == "rc") {
            uint32_t n = param(op);
            if (n < 4 || n > 128) throw std::runtime_error("rc parameter must be between 4 and 128");
            p.push_back(PAD2); push_op(p, h, 1); ext(p, {SWAP, DUP});
            hint.kind = H_RCSTART; hint.n = n; h[p.size()] = hint;
            p.resize(p.size() + n, BINACC);
            ext(p, {DUP, DROP4});
            Hint e; e.kind = H_EQSTART; h[p.size()] = e;
            ext(p, {READ, EQ});
        }
        else if (o == "isodd") {
            uint32_t n = param(op);
            if (n < 4 || n > 128) throw std::runtime_error("isodd parameter must be between 4 and 128");
            p.push_back(PAD2); push_op(p, h, 1); ext(p, {SWAP, DUP});
            hint.kind = H_RCSTART; hint.n = n; h[p.size()] = hint;
            ext(p, {BINACC, SWAP2, ROLL4, DUP});
            p.resize(p.size() + (n - 1), BINACC);
            ext(p, {DROP, DROP, SWAP, ROLL4, ASSERTEQ, DROP});
        }
        else if (o == "choose") { switch (param(op)) { case 1: p.push_back(CHOOSE); break; case 2: p.push_back(CHOOSE2); break; default: throw std::runtime_error("invalid choose parameter"); } }
        else if (o == "hash") {
            switch (param(op)) { case 1: ext(p, {PAD2, PAD2, PAD2, DROP}); break; case 2: ext(p, {PAD2, PAD2}); break; case 3: ext(p, {PAD2, PAD2, DROP}); break;
                case 4: ext(p, {PAD2}); break; default: throw std::runtime_error("invalid hash parameter"); }
            align16(p);
            p.resize(p.size() + 10, RESCR);
            p.push_back(DROP4);
        }
        else if (o == "smpath") {
            uint32_t n = param(op);
            if (n < 2 || n > 256) throw std::runtime_error("smpath parameter must be between 2 and 256");
            ext(p, {READ2, SWAP2, READ2, CSWAP2, PAD2});
            align16(p);
            static const uint8_t SUB[16] = { RESCR, RESCR, RESCR, RESCR, RESCR, RESCR, RESCR, RESCR, RESCR, RESCR, DROP4, READ2, SWAP2, READ2, CSWAP2, PAD2 };
            for (uint32_t i = 0; i < n - 2; i++) p.insert(p.end(), SUB, SUB + 16);
            p.insert(p.end(), SUB, SUB + 11);
        }
        else if (o == "pmpath") {
            uint32_t n = param(op);
            if (n < 2 || n > 256) throw std::runtime_error("pmpath parameter must be between 2 and 256");
            hint.kind = H_PMPATH; hint.n = n; h[p.size()] = hint;
            ext(p, {READ2, PAD2});
            push_op(p, h, 1);
            ext(p, {SWAP, DUP, BINACC, SWAP4, CSWAP2, PAD2});
            align16(p);
            static const uint8_t SUB[32] = { RESCR, RESCR, RESCR, RESCR, RESCR, RESCR, RESCR, RESCR, RESCR, RESCR, DROP4, PAD2, SWAP2, READ2, SWAP4, BINACC,
                SWAP4, CSWAP2, PAD2, NOOP, NOOP, NOOP, NOOP, NOOP, NOOP, NOOP, NOOP, NOOP, NOOP, NOOP, NOOP, NOOP };
            for (uint32_t i = 0; i < n - 2; i++) p.insert(p.end(), SUB, SUB + 32);
            p.insert(p.end(), SUB, SUB + 11);
            ext(p, {SWAP2, DROP, ROLL4, ASSERTEQ});
        }
        else throw std::runtime_error("invalid operation: " + o);
    }

    static void add_span(std::vector<Block> &body, std::vector<uint8_t> &ops, std::map<size_t, Hint> &hints, bool force) {
        if (ops.empty() && !force) return;
        std::vector<uint8_t> padded(ops);
        size_t pad = 16 - (padded.size() % 16) - 1;
        padded.resize(padded.size() + pad, NOOP);
        body.push_back(span_block(padded, hints));
        ops.clear(); hints.clear();
    }
    static Span merge_spans(const Span &a, const Span &b) {
        Span r; r.ops = a.ops; r.ops.push_back(NOOP); r.ops.insert(r.ops.end(), b.ops.begin(), b.ops.end());
        r.hints = a.hints;
        size_t off = a.ops.size() + 1;
        for (auto &kv : b.hints) r.hints[kv.first + off] = kv.second;
        check_span(r);
        return r;
    }
    static std::vector<Block> repeat_seq(const std::vector<Block> &tmpl, size_t iters) {
        std::vector<Block> body;
        if (tmpl.back().kind != B_SPAN) { for (size_t i = 0; i < iters; i++) body.insert(body.end(), tmpl.begin(), tmpl.end()); }
        else {
            body = tmpl;
            for (size_t i = 1; i < iters; i++) {
                body.back().span = merge_spans(body.back().span, tmpl[0].span);
                body.insert(body.end(), tmpl.begin() + 1, tmpl.end());
            }
        }
        return body;
    }

    size_t parse_block(std::vector<Block> &parent, size_t i) {
        std::vector<std::string> head = split(tokens[i], '.');
        if (head[0] == "block") {
            if (head.size() > 1) throw std::runtime_error("invalid block head");
            Block b; b.kind = B_GROUP;
            i = parse_branch(b.body, i);
            validate_block_list(b.body, {});
            parent.push_back(b);
            return i + 1;
        } else if (head[0] == "if") {
            if (head.size() == 1 || head[1] != "true") throw std::runtime_error("invalid if head");
            Block b; b.kind = B_SWITCH;
            i = parse_branch(b.body, i);
            if (tokens[i] == "else") i = parse_branch(b.alt, i);
            else b.alt.push_back(span_block(loop_skip_ops()));
            validate_block_list(b.body, {ASSERT});
            validate_block_list(b.alt, {NOT, ASSERT});
            parent.push_back(b);
            return i + 1;
        } else if (head[0] == "repeat") {
            if (head.size() != 2) throw std::runtime_error("invalid repeat head");
            size_t iters = std::stoul(head[1]);
            if (iters < 2) throw std::runtime_error("invalid number of iterations");
            std::vector<Block> tmpl;
            i = parse_branch(tmpl, i);
            Block b; b.kind = B_GROUP;
            b.body = repeat_seq(tmpl, iters);
            validate_block_list(b.body, {});
            parent.push_back(b);
            return i + 1;
        } else if (head[0] == "while") {
            if (head.size() == 1 || head[1] != "true") throw std::runtime_error("invalid while head");
            Block b; b.kind = B_LOOP;
            i = parse_branch(b.body, i);
            validate_block_list(b.body, {ASSERT});
            b.alt.push_back(span_block(loop_skip_ops()));
            parent.push_back(b);
            return i + 1;
        }
        throw std::runtime_error("invalid block head: " + tokens[i]);
    }
    size_t parse_branch(std::vector<Block> &body, size_t i) {
        std::vector<std::string> head = split(tokens[i], '.');
        std::vector<uint8_t> ops;
        if (head[0] == "begin") { head[0] = "block"; ops = {BEGIN}; }
        else if (head[0] == "block" || head[0] == "repeat") {}
        else if (head[0] == "if" || head[0] == "while") ops = {ASSERT};
        else if (head[0] == "else") ops = {NOT, ASSERT};
        else throw std::runtime_error("invalid block head: " + tokens[i]);
        std::map<size_t, Hint> hints;
        size_t first = i;
        i += 1;
        while (i < tokens.size()) {
            std::vector<std::string> op = split(tokens[i], '.');
            if (op[0] == "block" || op[0] == "if" || op[0] == "repeat" || op[0] == "while") {
                bool force = body.empty();
                add_span(body, ops, hints, force);
                i = parse_block(body, i);
            } else if (op[0] == "else") {
                if (head[0] != "if") throw std::runtime_error("dangling else");
                if (i - first < 2) throw std::runtime_error("empty block");
                add_span(body, ops, hints, false);
                return i;
            } else if (op[0] == "end") {
                if (i - first < 2) throw std::runtime_error("empty block");
                add_span(body, ops, hints, false);
                return i;
            } else { parse_op(op, ops, hints); i += 1; }
        }
        throw std::runtime_error("unmatched block");
    }
};

struct Program { Block root; u128 hash[2]; };

static Program compile(const std::string &source) {
    Asm a;
    std::istringstream ss(source);
    std::string t;
    while (ss >> t) a.tokens.push_back(t);
    if (a.tokens.empty()) throw std::runtime_error("empty program");
    if (a.tokens[0] != "begin") throw std::runtime_error("a program must start with 'begin'");
    if (a.tokens.back() != "end") throw std::runtime_error("a program must end with 'end'");
    Program p;
    p.root.kind = B_GROUP;
    size_t i = a.parse_branch(p.root.body, 0);
    validate_block_list(p.root.body, {});
    if (i < a.tokens.size() - 1) throw std::runtime_error("dangling instructions");
    if (p.root.body[0].span.ops[0] != BEGIN) throw std::runtime_error("a program must start with BEGIN operation");
    u128 v0, v1, st[4];
    block_hash(p.root, v0, v1);
    hash_acc(0, v0, v1, st);
    p.hash[0] = st[0]; p.hash[1] = st[1];
    return p;
}

// ---- processor (processor/decoder/mod.rs + processor/stack/mod.rs) ------------------------------------------------------
struct Machine {
    // decoder
    size_t step = 0, len = 16;
    std::vector<u128> op_counter;
    std::vector<u128> sponge_trace[4];
    u128 sponge[4] = {0, 0, 0, 0};
    std::vector<u128> cf[3], ld[5], hd[2];
    std::vector<std::vector<u128>> ctx_stack, loop_stack;
    size_t ctx_depth = 1, loop_depth = 0;
    // stack
    std::vector<std::vector<u128>> regs;
    std::vector<u128> tape_a, tape_b;
    size_t max_depth, depth;

    Machine(const std::vector<u128> &pub, std::vector<u128> sa, std::vector<u128> sb) {
        op_counter.assign(len, 0);
        for (auto &r : sponge_trace) r.assign(len, 0);
        for (auto &r : cf) r.assign(len, 0);
        for (auto &r : ld) r.assign(len, 0);
        for (auto &r : hd) r.assign(len, 0);
        ctx_stack.push_back(std::vector<u128>(len, 0));
        size_t init_depth = std::max(pub.size(), (size_t)8);
        for (size_t i = 0; i < init_depth; i++) { regs.push_back(std::vector<u128>(len, 0)); if (i < pub.size()) regs[i][0] = pub[i]; }
        std::reverse(sa.begin(), sa.end()); std::reverse(sb.begin(), sb.end());
        tape_a = std::move(sa); tape_b = std::move(sb);
        max_depth = depth = pub.size();
    }
    void fail(const std::string &m) const { throw std::runtime_error(m + " at step " + std::to_string(step)); }

    // both components advance in lock-step (decoder first, then stack), so one `step`/`len` serves both
    void advance(bool user_op) {
        step += 1;
        if (step >= len) {
            size_t nl = len * 2;
            op_counter.resize(nl, 0);
            for (auto &r : sponge_trace) r.resize(nl, 0);
            for (auto &r : cf) r.resize(nl, 0);
            for (auto &r : ld) r.resize(nl, 0);
            for (auto &r : hd) r.resize(nl, 0);
            for (auto &r : ctx_stack) r.resize(nl, 0);
            for (auto &r : loop_stack) r.resize(nl, 0);
            for (auto &r : regs) r.resize(nl, 0);
            len = nl;
        }
        op_counter[step] = op_counter[step - 1] + (user_op ? 1 : 0);
    }
    void set_op_bits(uint8_t flow, uint8_t user) {
        size_t s = step - 1;
        for (int i = 0; i < 3; i++) cf[i][s] = (flow >> i) & 1;
        for (int i = 0; i < 5; i++) ld[i][s] = (user >> i) & 1;
        for (int i = 0; i < 2; i++) hd[i][s] = (user >> (i + 5)) & 1;
    }
    void set_sponge(u128 a, u128 b, u128 c, u128 d) {
        sponge[0] = a; sponge[1] = b; sponge[2] = c; sponge[3] = d;
        for (int i = 0; i < 4; i++) sponge_trace[i][step] = sponge[i];
    }
    void save_context() {
        ctx_depth += 1;
        if (ctx_depth > 16) fail("context stack overflow");
        if (ctx_depth > ctx_stack.size()) ctx_stack.push_back(std::vector<u128>(len, 0));
        for (size_t i = 1; i < ctx_stack.size(); i++) ctx_stack[i][step] = ctx_stack[i - 1][step - 1];
        ctx_stack[0][step] = sponge[0];
    }
    u128 pop_context() {
        if (ctx_depth == 0) fail("context stack underflow");
        for (size_t i = 1; i < ctx_stack.size(); i++) ctx_stack[i - 1][step] = ctx_stack[i][step - 1];
        ctx_depth -= 1;
        return ctx_stack[0][step - 1];
    }
    void copy_ctx() { for (auto &r : ctx_stack) r[step] = r[step - 1]; }
    void copy_loop() { for (auto &r : loop_stack) r[step] = r[step - 1]; }
    void save_loop_image(u128 image) {
        loop_depth += 1;
        if (loop_depth > 8) fail("loop stack overflow");
        if (loop_depth > loop_stack.size()) loop_stack.push_back(std::vector<u128>(len, 0));
        for (size_t i = 1; i < loop_stack.size(); i++) loop_stack[i][step] = loop_stack[i - 1][step - 1];
        loop_stack[0][step] = image;
    }
    u128 peek_loop_image() { if (loop_depth == 0) fail("loop stack underflow"); copy_loop(); return loop_stack[0][step]; }
    u128 pop_loop_image() {
        if (loop_depth == 0) fail("loop stack underflow");
        for (size_t i = 1; i < loop_stack.size(); i++) loop_stack[i - 1][step] = loop_stack[i][step - 1];
        loop_depth -= 1;
        return loop_stack[0][step - 1];
    }

    // ---- decoder ops; each is followed by the matching stack op through `exec`
    void start_block() {
        if (step % 16 != 15) fail("cannot start context block: invalid alignment");
        advance(false); save_context(); copy_loop(); set_op_bits(F_BEGIN, NOOP); set_sponge(0, 0, 0, 0);
        stack_op(NOOP, Hint());
    }
    void end_block(u128 sibling, bool true_branch) {
        if (step % 16 != 0) fail("cannot exit context block: invalid alignment");
        advance(false);
        u128 ctx_hash = pop_context();
        copy_loop();
        u128 block_hash = sponge[0];
        if (true_branch) { set_op_bits(TEND, NOOP); set_sponge(ctx_hash, block_hash, sibling, 0); }
        else { set_op_bits(FEND, NOOP); set_sponge(ctx_hash, sibling, block_hash, 0); }
        stack_op(NOOP, Hint());
    }
    void start_loop(u128 image) {
        if (step % 16 != 15) fail("cannot start a loop: invalid alignment");
        advance(false); save_context(); save_loop_image(image); set_op_bits(LOOP, NOOP); set_sponge(0, 0, 0, 0);
        stack_op(NOOP, Hint());
    }
    void wrap_loop() {
        if (step % 16 != 15) fail("cannot wrap a loop: invalid alignment");
        advance(false); copy_ctx();
        if (sponge[0] != peek_loop_image()) fail("hash of the last iteration doesn't match loop image");
        set_op_bits(WRAP, NOOP); set_sponge(0, 0, 0, 0);
        stack_op(NOOP, Hint());
    }
    void break_loop() {
        if (step % 16 != 15) fail("cannot break a loop: invalid alignment");
        advance(false); copy_ctx();
        if (sponge[0] != pop_loop_image()) fail("hash of the last iteration doesn't match loop image");
        set_op_bits(BREAK, NOOP); set_sponge(sponge[0], sponge[1], sponge[2], sponge[3]);
        stack_op(NOOP, Hint());
    }
    void exec(uint8_t op, const Hint &hint) {
        u128 op_value = hint.kind == H_PUSH ? hint.value : 0;
        if (op_value != 0) {
            if (op != PUSH) fail("op_value is non-zero for a non-PUSH operation");
            if (step % 8 != 0) fail("invalid PUSH operation alignment");
        }
        advance(true); copy_ctx(); copy_loop(); set_op_bits(HACC, op);
        sponge_round(sponge, op, op_value, step - 1);
        for (int i = 0; i < 4; i++) sponge_trace[i][step] = sponge[i];
        stack_op(op, hint);
    }

    // ---- stack (processor/stack/mod.rs); operates on row `step` (already advanced by the decoder)
    u128 top() const { return regs[0][step]; }
    void copy_state(size_t start) { for (size_t i = start; i < depth; i++) regs[i][step] = regs[i][step - 1]; }
    void shift_left(size_t start, size_t cnt) {
        if (depth < cnt) fail("stack underflow");
        for (size_t i = start; i < depth; i++) regs[i - cnt][step] = regs[i][step - 1];
        for (size_t i = depth - cnt; i < depth; i++) regs[i][step] = 0;
        depth -= cnt;
    }
    void shift_right(size_t start, size_t cnt) {
        depth += cnt;
        if (depth > 32) fail("stack overflow");
        if (depth > max_depth) {
            max_depth += cnt;
            while (max_depth > regs.size()) regs.push_back(std::vector<u128>(len, 0));
        }
        for (size_t i = start; i < depth - cnt; i++) regs[i + cnt][step] = regs[i][step - 1];
    }
    void need(size_t d) { if (depth < d) fail("stack underflow"); }
    static bool is_bin(u128 v) { return v == 0 || v == 1; }
    static bool is_pow2(u128 v) { return v != 0 && (v & (v - 1)) == 0; }

    void stack_op(uint8_t op, const Hint &hint) {
        const size_t s = step, p = step - 1;
        auto R = [&](size_t i) -> u128 { return regs[i][p]; };
        switch (op) {
        case BEGIN: case NOOP: copy_state(0); break;
        case ASSERT: need(1); if (R(0) != 1) fail("ASSERT failed"); shift_left(1, 1); break;
        case ASSERTEQ: need(2); if (R(0) != R(1)) fail("ASSERTEQ failed"); shift_left(2, 2); break;
        case PUSH: if (hint.kind != H_PUSH) fail("invalid value for PUSH"); shift_right(0, 1); regs[0][s] = hint.value; break;
        case READ:
            if (hint.kind == H_EQSTART) {
                need(2);
                u128 x = R(0), y = R(1);
                tape_a.push_back(x == y ? (u128)1 : finv(fsub(x, y)));
            } else if (hint.kind == H_NONE) { if (tape_a.empty()) fail("attempt to read from empty tape A"); }
            else fail("invalid hint for READ");
            shift_right(0, 1);
            regs[0][s] = tape_a.back(); tape_a.pop_back();
            break;
        case READ2:
            if (hint.kind == H_PMPATH) {
                need(3);
                size_t n = hint.n - 1;
                if (tape_a.size() < n || tape_b.size() < n) fail("too few items on tapes for pmpath macro");
                u128 idx = R(2);
                std::vector<u128> va(tape_a.end() - n, tape_a.end());
                tape_a.resize(tape_a.size() - n);
                // bit k of the index, 0 from bit 128 on (a shift by 128 or more is undefined in C++; the GPU VM's bit_of does the same)
                for (size_t i = 0; i < n; i++) {
                    const size_t k = n - i - 1;
                    tape_a.push_back(k < 128 ? (idx >> k) & 1 : 0);
                    tape_a.push_back(va[i]);
                }
            } else if (hint.kind == H_NONE) { if (tape_a.empty() || tape_b.empty()) fail("attempt to read from empty tape"); }
            else fail("invalid hint for READ2");
            shift_right(0, 2);
            {
                u128 a = tape_a.back(); tape_a.pop_back();
                u128 b = tape_b.back(); tape_b.pop_back();
                regs[0][s] = b; regs[1][s] = a;
            }
            break;
        case DUP: need(1); shift_right(0, 1); regs[0][s] = R(0); break;
        case DUP2: need(2); shift_right(0, 2); regs[0][s] = R(0); regs[1][s] = R(1); break;
        case DUP4: need(4); shift_right(0, 4); for (int i = 0; i < 4; i++) regs[i][s] = R(i); break;
        case PAD2: shift_right(0, 2); regs[0][s] = 0; regs[1][s] = 0; break;
        case DROP: need(1); shift_left(1, 1); break;
        case DROP4: need(4); shift_left(4, 4); break;
        case SWAP: need(2); regs[0][s] = R(1); regs[1][s] = R(0); copy_state(2); break;
        case SWAP2: need(4); regs[0][s] = R(2); regs[1][s] = R(3); regs[2][s] = R(0); regs[3][s] = R(1); copy_state(4); break;
        case SWAP4: need(8); for (int i = 0; i < 4; i++) { regs[i][s] = R(4 + i); regs[4 + i][s] = R(i); } copy_state(8); break;
        case ROLL4: need(4); regs[0][s] = R(3); for (int i = 1; i < 4; i++) regs[i][s] = R(i - 1); copy_state(4); break;
        case ROLL8: need(8); regs[0][s] = R(7); for (int i = 1; i < 8; i++) regs[i][s] = R(i - 1); copy_state(8); break;
        case CHOOSE: {
            need(3);
            u128 c = R(2);
            if (c == 1) regs[0][s] = R(0); else if (c == 0) regs[0][s] = R(1); else fail("CHOOSE on a non-binary condition");
            shift_left(3, 2); break; }
        case CHOOSE2: {
            need(6);
            u128 c = R(4);
            if (c == 1) { regs[0][s] = R(0); regs[1][s] = R(1); } else if (c == 0) { regs[0][s] = R(2); regs[1][s] = R(3); }
            else fail("CHOOSE2 on a non-binary condition");
            shift_left(6, 4); break; }
        case CSWAP2: {
            need(6);
            u128 c = R(4);
            if (c == 0) { for (int i = 0; i < 4; i++) regs[i][s] = R(i); }
            else if (c == 1) { regs[0][s] = R(2); regs[1][s] = R(3); regs[2][s] = R(0); regs[3][s] = R(1); }
            else fail("CSWAP2 on a non-binary condition");
            shift_left(6, 2); break; }
        case ADD: need(2); regs[0][s] = fadd(R(0), R(1)); shift_left(2, 1); break;
        case MUL: need(2); regs[0][s] = fmul(R(0), R(1)); shift_left(2, 1); break;
        case INV: need(1); if (R(0) == 0) fail("cannot compute INV of 0"); regs[0][s] = finv(R(0)); copy_state(1); break;
        case NEG: need(1); regs[0][s] = fsub(0, R(0)); copy_state(1); break;
        case NOT: need(1); if (!is_bin(R(0))) fail("NOT of a non-binary value"); regs[0][s] = fsub(1, R(0)); copy_state(1); break;
        case AND: need(2); if (!is_bin(R(0)) || !is_bin(R(1))) fail("AND of a non-binary value");
            regs[0][s] = (R(0) == 1 && R(1) == 1) ? 1 : 0; shift_left(2, 1); break;
        case OR: need(2); if (!is_bin(R(0)) || !is_bin(R(1))) fail("OR of a non-binary value");
            regs[0][s] = (R(0) == 1 || R(1) == 1) ? 1 : 0; shift_left(2, 1); break;
        case EQ: {
            need(3);
            u128 aux = R(0), x = R(1), y = R(2);
            if (x == y) regs[0][s] = 1;
            else { if (aux != finv(fsub(x, y))) fail("invalid AUX value for EQ"); regs[0][s] = 0; }
            shift_left(3, 2); break; }
        case CMP: {
            if (hint.kind == H_CMPSTART) {
                need(10);
                u128 a = R(8), b = R(9);
                for (uint32_t i = 0; i < hint.n; i++) { tape_a.push_back((a >> i) & 1); tape_b.push_back((b >> i) & 1); }
            } else if (hint.kind == H_NONE) { need(8); if (tape_a.empty() || tape_b.empty()) fail("attempt to read from empty tape"); }
            else fail("invalid hint for CMP");
            u128 a_bit = tape_a.back(); tape_a.pop_back();
            u128 b_bit = tape_b.back(); tape_b.pop_back();
            if (!is_bin(a_bit) || !is_bin(b_bit)) fail("expected binary input");
            u128 bit_gt = fmul(a_bit, fsub(1, b_bit)), bit_lt = fmul(b_bit, fsub(1, a_bit));
            u128 p2 = R(0);
            if (!is_pow2(p2)) fail("expected top of the stack to be a power of 2");
            u128 np2 = p2 == 1 ? fmul(p2, finv(2)) : p2 >> 1;
            u128 gt = R(4), lt = R(5);
            u128 not_set = fmul(fsub(1, gt), fsub(1, lt));
            regs[0][s] = np2; regs[1][s] = a_bit; regs[2][s] = b_bit; regs[3][s] = not_set;
            regs[4][s] = fadd(gt, fmul(bit_gt, not_set)); regs[5][s] = fadd(lt, fmul(bit_lt, not_set));
            regs[6][s] = fadd(R(6), fmul(b_bit, p2)); regs[7][s] = fadd(R(7), fmul(a_bit, p2));
            copy_state(8); break; }
        case BINACC: {
            if (hint.kind == H_RCSTART) {
                need(5);
                u128 v = R(4);
                for (uint32_t i = 0; i < hint.n; i++) tape_a.push_back((v >> (hint.n - i - 1)) & 1);
            } else if (hint.kind == H_NONE) { need(4); if (tape_a.empty()) fail("attempt to read from empty tape A"); }
            else fail("invalid hint for BINACC");
            u128 bit = tape_a.back(); tape_a.pop_back();
            if (!is_bin(bit)) fail("expected binary input");
            u128 p2 = R(2);
            if (!is_pow2(p2)) fail("expected 3rd value from the top of the stack to be a power of 2");
            regs[0][s] = bit; regs[1][s] = 0; regs[2][s] = fmul(p2, 2); regs[3][s] = fadd(R(3), fmul(bit, p2));
            copy_state(4); break; }
        case RESCR: {
            need(6);
            u128 st[6];
            for (int i = 0; i < 6; i++) st[i] = R(i);
            hasher_round(st, p);
            for (int i = 0; i < 6; i++) regs[i][s] = st[i];
            copy_state(6); break; }
        default: fail("unknown opcode");
        }
    }

    // ---- processor/mod.rs:50-182
    void close_block(u128 sibling, bool true_branch) {
        exec(NOOP, Hint());
        end_block(sibling, true_branch);
        for (int i = 0; i < 14; i++) exec(NOOP, Hint());
    }
    void run_span(const Span &sp, bool is_first) {
        if (!is_first) exec(NOOP, Hint());
        for (size_t i = 0; i < sp.ops.size(); i++) exec(sp.ops[i], sp.hint(i));
    }
    void run_blocks(const std::vector<Block> &blocks) {
        if (blocks[0].kind != B_SPAN) fail("first block in a sequence must be a Span block");
        run_span(blocks[0].span, true);
        for (size_t k = 1; k < blocks.size(); k++) {
            const Block &b = blocks[k];
            switch (b.kind) {
            case B_SPAN: run_span(b.span, false); break;
            case B_GROUP: start_block(); run_blocks(b.body); close_block(0, true); break;
            case B_SWITCH: {
                start_block();
                u128 c = top();
                if (c == 0) { run_blocks(b.alt); close_block(b.has_hashes ? b.hashes[0] : hash_seq(b.body, BLOCK_SUFFIX, 15), false); }
                else if (c == 1) { run_blocks(b.body); close_block(b.has_hashes ? b.hashes[1] : hash_seq(b.alt, BLOCK_SUFFIX, 15), true); }
                else fail("cannot select a branch based on a non-binary condition");
                break; }
            case B_LOOP: {
                u128 c = top();
                if (c == 0) { start_block(); run_blocks(b.alt); close_block(b.has_hashes ? b.hashes[1] : hash_seq(b.body, loop_suffix(), 0), false); }
                else if (c == 1) {
                    u128 image = b.has_hashes ? b.hashes[0] : hash_seq(b.body, {}, 0);
                    u128 skip_hash = b.has_hashes ? b.hashes[2] : hash_seq(b.alt, BLOCK_SUFFIX, 15);
                    start_loop(image);
                    for (;;) {
                        run_blocks(b.body);
                        u128 cc = top();
                        if (cc == 0) { break_loop(); break; }
                        else if (cc == 1) wrap_loop();
                        else fail("cannot exit loop based on a non-binary condition");
                    }
                    run_span(b.alt[0].span, true);
                    close_block(skip_hash, true);
                } else fail("cannot enter loop based on a non-binary condition");
                break; }
            }
        }
    }
    static void fill(std::vector<u128> &r, size_t from, u128 v) { for (size_t i = from; i < r.size(); i++) r[i] = v; }
    void finalize() {
        u128 last = op_counter[step];
        fill(op_counter, step + 1, last);
        for (auto &r : cf) fill(r, step, 1);
        for (auto &r : ld) fill(r, step, 1);
        for (auto &r : hd) fill(r, step, 1);
        for (auto &r : sponge_trace) fill(r, step + 1, r[step]);
        for (auto &r : ctx_stack) fill(r, step + 1, r[step]);
        for (auto &r : loop_stack) fill(r, step + 1, r[step]);
        for (auto &r : regs) fill(r, step + 1, r[step]);
    }
};

struct Execution {
    std::vector<std::vector<u128>> registers;
    size_t ctx_depth, loop_depth, stack_depth;
    u128 program_hash[2];
    std::string error;
};

static Execution *run(const Program *prog, const std::string *source, const std::vector<u128> &pub, const std::vector<u128> &sa,
                      const std::vector<u128> &sb) {
    Execution *e = new Execution();
    try {
        if (pub.size() > 8) throw std::runtime_error("expected no more than 8 public inputs");
        if (sa.size() < sb.size()) throw std::runtime_error("tape A cannot be shorter than tape B");
        // the field arithmetic assumes canonical operands (the reference does not check; see include/distaff_gpu.h)
        auto check = [](const std::vector<u128> &v, const char *what) {
            for (size_t i = 0; i < v.size(); i++)
                if (v[i] >= M) throw std::runtime_error(std::string(what) + " " + std::to_string(i) + " is not a field element");
        };
        check(pub, "public input");
        check(sa, "tape A value");
        check(sb, "tape B value");
        Program compiled;
        if (!prog) { compiled = compile(*source); prog = &compiled; }
        Machine m(pub, sa, sb);
        m.run_blocks(prog->root.body);
        m.close_block(0, true);
        m.finalize();
        e->ctx_depth = m.ctx_stack.size() - 1;
        e->loop_depth = m.loop_stack.size();
        e->stack_depth = m.max_depth;
        auto &r = e->registers;
        r.push_back(std::move(m.op_counter));
        for (auto &x : m.sponge_trace) r.push_back(std::move(x));
        for (auto &x : m.cf) r.push_back(std::move(x));
        for (auto &x : m.ld) r.push_back(std::move(x));
        for (auto &x : m.hd) r.push_back(std::move(x));
        m.ctx_stack.pop_back();   // outer-most context is always 0 (decoder/mod.rs:149-151)
        for (auto &x : m.ctx_stack) r.push_back(std::move(x));
        for (auto &x : m.loop_stack) r.push_back(std::move(x));
        for (size_t i = 0; i < m.max_depth; i++) r.push_back(std::move(m.regs[i]));
        e->program_hash[0] = prog->hash[0]; e->program_hash[1] = prog->hash[1];
        // lib.rs:49-59
        size_t n = r[0].size();
        if (r[0][n - 1] < 16) throw std::runtime_error("a program must consist of at least 16 operations");
        if (r[1][n - 1] != prog->hash[0] || r[2][n - 1] != prog->hash[1]) throw std::runtime_error("program hash does not match trace hash");
    } catch (std::exception &ex) { e->error = ex.what(); }
    return e;
}
static Execution *execute(const std::string &source, const std::vector<u128> &pub, const std::vector<u128> &sa, const std::vector<u128> &sb) {
    return run(nullptr, &source, pub, sa, sb);
}

// ---- the flat program encoding of include/distaff_gpu.h (dg_program_t) ----------------------------------------------------------------
struct Encoded {
    std::vector<uint8_t> ops;
    std::vector<dg_op_hint_t> hints;
    std::vector<dg_block_t> blocks;
    std::vector<uint32_t> children;
    uint32_t root_first = 0, root_count = 0;
    uint8_t hash32[32];
    std::string error;
};
static void put128(uint8_t out[16], u128 v) { memcpy(out, &v, 16); }
static u128 get128(const uint8_t in[16]) { u128 v; memcpy(&v, in, 16); return v; }

static uint32_t encode_block(Encoded &e, const Block &b);
// encodes the blocks of a list (their own child lists first), then appends the list itself: returns its first index in `children`
static uint32_t encode_list(Encoded &e, const std::vector<Block> &list) {
    std::vector<uint32_t> idx;
    for (const Block &b : list) idx.push_back(encode_block(e, b));
    const uint32_t first = (uint32_t)e.children.size();
    e.children.insert(e.children.end(), idx.begin(), idx.end());
    return first;
}
static uint32_t encode_block(Encoded &e, const Block &b) {
    dg_block_t d;
    memset(&d, 0, sizeof d);
    switch (b.kind) {
    case B_SPAN:
        d.kind = DG_BLOCK_SPAN;
        d.first = (uint32_t)e.ops.size(); d.count = (uint32_t)b.span.ops.size();
        for (size_t i = 0; i < b.span.ops.size(); i++) {
            const Hint h = b.span.hint(i);
            dg_op_hint_t eh;
            memset(&eh, 0, sizeof eh);
            eh.kind = h.kind == H_NONE ? DG_HINT_NONE : h.kind == H_PUSH ? DG_HINT_PUSH : h.kind == H_EQSTART ? DG_HINT_EQ_START
                    : h.kind == H_RCSTART ? DG_HINT_RC_START : h.kind == H_CMPSTART ? DG_HINT_CMP_START : DG_HINT_PMPATH_START;
            eh.n = h.n;
            put128(eh.value16, h.value);
            e.ops.push_back(b.span.ops[i]);
            e.hints.push_back(eh);
        }
        break;
    case B_GROUP:
        d.kind = DG_BLOCK_GROUP;
        d.first = encode_list(e, b.body); d.count = (uint32_t)b.body.size();
        break;
    case B_SWITCH:
        d.kind = DG_BLOCK_SWITCH;
        d.first = encode_list(e, b.body); d.count = (uint32_t)b.body.size();
        d.alt_first = encode_list(e, b.alt); d.alt_count = (uint32_t)b.alt.size();
        put128(d.hash0, hash_seq(b.body, BLOCK_SUFFIX, 15));       // Switch::true_branch_hash
        put128(d.hash1, hash_seq(b.alt, BLOCK_SUFFIX, 15));        // Switch::false_branch_hash
        break;
    case B_LOOP:
        d.kind = DG_BLOCK_LOOP;
        d.first = encode_list(e, b.body); d.count = (uint32_t)b.body.size();
        d.alt_first = encode_list(e, b.alt); d.alt_count = (uint32_t)b.alt.size();
        put128(d.hash0, hash_seq(b.body, {}, 0));                  // Loop::image
        put128(d.hash1, hash_seq(b.body, loop_suffix(), 0));       // Loop::body_hash
        put128(d.hash2, hash_seq(b.alt, BLOCK_SUFFIX, 15));        // Loop::skip_hash
        break;
    }
    e.blocks.push_back(d);
    return (uint32_t)e.blocks.size() - 1;
}
static Encoded *encode(const std::string &source) {
    Encoded *e = new Encoded();
    try {
        Program p = compile(source);
        e->root_first = encode_list(*e, p.root.body);
        e->root_count = (uint32_t)p.root.body.size();
        put128(e->hash32, p.hash[0]);
        put128(e->hash32 + 16, p.hash[1]);
    } catch (std::exception &ex) { e->error = ex.what(); }
    return e;
}

// the block tree of an encoding, with its hashes; ranges are checked, nothing else (the VM reports what does not run)
static std::vector<Block> decode_list(const dg_program_t &p, uint32_t first, uint32_t count, int depth);
static Block decode_block(const dg_program_t &p, uint32_t index, int depth) {
    if (index >= p.n_blocks) throw std::runtime_error("block index out of range");
    if (depth > 64) throw std::runtime_error("blocks nested too deeply");
    const dg_block_t &d = p.blocks[index];
    Block b;
    switch (d.kind) {
    case DG_BLOCK_SPAN:
        b.kind = B_SPAN;
        if ((uint64_t)d.first + d.count > p.n_ops) throw std::runtime_error("span op range out of range");
        for (uint32_t i = 0; i < d.count; i++) {
            b.span.ops.push_back(p.ops[d.first + i]);
            const dg_op_hint_t &eh = p.hints[d.first + i];
            if (eh.kind == DG_HINT_NONE) continue;
            Hint h;
            h.kind = eh.kind == DG_HINT_PUSH ? H_PUSH : eh.kind == DG_HINT_EQ_START ? H_EQSTART : eh.kind == DG_HINT_RC_START ? H_RCSTART
                   : eh.kind == DG_HINT_CMP_START ? H_CMPSTART : H_PMPATH;
            h.n = eh.n;
            h.value = get128(eh.value16);
            b.span.hints[i] = h;
        }
        break;
    case DG_BLOCK_GROUP:
        b.kind = B_GROUP;
        b.body = decode_list(p, d.first, d.count, depth + 1);
        break;
    case DG_BLOCK_SWITCH: case DG_BLOCK_LOOP:
        b.kind = d.kind == DG_BLOCK_SWITCH ? B_SWITCH : B_LOOP;
        b.body = decode_list(p, d.first, d.count, depth + 1);
        b.alt = decode_list(p, d.alt_first, d.alt_count, depth + 1);
        b.has_hashes = true;
        b.hashes[0] = get128(d.hash0); b.hashes[1] = get128(d.hash1); b.hashes[2] = get128(d.hash2);
        break;
    default: throw std::runtime_error("unknown block kind");
    }
    return b;
}
static std::vector<Block> decode_list(const dg_program_t &p, uint32_t first, uint32_t count, int depth) {
    if (count == 0 || (uint64_t)first + count > p.n_children) throw std::runtime_error("child list out of range");
    std::vector<Block> list;
    for (uint32_t i = 0; i < count; i++) list.push_back(decode_block(p, p.children[first + i], depth));
    return list;
}

} // namespace vm

// ---- C-ABI ----------------------------------------------------------------------------------------------------------
extern "C" {
// field elements cross as 16 little-endian bytes
void *vm_execute(const char *source, const uint8_t *pub16, uint32_t n_pub, const uint8_t *a16, uint32_t n_a, const uint8_t *b16, uint32_t n_b) {
    auto rd = [](const uint8_t *p, uint32_t n) { std::vector<vm::u128> v(n); if (n) memcpy(v.data(), p, (size_t)n * 16); return v; };
    return vm::execute(source, rd(pub16, n_pub), rd(a16, n_a), rd(b16, n_b));
}
const char *vm_error(void *h) { auto *e = (vm::Execution *)h; return e->error.empty() ? nullptr : e->error.c_str(); }
uint32_t vm_width(void *h) { return (uint32_t)((vm::Execution *)h)->registers.size(); }
uint64_t vm_length(void *h) { auto *e = (vm::Execution *)h; return e->registers.empty() ? 0 : e->registers[0].size(); }
uint32_t vm_ctx_depth(void *h) { return (uint32_t)((vm::Execution *)h)->ctx_depth; }
uint32_t vm_loop_depth(void *h) { return (uint32_t)((vm::Execution *)h)->loop_depth; }
uint32_t vm_stack_depth(void *h) { return (uint32_t)((vm::Execution *)h)->stack_depth; }
void vm_program_hash(void *h, uint8_t *out32) { memcpy(out32, ((vm::Execution *)h)->program_hash, 32); }
// copies the column-major register traces: out must hold width*length*16 bytes
void vm_copy_trace(void *h, uint8_t *out) {
    auto *e = (vm::Execution *)h;
    size_t n = e->registers[0].size();
    for (size_t j = 0; j < e->registers.size(); j++) memcpy(out + j * n * 16, e->registers[j].data(), n * 16);
}
void vm_free(void *h) { delete (vm::Execution *)h; }

// compiles assembly into the program encoding of include/distaff_gpu.h; sizes = {n_ops, n_blocks, n_children, root_first, root_count}
void *vm_compile(const char *source) { return vm::encode(source); }
const char *vm_compile_error(void *h) { auto *e = (vm::Encoded *)h; return e->error.empty() ? nullptr : e->error.c_str(); }
void vm_compile_sizes(void *h, uint64_t sizes[5]) {
    auto *e = (vm::Encoded *)h;
    sizes[0] = e->ops.size(); sizes[1] = e->blocks.size(); sizes[2] = e->children.size(); sizes[3] = e->root_first; sizes[4] = e->root_count;
}
void vm_compile_copy(void *h, uint8_t *ops, dg_op_hint_t *hints, dg_block_t *blocks, uint32_t *children, uint8_t *hash32) {
    auto *e = (vm::Encoded *)h;
    if (!e->ops.empty()) { memcpy(ops, e->ops.data(), e->ops.size()); memcpy(hints, e->hints.data(), e->hints.size() * sizeof(dg_op_hint_t)); }
    memcpy(blocks, e->blocks.data(), e->blocks.size() * sizeof(dg_block_t));
    memcpy(children, e->children.data(), e->children.size() * 4);
    memcpy(hash32, e->hash32, 32);
}
void vm_compile_free(void *h) { delete (vm::Encoded *)h; }
// runs the VM on a program encoding decoded back into its block tree (the hashes the encoding carries close switches and loops)
void *vm_execute_program(const dg_program_t *program, const uint8_t *pub16, uint32_t n_pub, const uint8_t *a16, uint32_t n_a, const uint8_t *b16,
                         uint32_t n_b) {
    auto rd = [](const uint8_t *p, uint32_t n) { std::vector<vm::u128> v(n); if (n) memcpy(v.data(), p, (size_t)n * 16); return v; };
    vm::Program prog;
    try {
        prog.root.kind = vm::B_GROUP;
        prog.root.body = vm::decode_list(*program, program->root_first, program->root_count, 0);
    } catch (std::exception &ex) {
        auto *e = new vm::Execution();
        e->error = ex.what();
        return e;
    }
    prog.hash[0] = vm::get128(program->hash32);
    prog.hash[1] = vm::get128(program->hash32 + 16);
    return vm::run(&prog, nullptr, rd(pub16, n_pub), rd(a16, n_a), rd(b16, n_b));
}
}
