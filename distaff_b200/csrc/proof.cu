// bincode 1.3.1 encoding of StarkProof (proof.h): integers little-endian at their own width, a u64 length before every Vec, arrays
// (digests, rows of four values) raw, a field element as its u128.  The crate is not vendored with the reference; its layout is restated
// from the crate's documentation (DESIGN.md section 3).
#include "proof.h"

namespace dg {

namespace {

struct ByteWriter {
    std::vector<uint8_t> b;
    void u8(uint8_t v) { b.push_back(v); }
    void u32(uint32_t v) { for (int i = 0; i < 4; i++) b.push_back((uint8_t)(v >> (8 * i))); }
    void u64(uint64_t v) { for (int i = 0; i < 8; i++) b.push_back((uint8_t)(v >> (8 * i))); }
    void felt(fe v) { u64(v.lo); u64(v.hi); }
    void digest(const Digest &d) { b.insert(b.end(), d.begin(), d.end()); }
    void dvec(const std::vector<Digest> &v) { u64(v.size()); for (auto &d : v) digest(d); }
    void dvv(const std::vector<std::vector<Digest>> &v) { u64(v.size()); for (auto &x : v) dvec(x); }
    void fvec(const std::vector<fe> &v) { u64(v.size()); for (auto &x : v) felt(x); }
};

// Reads what ByteWriter writes.  After the first short read every read returns zeros and ok stays false.
struct Reader {
    const uint8_t *p, *end;
    bool ok = true;
    Reader(const uint8_t *b, size_t n) : p(b), end(b + n) {}
    bool need(size_t n) { if (!ok || (size_t)(end - p) < n) { ok = false; return false; } return true; }
    uint8_t u8() { if (!need(1)) return 0; return *p++; }
    uint32_t u32() { if (!need(4)) return 0; uint32_t v; memcpy(&v, p, 4); p += 4; return v; }
    uint64_t u64() { if (!need(8)) return 0; uint64_t v; memcpy(&v, p, 8); p += 8; return v; }
    fe felt() { fe v = fe_make(0, 0); if (!need(16)) return v; memcpy(&v, p, 16); p += 16; return v; }
    Digest digest() { Digest d; d.fill(0); if (!need(32)) return d; memcpy(d.data(), p, 32); p += 32; return d; }
    size_t len(size_t elem_bytes) {                              // a Vec length that the remaining bytes can actually hold
        uint64_t n = u64();
        if (!ok || n > (uint64_t)(end - p) / (elem_bytes ? elem_bytes : 1)) { ok = false; return 0; }
        return (size_t)n;
    }
    std::vector<Digest> dvec() { size_t n = len(32); std::vector<Digest> v(n); for (auto &x : v) x = digest(); return v; }
    std::vector<std::vector<Digest>> dvv() { size_t n = len(8); std::vector<std::vector<Digest>> v(n); for (auto &x : v) x = dvec(); return v; }
    std::vector<fe> fvec() { size_t n = len(16); std::vector<fe> v(n); for (auto &x : v) x = felt(); return v; }
};

}  // namespace

std::vector<uint8_t> write_proof(const StarkProof &P) {
    ByteWriter w;
    w.digest(P.trace_root);
    const TraceInfo &t = P.trace_info;
    w.u8(t.domain_depth); w.u8(t.ctx_depth); w.u8(t.loop_depth); w.u8(t.stack_depth);
    w.u32(t.op_count);
    w.dvv(P.trace_nodes);
    w.u64(P.trace_evaluations.size());
    for (auto &row : P.trace_evaluations) w.fvec(row);
    w.digest(P.constraint_root);
    w.dvec(P.constraint_proof.values); w.dvv(P.constraint_proof.nodes); w.u8(P.constraint_proof.depth);
    w.fvec(P.trace_at_z1); w.fvec(P.trace_at_z2);
    w.u64(P.degree_proof.layers.size());
    for (auto &l : P.degree_proof.layers) {
        w.digest(l.root);
        w.u64(l.values.size());
        for (auto &q : l.values) for (int j = 0; j < 4; j++) w.felt(q[j]);
        w.dvv(l.nodes);
        w.u8(l.depth);
    }
    w.digest(P.degree_proof.rem_root);
    w.fvec(P.degree_proof.rem_values);
    w.u64(P.pow_nonce);
    const ProofOptions &o = P.options;
    w.u8(o.log_extension_factor); w.u8(o.num_queries); w.u8(o.grinding_factor); w.u8(o.hash_fn);
    return std::move(w.b);
}

// Vec lengths are bounded by their least encoded element: 8 bytes for a Vec of Vecs, 16 for a value, 32 for a digest, 41 for a FRI
// layer (root, empty values and nodes, depth), 64 for a row of four values
bool read_proof(const uint8_t *bytes, size_t len, StarkProof &P) {
    Reader r(bytes, len);
    P.trace_root = r.digest();
    TraceInfo &t = P.trace_info;
    t.domain_depth = r.u8(); t.ctx_depth = r.u8(); t.loop_depth = r.u8(); t.stack_depth = r.u8();
    t.op_count = r.u32();
    P.trace_nodes = r.dvv();
    P.trace_evaluations.resize(r.len(8));
    for (auto &row : P.trace_evaluations) row = r.fvec();
    P.constraint_root = r.digest();
    P.constraint_proof.values = r.dvec(); P.constraint_proof.nodes = r.dvv(); P.constraint_proof.depth = r.u8();
    P.trace_at_z1 = r.fvec(); P.trace_at_z2 = r.fvec();
    P.degree_proof.layers.resize(r.len(41));
    for (auto &l : P.degree_proof.layers) {
        l.root = r.digest();
        l.values.resize(r.len(64));
        for (auto &q : l.values) for (int j = 0; j < 4; j++) q[j] = r.felt();
        l.nodes = r.dvv();
        l.depth = r.u8();
    }
    P.degree_proof.rem_root = r.digest();
    P.degree_proof.rem_values = r.fvec();
    P.pow_nonce = r.u64();
    ProofOptions &o = P.options;
    o.log_extension_factor = r.u8(); o.num_queries = r.u8(); o.grinding_factor = r.u8(); o.hash_fn = r.u8();
    return r.ok && r.p == r.end;
}

bool read_batch_proof(const uint8_t *bytes, size_t len, BatchMerkleProof &P) {
    Reader r(bytes, len);
    P.values = r.dvec(); P.nodes = r.dvv(); P.depth = r.u8();
    return r.ok && r.p == r.end;
}

}  // namespace dg
