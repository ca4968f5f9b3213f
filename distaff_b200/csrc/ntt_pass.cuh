// Pass kernels of the batched NTT / coset LDE (included by ntt.cu and ntt_inl.cu, which differ in how fe_mul is emitted:
// out of line -- one shared body, small code -- or inlined).  DG_NTT_TAG keeps the kernel symbols of the two translation units apart.
#pragma once
#include "common.cuh"

namespace dg {

// What a pass does besides its butterflies is fixed per instantiation, so that a kernel holds only its own input and output paths
// (and its registers are allocated for that path alone).  launch_pass (ntt.cu) picks the kind from the PassGeom flags.
enum PassKind {
    PK_TW,              // first / middle pass: output k of lane l times tw^(l*k)
    PK_COSET_TWFULL,    // first pass of a fold-1 LDE: input times cw_point, output times the streamed tw_full table
    PK_COSET_TW,        // the same, output factor from the two-level table cw (tw_full not built for this shape)
    PK_FOLD_TW,         // first pass of a fold > 1 LDE: Horner fold of the input, output times tw^(l*k)
    PK_LAST,            // last or only pass (lane-major), plain output
    PK_LAST_SCALE,      // last or only pass of an inverse transform: output times n^-1
    PK_COSET_ONE,       // only pass of a fold-1 LDE: input times cw_point
    PK_FOLD_ONE,        // only pass of a fold > 1 LDE: Horner fold of the input
    PK_COUNT
};
__host__ __device__ constexpr bool pk_lane_major(int k) { return k >= PK_LAST; }
__host__ __device__ constexpr bool pk_coset_in(int k) { return k == PK_COSET_TWFULL || k == PK_COSET_TW || k == PK_COSET_ONE; }
__host__ __device__ constexpr bool pk_fold_in(int k) { return k == PK_FOLD_TW || k == PK_FOLD_ONE; }

struct PassGeom {
    int log_t;                          // lanes per block (power of two)
    unsigned num_tiles;                 // blockIdx.x = outer * num_tiles + tile
    long long in_outer, in_lane, in_point;
    long long out_outer, out_lane, out_point;
    long long in_batch_y, out_batch_y, in_batch_z, out_batch_z;
    // the five flags below select the PassKind on the host; the kernels do not read them
    int lane_major;                     // shared-memory layout: 0 = [point][lane], 1 = [lane][point] (padded)
    int tw_on;                          // multiply output k of lane (tile*T+lane) by tw^((tile*T+lane)*k)
    int has_scale;
    int coset_on;                       // input transform of the LDE: sum_f src[j + f*fold_stride] * cw^(c*(j + f*fold_stride))
    int coset_fast;                     // fold == 1: input factor from a single-level table, lane factor merged into the output twiddle
    TwiddleRef tw;
    fe scale;
    int fold;
    long long fold_stride;
    TwiddleRef cw;
    const fe *cw_point;                 // cw_point[e] = (w_N^in_point)^e, e < cw_point_mask + 1
    unsigned cw_point_mask;
    const fe *tw_full;                  // coset_fast: tw_full[coset][k * out_point + lane] = cw^(lane * (k * blowup + coset)), or null
    long long tw_full_stride;           // elements per coset (= transform size n)
    int log_blowup;
    unsigned coset0;                    // first coset handled by this launch (blockIdx.y = coset - coset0)
    const fe *roots;                    // per-stage twiddle tables of the L-point transform: W_st[j] = w_L^(j << st), back to back
};

// The pass kernels' multiply.  ntt.cu: the shared out-of-line body.  ntt_inl.cu: v4 inlined with its rare canonicalisation as a plain
// branch, so that no multiply carries a call site (the call pins argument and result registers around every product).
__device__ __forceinline__ fe ntt_mul(fe a, fe b) {
#if defined(__CUDA_ARCH__) && !defined(DG_MUL_CALL)
    return ptx::fe_mul_v4t<false>(a, b);
#else
    return fe_mul(a, b);
#endif
}

__device__ __forceinline__ fe tw_lookup(const TwiddleRef &t, unsigned long long e) {
    unsigned ee = (unsigned)e & t.mask;
    fe a = t.lo[ee & ((1u << t.lo_bits) - 1u)];
    fe b = t.hi[ee >> t.lo_bits];
    return ntt_mul(a, b);
}

// ---- pass kernel -------------------------------------------------------------------------------------------------------
// One block transforms a tile of T lanes x L points.  The log2(L) decimation-in-frequency stages are grouped into rounds of
// up to RMAX stages that run entirely in registers on 2^rho elements per thread ("unit"); shared memory is touched only
// between rounds.  The first round reads its operands straight from global memory and the last one writes straight back.
// RMAX = 2: 4 elements per unit, 5 rounds for 1024 points (small unrolled bodies, few registers, many resident warps).
// Stage twiddles come from per-stage compact tables W_st[j] = w_L^(j << st) (unit-stride, conflict-free) staged in shared memory.
template <int LOG_L, int S0, int RHO>
__device__ __forceinline__ void dif_regs(fe *x, const fe *s_tw, int g_lo) {
    constexpr int L = 1 << LOG_L, R = 1 << RHO;
    constexpr int LOG_SP = LOG_L - S0 - RHO;
#pragma unroll
    for (int u = 0; u < RHO; u++) {
        const int hr = R >> (u + 1);
        const int st = S0 + u;
        const fe *W = s_tw + (L - (L >> st));
#pragma unroll
        for (int i = 0; i < R; i++) {
            if ((i & hr) == 0) {
                fe a = x[i], b = x[i + hr];
                x[i] = fe_add(a, b);
                fe d = fe_sub(a, b);
                // in the last round (LOG_SP == 0, g_lo == 0) the twiddle index is a compile-time constant: index 0 is w^0 = 1
                if (st != LOG_L - 1 && !(LOG_SP == 0 && (i & (hr - 1)) == 0)) d = ntt_mul(d, W[g_lo + ((i & (hr - 1)) << LOG_SP)]);
                x[i + hr] = d;
            }
        }
    }
}

template <int LOG_L, bool LANE_MAJOR>
__device__ __forceinline__ int sidx(int pos, int t, int T) {
    constexpr int L = 1 << LOG_L;
    constexpr int LS = L + (L >> 3) + 1;                 // padded lane stride, one pad element per 8 points
    return LANE_MAJOR ? (t * LS + pos + (pos >> 3)) : (pos * T + t);
}

template <int LOG_L, int S0, int RHO, bool FIRST, bool LAST, int KIND>
__device__ __forceinline__ void ntt_round(const fe *__restrict__ src, fe *__restrict__ dst, fe *s_data, const fe *s_tw, const PassGeom &g,
                                          unsigned tile, long long in_base) {
    constexpr bool LANE_MAJOR = pk_lane_major(KIND);
    constexpr int L = 1 << LOG_L, R = 1 << RHO;
    constexpr int LOG_B = LOG_L - S0, LOG_SP = LOG_B - RHO;
    constexpr int N_GLO = 1 << LOG_SP, N_GHI = 1 << S0;
    const int T = 1 << g.log_t;
    const int units = (L >> RHO) * T;
    for (int u = threadIdx.x; u < units; u += blockDim.x) {
        int t, g_lo, g_hi;
        if (!LANE_MAJOR || LAST) {             // lanes fastest: global accesses of neighbouring threads are contiguous across lanes
            t = u & (T - 1);
            const int rest = u >> g.log_t;
            g_lo = rest & (N_GLO - 1);
            g_hi = rest >> LOG_SP;
        } else {                               // points fastest: contiguous rows of the last pass / conflict-free shared accesses
            g_lo = u & (N_GLO - 1);
            const int rest = u >> LOG_SP;
            g_hi = rest & (N_GHI - 1);
            t = rest >> S0;
        }
        const int gbase = (g_hi << LOG_B) + g_lo;
        fe x[R];
#pragma unroll
        for (int m = 0; m < R; m++) {
            const int pos = gbase + (m << LOG_SP);
            if (FIRST) {
                const long long j = in_base + (long long)t * g.in_lane + (long long)pos * g.in_point;
                if (pk_coset_in(KIND)) {
                    // p[j] * w_N^(c*pos*in_point); the lane part w_N^(c*lane) rides on the output twiddle
                    x[m] = ntt_mul(src[j], g.cw_point[((g.coset0 + (unsigned)blockIdx.y) * (unsigned)pos) & g.cw_point_mask]);
                } else if (pk_fold_in(KIND)) {
                    // sum_f src[j + f n] w_N^(c (j + f n)) = w_N^(c j) * Horner_f(src[j + f n]; u),  u = w_N^(c n) (constant per coset)
                    const unsigned long long c = g.coset0 + blockIdx.y;
                    const fe u = tw_lookup(g.cw, c * (unsigned long long)g.fold_stride);
                    fe v = src[j + (long long)(g.fold - 1) * g.fold_stride];
                    for (int f = g.fold - 2; f >= 0; f--) v = fe_add(ntt_mul(v, u), src[j + (long long)f * g.fold_stride]);
                    x[m] = ntt_mul(v, tw_lookup(g.cw, c * (unsigned long long)j));
                } else {
                    x[m] = src[j];
                }
            } else {
                x[m] = s_data[sidx<LOG_L, LANE_MAJOR>(pos, t, T)];
            }
        }
        dif_regs<LOG_L, S0, RHO>(x, s_tw, g_lo);
#pragma unroll
        for (int m = 0; m < R; m++) {
            const int pos = gbase + (m << LOG_SP);
            if (LAST) {                        // position q holds X[bitrev(q)]
                const unsigned k = __brev((unsigned)pos) >> (32 - LOG_L);
                fe v = x[m];
                if (KIND == PK_COSET_TWFULL)   // streamed table in the layout of the output: one 16-byte load instead of two loads and a multiplication
                    v = ntt_mul(v, g.tw_full[(long long)(g.coset0 + blockIdx.y) * g.tw_full_stride + (long long)(tile * T + t) * g.out_lane + (long long)k * g.out_point]);
                else if (KIND == PK_COSET_TW)
                    v = ntt_mul(v, tw_lookup(g.cw, (unsigned long long)(tile * T + t) * (((unsigned long long)k << g.log_blowup) + g.coset0 + blockIdx.y)));
                else if (KIND == PK_TW || KIND == PK_FOLD_TW)
                    v = ntt_mul(v, tw_lookup(g.tw, (unsigned long long)(tile * T + t) * k));
                else if (KIND == PK_LAST_SCALE)
                    v = ntt_mul(v, g.scale);
                dst[(long long)t * g.out_lane + (long long)k * g.out_point] = v;
            } else {
                s_data[sidx<LOG_L, LANE_MAJOR>(pos, t, T)] = x[m];
            }
        }
    }
}

template <int LOG_L, int RMAX, int S0, int KIND>
__device__ __forceinline__ void ntt_rounds(const fe *__restrict__ src, fe *__restrict__ dst, fe *s_data, const fe *s_tw, const PassGeom &g,
                                           unsigned tile, long long in_base) {
    constexpr int REM = LOG_L - S0, LEFT = (REM + RMAX - 1) / RMAX, RHO = (REM + LEFT - 1) / LEFT;   // even split, largest round first
    ntt_round<LOG_L, S0, RHO, S0 == 0, S0 + RHO == LOG_L, KIND>(src, dst, s_data, s_tw, g, tile, in_base);
    if constexpr (S0 + RHO < LOG_L) {
        __syncthreads();
        ntt_rounds<LOG_L, RMAX, S0 + RHO, KIND>(src, dst, s_data, s_tw, g, tile, in_base);
    }
}

template <int LOG_L, int KIND, int RMAX, int BT, int MINB, int TAG>
__global__ void __launch_bounds__(BT, MINB) ntt_pass_kernel(const fe *__restrict__ src, fe *__restrict__ dst, const PassGeom g) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int L = 1 << LOG_L;
    fe *s_tw = reinterpret_cast<fe *>(smem_raw);          // L entries: per-stage tables back to back
    fe *s_data = s_tw + L;
    const int T = 1 << g.log_t;
    const unsigned tile = blockIdx.x % g.num_tiles, outer = blockIdx.x / g.num_tiles;
    const long long in_base = (long long)outer * g.in_outer + (long long)tile * T * g.in_lane;   // index inside the vector
    src += (long long)blockIdx.y * g.in_batch_y + (long long)blockIdx.z * g.in_batch_z;
    dst += (long long)blockIdx.y * g.out_batch_y + (long long)blockIdx.z * g.out_batch_z + (long long)outer * g.out_outer +
           (long long)tile * T * g.out_lane;
    for (int i = threadIdx.x; i < L - 1; i += blockDim.x) s_tw[i] = g.roots[i];
    if (KIND == PK_COSET_TWFULL) {
        // the streamed twiddles are consumed in the last round: start pulling this block's T*16-byte segments (one per output k) into L2 now
        const fe *tb = g.tw_full + (long long)(g.coset0 + blockIdx.y) * g.tw_full_stride + (long long)tile * T * g.out_lane;
        for (int k = threadIdx.x; k < L; k += blockDim.x)
            asm volatile("prefetch.global.L2 [%0];" :: "l"(tb + (long long)k * g.out_point));
    }
    __syncthreads();
    ntt_rounds<LOG_L, RMAX, 0, KIND>(src, dst, s_data, s_tw, g, tile, in_base);
}

typedef void (*PassKernel)(const fe *, fe *, const PassGeom);

// The shape of every pass kernel (ntt.cu gives the measurements): 4-element register rounds, 512 threads, 2 blocks per SM.  Passes of
// 2^PASS_INLINE_LOG_L points and more run the inline-multiply kernels of ntt_inl.cu, smaller ones the out-of-line kernels of ntt.cu.
static const int PASS_RMAX = 2, PASS_THREADS = 512, PASS_MINB = 2, PASS_INLINE_LOG_L = 8;
PassKernel pass_kernel_inline(int kind, int log_l);     // ntt_inl.cu: 2^PASS_INLINE_LOG_L .. 2^MAX_LOG_L points

// the instantiation for (kind, log2 L) with L in [2^LO, 2^HI], nullptr outside
template <int KIND, int RMAX, int BT, int MINB, int TAG, int LO, int HI> PassKernel pass_kernel_sized(int log_l) {
    if constexpr (LO > HI) return nullptr;
    else return log_l == LO ? ntt_pass_kernel<LO, KIND, RMAX, BT, MINB, TAG> : pass_kernel_sized<KIND, RMAX, BT, MINB, TAG, LO + 1, HI>(log_l);
}
template <int RMAX, int BT, int MINB, int TAG, int LO, int HI> PassKernel pass_kernel_of(int kind, int log_l) {
    switch (kind) {
        case PK_TW: return pass_kernel_sized<PK_TW, RMAX, BT, MINB, TAG, LO, HI>(log_l);
        case PK_COSET_TWFULL: return pass_kernel_sized<PK_COSET_TWFULL, RMAX, BT, MINB, TAG, LO, HI>(log_l);
        case PK_COSET_TW: return pass_kernel_sized<PK_COSET_TW, RMAX, BT, MINB, TAG, LO, HI>(log_l);
        case PK_FOLD_TW: return pass_kernel_sized<PK_FOLD_TW, RMAX, BT, MINB, TAG, LO, HI>(log_l);
        case PK_LAST: return pass_kernel_sized<PK_LAST, RMAX, BT, MINB, TAG, LO, HI>(log_l);
        case PK_LAST_SCALE: return pass_kernel_sized<PK_LAST_SCALE, RMAX, BT, MINB, TAG, LO, HI>(log_l);
        case PK_COSET_ONE: return pass_kernel_sized<PK_COSET_ONE, RMAX, BT, MINB, TAG, LO, HI>(log_l);
        case PK_FOLD_ONE: return pass_kernel_sized<PK_FOLD_ONE, RMAX, BT, MINB, TAG, LO, HI>(log_l);
    }
    return nullptr;
}

}  // namespace dg
