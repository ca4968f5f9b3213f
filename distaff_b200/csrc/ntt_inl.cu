// Inline-multiply instantiations of the NTT pass kernels (see ntt_pass.cuh): fe_mul is expanded at every butterfly instead of
// calling the shared out-of-line body of ntt.cu.  Only the sub-transform sizes of the large transforms are instantiated; the
// register rounds are small (RMAX 2) so that the unrolled code stays near the instruction-cache size.
#include "ntt_pass.cuh"

namespace dg {

PassKernel pass_kernel_inline(int kind, int log_l) {
    return pass_kernel_of<PASS_RMAX, PASS_THREADS, PASS_MINB, 1, PASS_INLINE_LOG_L, MAX_LOG_L>(kind, log_l);
}

}  // namespace dg
