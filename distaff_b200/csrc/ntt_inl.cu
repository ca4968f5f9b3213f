// Inline-multiply instantiations of the NTT pass kernels (see ntt_pass.cuh): fe_mul is expanded at every butterfly instead of
// calling the shared out-of-line body of ntt.cu.  Only the sub-transform sizes of the large transforms are instantiated; the
// register rounds are small (RMAX <= 3) so that the unrolled code stays near the instruction-cache size.
#include "ntt_pass.cuh"

namespace dg {

PassKernel pass_kernel_inline(int kind, int log_l, int rmax, int bt) {
    if (rmax == 3 && bt == 1024) return pass_kernel_of<3, 1024, 1, 1, 8, 10>(kind, log_l);
    if (rmax == 3 && bt == 512) return pass_kernel_of<3, 512, 2, 1, 8, 10>(kind, log_l);
    if (rmax == 3) return pass_kernel_of<3, 256, 3, 1, 8, 10>(kind, log_l);
    if (rmax == 2 && bt == 512) return pass_kernel_of<2, 512, 2, 1, 8, 10>(kind, log_l);
    if (rmax == 2) return pass_kernel_of<2, 256, 4, 1, 8, 10>(kind, log_l);
    return nullptr;
}

}  // namespace dg
