// The e4m3 x e4m3 -> fp32 instantiations of the persistent wgmma GEMM (gemm_kernel.cuh), kept in their own translation
// unit so that the 16-bit kernels of gemm.cu compile (and are checked) exactly as before.  Plain and grouped launches with
// tile widths 64 / 128 / 256 (m3r_gemm_e4m3 maps the other widths of pick_bn onto these).  The LayerNorm-emitting form
// has no e4m3 instantiation: the GEMMs that emit a LayerNorm (proj, cross-attention proj, fc2, the projector) take
// unbounded 16-bit A operands, and its 128-wide e4m3 tile spilled.
#include "gemm_kernel.cuh"

namespace m3r {

int launch_gemm_e4m3(int bn, int mode, const m3r_gemm_args* a, const m3r_gemm_e4m3_args* e8, cudaStream_t stream,
                     const m3r_gemm_group* grp) {
  switch (mode) {
    case MODE_GROUPED:
      if (bn == 256) return launch_gemm<256, MODE_GROUPED, true>(a, e8, stream, grp);
      if (bn == 128) return launch_gemm<128, MODE_GROUPED, true>(a, e8, stream, grp);
      return launch_gemm<64, MODE_GROUPED, true>(a, e8, stream, grp);
    default:
      if (bn == 256) return launch_gemm<256, MODE_PLAIN, true>(a, e8, stream);
      if (bn == 128) return launch_gemm<128, MODE_PLAIN, true>(a, e8, stream);
      return launch_gemm<64, MODE_PLAIN, true>(a, e8, stream);
  }
}

}  // namespace m3r
