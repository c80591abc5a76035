// Internal helpers shared by the kernels of libm3r_b200.so (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include "../../include/must3r_b200.h"

namespace m3r {

int set_error(const char* fmt, ...);           // records the message, returns 1
int num_sms();                                  // SM count of the current device (cached)
void count_launch();                            // bumps the kernel-launch counter (m3r_launch_count)

// Optional per-category device timing (m3r_prof_*): CUDA events recorded on the launch stream around each kernel.
// The attention kernel has one CTA shape; its two categories keep their historical names (bench.py prints them as
// "attn_kernel<QT=2>" and "attn_kernel<QT=1>+split-merge"): PROF_ATTN_QT2 = launches over the whole key range,
// PROF_ATTN_QT1 = launches with key splits and the in-kernel merge (the one-view update steps).
enum ProfCat { PROF_GEMM256 = 0, PROF_GEMM128 = 1, PROF_GEMM64 = 2, PROF_ATTN_QT2 = 3, PROF_ATTN_QT1 = 4, PROF_LN = 5, PROF_OTHER = 6, PROF_NCAT = 7 };
struct ProfScope {
  int slot;
  ProfScope(int cat, double flops, double bytes, cudaStream_t s);
  ~ProfScope();
  cudaStream_t stream;
};

// 2-D TMA descriptor over a row-major 16-bit matrix: inner extent `cols` (contiguous), outer extent `rows`,
// leading dimension `ld` elements, box = {box_cols, box_rows}, 128-byte swizzle, OOB reads return zeros.
int make_tmap_2d(CUtensorMap* out, const void* base, int is_bf16, uint64_t cols, uint64_t rows, uint64_t ld,
                 uint32_t box_cols, uint32_t box_rows);

// 3-D variant: {cols, rows, batches}; rows beyond `rows` read as zeros even when the batch stride is larger.
int make_tmap_3d(CUtensorMap* out, const void* base, int is_bf16, uint64_t cols, uint64_t rows, uint64_t batches,
                 uint64_t ld, uint64_t batch_stride_elems, uint32_t box_cols, uint32_t box_rows);

// Launch with the programmatic-stream-serialization attribute (PDL); M3R_PDL=0 in the environment disables it.
bool pdl_enabled();
unsigned long long* trace_buffer();            // device buffer set by m3r_debug_trace (nullptr = off)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace m3r
