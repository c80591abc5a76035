// Internal helpers shared by the kernels of libm3r_b200.so (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <mutex>
#include "../../include/must3r_b200.h"

namespace m3r {

int set_error(const char* fmt, ...);           // records the message, returns 1
void count_launch();                            // bumps the kernel-launch counter (m3r_launch_count)

// ---- registry of the library's host-side state (runtime.cu), per device and per (device, caller stream).  Every part
// is created on first use under the registry's one mutex and lives for the whole process: the number of entries is
// bounded by the devices and the caller streams that ever run these launches.
int num_sms();                                  // SM count of the current device
// Sets `fn`'s dynamic shared-memory limit to `smem_bytes` once per device.  Returns the kernel's registers per thread
// and how many CTAs of `threads` threads and `smem_bytes` bytes an SM holds; resident == 0 after set_error.
struct KernelInfo { int regs = 0, resident = 0; };
KernelInfo kernel_setup(const void* fn, size_t smem_bytes, int threads);
// What the launches on one caller stream own.  The registry only stores it: the files named below create the parts.
// One thread at a time enqueues on a stream, so once created the parts are used without the lock.
struct StreamState {
  // model.cu: `side` runs the decoder's feedback MLP and memory append next to its last block and the head, `copy`
  // moves the old memory rows; the fork / join events are used round robin
  cudaStream_t side = nullptr, copy = nullptr;
  cudaEvent_t ev[32] = {};
  int next_ev = 0;
  // gemm.cu: LayerNorm-emit partial statistics and counters, split-K hand-over
  float2* emit_stats = nullptr; unsigned int* emit_sync = nullptr; float4* emit_kpart = nullptr; unsigned int* emit_kflag = nullptr;
  // attention.cu: key-split counters and partials, grown on demand
  float* split_buf = nullptr; size_t split_cap = 0;
};
// The entry of caller stream `s` on the current device, with `lock` holding the registry mutex while the caller
// creates missing parts; nullptr (lock not taken) when there is no current device.
using RegistryLock = std::unique_lock<std::mutex>;
StreamState* stream_state(cudaStream_t s, RegistryLock& lock);

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

// 2-D TMA descriptor over a row-major 16-bit (or, with fp32, 32-bit float) matrix: inner extent `cols` (contiguous),
// outer extent `rows`, leading dimension `ld` elements, box = {box_cols, box_rows}, 128-byte swizzle, OOB reads return
// zeros and OOB writes are dropped.  is_bf16 == TMAP_E4M3: 1-byte e4m3 elements.
constexpr int TMAP_E4M3 = 2;
int make_tmap_2d(CUtensorMap* out, const void* base, int is_bf16, uint64_t cols, uint64_t rows, uint64_t ld,
                 uint32_t box_cols, uint32_t box_rows, bool fp32 = false);

// 3-D variant: {cols, rows, batches}; rows beyond `rows` read as zeros even when the batch stride is larger.
int make_tmap_3d(CUtensorMap* out, const void* base, int is_bf16, uint64_t cols, uint64_t rows, uint64_t batches,
                 uint64_t ld, uint64_t batch_stride_elems, uint32_t box_cols, uint32_t box_rows);

unsigned long long* trace_buffer();            // device buffer set by m3r_debug_trace (nullptr = off)
// Launch with the programmatic-stream-serialization attribute (PDL).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace m3r
