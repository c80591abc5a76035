// Runtime glue of libm3r_b200.so: error reporting, the per-device / per-stream state registry, TMA descriptor encoding.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <map>
#include <utility>
#include <vector>
#include "m3r_internal.h"

namespace m3r {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

int set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}

static unsigned long long* g_trace = nullptr;
unsigned long long* trace_buffer() { return g_trace; }

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

// ---- profiling: a ring of event pairs; disabled by default (zero overhead beyond one branch)
struct ProfRec { cudaEvent_t a, b; int cat; double flops, bytes; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;
static size_t g_prof_used = 0;

ProfScope::ProfScope(int cat, double flops, double bytes, cudaStream_t s) : slot(-1), stream(s) {
  if (!g_prof_on) return;
  if (g_prof_used == g_prof.size()) {
    ProfRec r; cudaEventCreate(&r.a); cudaEventCreate(&r.b); r.cat = 0; r.flops = r.bytes = 0;
    g_prof.push_back(r);
  }
  slot = (int)g_prof_used++;
  g_prof[slot].cat = cat; g_prof[slot].flops = flops; g_prof[slot].bytes = bytes;
  cudaEventRecord(g_prof[slot].a, s);
}
ProfScope::~ProfScope() { if (slot >= 0) cudaEventRecord(g_prof[slot].b, stream); }

// ---- the registry (m3r_internal.h)
struct DeviceState { int sms = 0; std::map<const void*, KernelInfo> kernels; };
static std::mutex g_mu;
static std::map<int, DeviceState> g_devices;
static std::map<std::pair<int, cudaStream_t>, StreamState> g_streams;

int num_sms() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  std::lock_guard<std::mutex> lock(g_mu);
  int& n = g_devices[dev].sms;
  if (n <= 0 && (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)) n = 132;
  return n;
}

KernelInfo kernel_setup(const void* fn, size_t smem_bytes, int threads) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return set_error("kernel setup: no current device: %s", cudaGetErrorString(e)), KernelInfo{};
  std::lock_guard<std::mutex> lock(g_mu);
  KernelInfo& k = g_devices[dev].kernels[fn];
  if (k.resident == 0) {
    cudaFuncAttributes fa;
    int n = 0;
    e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, fn);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, threads, smem_bytes);
    if (e != cudaSuccess || n < 1)
      return set_error("kernel setup (%zu B shared memory, %d threads): %s", smem_bytes, threads,
                       e != cudaSuccess ? cudaGetErrorString(e) : "no CTA fits on an SM"), KernelInfo{};
    k.regs = fa.numRegs; k.resident = n;
  }
  return k;
}

StreamState* stream_state(cudaStream_t s, RegistryLock& lock) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  lock = RegistryLock(g_mu);
  return &g_streams[std::make_pair(dev, s)];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int make_tmap_2d(CUtensorMap* out, const void* base, int is_bf16, uint64_t cols, uint64_t rows, uint64_t ld,
                 uint32_t box_cols, uint32_t box_rows, bool fp32) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error("cuTensorMapEncodeTiled is unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error("TMA base pointer must be 16-byte aligned");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * (fp32 ? 4 : 2)};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = fp32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                      : (is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
  CUresult r = enc(out, dt, 2,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled failed (%d): cols=%llu rows=%llu ld=%llu box=%ux%u",
                                          (int)r, (unsigned long long)cols, (unsigned long long)rows,
                                          (unsigned long long)ld, box_cols, box_rows);
  return 0;
}

int make_tmap_3d(CUtensorMap* out, const void* base, int is_bf16, uint64_t cols, uint64_t rows, uint64_t batches,
                 uint64_t ld, uint64_t batch_stride_elems, uint32_t box_cols, uint32_t box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error("cuTensorMapEncodeTiled is unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error("TMA base pointer must be 16-byte aligned");
  if (batches <= 1) batch_stride_elems = rows * ld;
  cuuint64_t dims[3] = {cols, rows, batches < 1 ? 1 : batches};
  cuuint64_t strides[2] = {ld * 2, batch_stride_elems * 2};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled(3d) failed (%d): cols=%llu rows=%llu nb=%llu ld=%llu bs=%llu",
                                          (int)r, (unsigned long long)cols, (unsigned long long)rows,
                                          (unsigned long long)batches, (unsigned long long)ld,
                                          (unsigned long long)batch_stride_elems);
  return 0;
}

}  // namespace m3r

extern "C" const char* m3r_last_error(void) { return m3r::g_err; }
extern "C" int m3r_abi_version(void) { return M3R_ABI_VERSION; }
extern "C" long long m3r_launch_count(void) { return m3r::g_launches.load(); }

// Enable (1) / disable (0) per-kernel event timing; enabling clears previous records.
extern "C" void m3r_prof_enable(int on) {
  m3r::g_prof_on = on != 0;
  if (on) m3r::g_prof_used = 0;
}
// Synchronise and sum the recorded kernels per category: out[cat*4 + {0: ms, 1: launches, 2: flops, 3: bytes}]
extern "C" int m3r_prof_read(double* out) {
  using namespace m3r;
  for (int i = 0; i < PROF_NCAT * 4; ++i) out[i] = 0.0;
  for (size_t i = 0; i < g_prof_used; ++i) {
    if (cudaEventSynchronize(g_prof[i].b) != cudaSuccess) return set_error("prof_read: event sync failed");
    float ms = 0.f;
    cudaEventElapsedTime(&ms, g_prof[i].a, g_prof[i].b);
    double* o = out + g_prof[i].cat * 4;
    o[0] += ms; o[1] += 1.0; o[2] += g_prof[i].flops; o[3] += g_prof[i].bytes;
  }
  return 0;
}

extern "C" int m3r_peer_alloc(int64_t bytes, void** ptr) {
  if (!ptr || bytes <= 0) return m3r::set_error("peer_alloc: bad arguments");
  cudaError_t e = cudaMalloc(ptr, (size_t)bytes);
  if (e != cudaSuccess) return m3r::set_error("peer_alloc: cudaMalloc(%lld) failed: %s", (long long)bytes, cudaGetErrorString(e));
  return 0;
}
extern "C" int m3r_peer_free(void* ptr) {
  cudaError_t e = cudaFree(ptr);
  return e == cudaSuccess ? 0 : m3r::set_error("peer_free: %s", cudaGetErrorString(e));
}
extern "C" int m3r_ipc_export(void* ptr, void* handle64) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaError_t e = cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle64), ptr);
  return e == cudaSuccess ? 0 : m3r::set_error("ipc_export: %s", cudaGetErrorString(e));
}
extern "C" int m3r_ipc_open(const void* handle64, void** ptr) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  cudaError_t e = cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
  return e == cudaSuccess ? 0 : m3r::set_error("ipc_open: %s", cudaGetErrorString(e));
}
extern "C" int m3r_ipc_close(void* ptr) {
  cudaError_t e = cudaIpcCloseMemHandle(ptr);
  return e == cudaSuccess ? 0 : m3r::set_error("ipc_close: %s", cudaGetErrorString(e));
}

// ---- device-side flag barrier for the multi-GPU schedule (engine/sharded.py): every rank owns a uint32 slot in every
// rank's flag array (peer-mapped memory).  m3r_peer_signal, enqueued after the kernels whose peer stores must be visible,
// publishes an epoch number into its slot on all ranks; m3r_peer_wait spins (on the GPU, never on the host) until the slots
// of the ranks in `rank_mask` have reached the epoch.  Stream order + system-scope release / acquire make the K|V rows
// that the GEMM epilogues stored into this GPU's memory visible to the kernels enqueued after the wait.
namespace m3r {
struct SlotList { unsigned int* p[M3R_MAX_PEERS]; };
__global__ void peer_signal_kernel(SlotList slots, int n, unsigned int value) {
  asm volatile("griddepcontrol.wait;" ::: "memory");          // the producing kernels of this stream have completed
  if ((int)threadIdx.x < n) {
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(slots.p[threadIdx.x]), "r"(value) : "memory");
  }
}
__global__ void peer_wait_kernel(const unsigned int* flags, unsigned int rank_mask, unsigned int value) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const unsigned int r = threadIdx.x;
  if (r < 32 && ((rank_mask >> r) & 1u)) {
    const long long t0 = clock64();
    for (;;) {
      unsigned int v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + r) : "memory");
      if ((int)(v - value) >= 0) break;
      if (clock64() - t0 > 60000000000ll) __trap();            // ~30 s: a peer died; fail the launch instead of hanging the box
      __nanosleep(100);
    }
  }
  __syncthreads();
  __threadfence_system();
}
}  // namespace m3r

extern "C" int m3r_peer_signal(void* const* flag_slots, int32_t n, uint32_t value, void* stream) {
  using namespace m3r;
  if (!flag_slots || n < 1 || n > M3R_MAX_PEERS) return set_error("peer_signal: 1..%d slots", M3R_MAX_PEERS);
  SlotList sl;
  for (int i = 0; i < M3R_MAX_PEERS; ++i) sl.p[i] = i < n ? reinterpret_cast<unsigned int*>(flag_slots[i]) : nullptr;
  cudaError_t e = launch_pdl(peer_signal_kernel, dim3(1), dim3(32), 0, reinterpret_cast<cudaStream_t>(stream), sl, (int)n, (unsigned int)value);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("peer_signal launch: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}
extern "C" int m3r_peer_wait(const void* local_flags, uint32_t rank_mask, uint32_t value, void* stream) {
  using namespace m3r;
  if (!local_flags) return set_error("peer_wait: null pointer");
  cudaError_t e = launch_pdl(peer_wait_kernel, dim3(1), dim3(32), 0, reinterpret_cast<cudaStream_t>(stream),
                             reinterpret_cast<const unsigned int*>(local_flags), (unsigned int)rank_mask, (unsigned int)value);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("peer_wait launch: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

// Debug hook (tools/trace_attn.py, tools/trace_gemm.py): device buffer that the next attention / GEMM launches fill with
// %globaltimer stamps (64 / 16 uint64 per CTA); nullptr switches it off.  The stamps are compiled in only with -DM3R_TRACE
// (M3R_TRACE=1 python -m must3r_b200.build): they cost registers in the hot loops.
extern "C" int m3r_debug_trace(void* buf) {
#ifdef M3R_TRACE
  m3r::g_trace = reinterpret_cast<unsigned long long*>(buf);
  return 0;
#else
  (void)buf;
  return m3r::set_error("kernel trace not compiled in (build with M3R_TRACE=1)");
#endif
}
