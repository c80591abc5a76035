// Confidence-filtered point clouds of a reconstructed scene (must3r_b200/engine/demo.py get_3D_model_from_scene).
//
// Two-pass ordered compaction over V views of any sizes and T <= 8 thresholds.  The pixels of every view are cut into
// tiles of kTile consecutive raster positions; tile i of view v is global tile first_tile[v] + i, so global tiles run
// view-major, then in raster order, which is the order numpy's `concatenate([p[m] for ...])` gives.
//  * m3r_scene_count: one CTA per tile reads conf once and counts, for every threshold, the pixels with conf >= thr
//    (NaN is never selected: the comparison is false, as in numpy).  A second kernel (one CTA per threshold) turns the
//    per-tile counts into exclusive offsets and the threshold's total.
//  * m3r_scene_points: one CTA per tile reads conf again, ranks each selected pixel inside its tile with warp ballots
//    and a scan of the per-warp counts, and writes the point (xyz, optionally transformed by the view's c2w) and its
//    colour (ImgNorm -> [0,1], dust3r's `rgb`) to base[t] + tile offset + rank.  base[t] = counts[0] + ... + counts[t-1].
#include "ptx.cuh"
#include "m3r_internal.h"

namespace m3r {

constexpr int kThreads = 256;
constexpr int kPerThread = 4;
constexpr int kTile = kThreads * kPerThread;     // pixel k*kThreads + tid of a tile: raster order is (k, tid) order
constexpr int kWarps = kThreads / 32;
constexpr int kScanThreads = 1024;

__device__ __forceinline__ int view_of_tile(const m3r_scene_view* __restrict__ views, int V, long long tile) {
  int lo = 0, hi = V - 1;                        // last view whose first tile is <= tile
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (views[mid].first_tile <= tile) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kThreads) scene_count_kernel(const m3r_scene_view* __restrict__ views, int V,
                                                               const float* __restrict__ thr, int T, long long n_tiles,
                                                               int* __restrict__ tile_counts) {
  griddep_wait();
  griddep_launch();
  __shared__ int warp_count[kWarps][M3R_SCENE_MAX_THR];
  const long long tile = blockIdx.x;
  const int v = view_of_tile(views, V, tile);
  const m3r_scene_view vw = views[v];
  const long long HW = (long long)vw.H * vw.W;
  const long long base = (tile - vw.first_tile) * kTile;
  float c[kPerThread];
#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    const long long p = base + k * kThreads + threadIdx.x;
    c[k] = p < HW ? __ldg(vw.conf + p) : __int_as_float(0x7fffffff);   // outside the view: NaN, never selected
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int t = 0; t < T; ++t) {
    const float th = __ldg(thr + t);
    int n = 0;
#pragma unroll
    for (int k = 0; k < kPerThread; ++k) n += c[k] >= th ? 1 : 0;
    n = __reduce_add_sync(0xffffffffu, n);
    if (lane == 0) warp_count[wid][t] = n;
  }
  __syncthreads();
  if (threadIdx.x < T) {
    int n = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) n += warp_count[w][threadIdx.x];
    tile_counts[(long long)threadIdx.x * n_tiles + tile] = n;
  }
}

// One CTA per threshold: tile_off[t][i] = sum of tile_counts[t][0..i), counts[t] = the total.
__global__ void __launch_bounds__(kScanThreads) scene_scan_kernel(const int* __restrict__ tile_counts, long long n_tiles,
                                                                  long long* __restrict__ tile_off, long long* __restrict__ counts) {
  griddep_wait();
  griddep_launch();
  __shared__ long long warp_sum[kScanThreads / 32];
  const int t = blockIdx.x;
  const int* in = tile_counts + (long long)t * n_tiles;
  long long* out = tile_off + (long long)t * n_tiles;
  const long long per = (n_tiles + kScanThreads - 1) / kScanThreads;    // each thread owns a contiguous run of tiles
  const long long lo = min(n_tiles, per * threadIdx.x), hi = min(n_tiles, lo + per);
  long long s = 0;
  for (long long i = lo; i < hi; ++i) s += in[i];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long incl = s;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const long long o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) warp_sum[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    long long w = warp_sum[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const long long o = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += o;
    }
    warp_sum[lane] = w;                                      // inclusive over warps
  }
  __syncthreads();
  long long run = incl - s + (wid ? warp_sum[wid - 1] : 0);
  for (long long i = lo; i < hi; ++i) {
    out[i] = run;
    run += in[i];
  }
  if (threadIdx.x == kScanThreads - 1) counts[t] = warp_sum[kScanThreads / 32 - 1];
}

__device__ __forceinline__ float unit_rgb(float x) {        // (x * 0.5) + 0.5, then clip to [0, 1]; NaN stays NaN
  const float v = __fadd_rn(__fmul_rn(x, 0.5f), 0.5f);
  return v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
}

__global__ void __launch_bounds__(kThreads) scene_points_kernel(const m3r_scene_view* __restrict__ views, int V,
                                                                const float* __restrict__ thr, int T, long long n_tiles,
                                                                const long long* __restrict__ tile_off,
                                                                const long long* __restrict__ counts,
                                                                float* __restrict__ pts_out, float* __restrict__ col_out) {
  griddep_wait();
  griddep_launch();
  // per threshold, the selected pixels of each (k, warp) slot in raster order, then their exclusive prefix
  __shared__ int slot[M3R_SCENE_MAX_THR][kPerThread * kWarps];
  const long long tile = blockIdx.x;
  const int v = view_of_tile(views, V, tile);
  const m3r_scene_view vw = views[v];
  const long long HW = (long long)vw.H * vw.W;
  const long long base = (tile - vw.first_tile) * kTile;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  float c[kPerThread];
  unsigned sel[kPerThread];                                  // bit t: pixel k passes threshold t
#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    const long long p = base + k * kThreads + threadIdx.x;
    c[k] = p < HW ? __ldg(vw.conf + p) : __int_as_float(0x7fffffff);
    sel[k] = 0;
  }
  unsigned rank[kPerThread][M3R_SCENE_MAX_THR];              // fully unrolled over t: the ranks stay in registers
#pragma unroll
  for (int t = 0; t < M3R_SCENE_MAX_THR; ++t) {
    if (t >= T) break;
    const float th = __ldg(thr + t);
#pragma unroll
    for (int k = 0; k < kPerThread; ++k) {
      const bool s = c[k] >= th;
      const unsigned b = __ballot_sync(0xffffffffu, s);
      sel[k] |= (s ? 1u : 0u) << t;
      rank[k][t] = __popc(b & lt_mask);
      if (lane == 0) slot[t][k * kWarps + wid] = __popc(b);
    }
  }
  __syncthreads();
  if (wid < T) {                                             // warp t scans the 32 slots of threshold t
    const int n = slot[wid][lane];
    int incl = n;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += o;
    }
    slot[wid][lane] = incl - n;
  }
  __syncthreads();
  unsigned any = 0;
#pragma unroll
  for (int k = 0; k < kPerThread; ++k) any |= sel[k];
  if (!any) return;
  float r[12];
  if (vw.c2w) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) r[4 * i + j] = __ldg(vw.c2w + 4 * i + j);
  }
#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    if (!sel[k]) continue;
    const long long p = base + k * kThreads + threadIdx.x;
    float x = __ldg(vw.pts3d + 3 * p), y = __ldg(vw.pts3d + 3 * p + 1), z = __ldg(vw.pts3d + 3 * p + 2);
    if (vw.c2w) {                                            // geotrf(c2w, pts3d_local): R x + t
      const float X = fmaf(r[0], x, fmaf(r[1], y, r[2] * z)) + r[3];
      const float Y = fmaf(r[4], x, fmaf(r[5], y, r[6] * z)) + r[7];
      const float Z = fmaf(r[8], x, fmaf(r[9], y, r[10] * z)) + r[11];
      x = X; y = Y; z = Z;
    }
    const float cr = unit_rgb(__ldg(vw.img + p)), cg = unit_rgb(__ldg(vw.img + HW + p)), cb = unit_rgb(__ldg(vw.img + 2 * HW + p));
    long long off = 0;
#pragma unroll
    for (int t = 0; t < M3R_SCENE_MAX_THR; ++t) {
      if (t >= T) break;
      if (sel[k] >> t & 1u) {
        const long long o = off + tile_off[(long long)t * n_tiles + tile] + slot[t][k * kWarps + wid] + rank[k][t];
        pts_out[3 * o] = x; pts_out[3 * o + 1] = y; pts_out[3 * o + 2] = z;
        col_out[3 * o] = cr; col_out[3 * o + 1] = cg; col_out[3 * o + 2] = cb;
      }
      off += __ldg(counts + t);
    }
  }
}

static int check_launch(cudaError_t e, const char* what) {
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("%s launch: %s", what, cudaGetErrorString(e));
  count_launch();
  return 0;
}

static int check_args(const char* what, const m3r_scene_view* views, int32_t V, const float* thr, int32_t T,
                      int64_t n_tiles) {
  if (!views || !thr) return set_error("%s: null pointer", what);
  if (V < 1) return set_error("%s: %d views", what, V);
  if (T < 1 || T > M3R_SCENE_MAX_THR) return set_error("%s: %d thresholds (1..%d)", what, T, M3R_SCENE_MAX_THR);
  if (n_tiles < 1 || n_tiles > 0x7fffffffLL) return set_error("%s: %lld tiles (1..2^31 - 1)", what, (long long)n_tiles);
  return 0;
}

}  // namespace m3r

using namespace m3r;

extern "C" int m3r_scene_count(const m3r_scene_view* views, int32_t V, const float* thr, int32_t T, int64_t n_tiles,
                               int32_t* tile_counts, int64_t* tile_off, int64_t* counts, void* stream) {
  if (int rc = check_args("scene_count", views, V, thr, T, n_tiles)) return rc;
  if (!tile_counts || !tile_off || !counts) return set_error("scene_count: null pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (int rc = check_launch(launch_pdl(scene_count_kernel, dim3((unsigned)n_tiles), dim3(kThreads), 0, s, views, (int)V, thr,
                                       (int)T, (long long)n_tiles, (int*)tile_counts), "scene_count"))
    return rc;
  return check_launch(launch_pdl(scene_scan_kernel, dim3((unsigned)T), dim3(kScanThreads), 0, s, (const int*)tile_counts,
                                 (long long)n_tiles, (long long*)tile_off, (long long*)counts), "scene_scan");
}

extern "C" int m3r_scene_points(const m3r_scene_view* views, int32_t V, const float* thr, int32_t T, int64_t n_tiles,
                                const int64_t* tile_off, const int64_t* counts, float* pts_out, float* col_out, void* stream) {
  if (int rc = check_args("scene_points", views, V, thr, T, n_tiles)) return rc;
  if (!tile_off || !counts || !pts_out || !col_out) return set_error("scene_points: null pointer");
  return check_launch(launch_pdl(scene_points_kernel, dim3((unsigned)n_tiles), dim3(kThreads), 0,
                                 reinterpret_cast<cudaStream_t>(stream), views, (int)V, thr, (int)T, (long long)n_tiles,
                                 (const long long*)tile_off, (const long long*)counts, pts_out, col_out), "scene_points");
}
