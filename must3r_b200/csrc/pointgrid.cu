// Exact nearest-neighbour grid index over the SLAM keyframe point map (the searchers of must3r_b200/engine/keyframes.py).
//
// Layout (built by engine/keyframes.py PointGrid from m3r_pointgrid_keys + torch.sort):
//  * every map point p with bucket b gets a 64-bit key: bits [62:54] = b, bits [53:0] = the Morton code (bits of x, y, z
//    interleaved) of its cell c = floor(p * inv_h), 18 bits per axis biased by 2^17.  Points whose cell does not fit
//    (|p * inv_h| out of range, or non-finite) get the bucket's overflow key (all 54 low bits set, a code no real cell
//    has), so they sort to the end of the bucket: the bucket's overflow list.
//  * pts [P,3]: the points sorted by key; cell_keys [C]: the distinct keys in order; cell_off [C+1]: each cell's point
//    range; bucket_cells [nb+1]: each bucket's cell range.
//  Because the code is a Morton code, the cells of an aligned block of 2^L x 2^L x 2^L cells are one contiguous range of
//  cell_keys, found with two binary searches.
//
// Query (one thread per query point): scan the overflow list, then visit blocks level by level (level L: blocks of
// 2^L cells per side), in Chebyshev rings 0..kRing around the query's block, skipping blocks and cells whose box cannot
// hold a point closer than the best so far.  Stop after ring r of level L once no unvisited cell can (the bound is about
// r * 2^L * h).  A level that does not stop has visited all its rings, so the next level skips the blocks whose eight
// children all lie in them; blocks only partly covered are visited again, which costs time but not exactness (fminf
// of a distance already taken changes nothing).  The last level is one block holding the whole bucket, so the search
// always terminates exactly; a query outside the key range visits the whole bucket directly.
// Distances use exactly the expression of nn_min_dist_kernel (elementwise.cu) and are combined with fminf, so the
// result is bitwise the brute-force scan of the bucket whatever order the cells are visited in, provided no cell holding
// a point that ties or beats the best is ever skipped.  The bounds below guarantee that:
//  * a point in cell c satisfies p/h in [c - 2^-6, c + 1 + 2^-6): |p * inv_h| < 2^17, and fl(p * inv_h) differs from
//    p/h by at most two roundings relative to 2^17;
//  * boxes are widened by h/16 per side, which also covers the rounding of (c -/+ 1/16) * h;
//  * the squared gap is shrunk by 2e-5 relatively, far more than the few roundings in it and in the distance itself
//    (every point in the box then has a rounded squared distance strictly above the bound).
#include "ptx.cuh"
#include "m3r_internal.h"

namespace m3r {

constexpr int kAxisBits = 18;
constexpr int kBias = 1 << (kAxisBits - 1);                       // cell c is stored as c + kBias in [0, 2^18 - 1)
constexpr float kCellLo = -(float)kBias, kCellHi = (float)(kBias - 1);
constexpr unsigned long long kOverflow = (1ull << (3 * kAxisBits)) - 1;
constexpr int kMaxBuckets = 1 << (63 - 3 * kAxisBits);           // 512: the key stays non-negative as int64
constexpr int kRing = 2;
constexpr float kSlack = 0.0625f;                                 // box widening, in cells
constexpr float kShrink = 0.99998f;

__device__ __forceinline__ bool cell_coord(float x, float inv_h, int& c) {
  const float v = x * inv_h;
  if (!(v >= kCellLo && v < kCellHi)) return false;              // also rejects NaN and inf
  c = (int)floorf(v);
  return true;
}

__device__ __forceinline__ unsigned long long spread3(unsigned long long x) {   // bit i -> bit 3i, for 21-bit x
  x &= 0x1fffffull;
  x = (x | x << 32) & 0x1f00000000ffffull;
  x = (x | x << 16) & 0x1f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}

__device__ __forceinline__ int compact3(unsigned long long x) {                 // inverse of spread3
  x &= 0x1249249249249249ull;
  x = (x ^ (x >> 2)) & 0x10c30c30c30c30c3ull;
  x = (x ^ (x >> 4)) & 0x100f00f00f00f00full;
  x = (x ^ (x >> 8)) & 0x1f0000ff0000ffull;
  x = (x ^ (x >> 16)) & 0x1f00000000ffffull;
  x = (x ^ (x >> 32)) & 0x1fffffull;
  return (int)x;
}

// Morton code of biased coordinates (ux, uy, uz)
__device__ __forceinline__ unsigned long long morton(unsigned ux, unsigned uy, unsigned uz) {
  return (spread3(ux) << 2) | (spread3(uy) << 1) | spread3(uz);
}

// Gap from q to the cells [lo, hi) of one axis (unbiased cell coordinates), boxes widened by kSlack cells.
__device__ __forceinline__ float axis_gap(float q, int lo, int hi, float h) {
  return fmaxf(0.f, fmaxf(((float)lo - kSlack) * h - q, q - ((float)hi + kSlack) * h));
}

// Lower bound of the rounded squared distance from q to any point stored in the cells [x0,x1) x [y0,y1) x [z0,z1).
__device__ __forceinline__ float box_lb2(float qx, float qy, float qz, int x0, int x1, int y0, int y1, int z0, int z1, float h) {
  const float gx = axis_gap(qx, x0, x1, h), gy = axis_gap(qy, y0, y1, h), gz = axis_gap(qz, z0, z1, h);
  return (gx * gx + gy * gy + gz * gz) * kShrink;
}

__device__ __forceinline__ float scan(float qx, float qy, float qz, const float* __restrict__ pts, int lo, int hi, float best) {
  for (int j = lo; j < hi; ++j) {
    const float dx = qx - __ldg(pts + 3 * j), dy = qy - __ldg(pts + 3 * j + 1), dz = qz - __ldg(pts + 3 * j + 2);
    best = fminf(best, fmaf(dx, dx, fmaf(dy, dy, dz * dz)));
  }
  return best;
}

// Scan the points of the cells [c0, c1) whose box may hold a point closer than `best`.
__device__ __forceinline__ float visit(float qx, float qy, float qz, const float* __restrict__ pts, const long long* __restrict__ keys,
                                       const int* __restrict__ cell_off, int c0, int c1, float h, float best) {
  for (int c = c0; c < c1; ++c) {
    const unsigned long long k = (unsigned long long)__ldg(keys + c) & kOverflow;   // the cell's Morton code
    const int x = compact3(k >> 2) - kBias, y = compact3(k >> 1) - kBias, z = compact3(k) - kBias;
    if (box_lb2(qx, qy, qz, x, x + 1, y, y + 1, z, z + 1, h) < best)
      best = scan(qx, qy, qz, pts, __ldg(cell_off + c), __ldg(cell_off + c + 1), best);
  }
  return best;
}

// First index in keys[lo, hi) whose key is >= `key`.
__device__ __forceinline__ int lower_bound(const long long* __restrict__ keys, int lo, int hi, long long key) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(keys + mid) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(256) pointgrid_keys_kernel(const float* __restrict__ pts, const int* __restrict__ bucket,
                                                             long long P, float inv_h, long long* __restrict__ keys) {
  griddep_wait();
  griddep_launch();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const unsigned long long b = (bucket ? (unsigned long long)bucket[i] : 0ull) << (3 * kAxisBits);
  int cx, cy, cz;
  const bool ok = cell_coord(pts[3 * i], inv_h, cx) & cell_coord(pts[3 * i + 1], inv_h, cy) & cell_coord(pts[3 * i + 2], inv_h, cz);
  keys[i] = (long long)(b | (ok ? morton(cx + kBias, cy + kBias, cz + kBias) : kOverflow));
}

__global__ void __launch_bounds__(128) pointgrid_query_kernel(const float* __restrict__ q, const int* __restrict__ qbucket, int Q,
                                                              const float* __restrict__ pts, const long long* __restrict__ keys,
                                                              const int* __restrict__ cell_off, const int* __restrict__ bucket_cells,
                                                              int nb, float h, float inv_h, float* __restrict__ out) {
  griddep_wait();
  griddep_launch();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Q) return;
  const float qx = q[3 * i], qy = q[3 * i + 1], qz = q[3 * i + 2];
  const int b = qbucket ? qbucket[i] : 0;
  float best = INFINITY;
  if (b < 0 || b >= nb) { out[i] = __int_as_float(0x7fffffff); return; }   // a bucket id out of range gives NaN
  const unsigned long long base = (unsigned long long)b << (3 * kAxisBits);
  int lo = __ldg(bucket_cells + b), hi = __ldg(bucket_cells + b + 1);
  if (lo < hi && (unsigned long long)__ldg(keys + hi - 1) == (base | kOverflow)) {
    --hi;
    best = scan(qx, qy, qz, pts, __ldg(cell_off + hi), __ldg(cell_off + hi + 1), best);
  }
  // A non-finite query is at infinite (or NaN, which fminf drops) distance from every point: the scan gives inf.
  if (lo < hi && isfinite(qx) && isfinite(qy) && isfinite(qz)) {
    int cx, cy, cz;
    if (cell_coord(qx, inv_h, cx) & cell_coord(qy, inv_h, cy) & cell_coord(qz, inv_h, cz)) {
      bool done = false;
      for (int L = 0; L <= kAxisBits && !done; ++L) {
        const int n = 1 << (kAxisBits - L);                        // blocks per axis at this level
        const int bx = (cx + kBias) >> L, by = (cy + kBias) >> L, bz = (cz + kBias) >> L;
        // the previous level's query block: blocks of this level whose children all lie within its rings were visited
        const int px = L ? (cx + kBias) >> (L - 1) : 0, py = L ? (cy + kBias) >> (L - 1) : 0, pz = L ? (cz + kBias) >> (L - 1) : 0;
        for (int r = 0; r <= kRing && !done; ++r) {
          for (int dz = -r; dz <= r; ++dz) {
            const int Z = bz + dz;
            if (Z < 0 || Z >= n) continue;
            const bool cov_z = L > 0 && 2 * Z >= pz - kRing && 2 * Z + 1 <= pz + kRing;
            for (int dy = -r; dy <= r; ++dy) {
              const int Y = by + dy;
              if (Y < 0 || Y >= n) continue;
              const bool cov_yz = cov_z && 2 * Y >= py - kRing && 2 * Y + 1 <= py + kRing;
              const int step = (dz == -r || dz == r || dy == -r || dy == r) ? 1 : 2 * r;
              for (int dx = -r; dx <= r; dx += step) {
                const int X = bx + dx;
                if (X < 0 || X >= n || (cov_yz && 2 * X >= px - kRing && 2 * X + 1 <= px + kRing)) continue;
                if (box_lb2(qx, qy, qz, (X << L) - kBias, ((X + 1) << L) - kBias, (Y << L) - kBias, ((Y + 1) << L) - kBias,
                            (Z << L) - kBias, ((Z + 1) << L) - kBias, h) >= best) continue;
                const unsigned long long first = base | (morton(X, Y, Z) << (3 * L));
                const int c0 = lower_bound(keys, lo, hi, (long long)first);
                const int c1 = lower_bound(keys, c0, hi, (long long)(first + (1ull << (3 * L))));
                best = visit(qx, qy, qz, pts, keys, cell_off, c0, c1, h, best);
              }
            }
          }
          // Every cell outside rings 0..r of this level is more than (r * 2^L - 2^-6 - 1/16) h away along one axis.
          const float bound = ((float)(r << L) - 0.125f) * h;
          done = r >= 1 && best < bound * bound * kShrink;
        }
      }
    } else {
      best = visit(qx, qy, qz, pts, keys, cell_off, lo, hi, h, best);
    }
  }
  out[i] = sqrtf(best);
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("%s launch: %s", what, cudaGetErrorString(e));
  count_launch();
  return 0;
}

}  // namespace m3r

using namespace m3r;

extern "C" int m3r_pointgrid_keys(const float* pts, const int32_t* bucket, int64_t P, float inv_h, int64_t* keys, void* stream) {
  if (P <= 0) return 0;
  if (!pts || !keys) return set_error("pointgrid_keys: null pointer");
  if (!(inv_h > 0.f) || !isfinite(inv_h)) return set_error("pointgrid_keys: bad inverse cell size %g", (double)inv_h);
  launch_pdl(pointgrid_keys_kernel, dim3((unsigned)((P + 255) / 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), pts,
             (const int*)bucket, (long long)P, inv_h, (long long*)keys);
  return check_launch("pointgrid_keys");
}

extern "C" int m3r_pointgrid_query(const float* queries, const int32_t* qbucket, int32_t Q, const float* pts, int64_t P,
                                   const int64_t* cell_keys, const int32_t* cell_off, int32_t C, const int32_t* bucket_cells,
                                   int32_t nb, float h, float inv_h, float* out, void* stream) {
  if (Q <= 0) return 0;
  if (!queries || !out || !bucket_cells) return set_error("pointgrid_query: null pointer");
  if (C > 0 && (!pts || !cell_keys || !cell_off)) return set_error("pointgrid_query: null pointer");
  if (nb < 1 || nb > kMaxBuckets) return set_error("pointgrid_query: %d buckets (1..%d)", nb, kMaxBuckets);
  if (P > 0x7fffffffLL) return set_error("pointgrid_query: %lld points (at most 2^31 - 1)", (long long)P);
  if (!(h > 0.f) || !isfinite(h) || !(inv_h > 0.f) || !isfinite(inv_h)) return set_error("pointgrid_query: bad cell size %g", (double)h);
  launch_pdl(pointgrid_query_kernel, dim3((Q + 127) / 128), dim3(128), 0, reinterpret_cast<cudaStream_t>(stream), queries,
             (const int*)qbucket, (int)Q, pts, (const long long*)cell_keys, (const int*)cell_off, (const int*)bucket_cells,
             (int)nb, h, inv_h, out);
  return check_launch("pointgrid_query");
}
