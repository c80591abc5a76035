// Per-frame camera and keyframe test of the SLAM front end (must3r_b200/engine/slam.py).
//
// m3r_slam_pose: each view is one cluster of kCluster CTAs; every CTA owns a contiguous slice of the view's pixels.
// The focal fit (1 + 10 dependent sums), the Procrustes centroids and cross-covariance and the radix selection of the
// median are all cluster-wide reductions: each CTA reduces its slice into shared memory, the cluster synchronises, and
// every CTA adds up the partials of all ranks through distributed shared memory in rank order, so all CTAs hold the
// same total without a second launch or a grid-wide barrier.  Partials and histograms are double-buffered: the buffer a
// reduction reads is only written again two reductions later, after a cluster barrier every reader has passed.
// Sums accumulate in double over fp32 per-pixel terms; the rotation is Horn's quaternion in double, in one thread.
//
// m3r_slam_keyframe: one cluster; the same reductions and the same selection pick the two order statistics of the
// percentile, which is interpolated in double exactly as np.percentile / torch.quantile do.
#include <cooperative_groups.h>
#include <float.h>
#include "ptx.cuh"
#include "m3r_internal.h"

namespace cg = cooperative_groups;

namespace m3r {

constexpr int kCluster = 8;                 // CTAs per view (portable cluster size)
constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxSum = 9;                  // widest reduction: the 3x3 cross-covariance

struct SlamShared {
  double part[2][kMaxSum];                  // this CTA's partial sums, read by the whole cluster
  double warp[kWarps][kMaxSum];
  double total[kMaxSum];
  unsigned int hist[2][256];                // this CTA's radix histogram, read by the whole cluster
  unsigned int count[256];                  // the cluster's histogram
  unsigned int sel_bin;
  unsigned long long sel_rank;
};

// Sums v[0..K) over every thread of the cluster; every thread gets the totals.
template <int K>
__device__ __forceinline__ void cluster_sum(cg::cluster_group& cluster, SlamShared& sh, int& buf, double (&v)[K]) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double x = v[k];
#pragma unroll
    for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (lane == 0) sh.warp[wid][k] = x;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += sh.warp[w][threadIdx.x];
    sh.part[buf][threadIdx.x] = s;
  }
  cluster.sync();
  if (threadIdx.x < K) {
    double s = 0.0;
    for (unsigned r = 0; r < cluster.num_blocks(); ++r) s += cluster.map_shared_rank(&sh.part[buf][0], r)[threadIdx.x];
    sh.total[threadIdx.x] = s;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = sh.total[k];
  buf ^= 1;
}

// Total order of the float bits: negative values reversed below the positive ones (NaN never reaches a selection).
__device__ __forceinline__ unsigned float_key(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Exact selection: the key of 0-based rank `k` among the keys that key_of(i, key) accepts for the elements
// i in [lo, hi) of every CTA of the cluster (k must be below their number).  Four 8-bit radix passes, most
// significant digit first; each pass histograms the keys that match the digits chosen so far.
template <class KeyOf>
__device__ __forceinline__ unsigned cluster_select(cg::cluster_group& cluster, SlamShared& sh, int& buf, long long lo, long long hi,
                                   unsigned long long k, KeyOf key_of) {
  unsigned prefix = 0, mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    unsigned* h = sh.hist[buf];
    for (int j = threadIdx.x; j < 256; j += blockDim.x) h[j] = 0;
    __syncthreads();
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      unsigned key;
      if (key_of(i, key) && (key & mask) == prefix) atomicAdd(&h[(key >> shift) & 255u], 1u);
    }
    cluster.sync();
    if (threadIdx.x < 256) {
      unsigned c = 0;
      for (unsigned r = 0; r < cluster.num_blocks(); ++r) c += cluster.map_shared_rank(h, r)[threadIdx.x];
      sh.count[threadIdx.x] = c;
    }
    __syncthreads();
    if (threadIdx.x < 32) {                 // the bin holding rank k: a scan over 32 lanes of 8 bins each
      const int l = threadIdx.x;
      unsigned long long s = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += sh.count[8 * l + j];
      unsigned long long inc = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
        if (l >= o) inc += t;
      }
      const unsigned ball = __ballot_sync(0xffffffffu, inc > k);
      const int owner = ball ? __ffs(ball) - 1 : 31;
      if (l == owner) {
        unsigned long long acc = inc - s;
        int b = 8 * l + 7;
        for (int j = 0; j < 8; ++j) {
          if (acc + sh.count[8 * l + j] > k) { b = 8 * l + j; break; }
          acc += sh.count[8 * l + j];
        }
        sh.sel_bin = (unsigned)b;
        sh.sel_rank = k - acc;
      }
    }
    __syncthreads();
    prefix |= sh.sel_bin << shift;
    mask |= 255u << shift;
    k = sh.sel_rank;
    buf ^= 1;
  }
  return prefix;
}

// The proper rotation maximising tr(R^T ...) for S = sum w (x - xc)(y - yc)^T, as engine/camera.py _rotation_horn:
// the dominant eigenvector of Horn's symmetric 4x4 matrix by ten squarings of the shifted, normalised matrix.
__device__ __forceinline__ void horn_rotation(const double* S, double* R) {
  const double Sxx = S[0], Sxy = S[1], Sxz = S[2], Syx = S[3], Syy = S[4], Syz = S[5], Szx = S[6], Szy = S[7], Szz = S[8];
  double P[16] = {Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx,
                  Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz,
                  Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy,
                  Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz};
  double n = 0.0;
  for (int i = 0; i < 16; ++i) n += P[i] * P[i];
  n = fmax(sqrt(n), 1e-300);
  for (int i = 0; i < 16; ++i) P[i] = P[i] / n + ((i % 5) == 0 ? 1.0 : 0.0);
#pragma unroll 1
  for (int it = 0; it < 10; ++it) {
    double Q[16];
    double m = 0.0;
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) {
        double v = 0.0;
        for (int j = 0; j < 4; ++j) v += P[4 * r + j] * P[4 * j + c];
        Q[4 * r + c] = v;
        m += v * v;
      }
    m = fmax(sqrt(m), 1e-300);
    for (int i = 0; i < 16; ++i) P[i] = Q[i] / m;
  }
  // P ~ v v^T: its column of largest norm is the eigenvector (up to sign)
  double best = -1.0, w = 0.0, x = 0.0, y = 0.0, z = 0.0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const double v = P[c] * P[c] + P[4 + c] * P[4 + c] + P[8 + c] * P[8 + c] + P[12 + c] * P[12 + c];
    if (v > best) { best = v; w = P[c]; x = P[4 + c]; y = P[8 + c]; z = P[12 + c]; }
  }
  const double qn = fmax(sqrt(w * w + x * x + y * y + z * z), 1e-300);
  w /= qn; x /= qn; y /= qn; z /= qn;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - w * z);     R[2] = 2 * (x * z + w * y);
  R[3] = 2 * (x * y + w * z);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - w * x);
  R[6] = 2 * (x * z - w * y);     R[7] = 2 * (y * z + w * x);     R[8] = 1 - 2 * (x * x + y * y);
}

// (x, y) / z with NaN and +-inf replaced by 0 (nan_to_num of the reference's focal fit), and the pixel minus the
// principal point.
__device__ __forceinline__ void ray_pixel(const float* __restrict__ loc, long long i, int W, float ppx, float ppy,
                                          float& rx, float& ry, float& px, float& py) {
  const float z = loc[3 * i + 2];
  rx = loc[3 * i] / z;
  ry = loc[3 * i + 1] / z;
  if (!isfinite(rx)) rx = 0.f;
  if (!isfinite(ry)) ry = 0.f;
  px = (float)(i % W) - ppx;
  py = (float)(i / W) - ppy;
}

// Per-view focal state of a batch of views from several cameras (m3r_slam_pose_views); m3r_slam_pose passes one value
// for all views and PER_VIEW = false.
struct ViewFlags {
  int has_seq_focal[M3R_MAX_COMMIT];
  float seq_focal[M3R_MAX_COMMIT];
  int is_first[M3R_MAX_COMMIT];
};

template <bool PER_VIEW>
__global__ void __cluster_dims__(kCluster, 1, 1) __launch_bounds__(kThreads)
slam_pose_kernel(const float* __restrict__ pts3d, float* __restrict__ pts3d_local, const float* __restrict__ conf, int H,
                 int W, float ppx, float ppy, int has_seq_focal_all, float seq_focal_all, int is_first_all,
                 const __grid_constant__ ViewFlags vf, m3r_slam_record* __restrict__ rec) {
  __shared__ SlamShared sh;
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank();
  const int view = blockIdx.x / kCluster;
  const int has_seq_focal = PER_VIEW ? vf.has_seq_focal[view] : has_seq_focal_all;
  const float seq_focal = PER_VIEW ? vf.seq_focal[view] : seq_focal_all;
  const int is_first = PER_VIEW ? vf.is_first[view] : is_first_all;
  const long long N = (long long)H * W;
  const long long chunk = (N + kCluster - 1) / kCluster;
  const long long lo = min(N, rank * chunk), hi = min(N, lo + chunk);
  const float* __restrict__ wp = pts3d + 3 * N * view;
  float* __restrict__ loc = pts3d_local + 3 * N * view;
  const float* __restrict__ cf = conf + N * view;
  int sbuf = 0, hbuf = 0;
  griddep_wait();
  griddep_launch();

  // closed-form L2 focal; the confidence sum and NaN count ride along
  double s0[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    float rx, ry, px, py;
    ray_pixel(loc, i, W, ppx, ppy, rx, ry, px, py);
    s0[0] += (double)(rx * px + ry * py);
    s0[1] += (double)(rx * rx + ry * ry);
    const float c = cf[i];
    s0[2] += (double)c;
    s0[3] += isnan(c) ? 1.0 : 0.0;
  }
  cluster_sum(cluster, sh, sbuf, s0);
  double focal = s0[0] / s0[1];
  // iteratively re-weighted least squares, weights 1 / distance
  for (int it = 0; it < 10; ++it) {
    const float f = (float)focal;
    double s[2] = {0.0, 0.0};
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      float rx, ry, px, py;
      ray_pixel(loc, i, W, ppx, ppy, rx, ry, px, py);
      const float dx = px - f * rx, dy = py - f * ry;
      const double w = (double)(1.f / fmaxf(sqrtf(dx * dx + dy * dy), 1e-8f));
      s[0] += w * (double)(rx * px + ry * py);
      s[1] += w * (double)(rx * rx + ry * ry);
    }
    cluster_sum(cluster, sh, sbuf, s);
    focal = s[0] / s[1];
  }
  const float focal_f = (float)(focal < 0.0 ? 0.0 : focal);

  double Rm[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0, 0, 0};
  if (!is_first) {
    const bool rectify = has_seq_focal != 0;
    const float ratio = rectify ? seq_focal / focal_f : 1.f;
    double s1[7] = {0, 0, 0, 0, 0, 0, 0};
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      float z = loc[3 * i + 2];
      if (rectify) { z *= ratio; loc[3 * i + 2] = z; }
      const double w = (double)(cf[i] - 1.f);
      s1[0] += w;
      s1[1] += w * loc[3 * i]; s1[2] += w * loc[3 * i + 1]; s1[3] += w * z;
      s1[4] += w * wp[3 * i]; s1[5] += w * wp[3 * i + 1]; s1[6] += w * wp[3 * i + 2];
    }
    cluster_sum(cluster, sh, sbuf, s1);
    const double xc[3] = {s1[1] / s1[0], s1[2] / s1[0], s1[3] / s1[0]};
    const double yc[3] = {s1[4] / s1[0], s1[5] / s1[0], s1[6] / s1[0]};
    double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      const double w = (double)(cf[i] - 1.f);
      const double x[3] = {loc[3 * i] - xc[0], loc[3 * i + 1] - xc[1], loc[3 * i + 2] - xc[2]};
      const double y[3] = {wp[3 * i] - yc[0], wp[3 * i + 1] - yc[1], wp[3 * i + 2] - yc[2]};
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) S[3 * a + b] += w * x[a] * y[b];
    }
    cluster_sum(cluster, sh, sbuf, S);
    if (rank == 0 && threadIdx.x == 0) {
      horn_rotation(S, Rm);
      for (int a = 0; a < 3; ++a) t[a] = yc[a] - (Rm[3 * a] * xc[0] + Rm[3 * a + 1] * xc[1] + Rm[3 * a + 2] * xc[2]);
    }
  }

  // lower median of conf (torch.median): rank (N - 1) / 2; NaN if any conf is NaN
  float median = __int_as_float(0x7fffffff);
  if (s0[3] == 0.0 && N > 0) {
    const unsigned key = cluster_select(cluster, sh, hbuf, lo, hi, (unsigned long long)((N - 1) / 2),
                                        [&](long long i, unsigned& k) { k = float_key(cf[i]); return true; });
    median = key_float(key);
  }

  if (rank == 0 && threadIdx.x == 0) {
    m3r_slam_record& r = rec[view];
    for (int a = 0; a < 4; ++a)
      for (int b = 0; b < 4; ++b) {
        const double c2w = a < 3 ? (b < 3 ? Rm[3 * a + b] : t[a]) : (b == 3 ? 1.0 : 0.0);
        // w2c = [R^T, -R^T t]
        const double w2c = a < 3 ? (b < 3 ? Rm[3 * b + a] : -(Rm[a] * t[0] + Rm[3 + a] * t[1] + Rm[6 + a] * t[2]))
                                 : (b == 3 ? 1.0 : 0.0);
        r.c2w[4 * a + b] = (float)c2w;
        r.w2c[4 * a + b] = (float)w2c;
      }
    r.focal = focal_f;
    r.conf_mean = (float)(s0[2] / (double)N);
    r.conf_median = median;
    r.n_conf = 0;
    r.score = 0.0;
    r.keyframe = 0;
    r.reserved = 0;
  }
  cluster.sync();                         // no CTA leaves while another may still read its shared memory
}

// One cluster per frame: frame blockIdx.x / kCluster reads its own rows of dists [F, Q], conf [F, H, W] and pts3d_local
// [F, H, W, 3] and writes rec[frame]; bit f of first_mask is frame f's is_first.  A single frame (F = 1) is
// m3r_slam_keyframe.
__global__ void __cluster_dims__(kCluster, 1, 1) __launch_bounds__(kThreads)
slam_keyframe_kernel(const float* __restrict__ dists_all, const float* __restrict__ conf_all,
                     const float* __restrict__ pts3d_local_all, int H, int W, int s, int mode, double q, double thr,
                     float min_conf, unsigned long long first_mask, m3r_slam_record* __restrict__ rec_all) {
  __shared__ SlamShared sh;
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank();
  const int frame = blockIdx.x / kCluster;
  const int is_first = (int)((first_mask >> frame) & 1ull);
  const int ws = (W + s - 1) / s;
  const long long Q = (long long)((H + s - 1) / s) * ws;
  const long long HW = (long long)H * W;
  // (a null dists / pts3d_local is never read: the conf modes do not look at them)
  const float* __restrict__ dists = dists_all + Q * frame;
  const float* __restrict__ conf = conf_all + HW * frame;
  const float* __restrict__ pts3d_local = pts3d_local_all + 3 * HW * frame;
  m3r_slam_record* __restrict__ rec = rec_all + frame;
  const long long chunk = (Q + kCluster - 1) / kCluster;
  const long long lo = min(Q, rank * chunk), hi = min(Q, lo + chunk);
  int sbuf = 0, hbuf = 0;
  griddep_wait();
  griddep_launch();
  const bool nn = mode == M3R_OVERLAP_NN || mode == M3R_OVERLAP_NN_NORM;
  auto pixel = [&](long long i) { return (i / ws) * s * (long long)W + (i % ws) * s; };
  auto value = [&](long long i) {
    float d = dists[i];
    if (mode == M3R_OVERLAP_NN_NORM) d = d / (pts3d_local[3 * pixel(i) + 2] + 1e-9f);
    return d == INFINITY ? FLT_MAX : d;
  };
  // Every CTA runs the same reductions whatever the mode and the data (they synchronise the cluster); the conf modes
  // count nothing and select nothing.
  auto masked = [&](long long i) { return nn && conf[pixel(i)] > min_conf; };
  double cnt[2] = {0.0, 0.0};
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    if (masked(i)) {
      cnt[0] += 1.0;
      cnt[1] += isnan(value(i)) ? 1.0 : 0.0;
    }
  }
  cluster_sum(cluster, sh, sbuf, cnt);
  const unsigned long long n = (unsigned long long)cnt[0];
  auto key_of = [&](long long i, unsigned& k) {
    if (!masked(i)) return false;
    k = float_key(value(i));
    return true;
  };
  // np.percentile / torch.quantile 'linear': index q (n - 1) between two order statistics, lerp in double
  const double idx = n ? q * (double)(n - 1) : 0.0;
  const unsigned long long below = (unsigned long long)floor(idx);
  const unsigned long long above = below + 1 < n ? below + 1 : below;
  const double g = idx - (double)below;
  const double a = key_float(cluster_select(cluster, sh, hbuf, lo, hi, below, key_of));
  const double b = key_float(cluster_select(cluster, sh, hbuf, lo, hi, above, key_of));
  const double diff = b - a;
  double score = 0.0;
  if (!nn) score = mode == M3R_OVERLAP_MEANCONF ? (double)rec->conf_mean : (double)rec->conf_median;
  else if (n > 0 && cnt[1] > 0.0) score = __longlong_as_double(0x7ff8000000000000LL);
  else if (n > 0) score = g >= 0.5 ? b - diff * (1.0 - g) : a + diff * g;
  if (rank == 0 && threadIdx.x == 0) {
    const bool choose = nn ? score > thr : score < thr;
    rec->n_conf = (int)cnt[0];
    rec->score = score;
    rec->keyframe = (is_first || (choose && rec->conf_median > min_conf)) ? 1 : 0;
  }
  cluster.sync();
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("%s launch: %s", what, cudaGetErrorString(e));
  count_launch();
  return 0;
}

}  // namespace m3r

using namespace m3r;

static int pose_args(const float* pts3d, const float* pts3d_local, const float* conf, int32_t B, int32_t H, int32_t W,
                     const m3r_slam_record* rec) {
  if (B <= 0 || H <= 0 || W <= 0) return set_error("slam_pose: bad shape B=%d H=%d W=%d", B, H, W);
  if (!pts3d || !pts3d_local || !conf || !rec) return set_error("slam_pose: null pointer");
  return 0;
}

extern "C" int m3r_slam_pose(const float* pts3d, float* pts3d_local, const float* conf, int32_t B, int32_t H, int32_t W,
                             float ppx, float ppy, int32_t has_seq_focal, float seq_focal, int32_t is_first,
                             m3r_slam_record* rec, void* stream) {
  if (pose_args(pts3d, pts3d_local, conf, B, H, W, rec)) return 1;
  const ViewFlags none = {};
  launch_pdl(slam_pose_kernel<false>, dim3(B * kCluster), dim3(kThreads), 0, reinterpret_cast<cudaStream_t>(stream), pts3d,
             pts3d_local, conf, (int)H, (int)W, ppx, ppy, (int)has_seq_focal, seq_focal, (int)is_first, none, rec);
  return check_launch("slam_pose");
}

extern "C" int m3r_slam_pose_views(const float* pts3d, float* pts3d_local, const float* conf, int32_t B, int32_t H,
                                   int32_t W, float ppx, float ppy, const int32_t* has_seq_focal, const float* seq_focal,
                                   const int32_t* is_first, m3r_slam_record* rec, void* stream) {
  if (pose_args(pts3d, pts3d_local, conf, B, H, W, rec)) return 1;
  if (B > M3R_MAX_COMMIT) return set_error("slam_pose_views: B = %d views, at most %d", B, M3R_MAX_COMMIT);
  if (!has_seq_focal || !seq_focal || !is_first) return set_error("slam_pose_views: null per-view array");
  ViewFlags vf = {};
  for (int v = 0; v < B; ++v) {
    vf.has_seq_focal[v] = has_seq_focal[v];
    vf.seq_focal[v] = seq_focal[v];
    vf.is_first[v] = is_first[v];
  }
  launch_pdl(slam_pose_kernel<true>, dim3(B * kCluster), dim3(kThreads), 0, reinterpret_cast<cudaStream_t>(stream), pts3d,
             pts3d_local, conf, (int)H, (int)W, ppx, ppy, 0, 0.f, 0, vf, rec);
  return check_launch("slam_pose_views");
}

static int keyframe_args(const float* dists, const float* conf, const float* pts3d_local, int32_t H, int32_t W,
                         int32_t subsamp, int32_t mode, double percentile, const m3r_slam_record* rec) {
  if (H <= 0 || W <= 0 || subsamp <= 0) return set_error("slam_keyframe: bad shape H=%d W=%d subsamp=%d", H, W, subsamp);
  if (mode < M3R_OVERLAP_NN || mode > M3R_OVERLAP_MEDIANCONF) return set_error("slam_keyframe: unknown overlap mode %d", mode);
  if (!(percentile >= 0.0 && percentile <= 100.0)) return set_error("slam_keyframe: percentile %g outside [0, 100]", percentile);
  if (!conf || !rec || (mode <= M3R_OVERLAP_NN_NORM && !dists) || (mode == M3R_OVERLAP_NN_NORM && !pts3d_local))
    return set_error("slam_keyframe: null pointer");
  return 0;
}

extern "C" int m3r_slam_keyframe(const float* dists, const float* conf, const float* pts3d_local, int32_t H, int32_t W,
                                 int32_t subsamp, int32_t mode, double percentile, double thr, float min_conf_keyframe,
                                 int32_t is_first, m3r_slam_record* rec, void* stream) {
  if (keyframe_args(dists, conf, pts3d_local, H, W, subsamp, mode, percentile, rec)) return 1;
  launch_pdl(slam_keyframe_kernel, dim3(kCluster), dim3(kThreads), 0, reinterpret_cast<cudaStream_t>(stream), dists, conf,
             pts3d_local, (int)H, (int)W, (int)subsamp, (int)mode, percentile / 100.0, thr, min_conf_keyframe,
             is_first ? 1ull : 0ull, rec);
  return check_launch("slam_keyframe");
}

extern "C" int m3r_slam_keyframe_frames(const float* dists, const float* conf, const float* pts3d_local, int32_t F,
                                        int32_t H, int32_t W, int32_t subsamp, int32_t mode, double percentile, double thr,
                                        float min_conf_keyframe, const int32_t* is_first, m3r_slam_record* rec,
                                        void* stream) {
  if (keyframe_args(dists, conf, pts3d_local, H, W, subsamp, mode, percentile, rec)) return 1;
  if (F <= 0 || F > M3R_MAX_COMMIT) return set_error("slam_keyframe_frames: F = %d frames, 1..%d", F, M3R_MAX_COMMIT);
  if (!is_first) return set_error("slam_keyframe_frames: null is_first");
  unsigned long long mask = 0;
  for (int f = 0; f < F; ++f) mask |= is_first[f] ? 1ull << f : 0ull;
  launch_pdl(slam_keyframe_kernel, dim3(F * kCluster), dim3(kThreads), 0, reinterpret_cast<cudaStream_t>(stream), dists,
             conf, pts3d_local, (int)H, (int)W, (int)subsamp, (int)mode, percentile / 100.0, thr, min_conf_keyframe, mask,
             rec);
  return check_launch("slam_keyframe_frames");
}
