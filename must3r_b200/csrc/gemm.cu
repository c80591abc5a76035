// Persistent warp-specialised wgmma GEMM for sm_90a:  out = epilogue(A[M,K] * W[N,K]^T).
//
//   warps 0..7 : two consumer warpgroups -- warpgroup w multiplies rows [64w, 64w + 64) of the 128-row tile with
//                wgmma.m64nBNk16 (operands straight from the 128B-swizzled smem ring, fp32 accumulator in registers),
//                then runs the epilogue: bias / RoPE / GELU / residual / image2-embed row bias, vectorised global stores
//   warp 8     : TMA producer (one elected lane) -- A and W tiles, 128B-swizzled, mbarrier ring
// The producer keeps filling the ring for the next tile while the consumers drain the current one.  Tiles are walked
// m-fastest so that co-resident CTAs share the weight tile in L2.
#include "ptx.cuh"
#include "m3r_internal.h"

namespace m3r {

constexpr int BM = 128;
constexpr int BK = 64;        // 64 x 16-bit = 128 B = one swizzle atom
constexpr int MMA_K = 16;
constexpr int GEMM_THREADS = 288;      // 2 consumer warpgroups + the TMA warp
constexpr int PRODUCER_WARP = 8;
constexpr int SMEM_MAX = 232448;       // 227 KB: the most dynamic shared memory an sm_90 block may opt in to

template <int BN>
struct GemmCfg {
  static constexpr int STAGE_BYTES = (BM + BN) * BK * 2;
  static constexpr int STG_BYTES = 2 * 2 * 64 * 33 * 4;        // epilogue transpose: [warpgroup][chunk][64 rows][33]
  static constexpr int PEER_STAGE_BYTES = 8 * 4096;          // per consumer warp 32 rows x 128 B: transposes peer stores (below)
  static constexpr int FIXED = 1024 /*align*/ + 256 /*barriers*/ + STG_BYTES + PEER_STAGE_BYTES;
  static constexpr int STAGES = (SMEM_MAX - FIXED) / STAGE_BYTES;   // 256:3  192:4  160:4  128:5  64:6  32:8
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256 + STG_BYTES;
  static constexpr int SMEM_BYTES_PEER = SMEM_BYTES + PEER_STAGE_BYTES;
};

struct GemmParams {
  int M, N, K;
  int is_bf16;
  const float* bias;
  int act;
  const float* residual;
  long long ldr;
  const float* rowbias;
  int rb_period, rb_first;
  const float* rope_tab;
  int rope_cols, rope_period;
  void* out;
  long long ldc;
  int out_dtype;
  int rows_per_batch;
  long long batch_stride_rows;
  int n_peer_out;
  void* peer_out[M3R_MAX_PEERS];
  unsigned long long* trace;   // debug only (m3r_debug_trace): 16 words per CTA; normally null
  int w_static;                // weights may be requested before the programmatic-dependency wait
  // ---- grouped GEMM: `groups` independent problems of M rows each that share the shapes: A rows [g*M, (g+1)*M) of one
  // [groups*M, K] matrix, W rows [g*w_group_rows, +N), bias + g*bias_group, outputs from GemmGroupTab (groups == 1: `out`)
  int groups;
  long long w_group_rows, bias_group;
  // ---- LayerNorm emitted by the epilogue (EMIT kernels): besides `out` (fp32 x = acc + bias + residual) the CTAs of one
  // m-tile exchange per-row (mean, M2) partials through `stats`, meet at a device-scope counter and write the normalised
  // row (x - mean) * rstd as 16-bit into norm_out - the A operand of the next GEMM, whose weights carry the affine.
  void* norm_out;
  long long ldn;
  float norm_eps;
  float2* stats;               // [tiles_m][2 * tiles_n][128]
  unsigned int* sync;          // [tiles_m][2]: arrivals, departures (both zero between launches)
  // split-K of the LayerNorm-emitting kernel (K >= 2048, i.e. fc2): CTA pairs (tile, ks = 0 / 1) each stream half of K;
  // the ks = 1 CTA hands its fp32 accumulator tile to the ks = 0 CTA through `kpart` and a flag, the ks = 0 CTA adds it and
  // runs the epilogue.  Halves the bytes ONE SM pulls from L2, which is what bounds these one-wave GEMMs.
  int ksplit;                  // 1 or 2
  float4* kpart;               // [tiles][2 column halves][8][128] float4
  unsigned int* kflag;         // [tiles], zero between launches
};

// output pointers of a grouped GEMM (passed by value: kernel parameter space)
struct GemmGroupTab {
  void* out[M3R_MAX_GROUPS];
  void* peer[M3R_MAX_GROUPS][M3R_MAX_PEERS];
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

// Epilogue arithmetic of one 32-column chunk of one accumulator row: bias, RoPE, row bias, GELU, residual -> v[32].
__device__ __forceinline__ void epilogue_math(const GemmParams& p, const float* bias, const uint32_t (&raw)[32], float (&v)[32], int row,
                                              bool row_ok, bool rb_on, const float* rope_row, int col0) {
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(raw[i]);
  if (bias) {
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(bias + col0 + i));
      v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
    }
  }
  if (rope_row != nullptr && col0 < p.rope_cols && row_ok) {
    // chunk = half a head: even chunks are the y half (u: 0..15, v: 16..31), odd chunks the x half
    const float* cs = rope_row + ((col0 >> 5) & 1) * 32;
#pragma unroll
    for (int i = 0; i < 16; i += 4) {
      const float4 c4 = __ldg(reinterpret_cast<const float4*>(cs + i));
      const float4 s4 = __ldg(reinterpret_cast<const float4*>(cs + 16 + i));
      const float cc[4] = {c4.x, c4.y, c4.z, c4.w};
      const float ss[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float u = v[i + j], w = v[i + j + 16];
        v[i + j] = u * cc[j] - w * ss[j];
        v[i + j + 16] = w * cc[j] + u * ss[j];
      }
    }
  }
  if (rb_on) {
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(p.rowbias + col0 + i));
      v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
    }
  }
  if (p.act == 1) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = gelu_erf(v[i]);
  }
  if (row_ok && p.residual) {
    const float4* r4 = reinterpret_cast<const float4*>(p.residual + (long long)row * p.ldr + col0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 r = r4[i];
      v[4 * i] += r.x; v[4 * i + 1] += r.y; v[4 * i + 2] += r.z; v[4 * i + 3] += r.w;
    }
  }
}

// Store of one chunk: fp32 or 16-bit row segment; the 16-bit form optionally also goes to the peers' buffers.
// A peer store instruction of a warp covers 32 rows x 16 B; the four uint4 of a thread complete a 64-byte segment per
// row back to back, so NVLink sees 64 B write bursts (the fused GEMM -> all-gather path).
__device__ __forceinline__ void epilogue_store(const GemmParams& p, void* out, void* const* peers, const float (&v)[32], long long orow, int col0) {
  if (p.out_dtype == 0) {
    float4* o4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + orow * p.ldc + col0);
#pragma unroll
    for (int i = 0; i < 8; ++i) o4[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
  } else {
    uint4 w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      w[i].x = pack16(v[8 * i], v[8 * i + 1], p.is_bf16);
      w[i].y = pack16(v[8 * i + 2], v[8 * i + 3], p.is_bf16);
      w[i].z = pack16(v[8 * i + 4], v[8 * i + 5], p.is_bf16);
      w[i].w = pack16(v[8 * i + 6], v[8 * i + 7], p.is_bf16);
    }
    uint4* o4 = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(out) + orow * p.ldc + col0);
#pragma unroll
    for (int i = 0; i < 4; ++i) o4[i] = w[i];
    for (int pr = 0; pr < p.n_peer_out; ++pr) {
      uint4* q4 = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(peers[pr]) + orow * p.ldc + col0);
#pragma unroll
      for (int i = 0; i < 4; ++i) q4[i] = w[i];
    }
  }
}

__device__ __forceinline__ void epilogue_chunk(const GemmParams& p, const uint32_t (&raw)[32], int row, bool row_ok, long long orow,
                                               bool rb_on, const float* rope_row, int col0) {
  float v[32];
  epilogue_math(p, p.bias, raw, v, row, row_ok, rb_on, rope_row, col0);
  if (row_ok) epilogue_store(p, p.out, p.peer_out, v, orow, col0);
}

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned int atom_add_release_u32(unsigned int* p, unsigned int v) {
  unsigned int o;
  asm volatile("atom.add.release.gpu.global.u32 %0, [%1], %2;" : "=r"(o) : "l"(p), "r"(v) : "memory");
  return o;
}

constexpr int MODE_PLAIN = 0, MODE_EMIT = 1, MODE_GROUPED = 2;
struct NoTab {};
template <int MODE> struct TabOf { using type = NoTab; };
template <> struct TabOf<MODE_GROUPED> { using type = GemmGroupTab; };

template <int BN, int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const GemmParams p,
            const __grid_constant__ typename TabOf<MODE>::type tab) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int NCHUNK = BN / 32;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                               // STAGES x [128 x 64] 16-bit
  uint8_t* sB = smem + STAGES * BM * BK * 2;        // STAGES x [BN x 64] 16-bit
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* full = bars;                  // [STAGES]
  uint64_t* empty = bars + STAGES;        // [STAGES]
  float* stg_all = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES + 256);    // [2 warpgroups][2 chunks][64][33]

  M3R_TR(unsigned long long* tr = p.trace ? p.trace + 16ull * blockIdx.x : nullptr;
         if (tr && threadIdx.x == 0) { tr[0] = gtime_ns(); tr[8] = smid(); })
  const int warp = threadIdx.x >> 5;
  const int tiles_mg = (p.M + BM - 1) / BM;          // m-tiles per group
  const int tiles_m = tiles_mg * p.groups;
  const int tiles_n = p.N / BN;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb_all = p.K / BK;
  // LayerNorm-emitting kernels own exactly one tile per CTA (or per CTA pair with split-K); the others walk tiles persistently
  const int ksplit = (MODE == MODE_EMIT) ? p.ksplit : 1;
  const int ks = (MODE == MODE_EMIT) ? (int)blockIdx.x / num_tiles : 0;
  const int tile0 = (MODE == MODE_EMIT) ? (int)blockIdx.x % num_tiles : (int)blockIdx.x;
  const int tile_step = (MODE == MODE_EMIT) ? num_tiles : (int)gridDim.x;
  const int num_kb = num_kb_all / ksplit;
  const int kb0 = ks * num_kb;
  // tile t -> (group g, m-tile inside the group, n-tile); m-fastest so that co-resident CTAs share the weight tile in L2
  auto a_row0 = [&](int tm) { return (tm / tiles_mg) * p.M + (tm % tiles_mg) * BM; };      // first A row of m-tile tm
  auto w_row0 = [&](int tm, int tn) { return (long long)(tm / tiles_mg) * p.w_group_rows + (long long)tn * BN; };

  if (warp == PRODUCER_WARP && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }   // empty: one arrival per warpgroup
    fence_mbar_init();
  }
  __syncthreads();
  M3R_TR(if (tr && threadIdx.x == 0) tr[1] = gtime_ns();)

  if (warp == PRODUCER_WARP) {
    // ------------------------------------------------------------ TMA producer
    if (elect_one()) {
      // The weights never depend on the kernel before this one, so the W halves of the first ring of stages are requested
      // BEFORE the programmatic-dependency wait: their (cold, HBM) latency overlaps the predecessor's tail.  The
      // activations follow after the wait; each stage's barrier expects both halves.
      int pre = 0;
      if (p.w_static && tile0 < num_tiles) {
        const int n0 = (int)w_row0(tile0 % tiles_m, tile0 / tiles_m);
        pre = num_kb < STAGES ? num_kb : STAGES;
        for (int kb = 0; kb < pre; ++kb) {
          mbar_arrive_expect_tx(&full[kb], Cfg::STAGE_BYTES);
          tma_load_2d(sB + kb * BN * BK * 2, &tmW, &full[kb], (kb0 + kb) * BK, n0);
        }
      }
      griddep_wait();
      griddep_launch();
      M3R_TR(if (tr) tr[2] = gtime_ns();)
      int stage = 0; uint32_t phase = 0;
      for (int t = tile0; t < num_tiles; t += tile_step) {
        const int m0 = a_row0(t % tiles_m);
        const int n0 = (int)w_row0(t % tiles_m, t / tiles_m);
        for (int kb = 0; kb < num_kb; ++kb) {
          if (pre > 0) {                      // stage already armed, W half in flight
            --pre;
            tma_load_2d(sA + stage * BM * BK * 2, &tmA, &full[stage], (kb0 + kb) * BK, m0);
          } else {
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full[stage], Cfg::STAGE_BYTES);
            tma_load_2d(sA + stage * BM * BK * 2, &tmA, &full[stage], (kb0 + kb) * BK, m0);
            tma_load_2d(sB + stage * BN * BK * 2, &tmW, &full[stage], (kb0 + kb) * BK, n0);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
      M3R_TR(if (tr) tr[3] = gtime_ns();)
    } else {
      griddep_wait();
      griddep_launch();
    }
    return;
  }

  // ------------------------------------------------------------ consumer warpgroups 0, 1: wgmma + epilogue
  griddep_wait();
  griddep_launch();
  const int wg = warp >> 2;                       // rows [64 wg, 64 wg + 64) of the tile
  const int ct = threadIdx.x & 127;
  const int wl = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int u = ct >> 6;                          // epilogue: which chunk of a pair this thread drains ...
  const int r = ct & 63;                          // ... for which row of the warpgroup's 64
  float* stg = stg_all + wg * (2 * 64 * 33);
  int stage = 0; uint32_t phase = 0;
  for (int t = tile0; t < num_tiles; t += tile_step) {
    const int tm = t % tiles_m, tn = t / tiles_m;
    const int g = tm / tiles_mg;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full[stage], phase);
      M3R_TR(if (tr && kb == 0 && t == tile0 && threadIdx.x == 0) tr[4] = gtime_ns();)
      const uint64_t adesc = smem_desc_sw128(smem_u32(sA + stage * BM * BK * 2 + wg * 64 * 128));
      const uint64_t bdesc = smem_desc_sw128(smem_u32(sB + stage * BN * BK * 2));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / MMA_K; ++k) {
        // advance 16 elements (32 bytes) along K inside the 128B swizzle atom: +2 in the >>4 address field
        if (p.is_bf16) Wgmma<BN, true>::ss(acc, adesc + 2 * k, bdesc + 2 * k, 1);
        else Wgmma<BN, false>::ss(acc, adesc + 2 * k, bdesc + 2 * k, 1);
      }
      wgmma_commit();
      wgmma_wait<1>();                            // the previous k-block's MMAs are done: its stage may be refilled
      reg_fence(acc);
      if (prev >= 0 && ct == 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (prev >= 0 && ct == 0) mbar_arrive(&empty[prev]);
    M3R_TR(if (tr && threadIdx.x == 0) tr[5] = gtime_ns();)

    const int lrow = (tm % tiles_mg) * BM + wg * 64 + r;              // row inside the group
    const int n0 = tn * BN;
    const bool row_ok = lrow < p.M;
    long long orow = lrow;
    if (p.rows_per_batch > 0) orow = (long long)(lrow / p.rows_per_batch) * p.batch_stride_rows + lrow % p.rows_per_batch;
    const bool rb_on = p.rowbias != nullptr && (lrow % p.rb_period) >= p.rb_first;
    const float* rope_row = p.rope_tab ? p.rope_tab + (long long)(lrow % p.rope_period) * 64 : nullptr;
    const float* bias = p.bias ? p.bias + (long long)g * p.bias_group : nullptr;
    void* out_g = p.out;
    void* const* peers_g = p.peer_out;
    if constexpr (MODE == MODE_GROUPED) { out_g = tab.out[g]; peers_g = tab.peer[g]; }

    // The accumulator fragments are transposed through shared memory two 32-column chunks at a time, so that each
    // epilogue thread owns 32 consecutive columns of ONE row (the layout the bias / RoPE / LayerNorm code works on):
    // chunks c and c + 1 of the warpgroup's 64 rows go to smem, thread (u, r) reads back row r of chunk c + u.
    auto stage_pair = [&](int c, uint32_t (&raw)[32]) {
      asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");        // the previous pair has been read
#pragma unroll
      for (int uu = 0; uu < 2; ++uu) {
        if (c + uu < NCHUNK) {
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int nb = (c + uu) * 4 + jj;
            float* s0 = stg + uu * (64 * 33) + (wl * 16 + (lane >> 2)) * 33 + jj * 8 + 2 * (lane & 3);
            s0[0] = acc[nb * 4]; s0[1] = acc[nb * 4 + 1];
            s0[8 * 33] = acc[nb * 4 + 2]; s0[8 * 33 + 1] = acc[nb * 4 + 3];
          }
        }
      }
      asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
      if (c + u < NCHUNK) {
        const float* s1 = stg + u * (64 * 33) + r * 33;
#pragma unroll
        for (int i = 0; i < 32; ++i) raw[i] = __float_as_uint(s1[i]);
      }
    };
    if constexpr (MODE == MODE_EMIT) {
      // ---- x = acc + bias + residual -> out (fp32); the thread keeps its values (chunks u, u + 2, ...) for the normalisation
      constexpr int CPT = BN / 64;                                 // 32-column chunks per thread
      uint32_t rawc[CPT][32];
#pragma unroll
      for (int pi = 0; pi < CPT; ++pi) stage_pair(2 * pi, rawc[pi]);
      const int rit = wg * 64 + r;                                 // row in tile
      if (ksplit > 1) {                                            // BN == 64 only (host)
        // [tile][column chunk][8 float4][128 rows]: lanes are consecutive rows -> 512 B per warp request
        uint32_t (&raw)[32] = rawc[0];
        float4* kp = p.kpart + ((long long)(t * NCHUNK + u) * 8) * BM + rit;
        if (ks == 1) {
#pragma unroll
          for (int i = 0; i < 8; ++i)
            kp[(long long)i * BM] = make_float4(__uint_as_float(raw[4 * i]), __uint_as_float(raw[4 * i + 1]), __uint_as_float(raw[4 * i + 2]), __uint_as_float(raw[4 * i + 3]));
          __threadfence();
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (threadIdx.x == 0) atom_add_release_u32(p.kflag + t, 1u);
          continue;                                           // the partner CTA finishes the tile
        }
        if (threadIdx.x == 0) {
          unsigned int spins = 0;
          while (ld_acquire_u32(p.kflag + t) == 0u) { if (++spins > (1u << 26)) __trap(); }
          p.kflag[t] = 0u;                                    // re-armed for the next launch (nobody else touches it any more)
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 o = __ldcg(kp + (long long)i * BM);
          raw[4 * i] = __float_as_uint(__uint_as_float(raw[4 * i]) + o.x); raw[4 * i + 1] = __float_as_uint(__uint_as_float(raw[4 * i + 1]) + o.y);
          raw[4 * i + 2] = __float_as_uint(__uint_as_float(raw[4 * i + 2]) + o.z); raw[4 * i + 3] = __float_as_uint(__uint_as_float(raw[4 * i + 3]) + o.w);
        }
      }
      const int parts = NCHUNK * tiles_n;                          // 32-column partials per row
      float2* st = p.stats + ((long long)tm * parts) * BM;
      float v[CPT][32];
#pragma unroll
      for (int pi = 0; pi < CPT; ++pi) {
        const int cc = 2 * pi + u;
        epilogue_math(p, bias, rawc[pi], v[pi], lrow, row_ok, rb_on, rope_row, n0 + cc * 32);
        if (!row_ok) {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[pi][i] = 0.f;
        }
        // two-pass statistics of the thread's 32 values, combined across the row's partials with Chan's formula (as
        // accurate as a two-pass LayerNorm over the whole row)
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int i = 0; i < 32; i += 2) { s0 += v[pi][i]; s1 += v[pi][i + 1]; }
        const float mu = (s0 + s1) * (1.0f / 32.0f);
        float q0 = 0.f, q1 = 0.f;
#pragma unroll
        for (int i = 0; i < 32; i += 2) { const float a = v[pi][i] - mu, b = v[pi][i + 1] - mu; q0 = fmaf(a, a, q0); q1 = fmaf(b, b, q1); }
        st[(long long)(tn * NCHUNK + cc) * BM + rit] = make_float2(mu, q0 + q1);
      }
      __threadfence();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      unsigned int* cnt = p.sync + 2 * tm;
      if (threadIdx.x == 0) atom_add_release_u32(cnt, 1u);
      // the fp32 residual stream goes out while the other CTAs of the row block arrive (its 32 KB per CTA would otherwise
      // sit in front of the fence above)
      if (row_ok) {
#pragma unroll
        for (int pi = 0; pi < CPT; ++pi) epilogue_store(p, p.out, p.peer_out, v[pi], orow, n0 + (2 * pi + u) * 32);
      }
      if (threadIdx.x == 0) {
        unsigned int spins = 0;
        while (ld_acquire_u32(cnt) < (unsigned int)tiles_n) { if (++spins > (1u << 26)) __trap(); }
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      float msum = 0.f;
      float2 pr[24];
      const int np = parts <= 24 ? parts : 24;                   // host guarantees parts <= 24
#pragma unroll
      for (int i = 0; i < 24; ++i) if (i < np) { pr[i] = __ldcg(st + (long long)i * BM + rit); msum += pr[i].x; }
      const float mean = msum / (float)np;
      float m2 = 0.f;
#pragma unroll
      for (int i = 0; i < 24; ++i) if (i < np) { const float d = pr[i].x - mean; m2 += pr[i].y + 32.0f * d * d; }
      const float rstd = rsqrtf(m2 / (32.0f * (float)np) + p.norm_eps);
      if (row_ok) {
#pragma unroll
        for (int pi = 0; pi < CPT; ++pi) {
          uint4* o4 = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.norm_out) + (long long)lrow * p.ldn + n0 + (2 * pi + u) * 32);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            uint4 w;
            w.x = pack16((v[pi][8 * i] - mean) * rstd, (v[pi][8 * i + 1] - mean) * rstd, p.is_bf16);
            w.y = pack16((v[pi][8 * i + 2] - mean) * rstd, (v[pi][8 * i + 3] - mean) * rstd, p.is_bf16);
            w.z = pack16((v[pi][8 * i + 4] - mean) * rstd, (v[pi][8 * i + 5] - mean) * rstd, p.is_bf16);
            w.w = pack16((v[pi][8 * i + 6] - mean) * rstd, (v[pi][8 * i + 7] - mean) * rstd, p.is_bf16);
            o4[i] = w;
          }
        }
      }
      // departure: the last CTA of the m-tile to have read the partials re-arms both counters for the next launch
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (threadIdx.x == 0) {
        if (atomicAdd(cnt + 1, 1u) == (unsigned int)tiles_n - 1u) { cnt[1] = 0u; __threadfence(); cnt[0] = 0u; }
      }
      continue;
    }
#pragma unroll
    for (int c = 0; c < NCHUNK; c += 2) {
      uint32_t raw[32];
      stage_pair(c, raw);
      const int cc = c + u;                                              // this thread's chunk
      if (p.n_peer_out > 0 && p.out_dtype != 0) {
        // ---- fused GEMM -> all-gather epilogue.  A thread owns one ROW of the chunk, so direct peer stores would be 32
        // scattered 16-byte pieces per instruction - partial sectors over NVLink.  The warp's 32 rows x 32 columns go
        // through a swizzled shared-memory tile and leave as 64-byte row segments: one store instruction = 8 rows x 64 B
        // (4 lanes per row), whole sectors, to every peer's buffer.  (u and cc are uniform across a warp.)
        if (cc < NCHUNK) {
          uint4* pst = reinterpret_cast<uint4*>(stg_all + 2 * (2 * 64 * 33)) + warp * 256;      // [32 rows][8 x 16 B]
          const int row_base = (tm % tiles_mg) * BM + wg * 64 + (r & ~31);
          float v[32];
          epilogue_math(p, bias, raw, v, lrow, row_ok, rb_on, rope_row, n0 + cc * 32);
          uint4* o4 = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(out_g) + orow * p.ldc + n0 + cc * 32);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            uint4 w;
            w.x = pack16(v[8 * i], v[8 * i + 1], p.is_bf16); w.y = pack16(v[8 * i + 2], v[8 * i + 3], p.is_bf16);
            w.z = pack16(v[8 * i + 4], v[8 * i + 5], p.is_bf16); w.w = pack16(v[8 * i + 6], v[8 * i + 7], p.is_bf16);
            if (row_ok) o4[i] = w;                                  // this GPU's copy: the thread's own row
            pst[lane * 8 + (i ^ (lane & 7))] = w;
          }
          __syncwarp();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int rr = k * 8 + lane / 4, piece = lane % 4;
            const int row_r = row_base + rr;
            if (row_r < p.M) {
              long long orow_r = row_r;
              if (p.rows_per_batch > 0) orow_r = (long long)(row_r / p.rows_per_batch) * p.batch_stride_rows + row_r % p.rows_per_batch;
              const uint4 val = pst[rr * 8 + (piece ^ (rr & 7))];
              for (int pr = 0; pr < p.n_peer_out; ++pr)
                reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(peers_g[pr]) + orow_r * p.ldc + n0 + cc * 32)[piece] = val;
            }
          }
          __syncwarp();
        }
      } else if (cc < NCHUNK) {
        float v[32];
        epilogue_math(p, bias, raw, v, lrow, row_ok, rb_on, rope_row, n0 + cc * 32);
        if (row_ok) epilogue_store(p, out_g, peers_g, v, orow, n0 + cc * 32);
      }
    }
    M3R_TR(if (tr && threadIdx.x == 0) tr[7] = gtime_ns();)
  }
  M3R_TR(if (tr && threadIdx.x == 0) tr[9] = gtime_ns();)
}

static void fill_params(GemmParams& p, const m3r_gemm_args* a) {
  p.M = a->M; p.N = a->N; p.K = a->K; p.is_bf16 = a->is_bf16;
  p.bias = a->bias; p.act = a->act; p.residual = a->residual; p.ldr = a->ldr;
  p.rowbias = a->rowbias; p.rb_period = a->rb_period > 0 ? a->rb_period : 1; p.rb_first = a->rb_first;
  p.rope_tab = a->rope_tab; p.rope_cols = a->rope_cols; p.rope_period = a->rope_period > 0 ? a->rope_period : 1;
  p.out = a->out; p.ldc = a->ldc; p.out_dtype = a->out_dtype;
  p.rows_per_batch = a->rows_per_batch; p.batch_stride_rows = a->batch_stride_rows;
  p.n_peer_out = a->n_peer_out;
  p.trace = trace_buffer();
  p.w_static = a->w_static;
  for (int i = 0; i < M3R_MAX_PEERS; ++i) p.peer_out[i] = i < a->n_peer_out ? a->peer_out[i] : nullptr;
  p.groups = 1; p.w_group_rows = 0; p.bias_group = 0;
  p.norm_out = nullptr; p.ldn = 0; p.norm_eps = 0.f; p.stats = nullptr; p.sync = nullptr;
  p.ksplit = 1; p.kpart = nullptr; p.kflag = nullptr;
}

// Scratch of the LayerNorm-emitting epilogue: partial row statistics + arrival / departure counters (+ split-K hand-over).
// The CTAs of a launch spin on each other, so launches sharing a scratch must be ordered: there is one scratch per caller
// stream (two host threads driving the model, as the reference's SLAM worker does, slam.py:533, must not share counters),
// and the model code emits on the caller's stream only, never on its side streams.
constexpr int EMIT_MAX_KSPLIT_TILES = 80;
constexpr int EMIT_MAX_TILES_M = 16, EMIT_MAX_PARTS = 24;
static const StreamState* emit_scratch(cudaStream_t stream) {
  RegistryLock lock;
  StreamState* st = stream_state(stream, lock);
  if (!st || st->emit_stats) return st;
  void *a = nullptr, *b = nullptr, *c = nullptr, *d = nullptr;
  const size_t sync_bytes = sizeof(unsigned int) * 2 * EMIT_MAX_TILES_M, kflag_bytes = sizeof(unsigned int) * EMIT_MAX_KSPLIT_TILES;
  // the kernels rely on the counters starting at zero: clear them in order with the launches that will use them
  if (cudaMalloc(&a, sizeof(float2) * EMIT_MAX_TILES_M * EMIT_MAX_PARTS * BM) != cudaSuccess ||
      cudaMalloc(&b, sync_bytes) != cudaSuccess || cudaMemsetAsync(b, 0, sync_bytes, stream) != cudaSuccess ||
      cudaMalloc(&c, sizeof(float) * EMIT_MAX_KSPLIT_TILES * BM * 64) != cudaSuccess ||
      cudaMalloc(&d, kflag_bytes) != cudaSuccess || cudaMemsetAsync(d, 0, kflag_bytes, stream) != cudaSuccess) {
    cudaFree(a); cudaFree(b); cudaFree(c); cudaFree(d);
    return nullptr;
  }
  st->emit_stats = reinterpret_cast<float2*>(a); st->emit_sync = reinterpret_cast<unsigned int*>(b);
  st->emit_kpart = reinterpret_cast<float4*>(c); st->emit_kflag = reinterpret_cast<unsigned int*>(d);
  return st;
}

template <int BN, int MODE>
static int launch_gemm(const m3r_gemm_args* a, cudaStream_t stream, const m3r_gemm_group* grp = nullptr) {
  using Cfg = GemmCfg<BN>;
  const int groups = (MODE == MODE_GROUPED) ? grp->groups : 1;
  CUtensorMap tmA, tmW;
  if (make_tmap_2d(&tmA, a->A, a->is_bf16, (uint64_t)a->K, (uint64_t)a->M * groups, (uint64_t)a->lda, BK, BM)) return 1;
  if (make_tmap_2d(&tmW, a->W, a->is_bf16, (uint64_t)a->K, MODE == MODE_GROUPED ? (uint64_t)((groups - 1) * grp->w_group_rows + a->N) : (uint64_t)a->N, (uint64_t)a->ldw, BK, BN)) return 1;
  GemmParams p;
  fill_params(p, a);
  typename TabOf<MODE>::type tab;
  const int tiles = ((a->M + BM - 1) / BM) * groups * (a->N / BN);
  if constexpr (MODE == MODE_GROUPED) {
    p.groups = groups; p.w_group_rows = grp->w_group_rows; p.bias_group = grp->bias_group;
    for (int g = 0; g < M3R_MAX_GROUPS; ++g) {
      tab.out[g] = g < groups ? grp->out[g] : nullptr;
      for (int r = 0; r < M3R_MAX_PEERS; ++r) tab.peer[g][r] = (g < groups && r < a->n_peer_out) ? grp->peer_out[g * M3R_MAX_PEERS + r] : nullptr;
    }
  }
  if constexpr (MODE == MODE_EMIT) {
    const StreamState* e = emit_scratch(stream);
    if (!e) return set_error("gemm: LayerNorm-emit scratch allocation failed");
    p.norm_out = a->norm_out; p.ldn = a->ldn; p.norm_eps = a->norm_eps; p.stats = e->emit_stats; p.sync = e->emit_sync;
    if (BN == 64 && a->K >= 2048 && (a->K / BK) % 2 == 0 && 2 * tiles <= num_sms() && tiles <= EMIT_MAX_KSPLIT_TILES) {
      p.ksplit = 2; p.kpart = e->emit_kpart; p.kflag = e->emit_kflag;
    }
  }
  if (kernel_setup((const void*)gemm_kernel<BN, MODE>, Cfg::SMEM_BYTES_PEER, GEMM_THREADS).resident == 0) return 1;
  int grid = tiles < num_sms() ? tiles : num_sms();
  if (MODE == MODE_EMIT) grid = tiles * p.ksplit;
  if (MODE == MODE_GROUPED && grp->max_ctas > 0 && grid > grp->max_ctas) grid = grp->max_ctas;
  if (MODE == MODE_EMIT && grid > num_sms()) return set_error("gemm: LayerNorm-emitting epilogue needs one tile per CTA (%d tiles, %d SMs)", tiles, grid);
  {
    const int cat = BN >= 256 ? PROF_GEMM256 : (BN >= 128 ? PROF_GEMM128 : PROF_GEMM64);
    ProfScope prof(cat, 2.0 * a->M * groups * (double)a->N * a->K, 2.0 * ((double)a->M * groups * a->K + (double)a->N * groups * a->K) + (double)a->M * groups * a->N * (a->out_dtype ? 2 : 4), stream);
    const size_t smem_bytes = (a->n_peer_out > 0 && a->out_dtype != 0) ? Cfg::SMEM_BYTES_PEER : Cfg::SMEM_BYTES;
    cudaError_t le = launch_pdl(gemm_kernel<BN, MODE>, dim3(grid), dim3(GEMM_THREADS), smem_bytes, stream, tmA, tmW, p, tab);
    if (le != cudaSuccess) return set_error("gemm launch: %s", cudaGetErrorString(le));
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("gemm launch: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

static int check_args(const m3r_gemm_args* a) {
  if (!a || !a->A || !a->W) return set_error("gemm: null pointer");
  if (a->N % 32 || a->K % 64 || a->N <= 0 || a->K <= 0) return set_error("gemm: N (%d) must be a multiple of 32 and K (%d) of 64", a->N, a->K);
  if (a->lda % 8 || a->ldw % 8) return set_error("gemm: lda/ldw must be multiples of 8 elements (16 B)");
  if ((a->out_dtype == M3R_OUT_F32 && a->ldc % 4) || (a->out_dtype == M3R_OUT_16 && a->ldc % 8)) return set_error("gemm: ldc alignment");
  if (a->residual && a->ldr % 4) return set_error("gemm: ldr alignment");
  if (a->rope_tab && (a->rope_cols % 64)) return set_error("gemm: rope_cols must be a multiple of 64");
  if (a->n_peer_out < 0 || a->n_peer_out > M3R_MAX_PEERS || (a->n_peer_out > 0 && a->out_dtype != M3R_OUT_16)) return set_error("gemm: peer outputs need 0..%d pointers and a 16-bit output", M3R_MAX_PEERS);
  return 0;
}

// Tile width for the 1-CTA kernel.  One-wave problems (the one-view chain) are bound by the per-SM L2->smem ingest, i.e. by
// the bytes ONE CTA has to pull: K * (128 + BN) * 2 - so the narrowest tile that still fits in one wave wins (most SMs
// busy, least bytes per SM).  Multi-wave problems take the widest tile that keeps every SM busy (fewer re-reads of A).
static int pick_bn(int M, int N, int groups) {
  const int tiles_m = ((M + BM - 1) / BM) * groups;
  const int sms = num_sms();
  static const int cand[] = {64, 128, 160, 192, 256};
  for (int bn : cand)
    if (N % bn == 0 && tiles_m * (N / bn) <= sms) return bn;
  if (N % 256 == 0 && tiles_m * (N / 256) >= sms) return 256;
  if (N % 128 == 0 && tiles_m * (N / 128) >= (sms * 2) / 3) return 128;
  if (N % 64 == 0) return 64;
  if (N % 160 == 0) return 160;
  return 32;
}

}  // namespace m3r

extern "C" int m3r_gemm(const m3r_gemm_args* a, void* stream) {
  using namespace m3r;
  if (check_args(a)) return 1;
  if (!a->out) return set_error("gemm: null pointer");
  if (a->M <= 0) return 0;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int sms = num_sms();
  if (a->norm_out) {
    // LayerNorm-emitting epilogue: fp32 out = the new residual stream, norm_out = its normalised 16-bit rows
    if (a->N % 64 || a->N > 32 * EMIT_MAX_PARTS || a->out_dtype != M3R_OUT_F32 || a->ldn % 8)
      return set_error("gemm: norm_out needs N %% 64 == 0, N <= %d, an fp32 output and ldn %% 8 == 0", 32 * EMIT_MAX_PARTS);
    // every CTA of the launch must be resident at once (they meet at a counter): 128x64 tiles, or 128x128 tiles when the
    // 64-wide ones would not fit on the SMs in one wave
    const int tiles_m = (a->M + BM - 1) / BM;
    if (tiles_m <= EMIT_MAX_TILES_M && tiles_m * (a->N / 64) <= sms) return launch_gemm<64, MODE_EMIT>(a, s);
    if (tiles_m <= EMIT_MAX_TILES_M && a->N % 128 == 0 && tiles_m * (a->N / 128) <= sms) return launch_gemm<128, MODE_EMIT>(a, s);
    return set_error("gemm: norm_out needs one 128x64 tile per SM (M=%d N=%d); normalise with m3r_layernorm instead", a->M, a->N);
  }
  int bn = pick_bn(a->M, a->N, 1);
  const char* force = getenv("M3R_GEMM_BN");
  if (force) { int f = atoi(force); if ((f == 32 || f == 64 || f == 128 || f == 160 || f == 192 || f == 256) && a->N % f == 0) bn = f; }
  switch (bn) {
    case 256: return launch_gemm<256, MODE_PLAIN>(a, s);
    case 192: return launch_gemm<192, MODE_PLAIN>(a, s);
    case 160: return launch_gemm<160, MODE_PLAIN>(a, s);
    case 128: return launch_gemm<128, MODE_PLAIN>(a, s);
    case 64: return launch_gemm<64, MODE_PLAIN>(a, s);
    default: return launch_gemm<32, MODE_PLAIN>(a, s);
  }
}

// `groups` GEMMs of identical shape in one launch (the post-feedback K|V projections of all decoder levels,
// must3r/model/decoder.py:323-330): A = [groups * M, K] (group g = rows [g*M, (g+1)*M)), W / bias stacked with strides
// w_group_rows / bias_group, one output (and one set of peer outputs) per group.
extern "C" int m3r_gemm_grouped(const m3r_gemm_args* a, const m3r_gemm_group* grp, void* stream) {
  using namespace m3r;
  if (check_args(a)) return 1;
  if (!grp || grp->groups < 1 || grp->groups > M3R_MAX_GROUPS) return set_error("gemm_grouped: 1..%d groups", M3R_MAX_GROUPS);
  if (a->norm_out || a->residual) return set_error("gemm_grouped: no residual / norm_out");
  for (int g = 0; g < grp->groups; ++g) if (!grp->out[g]) return set_error("gemm_grouped: out[%d] is null", g);
  if (a->M <= 0) return 0;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  int bn = pick_bn(a->M, a->N, grp->groups);
  if (bn != 256 && bn != 128) bn = a->N % 128 == 0 ? 128 : 64;
  if (a->N % bn) return set_error("gemm_grouped: N (%d) must be a multiple of 64", a->N);
  switch (bn) {
    case 256: return launch_gemm<256, MODE_GROUPED>(a, s, grp);
    case 128: return launch_gemm<128, MODE_GROUPED>(a, s, grp);
    default: return launch_gemm<64, MODE_GROUPED>(a, s, grp);
  }
}
