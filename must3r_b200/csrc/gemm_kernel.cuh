// Persistent warp-specialised wgmma GEMM for sm_90a:  out = epilogue(A[M,K] * W[N,K]^T).
//
//   warps 0..7 : two consumer warpgroups -- warpgroup w multiplies rows [64w, 64w + 64) of the 128-row tile with
//                wgmma.m64nBNk16 (operands straight from the 128B-swizzled smem ring, fp32 accumulator in registers),
//                then runs the epilogue on the accumulator fragment: bias / RoPE / GELU / residual / image2-embed row
//                bias in place, then 128-byte column chunks through a swizzled staging buffer to global memory (TMA
//                stores that drain during the next tile when a CTA owns several tiles, 16-byte thread stores otherwise)
//   warps 8..11: producer warpgroup -- one elected lane issues TMA (A and W tiles, 128B-swizzled, mbarrier ring); the
//                warpgroup gives its registers to the consumers (setmaxnreg), whose accumulator is 128 registers at BN = 256
// The producer keeps filling the ring for the next tile while the consumers drain the current one.  Tiles are walked
// m-fastest so that co-resident CTAs share the weight tile in L2.  The operand type (fp16 / bf16 / e4m3) is a template
// parameter: a run-time choice between two wgmma forms inside the k loop makes ptxas fence the accumulator between wgmma
// groups.  A k-block is one 128-byte swizzle atom per row whatever the type: 64 16-bit or 128 e4m3 elements, so the ring,
// the TMA boxes and the descriptors keep their byte geometry; only the elements per k-step (16 / 32) and the instruction
// change.  The e4m3 kernel multiplies the accumulator by a per-column weight scale before the (shared) epilogues.
#pragma once
#include "ptx.cuh"
#include "m3r_internal.h"

namespace m3r {

constexpr int BM = 128;
constexpr int BK = 64;        // 64 x 16-bit = 128 B = one swizzle atom
constexpr int MMA_K = 16;     // elements of a 16-bit k-step (32 B; an e4m3 k-step is 32 elements, the same 32 B)
// operand types of the kernel template; the elements of a 128-byte k-block row
constexpr int OP_F16 = 0, OP_BF16 = 1, OP_E4M3 = 2;
__host__ __device__ constexpr int kblock_elems(int op) { return op == OP_E4M3 ? 128 : BK; }
constexpr int GEMM_THREADS = 384;      // 2 consumer warpgroups + the producer warpgroup
constexpr int PRODUCER_WARP = 8;       // first warp of the producer warpgroup
constexpr int SMEM_MAX = 232448;       // 227 KB: the most dynamic shared memory an sm_90 block may opt in to
// Register split after setmaxnreg.  The warpgroups can only redistribute what the CTA was given at launch (the
// __launch_bounds__ cap, 168 x 384 threads): an increase the CTA cannot cover would wait forever.
constexpr int GEMM_LAUNCH_REGS = (65536 / GEMM_THREADS) / 8 * 8;
constexpr int GEMM_PRODUCER_REGS = 40;
constexpr int GEMM_CONSUMER_REGS = 232;
static_assert(128 * GEMM_PRODUCER_REGS + 256 * GEMM_CONSUMER_REGS <= GEMM_LAUNCH_REGS * GEMM_THREADS,
              "register split exceeds the launch allocation");

template <int BN>
struct GemmCfg {
  static constexpr int STAGE_BYTES = (BM + BN) * BK * 2;
  // epilogue staging after the ring: [warpgroup][2 buffers][64 rows x 128 B], 1024-aligned for the 128B swizzle
  static constexpr int EPI_BUF_BYTES = 64 * 128;
  static constexpr int FIXED = 1024 /*align*/ + 1024 /*barriers*/ + 2 * 2 * EPI_BUF_BYTES;
  static constexpr int STAGES = (SMEM_MAX - FIXED) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED;
  static_assert(2 * STAGES * 8 <= 1024, "ring barriers exceed their space");
  static_assert(STAGES == (BN == 256 ? 4 : BN == 192 ? 4 : BN == 160 ? 5 : BN == 128 ? 6 : BN == 64 ? 8 : 9),
                "operand ring depth changed");
};

struct GemmParams {
  int M, N, K;
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
  int tma_store;               // the epilogue stores through TMA and the output tensor map (persistent plain launches)
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
  float4* kpart;               // [tiles][BN / 8 accumulator quads][256 consumer threads] float4 (the fragment layout)
  unsigned int* kflag;         // [tiles], zero between launches
  // ---- e4m3 operands: the accumulator column of W row r is multiplied by w_scale[r] (the weight's per-channel scale)
  const float* w_scale;
  int norm_e4m3;               // norm_out rows are e4m3 bytes (the A operand of an e4m3 GEMM) instead of 16-bit
};

// output pointers of a grouped GEMM (passed by value: kernel parameter space)
struct GemmGroupTab {
  void* out[M3R_MAX_GROUPS];
  void* peer[M3R_MAX_GROUPS][M3R_MAX_PEERS];
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

// The epilogue works on the wgmma accumulator fragment.  Thread (warp w, lane l) of a consumer warpgroup holds rows
// 16w + l/4 and 16w + l/4 + 8 (h = 0, 1) of the warpgroup's 64, columns 8nb + 2(l%4) + {0, 1} in acc[4nb + 2h + {0, 1}].
// EpiRows is what the thread needs to know about its two rows (counted inside the group).
struct EpiRows {
  bool ok[2], rb_on[2];
  const float* rope[2];
  const float* res[2];
};
__device__ __forceinline__ EpiRows epi_rows(const GemmParams& p, int lrow) {
  EpiRows e;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = lrow + 8 * h;
    e.ok[h] = row < p.M;
    e.rb_on[h] = p.rowbias != nullptr && (row % p.rb_period) >= p.rb_first;
    e.rope[h] = p.rope_tab ? p.rope_tab + (long long)(row % p.rope_period) * 64 : nullptr;
    e.res[h] = p.residual ? p.residual + (long long)row * p.ldr : nullptr;
  }
  return e;
}

// Epilogue arithmetic of the 32-column chunk c of the fragment, in place: bias, RoPE, row bias, GELU, residual.  The RoPE
// partner of column c (c % 32 < 16) is column c + 16, block nb + 2 of the same thread.
template <int BN>
__device__ __forceinline__ void epilogue_apply(const GemmParams& p, const EpiRows& rows, const float* bias, float (&acc)[BN / 2],
                                               int n0, int c, int q) {
  const int col0 = n0 + 32 * c;
  if (bias) {
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int nb = 4 * c + jj;
      const float2 b = __ldg(reinterpret_cast<const float2*>(bias + n0 + 8 * nb + 2 * q));
#pragma unroll
      for (int h = 0; h < 2; ++h) { acc[4 * nb + 2 * h] += b.x; acc[4 * nb + 2 * h + 1] += b.y; }
    }
  }
  if (p.rope_tab != nullptr && col0 < p.rope_cols) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!rows.ok[h]) continue;
      // chunk = half a head: even chunks are the y half, odd chunks the x half
      const float* cs = rows.rope[h] + ((col0 >> 5) & 1) * 32;
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int i = 8 * jj + 2 * q;
        const float2 c2 = __ldg(reinterpret_cast<const float2*>(cs + i));
        const float2 s2 = __ldg(reinterpret_cast<const float2*>(cs + 16 + i));
        const float cc[2] = {c2.x, c2.y}, ss[2] = {s2.x, s2.y};
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& vu = acc[4 * (4 * c + jj) + 2 * h + e];
          float& vw = acc[4 * (4 * c + jj + 2) + 2 * h + e];
          const float u = vu, w = vw;
          vu = u * cc[e] - w * ss[e];
          vw = w * cc[e] + u * ss[e];
        }
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!rows.rb_on[h]) continue;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int nb = 4 * c + jj;
      const float2 b = __ldg(reinterpret_cast<const float2*>(p.rowbias + n0 + 8 * nb + 2 * q));
      acc[4 * nb + 2 * h] += b.x; acc[4 * nb + 2 * h + 1] += b.y;
    }
  }
  if (p.act == 1) {
#pragma unroll
    for (int i = 16 * c; i < 16 * c + 16; ++i) acc[i] = gelu_erf(acc[i]);
  }
  if (p.residual) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!rows.ok[h]) continue;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int nb = 4 * c + jj;
        const float2 r = *reinterpret_cast<const float2*>(rows.res[h] + n0 + 8 * nb + 2 * q);
        acc[4 * nb + 2 * h] += r.x; acc[4 * nb + 2 * h + 1] += r.y;
      }
    }
  }
}

// Writes column chunk sc of the fragment (128 B per row: 32 fp32 or 64 16-bit columns; the last 16-bit chunk of BN 32 and
// 160 is half as wide) into a 64-row staging buffer, row r's 16-byte unit k at r * 128 + ((k ^ (r % 8)) << 4): the
// SWIZZLE_128B layout of the output tensor map, in which the fragment writes are free of bank conflicts.
template <int BN, bool BF16, bool OUT16>
__device__ __forceinline__ void epilogue_stage(const float (&acc)[BN / 2], uint8_t* buf, int sc, int fr, int q) {
  const int sw = fr & 7;                             // (row % 8) of both rows: the swizzle phase
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    uint8_t* rowp = buf + (fr + 8 * h) * 128;
    if constexpr (OUT16) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int nb = 8 * sc + jj;
        if (nb < BN / 8)
          *reinterpret_cast<uint32_t*>(rowp + ((jj ^ sw) << 4) + 4 * q) = pack16(acc[4 * nb + 2 * h], acc[4 * nb + 2 * h + 1], BF16);
      }
    } else {
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int nb = 4 * sc + jj;
        *reinterpret_cast<float2*>(rowp + (((2 * jj + (q >> 1)) ^ sw) << 4) + 8 * (q & 1)) = make_float2(acc[4 * nb + 2 * h], acc[4 * nb + 2 * h + 1]);
      }
    }
  }
}

// Epilogue of the plain and grouped launches: each chunk is applied, staged in one of the warpgroup's two buffers (they
// alternate over the CTA's whole sequence of chunks, `nchunk`) and drained after one barrier per chunk.  The barrier of a
// chunk is passed only after every thread has finished with the chunk before it, so that chunk's buffer is free again.
// - TMA: one thread stores the chunk with a TMA store that neither the next chunk nor the next tile's MMAs wait for; it
//   first waits until the previous store has read the other buffer.  Rows past M are clipped by the tensor map.
// - otherwise every thread copies 16-byte units, 8 consecutive threads per 128-byte row segment, to the output row (after
//   the rows_per_batch remap; rows past M skipped) and the same unit to every peer's buffer.
template <int BN, bool BF16, bool OUT16, bool TMA>
__device__ __forceinline__ void epilogue_out(const GemmParams& p, const CUtensorMap* tmC, const EpiRows& rows, const float* bias,
                                             float (&acc)[BN / 2], uint8_t* stg, unsigned& nchunk, int lrow0, int n0, int wg, int ct,
                                             void* out, void* const* peers) {
  constexpr int CW = OUT16 ? 64 : 32;                // columns per chunk
  constexpr int NSC = (BN + CW - 1) / CW;
  const int lane = ct & 31, q = lane & 3;
  const int fr = (ct >> 5) * 16 + (lane >> 2);
  // thread copy: rows (ct / 8) + 16 j of the warpgroup's 64, unit ct % 8; byte offset of the unit in chunk 0, -1 past M
  long long off[4];
#pragma unroll
  for (int j = 0; j < 4 && !TMA; ++j) {
    const int lrow = lrow0 + (ct >> 3) + 16 * j;
    long long orow = lrow;
    if (p.rows_per_batch > 0) orow = (long long)(lrow / p.rows_per_batch) * p.batch_stride_rows + lrow % p.rows_per_batch;
    off[j] = lrow < p.M ? (orow * p.ldc + n0) * (OUT16 ? 2 : 4) + 16 * (ct & 7) : -1;
  }
#pragma unroll
  for (int sc = 0; sc < NSC; ++sc) {
#pragma unroll
    for (int c = sc * (CW / 32); c < (sc + 1) * (CW / 32) && c < BN / 32; ++c) epilogue_apply<BN>(p, rows, bias, acc, n0, c, q);
    // (a TMA launch has an even number of chunks per tile: its buffer follows from sc alone)
    uint8_t* buf = stg + ((TMA ? sc : nchunk + sc) & 1) * GemmCfg<BN>::EPI_BUF_BYTES;
    epilogue_stage<BN, BF16, OUT16>(acc, buf, sc, fr, q);
    if constexpr (TMA) {
      fence_proxy_async_smem();
      if (ct == 0) bulk_wait_group_read<0>();
    }
    asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
    if constexpr (TMA) {
      if (ct == 0) {
        tma_store_2d(tmC, buf, n0 + sc * CW, lrow0);
        bulk_commit_group();
      }
      continue;
    }
    if ((sc + 1) * CW > BN && (ct & 7) >= 4) continue;     // half chunk: 64 B per row
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (off[j] < 0) continue;
      const int rr = (ct >> 3) + 16 * j;
      const uint4 val = *reinterpret_cast<const uint4*>(buf + rr * 128 + (((ct & 7) ^ (rr & 7)) << 4));
      const long long o = off[j] + sc * 128;
      *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(out) + o) = val;
      for (int pr = 0; pr < p.n_peer_out; ++pr) *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(peers[pr]) + o) = val;
    }
  }
  nchunk += NSC;
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

template <int BN, int MODE, int OP>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
            const __grid_constant__ CUtensorMap tmC, const GemmParams p, const __grid_constant__ typename TabOf<MODE>::type tab) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int NCHUNK = BN / 32;
  constexpr bool BF16 = OP != OP_F16;              // 16-bit outputs of the e4m3 kernel are bf16
  constexpr int KB = kblock_elems(OP);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                               // STAGES x [128 x 64] 16-bit
  uint8_t* sB = smem + STAGES * BM * BK * 2;        // STAGES x [BN x 64] 16-bit
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* full = bars;                  // [STAGES]
  uint64_t* empty = bars + STAGES;        // [STAGES]
  uint8_t* epi_stg = smem + STAGES * Cfg::STAGE_BYTES + 1024;     // [2 warpgroups][2][64 rows x 128 B] epilogue staging

  M3R_TR(unsigned long long* tr = p.trace ? p.trace + 16ull * blockIdx.x : nullptr;
         if (tr && threadIdx.x == 0) { tr[0] = gtime_ns(); tr[8] = smid(); })
  const int warp = threadIdx.x >> 5;
  const int tiles_mg = (p.M + BM - 1) / BM;          // m-tiles per group
  const int tiles_m = tiles_mg * p.groups;
  const int tiles_n = p.N / BN;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb_all = p.K / KB;
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

  if (warp >= PRODUCER_WARP) {
    // ------------------------------------------------------------ TMA producer warpgroup
    setmaxnreg_dec<GEMM_PRODUCER_REGS>();
    if (warp == PRODUCER_WARP && elect_one()) {
      // The weights never depend on the kernel before this one, so the W halves of the first ring of stages are requested
      // BEFORE the programmatic-dependency wait: their (cold, HBM) latency overlaps the predecessor's tail.  The
      // activations follow after the wait; each stage's barrier expects both halves.
      int pre = 0;
      if (p.w_static && tile0 < num_tiles) {
        const int n0 = (int)w_row0(tile0 % tiles_m, tile0 / tiles_m);
        pre = num_kb < STAGES ? num_kb : STAGES;
        for (int kb = 0; kb < pre; ++kb) {
          mbar_arrive_expect_tx(&full[kb], Cfg::STAGE_BYTES);
          tma_load_2d(sB + kb * BN * BK * 2, &tmW, &full[kb], (kb0 + kb) * KB, n0);
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
            tma_load_2d(sA + stage * BM * BK * 2, &tmA, &full[stage], (kb0 + kb) * KB, m0);
          } else {
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full[stage], Cfg::STAGE_BYTES);
            tma_load_2d(sA + stage * BM * BK * 2, &tmA, &full[stage], (kb0 + kb) * KB, m0);
            tma_load_2d(sB + stage * BN * BK * 2, &tmW, &full[stage], (kb0 + kb) * KB, n0);
          }
          if constexpr (MODE == MODE_PLAIN) {
            // the tile's residual rows, spread over its k-blocks, go to L2 ahead of the epilogue's fragment-layout loads
            if (p.tma_store && p.residual) {
              for (int r = kb; r < BM; r += num_kb)
                if (m0 + r < p.M) prefetch_l2_bulk(p.residual + (long long)(m0 + r) * p.ldr + n0, BN * 4);
            }
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
  setmaxnreg_inc<GEMM_CONSUMER_REGS>();
  griddep_wait();
  griddep_launch();
  const int wg = warp >> 2;                       // rows [64 wg, 64 wg + 64) of the tile
  const int ct = threadIdx.x & 127;
  const int wl = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int fr = wl * 16 + (lane >> 2), q = lane & 3;   // the thread's fragment rows fr, fr + 8 and column pair 2q (epi_rows)
  uint8_t* stg = epi_stg + wg * 2 * Cfg::EPI_BUF_BYTES;
  unsigned nchunk = 0;                            // chunks staged so far: selects the staging buffer
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
        // advance one k-step (32 bytes) along K inside the 128B swizzle atom: +2 in the >>4 address field
        if constexpr (OP == OP_E4M3) WgmmaE4M3<BN>::ss(acc, adesc + 2 * k, bdesc + 2 * k, 1);
        else Wgmma<BN, BF16>::ss(acc, adesc + 2 * k, bdesc + 2 * k, 1);
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

    const int lrow0 = (tm % tiles_mg) * BM + wg * 64;                 // the warpgroup's first row, counted inside the group
    const int n0 = tn * BN;
    if constexpr (OP == OP_E4M3) {
      // dequantise: column 8nb + 2q + e of the thread's fragment is W row w_row0 + 8nb + 2q + e
      const float* sc = p.w_scale + w_row0(tm, tn) + 2 * q;
#pragma unroll
      for (int nb = 0; nb < BN / 8; ++nb) {
        const float2 s2 = __ldg(reinterpret_cast<const float2*>(sc + 8 * nb));
#pragma unroll
        for (int h = 0; h < 2; ++h) { acc[4 * nb + 2 * h] *= s2.x; acc[4 * nb + 2 * h + 1] *= s2.y; }
      }
    }
    const float* bias = p.bias ? p.bias + (long long)g * p.bias_group : nullptr;
    if constexpr (MODE == MODE_EMIT) {
      // ---- LayerNorm-emitting epilogue (one tile per CTA).  Split-K: the ks = 1 CTA hands its raw accumulator over in the
      // fragment layout ([tile][acc / 4][256 threads]: lanes are consecutive float4, 512 B per warp request) and is done.
      if (ksplit > 1) {
        float4* kp = p.kpart + (long long)t * (BN / 8) * 256 + threadIdx.x;
        if (ks == 1) {
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) kp[i * 256] = make_float4(acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]);
          __threadfence();
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (threadIdx.x == 0) atom_add_release_u32(p.kflag + t, 1u);
          continue;                                           // the partner CTA finishes the tile
        }
        if (threadIdx.x == 0) {
          unsigned int spins = 0;
          while (ld_acquire_u32(p.kflag + t) == 0u) { if (++spins > (1u << 26)) spin_timeout_trap(); }
          p.kflag[t] = 0u;                                    // re-armed for the next launch (nobody else touches it any more)
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const float4 o = __ldcg(kp + i * 256);
          acc[4 * i] += o.x; acc[4 * i + 1] += o.y; acc[4 * i + 2] += o.z; acc[4 * i + 3] += o.w;
        }
      }
      // x = acc + bias + residual -> out (fp32).  Chunks c and c + 1 are applied and staged (fp32) together; thread (u, r)
      // reads back row r of chunk c + u and keeps it (chunks u, u + 2, ...) for the normalisation.
      constexpr int CPT = BN / 64;                                 // 32-column chunks per thread
      const int u = ct >> 6, r = ct & 63;
      const int lrow = lrow0 + r;
      const bool row_ok = lrow < p.M;
      long long orow = lrow;
      if (p.rows_per_batch > 0) orow = (long long)(lrow / p.rows_per_batch) * p.batch_stride_rows + lrow % p.rows_per_batch;
      const int rit = wg * 64 + r;                                 // row in tile
      const EpiRows rows = epi_rows(p, lrow0 + fr);
      float v[CPT][32];
#pragma unroll
      for (int pi = 0; pi < CPT; ++pi) {
        if (pi > 0) asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");     // the previous pair has been read
#pragma unroll
        for (int uu = 0; uu < 2; ++uu) {
          epilogue_apply<BN>(p, rows, bias, acc, n0, 2 * pi + uu, q);
          epilogue_stage<BN, BF16, false>(acc, stg + uu * Cfg::EPI_BUF_BYTES, 2 * pi + uu, fr, q);
        }
        asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
        const uint8_t* rowp = stg + u * Cfg::EPI_BUF_BYTES + r * 128;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float4 x = *reinterpret_cast<const float4*>(rowp + ((k ^ (r & 7)) << 4));
          v[pi][4 * k] = x.x; v[pi][4 * k + 1] = x.y; v[pi][4 * k + 2] = x.z; v[pi][4 * k + 3] = x.w;
        }
      }
      const int parts = NCHUNK * tiles_n;                          // 32-column partials per row
      float2* st = p.stats + ((long long)tm * parts) * BM;
#pragma unroll
      for (int pi = 0; pi < CPT; ++pi) {
        const int cc = 2 * pi + u;
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
        for (int pi = 0; pi < CPT; ++pi) {
          float4* o4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + orow * p.ldc + n0 + (2 * pi + u) * 32);
#pragma unroll
          for (int i = 0; i < 8; ++i) o4[i] = make_float4(v[pi][4 * i], v[pi][4 * i + 1], v[pi][4 * i + 2], v[pi][4 * i + 3]);
        }
      }
      if (threadIdx.x == 0) {
        unsigned int spins = 0;
        while (ld_acquire_u32(cnt) < (unsigned int)tiles_n) { if (++spins > (1u << 26)) spin_timeout_trap(); }
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
      if (row_ok && p.norm_e4m3) {
#pragma unroll
        for (int pi = 0; pi < CPT; ++pi) {
          uint4* o4 = reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(p.norm_out) + (long long)lrow * p.ldn + n0 + (2 * pi + u) * 32);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float y[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] = (v[pi][16 * i + j] - mean) * rstd;
            o4[i] = make_uint4(pack_e4m3x4(y[0], y[1], y[2], y[3]), pack_e4m3x4(y[4], y[5], y[6], y[7]),
                               pack_e4m3x4(y[8], y[9], y[10], y[11]), pack_e4m3x4(y[12], y[13], y[14], y[15]));
          }
        }
      } else if (row_ok) {
#pragma unroll
        for (int pi = 0; pi < CPT; ++pi) {
          uint4* o4 = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.norm_out) + (long long)lrow * p.ldn + n0 + (2 * pi + u) * 32);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            uint4 w;
            w.x = pack16((v[pi][8 * i] - mean) * rstd, (v[pi][8 * i + 1] - mean) * rstd, BF16);
            w.y = pack16((v[pi][8 * i + 2] - mean) * rstd, (v[pi][8 * i + 3] - mean) * rstd, BF16);
            w.z = pack16((v[pi][8 * i + 4] - mean) * rstd, (v[pi][8 * i + 5] - mean) * rstd, BF16);
            w.w = pack16((v[pi][8 * i + 6] - mean) * rstd, (v[pi][8 * i + 7] - mean) * rstd, BF16);
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
    void* out_g = p.out;
    void* const* peers_g = p.peer_out;
    if constexpr (MODE == MODE_GROUPED) { out_g = tab.out[g]; peers_g = tab.peer[g]; }
    const EpiRows rows = epi_rows(p, lrow0 + fr);
    if (MODE == MODE_PLAIN && (BN == 128 || BN == 256) && p.tma_store) {
      if (p.out_dtype != 0) epilogue_out<BN, BF16, true, true>(p, &tmC, rows, bias, acc, stg, nchunk, lrow0, n0, wg, ct, out_g, peers_g);
      else epilogue_out<BN, BF16, false, true>(p, &tmC, rows, bias, acc, stg, nchunk, lrow0, n0, wg, ct, out_g, peers_g);
    } else {
      if (p.out_dtype != 0) epilogue_out<BN, BF16, true, false>(p, &tmC, rows, bias, acc, stg, nchunk, lrow0, n0, wg, ct, out_g, peers_g);
      else epilogue_out<BN, BF16, false, false>(p, &tmC, rows, bias, acc, stg, nchunk, lrow0, n0, wg, ct, out_g, peers_g);
    }
    M3R_TR(if (tr && threadIdx.x == 0) tr[7] = gtime_ns();)
  }
  if constexpr (MODE == MODE_PLAIN) {
    if (p.tma_store && ct == 0) bulk_wait_group<0>();   // the shared-memory sources must outlive the stores
  }
  M3R_TR(if (tr && threadIdx.x == 0) tr[9] = gtime_ns();)
}

static void fill_params(GemmParams& p, const m3r_gemm_args* a) {
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.bias = a->bias; p.act = a->act; p.residual = a->residual; p.ldr = a->ldr;
  p.rowbias = a->rowbias; p.rb_period = a->rb_period > 0 ? a->rb_period : 1; p.rb_first = a->rb_first;
  p.rope_tab = a->rope_tab; p.rope_cols = a->rope_cols; p.rope_period = a->rope_period > 0 ? a->rope_period : 1;
  p.out = a->out; p.ldc = a->ldc; p.out_dtype = a->out_dtype;
  p.rows_per_batch = a->rows_per_batch; p.batch_stride_rows = a->batch_stride_rows;
  p.n_peer_out = a->n_peer_out;
  p.trace = trace_buffer();
  p.w_static = a->w_static;
  p.tma_store = 0;
  for (int i = 0; i < M3R_MAX_PEERS; ++i) p.peer_out[i] = i < a->n_peer_out ? a->peer_out[i] : nullptr;
  p.groups = 1; p.w_group_rows = 0; p.bias_group = 0;
  p.norm_out = nullptr; p.ldn = 0; p.norm_eps = 0.f; p.stats = nullptr; p.sync = nullptr;
  p.ksplit = 1; p.kpart = nullptr; p.kflag = nullptr;
  p.w_scale = nullptr; p.norm_e4m3 = 0;
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

// E4M3: A and W are e4m3 and e8->w_scale scales the accumulator; otherwise a->is_bf16 selects the 16-bit kernel.  e8 (may be
// null) also carries the norm_out format of the LayerNorm-emitting launches.
template <int BN, int MODE, bool E4M3>
static int launch_gemm(const m3r_gemm_args* a, const m3r_gemm_e4m3_args* e8, cudaStream_t stream, const m3r_gemm_group* grp = nullptr) {
  using Cfg = GemmCfg<BN>;
  const int groups = (MODE == MODE_GROUPED) ? grp->groups : 1;
  const int op_type = E4M3 ? TMAP_E4M3 : a->is_bf16;
  constexpr int KB = E4M3 ? kblock_elems(OP_E4M3) : BK;
  CUtensorMap tmA, tmW;
  if (make_tmap_2d(&tmA, a->A, op_type, (uint64_t)a->K, (uint64_t)a->M * groups, (uint64_t)a->lda, KB, BM)) return 1;
  if (make_tmap_2d(&tmW, a->W, op_type, (uint64_t)a->K, MODE == MODE_GROUPED ? (uint64_t)((groups - 1) * grp->w_group_rows + a->N) : (uint64_t)a->N, (uint64_t)a->ldw, KB, BN)) return 1;
  GemmParams p;
  fill_params(p, a);
  if (e8) { p.w_scale = e8->w_scale; p.norm_e4m3 = e8->norm_e4m3; }
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
    if (BN == 64 && a->K >= 2048 && (a->K / KB) % 2 == 0 && 2 * tiles <= num_sms() && tiles <= EMIT_MAX_KSPLIT_TILES) {
      p.ksplit = 2; p.kpart = e->emit_kpart; p.kflag = e->emit_kflag;
    }
  }
  // A CTA with more than one tile stores through TMA, so that its tensor cores resume while the stores drain.  One-wave
  // launches, peer stores and the batch row remap store from the threads.
  CUtensorMap tmC;
  memset(&tmC, 0, sizeof(tmC));
  if (MODE == MODE_PLAIN && (BN == 128 || BN == 256) && tiles > num_sms() && a->n_peer_out == 0 && a->rows_per_batch <= 0) {
    const bool f32 = a->out_dtype == M3R_OUT_F32;
    if (make_tmap_2d(&tmC, a->out, a->is_bf16, (uint64_t)a->N, (uint64_t)a->M, (uint64_t)a->ldc, f32 ? 32 : 64, 64, f32)) return 1;
    p.tma_store = 1;
  }
  auto kernel = gemm_kernel<BN, MODE, E4M3 ? OP_E4M3 : OP_BF16>;
  if constexpr (!E4M3) { if (!a->is_bf16) kernel = gemm_kernel<BN, MODE, OP_F16>; }
  const KernelInfo k = kernel_setup((const void*)kernel, Cfg::SMEM_BYTES, GEMM_THREADS);
  if (k.resident == 0) return 1;
  if (k.regs < GEMM_LAUNCH_REGS) return set_error("gemm: kernel built with %d registers per thread, the register split needs %d", k.regs, GEMM_LAUNCH_REGS);
  int grid = tiles < num_sms() ? tiles : num_sms();
  if (MODE == MODE_EMIT) grid = tiles * p.ksplit;
  if (MODE == MODE_GROUPED && grp->max_ctas > 0 && grid > grp->max_ctas) grid = grp->max_ctas;
  if (MODE == MODE_EMIT && grid > num_sms()) return set_error("gemm: LayerNorm-emitting epilogue needs one tile per CTA (%d tiles, %d SMs)", tiles, grid);
  {
    const int cat = BN >= 256 ? PROF_GEMM256 : (BN >= 128 ? PROF_GEMM128 : PROF_GEMM64);
    ProfScope prof(cat, 2.0 * a->M * groups * (double)a->N * a->K, (E4M3 ? 1.0 : 2.0) * ((double)a->M * groups * a->K + (double)a->N * groups * a->K) + (double)a->M * groups * a->N * (a->out_dtype ? 2 : 4), stream);
    cudaError_t le = launch_pdl(kernel, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream, tmA, tmW, tmC, p, tab);
    if (le != cudaSuccess) return set_error("gemm launch: %s", cudaGetErrorString(le));
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("gemm launch: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

// the e4m3 instantiations live in their own translation unit (gemm_e4m3.cu): bn in {64, 128, 256}
int launch_gemm_e4m3(int bn, int mode, const m3r_gemm_args* a, const m3r_gemm_e4m3_args* e8, cudaStream_t stream,
                     const m3r_gemm_group* grp);

}  // namespace m3r
