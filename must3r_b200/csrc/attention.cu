// FlashAttention-style softmax(Q K^T * scale) V for head_dim 64 on sm_90a tensor cores (wgmma).
//
// One CTA = one (batch, head, 128 queries [, key split]), one CTA per SM; the two consumer warpgroups share every K / V
// tile that TMA brings in.  (A 192-row form with three consumer warpgroups fits only 128 registers per thread: it
// spills and measured slower on H100.)  Roles:
//   warpgroup 2     : TMA producer -- Q once, then K and V tiles (128 keys x 64) through mbarrier rings.  It gives its
//                     registers back (setmaxnreg.dec) so that the consumers can hold two score tiles' worth of state.
//                     3-D tensor maps: rows beyond Nk read as zeros even inside over-allocated memory buffers.
//   warpgroups 0, 1 : consumers, 64 query rows each, one whole 128-key tile per pass:
//                     S[64 x 128] = Q K^T (m64n128 wgmma, both operands K-major smem, fp32 scores in registers), row max
//                     over the quad of threads sharing a row, exp2 with the scale folded in, row sums, P packed to 16-bit
//                     straight into the register A operand of O += P V (wgmma with V as an MN-major smem B operand:
//                     V is consumed in its natural [keys, d] layout -- no transpose anywhere in the pipeline).
//                     Software pipeline inside the warpgroup: S of tile j+1 and O += P V of tile j are issued together,
//                     and the softmax of tile j+1 runs while P V of tile j is still on the tensor cores.  A K stage is
//                     released as soon as its scores are in registers, a V stage when its P V has completed.
//                     (Making the two warpgroups also take turns at the tensor cores through named barriers
//                     ("ping-pong") measured 1-2 % slower on H100 for the C3 shapes, so they run independently.  With
//                     every ex2 removed, the render cross-attention ran only 12 % faster: the kernel is not bound by
//                     the MUFU, and no exponentials are moved to the FMA pipe.)
// O accumulates in registers across key tiles.  The running max used in the exponent is only refreshed when the true
// row max grew by more than 2^8 (lazy rescaling); the final O / l is mathematically unchanged.
//
// Keys come from two segments (stored memory + this step's new tokens) so the reference's torch.cat of the memory
// (decoder.py:306) never happens; a per-batch skip range implements make_mem_mask (decoder.py:119-139): fully
// masked key tiles are never loaded.  Small grids (one view per step) split the key range over several CTAs; the
// last CTA to finish a (batch, head, 64-row query tile) merges the partial (O, m, l) in-kernel.  The split
// count comes from a wave-count cost model (m3r_attention).
//
// Ragged segment 0 (m3r_attention_ragged): K/V batch b attends to rows j < nk0_b[b] of segment 0 only (the memories of
// several SLAM sessions, each of its own length, behind one decoder call).  The tensor maps span the longest batch, so the
// tiles of a shorter batch are enumerated from its own length and its last partial tile loads real rows behind its end.
// Their scores are masked like any padding; their V rows are zeroed in shared memory before P V, because P = 0 times a
// stale NaN / inf V element is still NaN.  Splits are planned for the longest batch; each batch divides its own tiles
// over them, and a CTA left without a tile contributes the empty state (m = -inf, l = 0) to the merge.
//
// Shared segment 0 (kv_bstride0 = 0 with several key batches): every batch reads the same K/V rows, so the batch becomes
// the fastest grid dimension and the CTAs that read the same key tiles run together; each CTA computes exactly what it
// computes in the usual order.
#include <math.h>
#include "ptx.cuh"
#include "m3r_internal.h"

namespace m3r {

constexpr int AT_BM = 64;                    // query rows per consumer warpgroup: the unit of the epilogue, splits and merge
constexpr int AT_BN = 128;
constexpr int HD = 64;
constexpr int TILE_BYTES = 128 * HD * 2;     // 16 KB: one K or V tile
constexpr int QTILE_BYTES = AT_BM * HD * 2;  // 8 KB: one warpgroup's Q rows
constexpr float RESCALE_THRESHOLD = 8.0f;    // log2 units

struct AttnCfg {
  static constexpr int NWG = 2;                                    // consumer warpgroups
  static constexpr int KS = 3;                                     // K / V ring depth
  static constexpr int THREADS = 128 * (NWG + 1);                  // consumer warpgroups + producer warpgroup
  static constexpr int SMEM = NWG * QTILE_BYTES + 2 * KS * TILE_BYTES + 1024 + 256;
  // Register split after setmaxnreg.  The warpgroups can only redistribute what the CTA was given at launch (the
  // __launch_bounds__ cap, 168 x 384 threads): an increase the CTA cannot cover would wait forever.
  static constexpr int LAUNCH_REGS = (65536 / THREADS) / 8 * 8;
  static constexpr int PRODUCER_REGS = 24;
  static constexpr int CONSUMER_REGS = 240;
  static_assert(128 * PRODUCER_REGS + 128 * NWG * CONSUMER_REGS <= LAUNCH_REGS * THREADS, "register split exceeds the launch allocation");
};
constexpr int OSTR = HD + 1;                 // fp32 row stride of the O tile staged for the epilogue (conflict-free reads)
// the staged O tiles + (m, l) rows overlay the Q and K stages
static_assert(AttnCfg::NWG * (AT_BM * OSTR * 4 + AT_BM * 8) <= AttnCfg::NWG * QTILE_BYTES + AttnCfg::KS * TILE_BYTES,
              "O staging must fit over the Q / K stages");

struct AttnParams {
  int Nq, Nk0, Nk1;
  int kv_group;
  int skip_lo, skip_step, skip_len;
  int splits;                // key-range splits (>=1); blockIdx.z = b * splits + split
  int batch_minor;           // shared segment 0: grid (B, H, query tiles * splits), blockIdx.z = query tile * splits + split
  const int* nk0_b;          // ragged: [B / kv_group] segment-0 lengths, clamped to [0, Nk0]; null = Nk0 for every batch
  float sl2;                 // scale * log2(e)
  void* O;                   // [B*Nq, H*64] 16-bit                     (splits == 1)
  long long ldo;
  float* part_o;             // [splits, B*Nq, H*64] fp32 unnormalised  (splits > 1)
  float* part_ml;            // [splits, B*Nq, H, 2]  (m_used * sl2, l)
  int* split_cnt;            // [B, H, ceil(Nq/64)] arrival counters (zero on entry, reset by the last arriver)
  int H;
  long long rows_total;      // B * Nq
  unsigned long long* trace; // debug only (m3r_debug_trace): per-CTA clock stamps, 64 words per CTA; normally null
  // export mode (context-parallel cross-attention): instead of the normalised 16-bit O, write this launch's UNNORMALISED
  // (O, m * sl2, l) - after the in-kernel merge of its own key splits - for a later merge with other key shards
  float* exp_o;              // [B*Nq, H*64] fp32
  float2* exp_ml;            // [B*Nq, H]
};


struct TileIt {
  int seg, t;          // current tile
  int g0;              // global index of its first key
  int nvalid;          // valid local keys in the tile (<=128)
  bool mask;           // needs element masking
};

// Key tiles in visiting order, without the ones entirely inside the skip range [lo, hi) (a view's own new tokens:
// never loaded nor multiplied).  Closed form: the fully masked tiles are one contiguous run [s0, s0 + ns) of the linear
// tile index (segment 0 tiles, then segment 1 tiles), so tile i of the visit is linear tile i (+ ns past the run).
// Every warp role maps indices the same way; no per-thread walk over the (possibly thousands of) tiles.
struct TileMap {
  int nk0, base1, nk1, lo, hi;      // base1: global index of segment 1's first key (Nk0 of the call, >= nk0 when ragged)
  int T0, s0, ns, n_all;
  __device__ static void masked_run(int n, int base, int T, int lo, int hi, int& a, int& c) {
    const int l = lo - base, h = hi - base;
    a = l <= 0 ? 0 : (l + AT_BN - 1) / AT_BN;                 // first tile with g0 >= lo
    const int b = h >= n ? T : (h <= 0 ? 0 : h / AT_BN);       // one past the last tile with g1 <= hi
    c = max(0, min(b, T) - a);
  }
  __device__ TileMap(int nk0_, int base1_, int nk1_, int lo_, int hi_) : nk0(nk0_), base1(base1_), nk1(nk1_), lo(lo_), hi(hi_) {
    T0 = (nk0 + AT_BN - 1) / AT_BN;
    const int T1 = (nk1 + AT_BN - 1) / AT_BN;
    int a0 = 0, c0 = 0, a1 = 0, c1 = 0;
    if (hi > lo) {
      masked_run(nk0, 0, T0, lo, hi, a0, c0);
      masked_run(nk1, base1, T1, lo, hi, a1, c1);
    }
    s0 = c0 > 0 ? a0 : T0 + a1;       // (a range covering both segments ends segment 0 and starts segment 1: contiguous)
    ns = c0 + c1;
    n_all = T0 + T1 - ns;
  }
  __device__ __forceinline__ TileIt get(int i) const {
    const int u = i + (i >= s0 ? ns : 0);
    TileIt it;
    it.seg = u >= T0 ? 1 : 0;
    it.t = u - (it.seg ? T0 : 0);
    const int n = it.seg ? nk1 : nk0;
    const int l0 = it.t * AT_BN;
    it.nvalid = min(AT_BN, n - l0);
    it.g0 = (it.seg ? base1 : 0) + l0;
    it.mask = (it.nvalid < AT_BN) || (it.g0 < hi && it.g0 + it.nvalid > lo);
    return it;
  }
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <bool BF16> __device__ __forceinline__ uint32_t packp(float lo, float hi) {
  uint32_t r;
  if (BF16) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}


// Online softmax of one 128-key score tile, in place: s <- 2^(s * sl2 - m_used * sl2), with masking, the lazy max
// refresh and the row sums.  alpha = the factor O must be rescaled by before P V of this tile is added.
__device__ __forceinline__ void softmax_tile(float (&s)[64], const TileIt& it, int lo, int hi, int fc, float sl2,
                                             float (&m_used)[2], float (&l_run)[2], float (&alpha)[2]) {
  if (it.mask) {
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int lc = (i >> 2) * 8 + fc + (i & 1);
      const int g = it.g0 + lc;
      if (!(lc < it.nvalid && !(g >= lo && g < hi))) s[i] = -INFINITY;
    }
  }
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < 32; ++i) mx = fmaxf(mx, s[(i >> 1) * 4 + rr * 2 + (i & 1)]);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    // lazy rescaling: refresh the folded max only when it is stale by more than 2^8
    alpha[rr] = 1.f;
    if (mx > -INFINITY && (m_used[rr] == -INFINITY || (mx - m_used[rr]) * sl2 > RESCALE_THRESHOLD)) {
      alpha[rr] = (m_used[rr] == -INFINITY) ? 0.f : ex2((m_used[rr] - mx) * sl2);
      m_used[rr] = mx;
    }
    l_run[rr] *= alpha[rr];
  }
  const float moff0 = (m_used[0] == -INFINITY) ? 0.f : m_used[0] * sl2;
  const float moff1 = (m_used[1] == -INFINITY) ? 0.f : m_used[1] * sl2;
#pragma unroll
  for (int nb = 0; nb < 16; ++nb) {
    s[nb * 4] = ex2(fmaf(s[nb * 4], sl2, -moff0)); s[nb * 4 + 1] = ex2(fmaf(s[nb * 4 + 1], sl2, -moff0));
    s[nb * 4 + 2] = ex2(fmaf(s[nb * 4 + 2], sl2, -moff1)); s[nb * 4 + 3] = ex2(fmaf(s[nb * 4 + 3], sl2, -moff1));
    l_run[0] += s[nb * 4] + s[nb * 4 + 1];
    l_run[1] += s[nb * 4 + 2] + s[nb * 4 + 3];
  }
}

// P in the A-operand fragment order: k-step kk covers keys 16 kk .. 16 kk + 15 = score blocks 2 kk, 2 kk + 1
// pa[4 kk ..] = {rows fr: keys 16kk + fc.., rows fr+8: same, rows fr: keys 16kk + 8 + fc.., rows fr+8: same}
template <bool BF16> __device__ __forceinline__ void pack_p(const float (&s)[64], uint32_t (&pa)[32]) {
#pragma unroll
  for (int nb = 0; nb < 16; ++nb) {
    pa[(nb >> 1) * 4 + (nb & 1) * 2] = packp<BF16>(s[nb * 4], s[nb * 4 + 1]);
    pa[(nb >> 1) * 4 + (nb & 1) * 2 + 1] = packp<BF16>(s[nb * 4 + 2], s[nb * 4 + 3]);
  }
}

// S[64 x 128] = Q K^T over the 4 k16 steps of head_dim 64 (16 head dims: +32 B inside the swizzle atom)
template <bool BF16> __device__ __forceinline__ void issue_qk(float (&s)[64], uint64_t qdesc, uint64_t kdesc) {
#pragma unroll
  for (int k = 0; k < HD / 16; ++k) Wgmma<128, BF16>::ss(s, qdesc + 2 * k, kdesc + 2 * k, k ? 1 : 0);
}

// O[64 x 64] += P[64 x 128] V[128 x 64] over 8 k16 steps (16 V rows: +2048 B)
template <bool BF16> __device__ __forceinline__ void issue_pv(float (&o)[32], const uint32_t (&pa)[32], uint64_t vdesc) {
#pragma unroll
  for (int kk = 0; kk < AT_BN / 16; ++kk) {
    const uint32_t a[4] = {pa[kk * 4], pa[kk * 4 + 1], pa[kk * 4 + 2], pa[kk * 4 + 3]};
    WgmmaRS<BF16>::n64_tb(o, a, vdesc + (uint64_t)((kk * 16 * 128) >> 4));
  }
}

// Ragged batch, last partial tile of segment 0: zero the V rows [nvalid, 128) of the stage (rows of another, longer batch's
// length that TMA did load) so that P V reads exact zeros there.  SW128 keeps each 128-byte row in place, so the rows
// are one contiguous byte range.  Every consumer thread of both warpgroups takes part, then the generic-proxy stores
// are made visible to wgmma and the warpgroups meet before either multiplies the stage.
template <int CT> __device__ __forceinline__ void zero_v_tail(uint8_t* sv, int nvalid) {
  uint4* v = reinterpret_cast<uint4*>(sv + nvalid * HD * 2);
  const int n = (AT_BN - nvalid) * (HD * 2 / 16);
  for (int i = threadIdx.x; i < n; i += CT) v[i] = make_uint4(0u, 0u, 0u, 0u);
  fence_proxy_async_smem();
  asm volatile("bar.sync 1, %0;" ::"n"(CT) : "memory");
}

template <bool BF16>
__global__ void __launch_bounds__(AttnCfg::THREADS, 1)
attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0,
            const __grid_constant__ CUtensorMap tmV0, const __grid_constant__ CUtensorMap tmK1,
            const __grid_constant__ CUtensorMap tmV1, const AttnParams p) {
  using Cfg = AttnCfg;
  constexpr int NWG = Cfg::NWG;
  constexpr int KS = Cfg::KS;
  constexpr int CT = 128 * NWG;                                 // consumer threads
  constexpr int TMA_WARP = 4 * NWG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                                   // NWG x 64 rows
  uint8_t* sK = smem + NWG * QTILE_BYTES;               // KS tiles
  uint8_t* sV = sK + KS * TILE_BYTES;                   // KS tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + KS * TILE_BYTES);
  uint64_t* q_full = bars;             // [1]
  uint64_t* k_full = bars + 1;         // [KS]
  uint64_t* k_empty = k_full + KS;     // [KS]
  uint64_t* v_full = k_empty + KS;     // [KS]
  uint64_t* v_empty = v_full + KS;     // [KS]

  M3R_TR(const unsigned long long t_entry = p.trace ? gtime_ns() : 0ull;)
  const int warp = threadIdx.x >> 5;
  const int wg = threadIdx.x >> 7;
  const int h = blockIdx.y;
  const int b = p.batch_minor ? blockIdx.x : blockIdx.z / p.splits, split = blockIdx.z % p.splits;
  const int kvb = b / p.kv_group;
  const int lo = p.skip_len > 0 ? p.skip_lo + (b % p.kv_group) * p.skip_step : 0;
  const int hi = p.skip_len > 0 ? lo + p.skip_len : 0;
  const int q0 = (p.batch_minor ? blockIdx.z / p.splits : blockIdx.x) * NWG * AT_BM;

  if (warp == TMA_WARP && elect_one()) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK0); tma_prefetch_desc(&tmV0);
    if (p.Nk1 > 0) { tma_prefetch_desc(&tmK1); tma_prefetch_desc(&tmV1); }
    mbar_init(q_full, 1);
    for (int s = 0; s < KS; ++s) { mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], NWG); mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], NWG); }
    fence_mbar_init();
  }
  __syncthreads();
  griddep_wait();
  griddep_launch();

  // this CTA's share [i0, i1) of the enumerated key tiles (the ragged lengths may come from the preceding kernel: read
  // after the dependency wait)
  const int nk0 = p.nk0_b ? min(max(__ldg(p.nk0_b + kvb), 0), p.Nk0) : p.Nk0;
  const TileMap tiles(nk0, p.Nk0, p.Nk1, lo, hi);
  const int n_all = tiles.n_all;
  const int chunk = (n_all + p.splits - 1) / p.splits;
  const int i0 = split * chunk;
  const int i1 = min(n_all, i0 + chunk);
  const int n_tiles = max(i1 - i0, 0);

  if (wg == NWG) {
    // ------------------------------------------------------------------ TMA producer warpgroup
    setmaxnreg_dec<Cfg::PRODUCER_REGS>();
    if (warp == TMA_WARP && elect_one() && n_tiles > 0) {
      mbar_arrive_expect_tx(q_full, NWG * QTILE_BYTES);
      for (int x = 0; x < NWG; ++x) tma_load_3d(sQ + x * QTILE_BYTES, &tmQ, q_full, h * HD, q0 + x * AT_BM, b);
      for (int j = 0; j < n_tiles; ++j) {
        const TileIt it = tiles.get(i0 + j);
        const int st = j % KS;
        const uint32_t ph = (j / KS) & 1;
        const CUtensorMap* mk = it.seg == 0 ? &tmK0 : &tmK1;
        const CUtensorMap* mv = it.seg == 0 ? &tmV0 : &tmV1;
        mbar_wait(&k_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&k_full[st], TILE_BYTES);
        tma_load_3d(sK + st * TILE_BYTES, mk, &k_full[st], h * HD, it.t * AT_BN, kvb);
        mbar_wait(&v_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&v_full[st], TILE_BYTES);
        tma_load_3d(sV + st * TILE_BYTES, mv, &v_full[st], h * HD, it.t * AT_BN, kvb);
      }
    }
    return;
  }
  setmaxnreg_inc<Cfg::CONSUMER_REGS>();

  // ------------------------------------------------------------------ consumer warpgroup: 64 query rows
  const int wl = warp & 3, lane = threadIdx.x & 31;
  const int fr = wl * 16 + (lane >> 2);                     // fragment rows fr and fr + 8 of the warpgroup's 64 rows
  const int fc = 2 * (lane & 3);                            // fragment column offset inside every 8-column block
  const bool leader = wl == 0 && lane == 0;                 // arrives on the ring's empty barriers for the warpgroup
  float o[32];                                 // O[64 x 64] fragment
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_used[2] = {-INFINITY, -INFINITY};    // max currently folded into the exponent (raw score units), rows fr, fr + 8
  float l_run[2] = {0.f, 0.f};                 // this thread's share of the row sums (reduced over the quad at the end)
  M3R_TR(unsigned long long* tr = nullptr;
         if (p.trace && threadIdx.x == 0)
           tr = p.trace + 128ull * ((blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x);
         if (tr) { tr[0] = t_entry; tr[1] = gtime_ns(); tr[2] = smid(); tr[3] = (unsigned long long)n_tiles; })
  if (n_tiles > 0) {
    const uint64_t qdesc = smem_desc_sw128(smem_u32(sQ + wg * QTILE_BYTES));
    float s[64];                               // S / P of the tile in flight (fp32)
    uint32_t pa[32];                           // P of the previous tile, packed: the A operand of its P V
    float alpha[2];
    mbar_wait(q_full, 0);
    // tile 0: scores and softmax only
    mbar_wait(&k_full[0], 0);
    wgmma_fence();
    issue_qk<BF16>(s, qdesc, smem_desc_sw128(smem_u32(sK)));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    if (leader) mbar_arrive(&k_empty[0]);
    softmax_tile(s, tiles.get(i0), lo, hi, fc, p.sl2, m_used, l_run, alpha);
    pack_p<BF16>(s, pa);
    for (int j = 1; j < n_tiles; ++j) {
      const int st = j % KS, pst = (j - 1) % KS;
      M3R_TR(if (tr && j < 12) tr[8 + 4 * j] = gtime_ns();)
      mbar_wait(&k_full[st], (j / KS) & 1);
      mbar_wait(&v_full[pst], ((j - 1) / KS) & 1);
      if (p.nk0_b) {
        const TileIt pt = tiles.get(i0 + j - 1);
        if (pt.seg == 0 && pt.nvalid < AT_BN) zero_v_tail<CT>(sV + pst * TILE_BYTES, pt.nvalid);
      }
      wgmma_fence();
      issue_qk<BF16>(s, qdesc, smem_desc_sw128(smem_u32(sK + st * TILE_BYTES)));
      wgmma_commit();
      issue_pv<BF16>(o, pa, smem_desc_sw128(smem_u32(sV + pst * TILE_BYTES)));
      wgmma_commit();
      wgmma_wait<1>();                          // the scores of tile j are in; P V of tile j - 1 may still run
      reg_fence(s);
      if (leader) mbar_arrive(&k_empty[st]);
      softmax_tile(s, tiles.get(i0 + j), lo, hi, fc, p.sl2, m_used, l_run, alpha);
      wgmma_wait<0>();
      reg_fence(o);
      reg_fence(pa);
      if (leader) mbar_arrive(&v_empty[pst]);
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
      pack_p<BF16>(s, pa);
    }
    const int lst = (n_tiles - 1) % KS;
    mbar_wait(&v_full[lst], ((n_tiles - 1) / KS) & 1);
    if (p.nk0_b) {
      const TileIt pt = tiles.get(i0 + n_tiles - 1);
      if (pt.seg == 0 && pt.nvalid < AT_BN) zero_v_tail<CT>(sV + lst * TILE_BYTES, pt.nvalid);
    }
    wgmma_fence();
    issue_pv<BF16>(o, pa, smem_desc_sw128(smem_u32(sV + lst * TILE_BYTES)));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    reg_fence(pa);
    if (leader) mbar_arrive(&v_empty[lst]);
  }
  M3R_TR(if (tr) tr[4] = gtime_ns();)
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    l_run[rr] += __shfl_xor_sync(0xffffffffu, l_run[rr], 1);
    l_run[rr] += __shfl_xor_sync(0xffffffffu, l_run[rr], 2);
  }

  // ---- O fragments -> shared memory (over the Q / K stages: every consumer has finished its MMAs), then each thread
  // takes one row and 32 of its 64 columns: the layout of the stores, the split partials and the merge below.
  asm volatile("bar.sync 1, %0;" ::"n"(CT) : "memory");
  {
    float* so = reinterpret_cast<float*>(smem) + wg * (AT_BM * OSTR);
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      so[fr * OSTR + nb * 8 + fc] = o[nb * 4]; so[fr * OSTR + nb * 8 + fc + 1] = o[nb * 4 + 1];
      so[(fr + 8) * OSTR + nb * 8 + fc] = o[nb * 4 + 2]; so[(fr + 8) * OSTR + nb * 8 + fc + 1] = o[nb * 4 + 3];
    }
    float2* sml = reinterpret_cast<float2*>(reinterpret_cast<float*>(smem) + NWG * AT_BM * OSTR) + wg * AT_BM;
    if ((lane & 3) == 0) { sml[fr] = make_float2(m_used[0], l_run[0]); sml[fr + 8] = make_float2(m_used[1], l_run[1]); }
  }
  asm volatile("bar.sync 1, %0;" ::"n"(CT) : "memory");
  const int row = threadIdx.x & (AT_BM - 1);
  const int half = (threadIdx.x >> 6) & 1;
  const int q_idx = q0 + wg * AT_BM + row;
  constexpr int OC = HD / 2;
  float acc[OC];
  float m_row, l_row;
  {
    const float* so = reinterpret_cast<const float*>(smem) + wg * (AT_BM * OSTR) + row * OSTR + half * OC;
#pragma unroll
    for (int d = 0; d < OC; ++d) acc[d] = so[d];
    const float2 ml = (reinterpret_cast<const float2*>(reinterpret_cast<const float*>(smem) + NWG * AT_BM * OSTR) + wg * AT_BM)[row];
    m_row = ml.x; l_row = ml.y;
  }
  if (q_idx < p.Nq && p.splits == 1 && p.exp_o != nullptr) {
    const long long grow = (long long)b * p.Nq + q_idx;
    float4* e4 = reinterpret_cast<float4*>(p.exp_o + (grow * p.H + h) * HD + half * OC);
#pragma unroll
    for (int t = 0; t < OC / 4; ++t) e4[t] = make_float4(acc[4 * t], acc[4 * t + 1], acc[4 * t + 2], acc[4 * t + 3]);
    if (half == 0) p.exp_ml[grow * p.H + h] = make_float2(m_row == -INFINITY ? -INFINITY : m_row * p.sl2, l_row);
  } else if (q_idx < p.Nq && p.splits == 1) {
    const long long grow = (long long)b * p.Nq + q_idx;
    const float inv = l_row > 0.f ? 1.0f / l_row : 0.f;
    uint4* o4 = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.O) + grow * p.ldo + h * HD + half * OC);
#pragma unroll
    for (int t = 0; t < OC / 8; ++t) {
      uint4 w;
      w.x = packp<BF16>(acc[8 * t] * inv, acc[8 * t + 1] * inv);
      w.y = packp<BF16>(acc[8 * t + 2] * inv, acc[8 * t + 3] * inv);
      w.z = packp<BF16>(acc[8 * t + 4] * inv, acc[8 * t + 5] * inv);
      w.w = packp<BF16>(acc[8 * t + 6] * inv, acc[8 * t + 7] * inv);
      o4[t] = w;
    }
  }
  // key-range splits: unnormalised partial (O, m, l) of this CTA.  Layout [split][unit = (b, h, 64-row query tile)]
  // [16 column chunks][64 rows] float4 (and [split][unit][64 rows] float2): lanes are consecutive rows, so both these
  // stores and the merge's loads are fully coalesced 512 B requests.
  constexpr int CH = 8;                   // float4 column chunks per thread
  const int n_qtiles = (p.Nq + AT_BM - 1) / AT_BM;
  const long long unit = ((long long)b * p.H + h) * n_qtiles + (q0 / AT_BM + wg);
  const long long n_units = p.rows_total / p.Nq * p.H * n_qtiles;
  // (a warpgroup whose rows are all past Nq has no unit of its own: it takes no part in the split bookkeeping)
  if (p.splits > 1 && q0 + wg * AT_BM < p.Nq) {
    float4* o4 = reinterpret_cast<float4*>(p.part_o) + ((long long)split * n_units + unit) * (16 * AT_BM) + (half * CH) * AT_BM + row;
#pragma unroll
    for (int t = 0; t < CH; ++t) o4[t * AT_BM] = make_float4(acc[4 * t], acc[4 * t + 1], acc[4 * t + 2], acc[4 * t + 3]);
    if (half == 0)
      reinterpret_cast<float2*>(p.part_ml)[((long long)split * n_units + unit) * AT_BM + row] =
          make_float2(m_row == -INFINITY ? -INFINITY : m_row * p.sl2, l_row);
  }
  M3R_TR(if (tr) tr[5] = gtime_ns();)
  if (p.splits > 1 && q0 + wg * AT_BM < p.Nq) {
    // ---- merge of the key-range splits by the last CTA to finish this (batch, head, query tile):
    // out = sum_s O_s 2^(m_s - m) / sum_s l_s 2^(m_s - m).  No extra kernel launch on the one-view-per-step chain.
    // Named barriers 2 .. 2 + NWG - 1: one per warpgroup (barrier 1 is the consumers' O staging above).
    __shared__ int s_last[NWG];
    __threadfence();                                              // partials visible device-wide
    asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
    int* cnt = p.split_cnt + unit;
    if ((threadIdx.x & 127) == 0) {
      const int prev = atomicAdd(cnt, 1);
      s_last[wg] = (prev == p.splits - 1);
      if (prev == p.splits - 1) *cnt = 0;                         // self-cleaning for the next launch
    }
    asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
    if (s_last[wg]) {
      __threadfence();
      const float2* mlp = reinterpret_cast<const float2*>(p.part_ml) + unit * AT_BM + row;
      const float4* op = reinterpret_cast<const float4*>(p.part_o) + unit * (16 * AT_BM) + (half * CH) * AT_BM + row;
      const long long ml_stride = n_units * AT_BM, o_stride = n_units * (16 * AT_BM);
      float m = -INFINITY;
#pragma unroll 4
      for (int sp = 0; sp < p.splits; ++sp) m = fmaxf(m, __ldcg(mlp + sp * ml_stride).x);
      float l = 0.f;
      const long long grow = (long long)b * p.Nq + q_idx;
      // 16 columns at a time: 4 splits x 4 float4 loads in flight per thread, few L2 round trips
#pragma unroll 1
      for (int qd = 0; qd < CH / 4; ++qd) {
        float a16[16];
#pragma unroll
        for (int d = 0; d < 16; ++d) a16[d] = 0.f;
        for (int sp0 = 0; sp0 < p.splits; sp0 += 4) {
          float4 v[4][4];
          float w[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int sp = min(sp0 + u, p.splits - 1);
            const float2 ml = __ldcg(mlp + sp * ml_stride);
            w[u] = (sp0 + u < p.splits && ml.x != -INFINITY) ? ex2(ml.x - m) : 0.f;
            if (qd == 0) l += ml.y * w[u];
#pragma unroll
            for (int t = 0; t < 4; ++t) v[u][t] = __ldcg(op + sp * o_stride + (qd * 4 + t) * AT_BM);
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
#pragma unroll
            for (int t = 0; t < 4; ++t) {
              a16[4 * t] = fmaf(v[u][t].x, w[u], a16[4 * t]); a16[4 * t + 1] = fmaf(v[u][t].y, w[u], a16[4 * t + 1]);
              a16[4 * t + 2] = fmaf(v[u][t].z, w[u], a16[4 * t + 2]); a16[4 * t + 3] = fmaf(v[u][t].w, w[u], a16[4 * t + 3]);
            }
          }
        }
        const float inv = l > 0.f ? 1.0f / l : 0.f;      // l is complete after the first pass
        if (q_idx < p.Nq && p.exp_o != nullptr) {
          float4* e4 = reinterpret_cast<float4*>(p.exp_o + (grow * p.H + h) * HD + half * OC + qd * 16);
#pragma unroll
          for (int t = 0; t < 4; ++t) e4[t] = make_float4(a16[4 * t], a16[4 * t + 1], a16[4 * t + 2], a16[4 * t + 3]);
          if (half == 0 && qd == 0) p.exp_ml[grow * p.H + h] = make_float2(m, l);
        } else if (q_idx < p.Nq) {
          uint4* o4 = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.O) + grow * p.ldo + h * HD + half * OC + qd * 16);
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            uint4 wv;
            wv.x = packp<BF16>(a16[8 * t] * inv, a16[8 * t + 1] * inv);
            wv.y = packp<BF16>(a16[8 * t + 2] * inv, a16[8 * t + 3] * inv);
            wv.z = packp<BF16>(a16[8 * t + 4] * inv, a16[8 * t + 5] * inv);
            wv.w = packp<BF16>(a16[8 * t + 6] * inv, a16[8 * t + 7] * inv);
            o4[t] = wv;
          }
        }
      }
    }
  }
M3R_TR(if (p.trace && threadIdx.x == 0)
         p.trace[128ull * ((blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) + 6] = gtime_ns();)
}

// How many CTAs an SM holds, from the kernel's actual registers and shared memory (-1 after set_error); checks that the
// launch allocation covers the register split.
template <bool BF16> static int attn_resident_ctas() {
  using Cfg = AttnCfg;
  const KernelInfo k = kernel_setup((const void*)attn_kernel<BF16>, Cfg::SMEM, Cfg::THREADS);
  if (k.resident == 0) return -1;
  if (k.regs < Cfg::LAUNCH_REGS)
    return set_error("attention: kernel built with %d registers per thread, the register split needs %d", k.regs, Cfg::LAUNCH_REGS), -1;
  return k.resident;
}

template <bool BF16>
static int launch_attn(const CUtensorMap& tmQ, const CUtensorMap& tmK0, const CUtensorMap& tmV0, const CUtensorMap& tmK1,
                       const CUtensorMap& tmV1, const AttnParams& p, int B, cudaStream_t s) {
  using Cfg = AttnCfg;
  const int qtiles = (p.Nq + Cfg::NWG * AT_BM - 1) / (Cfg::NWG * AT_BM);
  const dim3 grid = p.batch_minor ? dim3(B, p.H, qtiles * p.splits) : dim3(qtiles, p.H, B * p.splits);
  cudaError_t e = launch_pdl(attn_kernel<BF16>, grid, dim3(Cfg::THREADS), Cfg::SMEM, s, tmQ, tmK0, tmV0, tmK1, tmV1, p);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("attention launch: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}


static int attention(const m3r_attn_args* a, const int32_t* nk0_b, void* stream) {
  if (!a || !a->Q || !a->K0 || !a->V0 || (!a->O && !a->export_o)) return set_error("attention: null pointer");
  if ((a->export_o == nullptr) != (a->export_ml == nullptr)) return set_error("attention: export_o and export_ml go together");
  if (a->B <= 0 || a->H <= 0 || a->Nq <= 0) return 0;
  if (a->kv_group < 1 || a->B % a->kv_group) return set_error("attention: B (%d) must be a multiple of kv_group (%d)", a->B, a->kv_group);
  if (a->Nk0 < 0 || a->Nk1 < 0 || a->Nk0 + a->Nk1 <= 0) return set_error("attention: no keys");
  if (a->Nk1 > 0 && (!a->K1 || !a->V1)) return set_error("attention: segment 1 pointers missing");
  if (a->ldq % 8 || a->ldk0 % 8 || (a->Nk1 > 0 && a->ldk1 % 8) || a->ldo % 8) return set_error("attention: leading dims must be multiples of 8");
  {
    // a row whose keys are all skipped would be 0/0; the reference never produces one (decoder.py:291-296)
    const int tot = a->Nk0 + a->Nk1;
    if (a->skip_len >= tot && a->skip_len > 0) return set_error("attention: skip range covers every key");
  }
  cudaStream_t cs = reinterpret_cast<cudaStream_t>(stream);
  const int Bkv = a->B / a->kv_group;
  CUtensorMap tmQ, tmK0, tmV0, tmK1, tmV1;
  auto mk3 = [&](CUtensorMap* m, const void* base, int64_t ld, int64_t rows, int64_t bstride_rows, int64_t nb, uint32_t box_rows) {
    return make_tmap_3d(m, base, a->is_bf16, (uint64_t)a->H * HD, (uint64_t)rows, (uint64_t)nb, (uint64_t)ld,
                        (uint64_t)bstride_rows * (uint64_t)ld, HD, box_rows);
  };
  if (mk3(&tmQ, a->Q, a->ldq, a->Nq, a->Nq, a->B, AT_BM)) return 1;
  if (a->Nk0 > 0) {
    if (mk3(&tmK0, a->K0, a->ldk0, a->Nk0, a->kv_bstride0, Bkv, AT_BN)) return 1;
    if (mk3(&tmV0, a->V0, a->ldk0, a->Nk0, a->kv_bstride0, Bkv, AT_BN)) return 1;
  } else { tmK0 = tmQ; tmV0 = tmQ; }
  if (a->Nk1 > 0) {
    if (mk3(&tmK1, a->K1, a->ldk1, a->Nk1, a->kv_bstride1, Bkv, AT_BN)) return 1;
    if (mk3(&tmV1, a->V1, a->ldk1, a->Nk1, a->kv_bstride1, Bkv, AT_BN)) return 1;
  } else { tmK1 = tmK0; tmV1 = tmV0; }

  // ---- key splits, from a cost model in units of one CTA's pass over one key tile (CTAs of 128 query rows, one per
  // SM).  CTAs run in waves of (resident CTAs per SM x SMs); each CTA pays about 4 tile passes of prologue (Q load,
  // pipeline fill) and epilogue; a split launch pays the partial stores plus the merge, which reads every split's
  // partial.  Both constants were fitted to tools/prof_attn.py `sweep` / `longmem` on H100 SXM (132 SMs), where this
  // picks the measured best split count or one within 5 % of it.  M3R_ATTN_SPLITS forces a split count.
  const int sms = num_sms();
  const int key_tiles = (a->Nk0 + AT_BN - 1) / AT_BN + (a->Nk1 + AT_BN - 1) / AT_BN;   // upper bound
  const bool split_ok = (long long)a->B * a->H * ((a->Nq + AT_BM - 1) / AT_BM) <= 16384;   // counter table of the split path
  const int resident = a->is_bf16 ? attn_resident_ctas<true>() : attn_resident_ctas<false>();
  if (resident < 0) return 1;
  int splits = 1;
  if (const char* f = getenv("M3R_ATTN_SPLITS")) { const int v = atoi(f); if (v >= 1) splits = min(v, min(32, key_tiles)); }
  else if (split_ok) {
    const long long ctas = (long long)((a->Nq + AttnCfg::NWG * AT_BM - 1) / (AttnCfg::NWG * AT_BM)) * a->H * a->B;
    const long long slots = (long long)resident * sms;
    double best = 0.0;
    for (int sp = 1; sp <= 32 && sp <= key_tiles; ++sp) {
      const int chunk = (key_tiles + sp - 1) / sp;
      const long long waves = (ctas * sp + slots - 1) / slots;
      const double cost = waves * (chunk + 4.0) + (sp > 1 ? 4.0 + sp / 4.0 : 0.0);
      if (sp == 1 || cost < best) { best = cost; splits = sp; }
    }
  }
  { const int chunk = (key_tiles + splits - 1) / splits; splits = (key_tiles + chunk - 1) / chunk; }   // no empty splits

  AttnParams p;
  p.Nq = a->Nq; p.Nk0 = a->Nk0; p.Nk1 = a->Nk1; p.kv_group = a->kv_group;
  p.skip_lo = a->skip_lo; p.skip_step = a->skip_step; p.skip_len = a->skip_len;
  p.splits = splits; p.sl2 = a->scale * 1.4426950408889634f; p.nk0_b = nk0_b;
  // one segment-0 K/V for every key batch (kv_bstride0 = 0, e.g. the frames of several cameras against one SLAM memory):
  // the batches of one (head, query tile, key split) are launched next to each other, so that the K/V tiles they all read
  // can be fetched from HBM once and served from L2 to the others (the effect on speed has not been measured)
  p.batch_minor = a->Nk0 > 0 && a->kv_bstride0 == 0 && Bkv > 1 &&
                  (long long)((a->Nq + AttnCfg::NWG * AT_BM - 1) / (AttnCfg::NWG * AT_BM)) * splits <= 65535 ? 1 : 0;
  p.O = a->O; p.ldo = a->ldo; p.H = a->H; p.rows_total = (long long)a->B * a->Nq;
  p.part_o = nullptr; p.part_ml = nullptr; p.split_cnt = nullptr;
  p.exp_o = a->export_o; p.exp_ml = reinterpret_cast<float2*>(a->export_ml);
  p.trace = trace_buffer();
  if (splits > 1) {
    // scratch layout: [16384 arrival counters | partial O | partial (m, l)].  The counters sit at a fixed place, are
    // zeroed once when the buffer is (re)allocated and every launch leaves them zero again (last arriver resets).
    constexpr size_t CNT = 16384;
    const size_t n_cnt = (size_t)a->B * a->H * ((a->Nq + AT_BM - 1) / AT_BM);
    if (n_cnt > CNT) return set_error("attention: too many (batch, head, tile) groups for the split path");
    const size_t need = CNT + (size_t)splits * n_cnt * AT_BM * (HD + 2);     // partial O + (m, l), padded to whole query tiles
    RegistryLock lock;
    StreamState* sc = stream_state(cs, lock);
    if (!sc) return set_error("attention: no current device");
    if (need > sc->split_cap) {
      if (sc->split_buf) cudaFreeAsync(sc->split_buf, cs);
      sc->split_buf = nullptr; sc->split_cap = 0;
      const size_t cap = need + need / 2;
      if (cudaMallocAsync(&sc->split_buf, cap * sizeof(float), cs) != cudaSuccess) return set_error("attention: split scratch allocation failed");
      if (cudaMemsetAsync(sc->split_buf, 0, CNT * sizeof(int), cs) != cudaSuccess) return set_error("attention: counter memset failed");
      sc->split_cap = cap;
    }
    p.split_cnt = reinterpret_cast<int*>(sc->split_buf);
    p.part_o = sc->split_buf + CNT;
    p.part_ml = p.part_o + (size_t)splits * n_cnt * AT_BM * HD;
  }
  {
    const double nk_eff = (double)(a->Nk0 + a->Nk1 - a->skip_len);
    // profiling categories: launches over the whole key range, and launches with key splits + in-kernel merge
    ProfScope prof(splits == 1 ? PROF_ATTN_QT2 : PROF_ATTN_QT1, 4.0 * a->B * (double)a->H * a->Nq * nk_eff * HD,
                   2.0 * ((double)a->B * a->Nq * a->H * HD * 2 + (double)Bkv * (a->Nk0 + a->Nk1) * a->H * HD * 2), cs);
    const int rc = a->is_bf16 ? launch_attn<true>(tmQ, tmK0, tmV0, tmK1, tmV1, p, a->B, cs)
                              : launch_attn<false>(tmQ, tmK0, tmV0, tmK1, tmV1, p, a->B, cs);
    if (rc) return rc;
  }
  return 0;
}
}  // namespace m3r

extern "C" int m3r_attention(const m3r_attn_args* a, void* stream) { return m3r::attention(a, nullptr, stream); }

extern "C" int m3r_attention_ragged(const m3r_attn_args* a, const int32_t* nk0_b, void* stream) {
  using namespace m3r;
  if (!nk0_b) return set_error("attention_ragged: null nk0_b");
  if (reinterpret_cast<uintptr_t>(nk0_b) % 4) return set_error("attention_ragged: nk0_b must be 4-byte aligned");
  if (a && (a->export_o || a->export_ml)) return set_error("attention_ragged: export mode is not supported with ragged lengths");
  if (a && a->Nk0 < 1) return set_error("attention_ragged: Nk0 (the longest batch, %d) must be >= 1", a->Nk0);
  return attention(a, nk0_b, stream);
}
