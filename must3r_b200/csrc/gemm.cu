#include "gemm_kernel.cuh"

namespace m3r {

static bool misaligned(const void* ptr, unsigned bytes) { return ptr && (reinterpret_cast<uintptr_t>(ptr) % bytes) != 0; }

// The epilogue reads bias / rowbias / rope_tab / residual as float2 and stores out / peers / norm_out in 16-byte units;
// a base pointer off that grid would fault on the device, so it is refused here, before any CUDA call.
static int check_args(const m3r_gemm_args* a) {
  if (!a || !a->A || !a->W) return set_error("gemm: null pointer");
  if (a->N % 32 || a->K % 64 || a->N <= 0 || a->K <= 0) return set_error("gemm: N (%d) must be a multiple of 32 and K (%d) of 64", a->N, a->K);
  if (a->lda % 8 || a->ldw % 8) return set_error("gemm: lda/ldw must be multiples of 8 elements (16 B)");
  if ((a->out_dtype == M3R_OUT_F32 && a->ldc % 4) || (a->out_dtype == M3R_OUT_16 && a->ldc % 8)) return set_error("gemm: ldc alignment");
  if (a->residual && a->ldr % 4) return set_error("gemm: ldr alignment");
  if (a->rope_tab && (a->rope_cols % 64)) return set_error("gemm: rope_cols must be a multiple of 64");
  if (a->n_peer_out < 0 || a->n_peer_out > M3R_MAX_PEERS || (a->n_peer_out > 0 && a->out_dtype != M3R_OUT_16)) return set_error("gemm: peer outputs need 0..%d pointers and a 16-bit output", M3R_MAX_PEERS);
  if (misaligned(a->bias, 8)) return set_error("gemm: bias must be 8-byte aligned");
  if (misaligned(a->rowbias, 8)) return set_error("gemm: rowbias must be 8-byte aligned");
  if (misaligned(a->rope_tab, 8)) return set_error("gemm: rope_tab must be 8-byte aligned");
  if (misaligned(a->residual, 8)) return set_error("gemm: residual must be 8-byte aligned");
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

// e4m3 options: refused before any CUDA call when they do not fit the kernel
static int check_e4m3(const m3r_gemm_args* a, const m3r_gemm_e4m3_args* e8) {
  if (!e8) return 0;
  if (e8->a_e4m3) {
    if (!e8->w_scale) return set_error("gemm: e4m3 operands need w_scale");
    if (misaligned(e8->w_scale, 8)) return set_error("gemm: w_scale must be 8-byte aligned");
    if (!a->is_bf16) return set_error("gemm: e4m3 operands need is_bf16 = 1 (their 16-bit outputs are bf16)");
    if (a->K % 128 || a->N % 64) return set_error("gemm: e4m3 operands need K %% 128 == 0 (K = %d) and N %% 64 == 0 (N = %d)", a->K, a->N);
    if (a->lda % 16 || a->ldw % 16) return set_error("gemm: e4m3 lda/ldw must be multiples of 16 elements (16 B)");
  }
  if (e8->norm_e4m3 && !a->norm_out) return set_error("gemm: norm_e4m3 without norm_out");
  if (e8->a_e4m3 && a->norm_out) return set_error("gemm: norm_out takes 16-bit operands only (e4m3 operands with norm_out)");
  return 0;
}

// e4m3 operand launches: the tile widths the e4m3 kernel is instantiated for
static int e4m3_bn(int bn, int N) {
  if (bn == 32) return 64;
  if (bn == 160 || bn == 192) return N % 128 == 0 ? 128 : 64;
  return bn;
}

static int gemm_impl(const m3r_gemm_args* a, const m3r_gemm_e4m3_args* e8, cudaStream_t s) {
  if (check_args(a) || check_e4m3(a, e8)) return 1;
  if (!a->out) return set_error("gemm: null pointer");
  if (misaligned(a->out, 16)) return set_error("gemm: out must be 16-byte aligned");
  for (int r = 0; r < a->n_peer_out; ++r)
    if (!a->peer_out[r] || misaligned(a->peer_out[r], 16)) return set_error("gemm: peer_out[%d] must be a 16-byte aligned pointer", r);
  if (a->norm_out && misaligned(a->norm_out, 16)) return set_error("gemm: norm_out must be 16-byte aligned");
  if (a->norm_out && a->rows_per_batch > 0) return set_error("gemm: norm_out does not take the rows_per_batch remap");
  if (a->M <= 0) return 0;
  const int sms = num_sms();
  if (a->norm_out) {
    // LayerNorm-emitting epilogue: fp32 out = the new residual stream, norm_out = its normalised 16-bit (or e4m3) rows
    const int ldn_align = (e8 && e8->norm_e4m3) ? 16 : 8;
    if (a->N % 64 || a->N > 32 * EMIT_MAX_PARTS || a->out_dtype != M3R_OUT_F32 || a->ldn % ldn_align)
      return set_error("gemm: norm_out needs N %% 64 == 0, N <= %d, an fp32 output and ldn %% %d == 0", 32 * EMIT_MAX_PARTS, ldn_align);
    // every CTA of the launch must be resident at once (they meet at a counter): 128x64 tiles, or 128x128 tiles when the
    // 64-wide ones would not fit on the SMs in one wave
    const int tiles_m = (a->M + BM - 1) / BM;
    if (tiles_m <= EMIT_MAX_TILES_M && tiles_m * (a->N / 64) <= sms) return launch_gemm<64, MODE_EMIT, false>(a, e8, s);
    if (tiles_m <= EMIT_MAX_TILES_M && a->N % 128 == 0 && tiles_m * (a->N / 128) <= sms) return launch_gemm<128, MODE_EMIT, false>(a, e8, s);
    return set_error("gemm: norm_out needs one 128x64 tile per SM (M=%d N=%d); normalise with m3r_layernorm instead", a->M, a->N);
  }
  int bn = pick_bn(a->M, a->N, 1);
  const char* force = getenv("M3R_GEMM_BN");
  if (force) { int f = atoi(force); if ((f == 32 || f == 64 || f == 128 || f == 160 || f == 192 || f == 256) && a->N % f == 0) bn = f; }
  if (e8 && e8->a_e4m3) return launch_gemm_e4m3(e4m3_bn(bn, a->N), MODE_PLAIN, a, e8, s, nullptr);
  switch (bn) {
    case 256: return launch_gemm<256, MODE_PLAIN, false>(a, e8, s);
    case 192: return launch_gemm<192, MODE_PLAIN, false>(a, e8, s);
    case 160: return launch_gemm<160, MODE_PLAIN, false>(a, e8, s);
    case 128: return launch_gemm<128, MODE_PLAIN, false>(a, e8, s);
    case 64: return launch_gemm<64, MODE_PLAIN, false>(a, e8, s);
    default: return launch_gemm<32, MODE_PLAIN, false>(a, e8, s);
  }
}

static int gemm_grouped_impl(const m3r_gemm_args* a, const m3r_gemm_group* grp, const m3r_gemm_e4m3_args* e8, cudaStream_t s) {
  if (check_args(a) || check_e4m3(a, e8)) return 1;
  if (!grp || grp->groups < 1 || grp->groups > M3R_MAX_GROUPS) return set_error("gemm_grouped: 1..%d groups", M3R_MAX_GROUPS);
  if (a->norm_out || a->residual) return set_error("gemm_grouped: no residual / norm_out");
  if (a->bias && grp->bias_group % 2) return set_error("gemm_grouped: bias_group must keep every group's bias 8-byte aligned");
  if (e8 && e8->a_e4m3 && grp->w_group_rows % 2) return set_error("gemm_grouped: w_group_rows must keep every group's w_scale 8-byte aligned");
  for (int g = 0; g < grp->groups; ++g) {
    if (!grp->out[g]) return set_error("gemm_grouped: out[%d] is null", g);
    if (misaligned(grp->out[g], 16)) return set_error("gemm_grouped: out[%d] must be 16-byte aligned", g);
    for (int r = 0; r < a->n_peer_out; ++r) {
      const void* pr = grp->peer_out[g * M3R_MAX_PEERS + r];
      if (!pr || misaligned(pr, 16)) return set_error("gemm_grouped: peer_out[%d] must be a 16-byte aligned pointer", g * M3R_MAX_PEERS + r);
    }
  }
  if (a->M <= 0) return 0;
  int bn = pick_bn(a->M, a->N, grp->groups);
  if (bn != 256 && bn != 128) bn = a->N % 128 == 0 ? 128 : 64;
  if (a->N % bn) return set_error("gemm_grouped: N (%d) must be a multiple of 64", a->N);
  if (e8 && e8->a_e4m3) return launch_gemm_e4m3(bn, MODE_GROUPED, a, e8, s, grp);
  switch (bn) {
    case 256: return launch_gemm<256, MODE_GROUPED, false>(a, e8, s, grp);
    case 128: return launch_gemm<128, MODE_GROUPED, false>(a, e8, s, grp);
    default: return launch_gemm<64, MODE_GROUPED, false>(a, e8, s, grp);
  }
}

}  // namespace m3r

extern "C" int m3r_gemm(const m3r_gemm_args* a, void* stream) {
  return m3r::gemm_impl(a, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int m3r_gemm_e4m3(const m3r_gemm_args* a, const m3r_gemm_e4m3_args* e8, void* stream) {
  return m3r::gemm_impl(a, e8, reinterpret_cast<cudaStream_t>(stream));
}

// `groups` GEMMs of identical shape in one launch (the post-feedback K|V projections of all decoder levels,
// must3r/model/decoder.py:323-330): A = [groups * M, K] (group g = rows [g*M, (g+1)*M)), W / bias stacked with strides
// w_group_rows / bias_group, one output (and one set of peer outputs) per group.
extern "C" int m3r_gemm_grouped(const m3r_gemm_args* a, const m3r_gemm_group* grp, void* stream) {
  return m3r::gemm_grouped_impl(a, grp, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int m3r_gemm_grouped_e4m3(const m3r_gemm_args* a, const m3r_gemm_group* grp, const m3r_gemm_e4m3_args* e8, void* stream) {
  return m3r::gemm_grouped_impl(a, grp, e8, reinterpret_cast<cudaStream_t>(stream));
}
