// Whole-model forward passes: every kernel of an encoder / decoder call is enqueued from here, so a step costs
// one C-ABI call instead of ~15 Python->ctypes round trips per layer.
//
// Data layout in HBM (per call, inside the caller-provided workspace):
//   residual stream  x      fp32  [M, D]        (M = all tokens of the call, rows ordered group/scene/view/token)
//   GEMM operands    h16    16b   [M, D]        LayerNorm output
//                    qkv16  16b   [M, 3D]       fused q|k|v, RoPE already applied to q,k by the GEMM epilogue
//                    att16  16b   [M, D]        attention output (heads merged), operand of proj
//                    mlp16  16b   [M, 4D]       GELU(fc1) output
//   decoder only     snap   fp32  [depth][M,D]  block inputs (= new_mem[l], decoder.py:304) kept for the feedback
//                    kvnew  16b   [B, Nt, 2D]   this step's pre-feedback K|V (second key segment of the CA)
#include <stdio.h>
#include <algorithm>
#include <vector>
#include "m3r_internal.h"
#include "ptx.cuh"

namespace m3r {

struct Arena {
  uint8_t* base; int64_t off; int64_t cap;
  Arena(void* p, int64_t c) : base(reinterpret_cast<uint8_t*>(p)), off(0), cap(c) {}
  template <typename T> T* take(int64_t n_elems) {
    off = (off + 255) & ~int64_t(255);
    T* p = reinterpret_cast<T*>(base ? base + off : nullptr);
    off += n_elems * (int64_t)sizeof(T);
    return p;
  }
};

#define M3R_TRY(x) do { if ((x) != 0) return 1; } while (0)

static int gemm(const void* A, int64_t lda, const void* W, int64_t ldw, int M, int N, int K, int is_bf16,
                const float* bias, int act, const float* residual, int64_t ldr, void* out, int64_t ldc, int out_dtype,
                void* stream, const float* rope_tab = nullptr, int rope_cols = 0, int rope_period = 0,
                const float* rowbias = nullptr, int rb_period = 1, int rb_first = 0, int rows_per_batch = 0,
                int64_t batch_stride_rows = 0, int n_peer_out = 0, void* const* peer_out = nullptr,
                const float* w_scale = nullptr) {
  m3r_gemm_args a = {};
  a.n_peer_out = n_peer_out;
  a.w_static = 1;                  // every GEMM of the model multiplies by checkpoint weights
  for (int i = 0; i < M3R_MAX_PEERS; ++i) a.peer_out[i] = i < n_peer_out ? peer_out[i] : nullptr;
  a.A = A; a.lda = lda; a.W = W; a.ldw = ldw; a.M = M; a.N = N; a.K = K; a.is_bf16 = is_bf16;
  a.bias = bias; a.act = act; a.residual = residual; a.ldr = ldr;
  a.rowbias = rowbias; a.rb_period = rb_period; a.rb_first = rb_first;
  a.rope_tab = rope_tab; a.rope_cols = rope_cols; a.rope_period = rope_period;
  a.out = out; a.ldc = ldc; a.out_dtype = out_dtype;
  a.rows_per_batch = rows_per_batch; a.batch_stride_rows = batch_stride_rows;
  if (!w_scale) return m3r_gemm(&a, stream);
  m3r_gemm_e4m3_args e8 = {};                // A and W are e4m3, W row n scaled by w_scale[n]
  e8.a_e4m3 = 1; e8.w_scale = w_scale;
  return m3r_gemm_e4m3(&a, &e8, stream);
}

// The affine-free LayerNorm of the rows feeding the next GEMM: e4m3 bytes when that GEMM takes e4m3 operands
static int normalize(bool e4m3, const float* x, const float* add, int add_rows, int add_period, float eps, int M, int D,
                     void* out, int bf, void* stream) {
  if (e4m3) return m3r_normalize8(x, D, add, D, add_rows, add_period, eps, M, D, out, D, stream);
  return m3r_normalize16(x, D, add, D, add_rows, add_period, eps, M, D, out, D, bf, stream);
}

struct EncWs { uint16_t *cols16, *h16, *qkv16, *att16, *mlp16; float *x, *rope; };

static int64_t enc_layout(const m3r_encoder_weights* w, int V, int H, int W, void* base, int64_t cap, EncWs* ws) {
  const int64_t N = (int64_t)(H / 16) * (W / 16), M = V * N, D = w->embed_dim;
  Arena a(base, cap);
  ws->rope = a.take<float>(N * 64);
  ws->cols16 = a.take<uint16_t>(M * 768);
  ws->x = a.take<float>(M * D);
  ws->h16 = a.take<uint16_t>(M * D);
  ws->qkv16 = a.take<uint16_t>(M * 3 * D);
  ws->att16 = a.take<uint16_t>(M * D);
  ws->mlp16 = a.take<uint16_t>(M * w->mlp_hidden);
  return a.off + 256;
}

}  // namespace m3r

using namespace m3r;

extern "C" int64_t m3r_encoder_workspace_bytes(const m3r_encoder_weights* w, int32_t V, int32_t H, int32_t W) {
  EncWs ws;
  return enc_layout(w, V, H, W, nullptr, 0, &ws);
}

namespace m3r {

// b8 != null: qkv and fc1 take e4m3 operands (their LayerNorms folded into the weights, the rows normalised to e4m3)
static int encoder_forward(const m3r_encoder_weights* w, const m3r_enc_block_e4m3* b8, const float* img, int32_t V, int32_t H,
                           int32_t W, const int64_t* pos, float* out_x, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!w || !img || !pos || !out_x || !workspace) return set_error("encoder_forward: null pointer");
  if (H % 16 || W % 16) return set_error("Input image size (%d,%d) is not a multiple of patch size 16", H, W);  // patch_embed.py:22-23
  if (w->embed_dim != w->num_heads * 64) return set_error("encoder_forward: head_dim must be 64");
  if (V <= 0) return 0;
  EncWs ws;
  const int64_t need = enc_layout(w, V, H, W, workspace, workspace_bytes, &ws);
  if (need > workspace_bytes) return set_error("encoder_forward: workspace too small (%lld < %lld)", (long long)workspace_bytes, (long long)need);
  const int N = (H / 16) * (W / 16), M = V * N, D = w->embed_dim, Hh = w->num_heads, bf = w->is_bf16;

  M3R_TRY(m3r_rope_table(pos, N, w->rope_base, w->rope_f0, ws.rope, stream));
  // patch embedding = im2col + GEMM (+bias) -> fp32 residual stream
  M3R_TRY(m3r_im2col16(img, V, H, W, ws.cols16, bf, stream));
  M3R_TRY(gemm(ws.cols16, 768, w->patch_w, 768, M, D, 768, bf, w->patch_b, 0, nullptr, 0, ws.x, D, M3R_OUT_F32, stream));
  for (int l = 0; l < w->depth; ++l) {
    const m3r_enc_block& b = w->blocks[l];
    if (b8) M3R_TRY(m3r_normalize8(ws.x, D, nullptr, 0, 0, 1, w->ln_eps, M, D, ws.h16, D, stream));
    else M3R_TRY(m3r_layernorm(ws.x, D, nullptr, 0, b.norm1_w, b.norm1_b, w->ln_eps, M, D, ws.h16, D, M3R_OUT_16, bf, stream));
    M3R_TRY(gemm(ws.h16, D, b.qkv_w, D, M, 3 * D, D, bf, b.qkv_b, 0, nullptr, 0, ws.qkv16, 3 * D, M3R_OUT_16, stream,
                 ws.rope, 2 * D, N, nullptr, 1, 0, 0, 0, 0, nullptr, b8 ? b8[l].qkv_s : nullptr));
    m3r_attn_args at = {};
    at.Q = ws.qkv16; at.ldq = 3 * D;
    at.K0 = ws.qkv16 + D; at.V0 = ws.qkv16 + 2 * D; at.ldk0 = 3 * D; at.kv_bstride0 = N; at.Nk0 = N;
    at.O = ws.att16; at.ldo = D; at.B = V; at.H = Hh; at.Nq = N; at.kv_group = 1; at.is_bf16 = bf; at.scale = 0.125f;
    M3R_TRY(m3r_attention(&at, stream));
    M3R_TRY(gemm(ws.att16, D, b.proj_w, D, M, D, D, bf, b.proj_b, 0, ws.x, D, ws.x, D, M3R_OUT_F32, stream));
    if (b8) M3R_TRY(m3r_normalize8(ws.x, D, nullptr, 0, 0, 1, w->ln_eps, M, D, ws.h16, D, stream));
    else M3R_TRY(m3r_layernorm(ws.x, D, nullptr, 0, b.norm2_w, b.norm2_b, w->ln_eps, M, D, ws.h16, D, M3R_OUT_16, bf, stream));
    M3R_TRY(gemm(ws.h16, D, b.fc1_w, D, M, w->mlp_hidden, D, bf, b.fc1_b, M3R_ACT_GELU, nullptr, 0, ws.mlp16,
                 w->mlp_hidden, M3R_OUT_16, stream, nullptr, 0, 0, nullptr, 1, 0, 0, 0, 0, nullptr, b8 ? b8[l].fc1_s : nullptr));
    M3R_TRY(gemm(ws.mlp16, w->mlp_hidden, b.fc2_w, w->mlp_hidden, M, D, w->mlp_hidden, bf, b.fc2_b, 0, ws.x, D, ws.x, D,
                 M3R_OUT_F32, stream));
  }
  M3R_TRY(m3r_layernorm(ws.x, D, nullptr, 0, w->norm_w, w->norm_b, w->ln_eps, M, D, out_x, D, M3R_OUT_F32, 0, stream));
  return 0;
}

}  // namespace m3r

extern "C" int m3r_encoder_forward(const m3r_encoder_weights* w, const float* img, int32_t V, int32_t H, int32_t W,
                                   const int64_t* pos, float* out_x, void* workspace, int64_t workspace_bytes,
                                   void* stream) {
  return encoder_forward(w, nullptr, img, V, H, W, pos, out_x, workspace, workspace_bytes, stream);
}

extern "C" int m3r_encoder_forward_e4m3(const m3r_encoder_weights* w, const m3r_enc_block_e4m3* blocks8, const float* img,
                                        int32_t V, int32_t H, int32_t W, const int64_t* pos, float* out_x, void* workspace,
                                        int64_t workspace_bytes, void* stream) {
  if (!blocks8) return set_error("encoder_forward_e4m3: null pointer");
  if (!w || !w->is_bf16) return set_error("encoder_forward_e4m3: the 16-bit operands of the e4m3 encoder are bf16 (is_bf16 = 1)");
  for (int l = 0; l < w->depth; ++l)
    if (!blocks8[l].qkv_s || !blocks8[l].fc1_s) return set_error("encoder_forward_e4m3: block %d has no weight scales", l);
  return encoder_forward(w, blocks8, img, V, H, W, pos, out_x, workspace, workspace_bytes, stream);
}

// ------------------------------------------------------------------------------------------------ decoder
namespace m3r {

// The side streams of caller stream `cs` (StreamState::side / copy and their events), created on its first update call.
// They belong to the caller's stream: host threads that drive the model on their own streams never wait on each other.
static StreamState* side_streams_of(cudaStream_t cs) {
  RegistryLock lock;
  StreamState* st = stream_state(cs, lock);
  if (!st) return set_error("decoder_forward: no current device"), nullptr;
  if (st->side) return st;                                      // created last: the set is complete
  cudaError_t e = st->copy ? cudaSuccess : cudaStreamCreateWithFlags(&st->copy, cudaStreamNonBlocking);
  for (int i = 0; i < 32 && e == cudaSuccess; ++i) if (!st->ev[i]) e = cudaEventCreateWithFlags(&st->ev[i], cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&st->side, cudaStreamNonBlocking);
  return e == cudaSuccess ? st : (set_error("decoder_forward: side stream creation failed: %s", cudaGetErrorString(e)), nullptr);
}
// make `to` wait for everything enqueued on `from` so far
static int link(StreamState* st, cudaStream_t from, cudaStream_t to) {
  cudaEvent_t e = st->ev[st->next_ev]; st->next_ev = (st->next_ev + 1) & 31;
  cudaError_t r = cudaEventRecord(e, from);
  if (r == cudaSuccess) r = cudaStreamWaitEvent(to, e, 0);
  return r == cudaSuccess ? 0 : set_error("decoder_forward: stream fork/join failed: %s", cudaGetErrorString(r));
}
// Joins whatever was forked onto the side / copy streams when the enclosing call returns early (an M3R_TRY error path):
// the caller's stream must never be left without a dependency on work that touches its buffers.
struct SideJoin {
  StreamState* sd = nullptr;
  cudaStream_t cs = nullptr;
  bool forked = false, copying = false, done = false;
  ~SideJoin() {
    if (done || !sd) return;
    if (forked) link(sd, sd->side, cs);
    if (copying) link(sd, sd->copy, cs);
  }
};

struct DecWs {
  uint16_t *enc16, *h16, *big16, *q16, *att16, *mlp16, *kvnew;
  uint16_t *hfb16, *mlpfb16, *hpost16;   // side stream: feedback MLP operands, normalised (new_mem[l] + offset) of every level
  uint16_t *kvmem, *memln;     // memory_mode norm_y / raw: K|V of the stored memory projected at use; LN_y of raw rows
  float *x, *tmp, *snap, *off, *rope, *headout;
  float *cp_o, *cp_ml;         // context parallel: this rank's exported attention state [M, D] + [M, H, 2], one contiguous block
  int64_t M, Nt;
  int nbm;                     // distinct memory batches behind kvmem (1 when the memory is a stride-0 expand)
  bool merged;                 // one scene, one aspect ratio: K|V of the new tokens live in big16 (no kvnew buffer)
  std::vector<int64_t> row0;   // first row of each group
  std::vector<int64_t> tok0;   // first new-token index (per scene) of each group
};

static int64_t dec_layout(const m3r_decoder_weights* w, const m3r_decoder_call* c, void* base, int64_t cap, DecWs* ws) {
  const int64_t D = w->embed_dim;
  int64_t M = 0, Nt = 0;
  ws->row0.assign(c->G, 0); ws->tok0.assign(c->G, 0);
  for (int g = 0; g < c->G; ++g) {
    ws->row0[g] = M; ws->tok0[g] = Nt;
    M += (int64_t)c->B * c->groups[g].n_views * c->groups[g].N;
    Nt += (int64_t)c->groups[g].n_views * c->groups[g].N;
  }
  ws->M = M; ws->Nt = Nt;
  ws->merged = !c->render && c->B == 1 && c->G == 1;
  Arena a(base, cap);
  ws->rope = a.take<float>(M * 64);
  ws->enc16 = a.take<uint16_t>(M * w->enc_dim);
  ws->x = a.take<float>(M * D);
  ws->tmp = a.take<float>(M * D);
  ws->h16 = a.take<uint16_t>(M * D);
  ws->big16 = a.take<uint16_t>(M * (ws->merged ? 5 : 3) * D);
  ws->q16 = a.take<uint16_t>(M * D);
  ws->att16 = a.take<uint16_t>(M * D);
  const int64_t hid = w->mlp_hidden > 4 * D ? w->mlp_hidden : 4 * D;
  ws->mlp16 = a.take<uint16_t>(M * hid);
  ws->headout = a.take<float>(M * w->out_dim);
  ws->snap = nullptr; ws->off = nullptr; ws->kvnew = nullptr; ws->hfb16 = ws->mlpfb16 = ws->hpost16 = nullptr;
  if (!c->render) {
    ws->snap = a.take<float>((int64_t)w->depth * M * D);
    ws->off = a.take<float>(M * D);
    if (!ws->merged) ws->kvnew = a.take<uint16_t>((int64_t)c->B * Nt * 2 * D);
    ws->hfb16 = a.take<uint16_t>(M * D);
    ws->mlpfb16 = a.take<uint16_t>(M * 4 * D);
    ws->hpost16 = a.take<uint16_t>((int64_t)w->depth * M * D);
  }
  ws->cp_o = ws->cp_ml = nullptr;
  if (c->cp_world > 1) {
    ws->cp_o = a.take<float>(M * D + M * (int64_t)w->num_heads * 2);
    ws->cp_ml = ws->cp_o + M * D;
  }
  ws->kvmem = ws->memln = nullptr; ws->nbm = 0;
  if (c->mem_mode != M3R_MEM_KV && c->Nm > 0) {
    ws->nbm = (c->B > 1 && c->mem_bstride_rows == 0) ? 1 : c->B;
    ws->kvmem = a.take<uint16_t>((int64_t)ws->nbm * c->Nm * 2 * D);
    if (c->mem_mode == M3R_MEM_RAW) ws->memln = a.take<uint16_t>((int64_t)ws->nbm * c->Nm * D);
  }
  return a.off + 256;
}

}  // namespace m3r

extern "C" int64_t m3r_decoder_cp_slot_bytes(const m3r_decoder_weights* w, int64_t M) {
  const int64_t b = M * (int64_t)w->embed_dim * 4 + M * (int64_t)w->num_heads * 8;
  return (b + 255) / 256 * 256;
}

extern "C" int64_t m3r_decoder_workspace_bytes(const m3r_decoder_weights* w, const m3r_decoder_call* c) {
  DecWs ws;
  return dec_layout(w, c, nullptr, 0, &ws);
}

namespace m3r {

// nm_scene != null: the ragged update of m3r_decoder_forward_ragged (checked there).  w8 != null: the GEMMs fed by an
// affine-free LayerNorm (a_w, q_w, fc1_w, fb1_w) take e4m3 operands, and the LayerNorms feeding them write e4m3 rows.
static int decoder_forward(const m3r_decoder_weights* w, const m3r_decoder_e4m3* w8, const m3r_decoder_call* c,
                           const int32_t* nm_scene, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!w || !c || !workspace || !c->groups) return set_error("decoder_forward: null pointer");
  if (c->B <= 0 || c->G <= 0) return set_error("decoder_forward: empty call");
  if (w->embed_dim != w->num_heads * 64) return set_error("decoder_forward: head_dim must be 64");
  if (c->render && c->Nm <= 0 && c->cp_world <= 1) return set_error("decoder_forward: render needs a memory (decoder.py:278)");
  if (c->Nm > 0 && !c->mem) return set_error("decoder_forward: memory pointers missing");
  const bool store_new = !c->render && !(c->cp_world > 1 && !c->cp_owner);     // context parallel: only the owner appends
  if (store_new && !c->mem_out) return set_error("decoder_forward: mem_out missing");
  if (c->n_peers < 0 || c->n_peers > M3R_MAX_PEERS || (c->n_peers > 0 && (!c->peer_mem || !c->new_only || c->B != 1)))
    return set_error("decoder_forward: peer output needs new_only, one scene and 1..%d peers", M3R_MAX_PEERS);
  if (c->mem_mode < M3R_MEM_KV || c->mem_mode > M3R_MEM_RAW) return set_error("decoder_forward: bad mem_mode %d", c->mem_mode);
  if (c->n_peers > 0 && c->mem_mode != M3R_MEM_KV) return set_error("decoder_forward: peer output needs mem_mode kv");
  const bool cp = c->cp_world > 1;
  if (cp) {
    if (c->cp_world > M3R_MAX_PEERS || c->cp_rank < 0 || c->cp_rank >= c->cp_world) return set_error("decoder_forward: context parallel over 2..%d ranks", M3R_MAX_PEERS);
    if (c->B != 1 || c->mem_mode != M3R_MEM_KV || c->n_peers > 0 || c->is_init) return set_error("decoder_forward: context parallel needs one scene, mem_mode kv, a continuation call and no peer output");
    if (!c->cp_stage || !c->cp_flag_slots || !c->cp_flags_local) return set_error("decoder_forward: context-parallel buffers missing");
  }
  DecWs ws;
  const int64_t need = dec_layout(w, c, workspace, workspace_bytes, &ws);
  if (need > workspace_bytes) return set_error("decoder_forward: workspace too small (%lld < %lld)", (long long)workspace_bytes, (long long)need);
  cudaStream_t cs = reinterpret_cast<cudaStream_t>(stream);
  const int D = w->embed_dim, Hh = w->num_heads, bf = w->is_bf16, B = c->B, G = c->G, Nm = c->Nm;
  const int depth = w->depth;
  const bool f8 = w8 != nullptr;
  const int64_t asz = f8 ? 1 : 2;                          // bytes per element of a_w
  auto a_kv = [&](const m3r_dec_block& b) { return reinterpret_cast<const uint8_t*>(b.a_w) + 3 * D * D * asz; };   // rows [3D, 5D)
  auto s_of = [&](int l, int which) -> const float* {      // per-row weight scales (null in 16-bit mode)
    if (!f8) return nullptr;
    const m3r_dec_block_e4m3& e = w8->blocks[l];
    return which == 0 ? e.a_s : which == 1 ? e.a_s + 3 * D : which == 2 ? e.q_s : e.fc1_s;
  };
  const int M = (int)ws.M;
  const int Nt = (int)ws.Nt;
  const int mode = c->mem_mode;
  const int mw = mode == M3R_MEM_KV ? 2 * D : D;         // width of a memory row (decoder.py:189,277)
  if (mode != M3R_MEM_KV) for (int l = 0; l < depth; ++l)
    if (!w->blocks[l].kv_w || !w->blocks[l].normy_w) return set_error("decoder_forward: memory_mode norm_y / raw needs the unfolded kv_w and the norm_y affine");
  int n_total = 0;
  for (int g = 0; g < G; ++g) n_total += c->groups[g].n_views;
  // make_mem_mask rule (decoder.py:199-204, 291-296): skip own tokens unless rendering or a lone first image
  // (context parallel: the scene's memory is non-empty even when this rank's shard is)
  const bool use_skip = !c->render && (Nm > 0 || n_total > 1 || cp);
  if (cp && c->cp_slot_bytes < m3r_decoder_cp_slot_bytes(w, M)) return set_error("decoder_forward: cp_slot_bytes too small");
  StreamState* sd = nullptr;
  if (store_new && !(sd = side_streams_of(cs))) return 1;
  SideJoin join_guard;
  join_guard.sd = sd; join_guard.cs = cs;
  if (store_new && Nm > 0 && !c->new_only) {
    // old memory rows -> output memory tensors (the reference's torch.cat, decoder.py:330) unless the caller appends in
    // place (mem_out[l] == mem[l]); independent of the whole step: copy stream, joined at the end
    cudaStream_t cps = sd->copy;
    bool linked = false;
    for (int l = 0; l < depth; ++l) {
      if (!c->mem_out[l]) return set_error("decoder_forward: mem_out[%d] is null", l);
      if (c->mem[l] == c->mem_out[l]) continue;
      if (!linked) { M3R_TRY(link(sd, cs, cps)); linked = true; join_guard.copying = true; }
      cudaError_t e = cudaSuccess;
      if (c->mem_bstride_rows == 0 && B > 1) {            // stride-0 (expanded) memory: one source block for every scene
        for (int bb = 0; bb < B && e == cudaSuccess; ++bb)
          e = cudaMemcpyAsync(reinterpret_cast<uint8_t*>(c->mem_out[l]) + (size_t)bb * c->mem_out_bstride_rows * mw * 2, c->mem[l],
                              (size_t)Nm * mw * 2, cudaMemcpyDeviceToDevice, cps);
      } else {
        e = cudaMemcpy2DAsync(c->mem_out[l], (size_t)c->mem_out_bstride_rows * mw * 2, c->mem[l],
                              (size_t)c->mem_bstride_rows * mw * 2, (size_t)Nm * mw * 2, B, cudaMemcpyDeviceToDevice, cps);
      }
      if (e != cudaSuccess) return set_error("decoder_forward: memory copy failed: %s", cudaGetErrorString(e));
    }
  }

  // LayerNorm placement: when the [M, D] residual stream fits in one wave of 128x64 tiles, every GEMM that produces it
  // also emits the normalised rows for its consumer (m3r_gemm_args.norm_out); otherwise a separate affine-free pass runs.
  const int tiles_m = (M + 127) / 128;
  const bool emit = D % 64 == 0 && D <= 768 && tiles_m <= 16 && tiles_m * (D / 64) <= num_sms();
  // residual-stream GEMM: xo = xr + A W^T + b, followed by (or fused with) the normalisation of xo into h16
  // norm8: the normalised rows feed an e4m3 GEMM
  auto res_gemm = [&](const void* A, int64_t lda, const void* W, int K, const float* bias, const float* xr, float* xo,
                      const float* rowbias, int rb_period, int rb_first, int Mrows, int64_t row_off, bool norm8) -> int {
    m3r_gemm_args a = {};
    a.A = A; a.lda = lda; a.W = W; a.ldw = K; a.M = Mrows; a.N = D; a.K = K; a.is_bf16 = bf; a.bias = bias;
    a.residual = xr ? xr + row_off * D : nullptr; a.ldr = D; a.out = xo + row_off * D; a.ldc = D; a.out_dtype = M3R_OUT_F32;
    a.rowbias = rowbias; a.rb_period = rb_period; a.rb_first = rb_first; a.w_static = 1;
    if (emit && Mrows == M) { a.norm_out = ws.h16; a.ldn = D; a.norm_eps = w->ln_eps; }
    m3r_gemm_e4m3_args e8 = {};
    e8.norm_e4m3 = norm8 && a.norm_out;
    M3R_TRY(m3r_gemm_e4m3(&a, &e8, stream));
    if (!(emit && Mrows == M) && row_off + Mrows == M)      // (grouped prologue: normalise once, after the last group)
      M3R_TRY(normalize(norm8, xo, nullptr, 0, 1, w->ln_eps, M, D, ws.h16, bf, stream));
    return 0;
  };

  // ---- prologue: projector + image2_embed, RoPE table (decoder.py:168-187, 272-289); X_0 -> snap[0] (update) or x (render)
  float* x0 = c->render ? ws.x : ws.snap;
  for (int g = 0; g < G; ++g) {
    const m3r_dec_group& gr = c->groups[g];
    const int Mg = B * gr.n_views * gr.N;
    if (gr.H % 16 || gr.W % 16 || (gr.H / 16) * (gr.W / 16) != gr.N) return set_error("decoder_forward: group %d: N=%d does not match true_shape (%d,%d)", g, gr.N, gr.H, gr.W);
    M3R_TRY(m3r_rope_table(gr.pos, Mg, w->rope_base, w->rope_f0, ws.rope + ws.row0[g] * 64, stream));
    M3R_TRY(m3r_cast16(gr.x_enc, w->enc_dim, Mg, w->enc_dim, ws.enc16 + ws.row0[g] * w->enc_dim, w->enc_dim, bf, stream));
    const int first = (c->is_init && g == 0) ? gr.N : 0;    // rows of view 0 of every scene get no embed at init
    M3R_TRY(res_gemm(ws.enc16 + ws.row0[g] * w->enc_dim, w->enc_dim, w->embed_w, w->enc_dim, w->embed_b, nullptr, x0,
                     w->image2_embed, gr.n_views * gr.N, first, Mg, ws.row0[g], f8));
  }

  // ---- feedback + memory append (feedback_mechanism.py:39-53, decoder.py:323-330), enqueued on stream `st` once
  // new_mem[depth-1] (the input of the last block) exists: offset = Mlp(LN_fb(new_mem[-1])); level l < depth-1 stores
  // K|V(LN_y(new_mem[l] + offset)), the last level K|V(LN_y(new_mem[-1])).
  auto append_memory = [&](void* st) -> int {
    const float* off = nullptr;
    if (w->feedback) {
      const float* last = ws.snap + (int64_t)(depth - 1) * M * D;
      const float* fb1_s = f8 ? w8->fb1_s : nullptr;
      M3R_TRY(normalize(f8, last, nullptr, 0, 1, w->fb_ln_eps, M, D, ws.hfb16, bf, st));
      if (w->feedback == 1) {
        M3R_TRY(gemm(ws.hfb16, D, w->fb1_w, D, M, 4 * D, D, bf, w->fb1_b, M3R_ACT_GELU, nullptr, 0, ws.mlpfb16, 4 * D, M3R_OUT_16, st,
                     nullptr, 0, 0, nullptr, 1, 0, 0, 0, 0, nullptr, fb1_s));
        M3R_TRY(gemm(ws.mlpfb16, 4 * D, w->fb2_w, 4 * D, M, D, 4 * D, bf, w->fb2_b, 0, nullptr, 0, ws.off, D, M3R_OUT_F32, st));
      } else {
        M3R_TRY(gemm(ws.hfb16, D, w->fb1_w, D, M, D, D, bf, w->fb1_b, 0, nullptr, 0, ws.off, D, M3R_OUT_F32, st,
                     nullptr, 0, 0, nullptr, 1, 0, 0, 0, 0, nullptr, fb1_s));
      }
      off = ws.off;
    }
    for (int l = 0; l < depth; ++l) if (!c->mem_out[l]) return set_error("decoder_forward: mem_out[%d] is null", l);
    if (mode != M3R_MEM_KV) {
      // norm_y stores LN_y(new_mem + off), raw stores new_mem + off (layers.py:81-86), D-wide rows
      for (int l = 0; l < depth; ++l) {
        const m3r_dec_block& b = w->blocks[l];
        uint16_t* mo = reinterpret_cast<uint16_t*>(c->mem_out[l]);
        const float* add = (off && l < depth - 1) ? off : nullptr;
        for (int g = 0; g < G; ++g) {
          const m3r_dec_group& gr = c->groups[g];
          const int rows = gr.n_views * gr.N;
          for (int bb = 0; bb < B; ++bb) {
            const int64_t in_row = ws.row0[g] + (int64_t)bb * rows;
            const float* xs = ws.snap + ((int64_t)l * M + in_row) * D;
            const float* as = add ? add + in_row * D : nullptr;
            uint16_t* dst = mo + ((int64_t)bb * c->mem_out_bstride_rows + (c->new_only ? 0 : Nm) + ws.tok0[g]) * D;
            if (mode == M3R_MEM_NORM_Y)
              M3R_TRY(m3r_layernorm(xs, D, as, D, b.normy_w, b.normy_b, w->ln_eps, rows, D, dst, D, M3R_OUT_16, bf, st));
            else
              M3R_TRY(m3r_add_cast16(xs, D, as, D, rows, D, dst, D, bf, st));
          }
        }
      }
      return 0;
    }
    // kv: ONE normalisation over the [depth * M] rows of all levels, then the K|V projections of all levels as one
    // grouped GEMM (weights = rows [3D,5D) of each block's stacked a_w) whose epilogue writes the stored rows - and, in the
    // multi-GPU schedule, every rank's copy of them - in place
    M3R_TRY(normalize(f8, ws.snap, off, (depth - 1) * M, M, w->ln_eps, depth * M, D, ws.hpost16, bf, st));
    bool stacked = depth <= M3R_MAX_GROUPS;
    for (int l = 1; l < depth && stacked; ++l)
      stacked = w->blocks[l].a_w == reinterpret_cast<const uint8_t*>(w->blocks[0].a_w) + (int64_t)l * 5 * D * D * asz &&
                w->blocks[l].a_b == w->blocks[0].a_b + (int64_t)l * 5 * D &&
                (!f8 || w8->blocks[l].a_s == w8->blocks[0].a_s + (int64_t)l * 5 * D);
    for (int g = 0; g < G; ++g) {
      const m3r_dec_group& gr = c->groups[g];
      const int Mg = B * gr.n_views * gr.N;
      m3r_gemm_args a = {};
      a.lda = D; a.ldw = D; a.M = Mg; a.N = 2 * D; a.K = D; a.is_bf16 = bf; a.ldc = 2 * D; a.out_dtype = M3R_OUT_16;
      a.rows_per_batch = gr.n_views * gr.N; a.batch_stride_rows = c->mem_out_bstride_rows; a.w_static = 1; a.n_peer_out = c->n_peers;
      m3r_gemm_e4m3_args e8 = {};
      e8.a_e4m3 = f8;
      const int64_t orow = (int64_t)(c->new_only ? 0 : Nm) + ws.tok0[g];
      if (stacked && G == 1) {
        m3r_gemm_group grp = {};
        grp.groups = depth; grp.w_group_rows = 5 * D; grp.bias_group = 5 * D;
        // next to the main chain (side stream): leave the SMs a LayerNorm-emitting GEMM needs (one wave of 128x64 tiles)
        const int left = num_sms() - tiles_m * (D / 64);
        grp.max_ctas = left > 32 ? left : 32;
        a.A = ws.hpost16; a.W = a_kv(w->blocks[0]); a.bias = w->blocks[0].a_b + 3 * D;
        e8.w_scale = s_of(0, 1);                            // indexed by the stacked W row, like W: group l at l * 5D
        for (int l = 0; l < depth; ++l) {
          grp.out[l] = reinterpret_cast<uint16_t*>(c->mem_out[l]) + orow * 2 * D;
          for (int r = 0; r < c->n_peers; ++r)
            grp.peer_out[l * M3R_MAX_PEERS + r] = reinterpret_cast<uint16_t*>(c->peer_mem[r * depth + l]) + ws.tok0[g] * 2 * D;
        }
        M3R_TRY(m3r_gemm_grouped_e4m3(&a, &grp, &e8, st));
      } else {
        for (int l = 0; l < depth; ++l) {
          const m3r_dec_block& b = w->blocks[l];
          a.A = reinterpret_cast<const uint8_t*>(ws.hpost16) + ((int64_t)l * M + ws.row0[g]) * D * (f8 ? 1 : 2);
          a.W = a_kv(b); a.bias = b.a_b + 3 * D;
          e8.w_scale = s_of(l, 1);
          a.out = reinterpret_cast<uint16_t*>(c->mem_out[l]) + orow * 2 * D;
          for (int r = 0; r < c->n_peers; ++r) a.peer_out[r] = reinterpret_cast<uint16_t*>(c->peer_mem[r * depth + l]) + ws.tok0[g] * 2 * D;
          M3R_TRY(m3r_gemm_e4m3(&a, &e8, st));
        }
      }
    }
    return 0;
  };
  bool appended = false;
  auto maybe_append = [&](int ready_level) -> int {      // called when X_{ready_level} has been enqueued
    if (!store_new || appended || ready_level != depth - 1) return 0;
    appended = true;
    M3R_TRY(link(sd, cs, sd->side));
    join_guard.forked = true;
    return append_memory(sd->side);
  };
  M3R_TRY(maybe_append(0));

  for (int l = 0; l < depth; ++l) {
    const m3r_dec_block& b = w->blocks[l];
    float* xin = c->render ? ws.x : ws.snap + (int64_t)l * M * D;                     // block input X_l (= new_mem[l], decoder.py:304)
    float* xout = c->render ? ws.x : (l + 1 < depth ? ws.snap + (int64_t)(l + 1) * M * D : ws.x);
    float* xt = c->render ? xin : ws.tmp;                                             // X_l must survive in update mode
    const int ldb = ws.merged ? 5 * D : 3 * D;
    // ---- h16 = n(X_l): first GEMM = self-attention q|k|v (RoPE on q,k) [+ pre-feedback K|V of the new tokens, the second
    // key segment of the cross-attention (decoder.py:306, layers.py:81-88)]
    M3R_TRY(gemm(ws.h16, D, b.a_w, D, M, ldb, D, bf, b.a_b, 0, nullptr, 0, ws.big16, ldb, M3R_OUT_16, stream, ws.rope, 2 * D, M,
                 nullptr, 1, 0, 0, 0, 0, nullptr, s_of(l, 0)));
    if (!c->render && !ws.merged) {
      for (int g = 0; g < G; ++g) {
        const m3r_dec_group& gr = c->groups[g];
        const int Mg = B * gr.n_views * gr.N;
        M3R_TRY(gemm(reinterpret_cast<const uint8_t*>(ws.h16) + ws.row0[g] * D * asz, D, a_kv(b), D, Mg, 2 * D, D, bf, b.a_b + 3 * D, 0,
                     nullptr, 0, ws.kvnew + ws.tok0[g] * 2 * D, 2 * D, M3R_OUT_16, stream, nullptr, 0, 0, nullptr, 1, 0,
                     gr.n_views * gr.N, Nt, 0, nullptr, s_of(l, 1)));
      }
    }
    if (mode != M3R_MEM_KV && Nm > 0) {
      // memory_mode norm_y / raw: K|V of the stored rows are projected at use (layers.py:92-96)
      for (int bm = 0; bm < ws.nbm; ++bm) {
        const uint16_t* src = reinterpret_cast<const uint16_t*>(c->mem[l]) + (int64_t)bm * c->mem_bstride_rows * D;
        if (mode == M3R_MEM_RAW) {
          uint16_t* ln = ws.memln + (int64_t)bm * Nm * D;
          M3R_TRY(m3r_layernorm16(src, D, b.normy_w, b.normy_b, w->ln_eps, Nm, D, ln, D, bf, stream));
          src = ln;
        }
        M3R_TRY(gemm(src, D, b.kv_w, D, Nm, 2 * D, D, bf, b.kv_b, 0, nullptr, 0, ws.kvmem + (int64_t)bm * Nm * 2 * D, 2 * D,
                     M3R_OUT_16, stream));
      }
    }
    // ---- self-attention (layers.py:91)
    for (int g = 0; g < G; ++g) {
      const m3r_dec_group& gr = c->groups[g];
      uint16_t* qkv = ws.big16 + ws.row0[g] * ldb;
      m3r_attn_args at = {};
      at.Q = qkv; at.ldq = ldb;
      at.K0 = qkv + D; at.V0 = qkv + 2 * D; at.ldk0 = ldb; at.kv_bstride0 = gr.N; at.Nk0 = gr.N;
      at.O = ws.att16 + ws.row0[g] * D; at.ldo = D; at.B = B * gr.n_views; at.H = Hh; at.Nq = gr.N; at.kv_group = 1;
      at.is_bf16 = bf; at.scale = 0.125f;
      M3R_TRY(m3r_attention(&at, stream));
    }
    // x_t = X_l + proj(SA), h16 = n(x_t)
    M3R_TRY(res_gemm(ws.att16, D, b.proj_w, D, b.proj_b, xin, xt, nullptr, 1, 0, M, 0, f8));
    // ---- memory cross-attention (layers.py:92-97, attention.py:139-149): q = projq(LN2(x)), K|V = memory (+ new)
    M3R_TRY(gemm(ws.h16, D, b.q_w, D, M, D, D, bf, b.q_b, 0, nullptr, 0, ws.q16, D, M3R_OUT_16, stream,
                 nullptr, 0, 0, nullptr, 1, 0, 0, 0, 0, nullptr, s_of(l, 2)));
    // context parallel: does this rank hold any key for this call?  (its memory shard, or - on rank 0 - the other views'
    // new tokens of a multi-view call)
    const bool cp_new_keys = cp && !c->render && c->cp_rank == 0 && n_total > 1;
    const bool cp_has_keys = Nm > 0 || cp_new_keys;
    if (cp && !cp_has_keys) M3R_TRY(m3r_attn_state_fill(ws.cp_o, ws.cp_ml, M, Hh, stream));
    for (int g = 0; g < G && (!cp || cp_has_keys); ++g) {
      const m3r_dec_group& gr = c->groups[g];
      m3r_attn_args at = {};
      at.Q = ws.q16 + ws.row0[g] * D; at.ldq = D;
      const uint16_t* mem_l = Nm > 0 ? reinterpret_cast<const uint16_t*>(c->mem[l]) : nullptr;
      const uint16_t* kn = ws.merged ? ws.big16 + 3 * D : ws.kvnew;       // this call's K|V rows
      const int64_t ldn = ws.merged ? 5 * D : 2 * D;
      if (cp) { at.export_o = ws.cp_o + ws.row0[g] * D; at.export_ml = ws.cp_ml + ws.row0[g] * Hh * 2; }
      if (Nm > 0) {
        if (mode == M3R_MEM_KV) {
          at.K0 = mem_l; at.V0 = mem_l + D; at.ldk0 = 2 * D; at.kv_bstride0 = c->mem_bstride_rows; at.Nk0 = Nm;
        } else {
          at.K0 = ws.kvmem; at.V0 = ws.kvmem + D; at.ldk0 = 2 * D; at.kv_bstride0 = ws.nbm > 1 ? Nm : 0; at.Nk0 = Nm;
        }
        if (!c->render && (!cp || cp_new_keys)) { at.K1 = kn; at.V1 = kn + D; at.ldk1 = ldn; at.kv_bstride1 = Nt; at.Nk1 = Nt; }
      } else {
        at.K0 = kn; at.V0 = kn + D; at.ldk0 = ldn; at.kv_bstride0 = Nt; at.Nk0 = Nt;   // first call: only new tokens
      }
      at.O = ws.att16 + ws.row0[g] * D; at.ldo = D; at.B = B * gr.n_views; at.H = Hh; at.Nq = gr.N;
      at.kv_group = gr.n_views; at.is_bf16 = bf; at.scale = 0.125f;
      if (use_skip && at.Nk0 + at.Nk1 > (Nm > 0 ? Nm : 0) ) { at.skip_lo = Nm + (int)ws.tok0[g]; at.skip_step = gr.N; at.skip_len = gr.N; }
      M3R_TRY(nm_scene ? m3r_attention_ragged(&at, nm_scene, stream) : m3r_attention(&at, stream));
    }
    if (cp) {
      // exchange: my state -> slot cp_rank of every rank's staging buffer (parity alternates so that a rank one layer ahead
      // never overwrites what a slower rank still merges), flag barrier, merge of the cp_world states into att16
      const int par = (int)((c->cp_epoch0 + (uint32_t)l) & 1u);
      const int64_t bytes = ((int64_t)M * D * 4 + (int64_t)M * Hh * 8 + 15) / 16 * 16;
      void* dsts[M3R_MAX_PEERS];
      for (int q = 0; q < c->cp_world; ++q)
        dsts[q] = reinterpret_cast<uint8_t*>(c->cp_stage[q]) + (int64_t)(par * c->cp_world + c->cp_rank) * c->cp_slot_bytes;
      M3R_TRY(m3r_peer_bcast(ws.cp_o, dsts, c->cp_world, bytes, stream));
      const uint32_t epoch = c->cp_epoch0 + (uint32_t)l + 1u;
      M3R_TRY(m3r_peer_signal(c->cp_flag_slots, c->cp_world, epoch, stream));
      M3R_TRY(m3r_peer_wait(c->cp_flags_local, (1u << c->cp_world) - 1u, epoch, stream));
      const float* po[M3R_MAX_PEERS]; const float* pml[M3R_MAX_PEERS];
      for (int q = 0; q < c->cp_world; ++q) {
        po[q] = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(c->cp_stage[c->cp_rank]) + (int64_t)(par * c->cp_world + q) * c->cp_slot_bytes);
        pml[q] = po[q] + (int64_t)M * D;
      }
      M3R_TRY(m3r_attn_merge(po, pml, c->cp_world, M, Hh, ws.att16, D, bf, stream));
    }
    M3R_TRY(res_gemm(ws.att16, D, b.cproj_w, D, b.cproj_b, xt, xt, nullptr, 1, 0, M, 0, f8));
    // ---- MLP (layers.py:98)
    M3R_TRY(gemm(ws.h16, D, b.fc1_w, D, M, w->mlp_hidden, D, bf, b.fc1_b, M3R_ACT_GELU, nullptr, 0, ws.mlp16, w->mlp_hidden,
                 M3R_OUT_16, stream, nullptr, 0, 0, nullptr, 1, 0, 0, 0, 0, nullptr, s_of(l, 3)));
    // (the last block's LayerNorm feeds the 16-bit head)
    M3R_TRY(res_gemm(ws.mlp16, w->mlp_hidden, b.fc2_w, w->mlp_hidden, b.fc2_b, xt, xout, nullptr, 1, 0, M, 0, f8 && l + 1 < depth));
    M3R_TRY(maybe_append(l + 1));
  }

  // ---- prediction head (decoder.py:149-156, head.py:69-72): LN (emitted by the last fc2) -> Linear(768->1792) fp32 -> pixel shuffle
  M3R_TRY(gemm(ws.h16, D, w->head_w, D, M, w->out_dim, D, bf, w->head_b, 0, nullptr, 0, ws.headout, w->out_dim, M3R_OUT_F32, stream));
  for (int g = 0; g < G; ++g) {
    const m3r_dec_group& gr = c->groups[g];
    M3R_TRY(m3r_unpatchify(ws.headout + ws.row0[g] * w->out_dim, B * gr.n_views, gr.H, gr.W, w->out_dim / 256, gr.pointmaps, stream));
  }

  if (store_new) {
    M3R_TRY(link(sd, sd->side, cs));                                // join the side stream
    if (Nm > 0 && !c->new_only) M3R_TRY(link(sd, sd->copy, cs));    // and the old-memory copies
  }
  join_guard.done = true;
  return 0;
}

struct CommitArgs {
  uint4* dst[M3R_MAX_GROUPS];
  const uint4* src[M3R_MAX_GROUPS];
  long long dst_row[M3R_MAX_COMMIT];
};

// grid (chunks, B, depth): level blockIdx.z of scene blockIdx.y, if its flag is set; rows * width / 8 uint4 per scene,
// read from scene b's staged block (src_stride rows apart; a.src already points at the first row copied)
__global__ void mem_commit_kernel(const __grid_constant__ CommitArgs a, const int* keep, long long keep_stride, int Nt, int w16,
                                  long long src_stride) {
  griddep_wait();
  const int b = blockIdx.y, l = blockIdx.z;
  if (keep[(long long)b * keep_stride] == 0) return;
  const long long n = (long long)Nt * w16;
  const uint4* src = a.src[l] + (long long)b * src_stride * w16;
  uint4* dst = a.dst[l] + a.dst_row[b] * w16;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i];
}

// grid (chunks, F, depth): frame blockIdx.y of a step whose frames share one memory, if its flag is set, goes behind the
// kept frames before it: row row0 + Nt * (flags set among frames < blockIdx.y).  The flags are read here, after the
// dependency wait, so the records written by the preceding keyframe kernels need no trip through the host.
__global__ void mem_commit_ordered_kernel(const __grid_constant__ CommitArgs a, const int* keep, long long keep_stride,
                                          int Nt, int w16, long long row0) {
  griddep_wait();
  const int k = blockIdx.y, l = blockIdx.z;
  if (keep[(long long)k * keep_stride] == 0) return;
  int before = 0;
  for (int j = 0; j < k; ++j) before += keep[(long long)j * keep_stride] != 0;
  const long long n = (long long)Nt * w16;
  const uint4* src = a.src[l] + (long long)k * n;
  uint4* dst = a.dst[l] + (row0 + (long long)before * Nt) * w16;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i];
}

struct CompactArgs {
  uint4* buf[M3R_MAX_GROUPS];
  long long base[M3R_MAX_COMMIT];
  int run0[M3R_MAX_COMMIT + 1];
  int3 runs[M3R_MAX_COMPACT_RUNS];      // (src_row, dst_row, rows) relative to the scene's base row
};

constexpr int COMPACT_COLS = 8;         // uint4 columns per CTA (128 bytes of a row)
constexpr int COMPACT_LANES = 32;       // rows in flight per unrolled slot
constexpr int COMPACT_UNROLL = 8;       // -> up to 256 rows moved per iteration

// grid (column chunks, B, depth), COMPACT_COLS * COMPACT_LANES threads: columns [8 * blockIdx.x, + 8) of level blockIdx.z
// of scene blockIdx.y, every run in order.  A CTA owns its columns for all rows, so the only hazard is inside the CTA:
// each iteration moves m <= shift = src - dst destination rows, whose sources lie at or past the iteration's last
// destination row (no read of the iteration meets one of its writes), and the barrier keeps the next iteration's writes
// (which may land on rows this one read) behind this iteration's reads.  Every row moves once, no scratch.
__global__ void __launch_bounds__(COMPACT_COLS * COMPACT_LANES) mem_compact_kernel(const __grid_constant__ CompactArgs a, int w16) {
  griddep_wait();
  const int b = blockIdx.y, l = blockIdx.z;
  const int col = blockIdx.x * COMPACT_COLS + (threadIdx.x % COMPACT_COLS), lane = threadIdx.x / COMPACT_COLS;
  const bool on = col < w16;
  uint4* buf = a.buf[l] + a.base[b] * w16 + col;
  for (int k = a.run0[b]; k < a.run0[b + 1]; ++k) {
    const int src = a.runs[k].x, dst = a.runs[k].y, n = a.runs[k].z;
    const int shift = src - dst;
    if (shift == 0) continue;
    const int step = min(shift, COMPACT_LANES * COMPACT_UNROLL);
    for (int r0 = 0; r0 < n; r0 += step) {
      const int m = min(step, n - r0);
      uint4 v[COMPACT_UNROLL];
#pragma unroll
      for (int u = 0; u < COMPACT_UNROLL; ++u) {
        const int r = lane + u * COMPACT_LANES;
        if (on && r < m) v[u] = buf[(long long)(src + r0 + r) * w16];
      }
#pragma unroll
      for (int u = 0; u < COMPACT_UNROLL; ++u) {
        const int r = lane + u * COMPACT_LANES;
        if (on && r < m) buf[(long long)(dst + r0 + r) * w16] = v[u];
      }
      __syncthreads();
    }
  }
}

}  // namespace m3r

extern "C" int m3r_decoder_forward(const m3r_decoder_weights* w, const m3r_decoder_call* c, void* workspace,
                                   int64_t workspace_bytes, void* stream) {
  return decoder_forward(w, nullptr, c, nullptr, workspace, workspace_bytes, stream);
}

static int check_ragged(const m3r_decoder_call* c, const int32_t* nm_scene) {
  if (!c || !nm_scene) return set_error("decoder_forward_ragged: null pointer");
  if (c->mem_mode != M3R_MEM_KV || !c->new_only || c->render || c->n_peers != 0 || c->cp_world > 1)
    return set_error("decoder_forward_ragged: only memory_mode kv with new_only (no render, peers or context parallel)");
  if (c->Nm < 1 || c->is_init) return set_error("decoder_forward_ragged: needs a memory (Nm = the longest, >= 1)");
  return 0;
}

extern "C" int m3r_decoder_forward_ragged(const m3r_decoder_weights* w, const m3r_decoder_call* c, const int32_t* nm_scene,
                                          void* workspace, int64_t workspace_bytes, void* stream) {
  if (check_ragged(c, nm_scene)) return 1;
  return decoder_forward(w, nullptr, c, nm_scene, workspace, workspace_bytes, stream);
}

static int check_e4m3(const m3r_decoder_weights* w, const m3r_decoder_e4m3* w8) {
  if (!w || !w8 || !w8->blocks) return set_error("decoder_forward_e4m3: null pointer");
  if (!w->is_bf16) return set_error("decoder_forward_e4m3: the 16-bit operands of the e4m3 decoder are bf16 (is_bf16 = 1)");
  for (int l = 0; l < w->depth; ++l)
    if (!w8->blocks[l].a_s || !w8->blocks[l].q_s || !w8->blocks[l].fc1_s) return set_error("decoder_forward_e4m3: block %d has no weight scales", l);
  if (w->feedback && !w8->fb1_s) return set_error("decoder_forward_e4m3: feedback weights have no scales");
  return 0;
}

extern "C" int m3r_decoder_forward_e4m3(const m3r_decoder_weights* w, const m3r_decoder_e4m3* w8, const m3r_decoder_call* c,
                                        const int32_t* nm_scene, void* workspace, int64_t workspace_bytes, void* stream) {
  if (check_e4m3(w, w8)) return 1;
  if (nm_scene && check_ragged(c, nm_scene)) return 1;
  return decoder_forward(w, w8, c, nm_scene, workspace, workspace_bytes, stream);
}

extern "C" int m3r_decoder_render_ragged(const m3r_decoder_weights* w, const m3r_decoder_e4m3* w8, const m3r_decoder_call* c,
                                         const int32_t* nm_scene, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!c || !nm_scene) return set_error("decoder_render_ragged: null pointer");
  if (!c->render || c->mem_mode != M3R_MEM_KV || c->n_peers != 0 || c->cp_world > 1 || c->is_init)
    return set_error("decoder_render_ragged: only a render call (render = 1, is_init = 0) with memory_mode kv, no peers and no context parallel");
  if (c->Nm < 1) return set_error("decoder_render_ragged: needs a memory (Nm = the longest, >= 1)");
  if (w8 && check_e4m3(w, w8)) return 1;
  return decoder_forward(w, w8, c, nm_scene, workspace, workspace_bytes, stream);
}

static int mem_commit(void* const* arena, const void* const* staged, int32_t depth, int32_t B, int32_t row0, int32_t Nt,
                      int32_t src_stride, int32_t width, const int64_t* dst_row, const int32_t* keep, int64_t keep_stride,
                      void* stream) {
  if (!arena || !staged || !dst_row || !keep) return set_error("mem_commit: null pointer");
  if (B < 0 || B > M3R_MAX_COMMIT || depth < 1 || depth > M3R_MAX_GROUPS || Nt < 0 || width < 8 || width % 8)
    return set_error("mem_commit: B in [0, %d], depth in [1, %d], Nt >= 0 and width a positive multiple of 8", M3R_MAX_COMMIT, M3R_MAX_GROUPS);
  if (row0 < 0 || (int64_t)row0 + Nt > src_stride) return set_error("mem_commit: rows [%d, %d) outside a staged block of %d rows", row0, row0 + Nt, src_stride);
  if (reinterpret_cast<uintptr_t>(keep) % 4) return set_error("mem_commit: keep must be 4-byte aligned");
  CommitArgs a = {};
  for (int l = 0; l < depth; ++l) {
    if (!arena[l] || !staged[l] || reinterpret_cast<uintptr_t>(arena[l]) % 16 || reinterpret_cast<uintptr_t>(staged[l]) % 16)
      return set_error("mem_commit: arena[%d] / staged[%d] null or not 16-byte aligned", l, l);
    a.dst[l] = reinterpret_cast<uint4*>(arena[l]);
    a.src[l] = reinterpret_cast<const uint4*>(staged[l]) + (int64_t)row0 * (width / 8);
  }
  for (int b = 0; b < B; ++b) {
    if (dst_row[b] < 0) return set_error("mem_commit: dst_row[%d] < 0", b);
    a.dst_row[b] = dst_row[b];
  }
  if (B == 0 || Nt == 0) return 0;
  const int w16 = width / 8;
  const long long n = (long long)Nt * w16;
  const int threads = 256;
  const int chunks = (int)std::min<long long>((n + threads - 1) / threads, 64);
  cudaError_t e = launch_pdl(mem_commit_kernel, dim3(chunks, B, depth), dim3(threads), 0, reinterpret_cast<cudaStream_t>(stream),
                             a, keep, (long long)keep_stride, (int)Nt, w16, (long long)src_stride);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("mem_commit launch: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

extern "C" int m3r_mem_commit(void* const* arena, const void* const* staged, int32_t depth, int32_t B, int32_t Nt, int32_t width,
                              const int64_t* dst_row, const int32_t* keep, int64_t keep_stride, void* stream) {
  return mem_commit(arena, staged, depth, B, 0, Nt, Nt, width, dst_row, keep, keep_stride, stream);
}

extern "C" int m3r_mem_commit_rows(void* const* arena, const void* const* staged, int32_t depth, int32_t B, int32_t row0,
                                   int32_t rows, int32_t src_stride_rows, int32_t width, const int64_t* dst_row,
                                   const int32_t* keep, int64_t keep_stride, void* stream) {
  return mem_commit(arena, staged, depth, B, row0, rows, src_stride_rows, width, dst_row, keep, keep_stride, stream);
}

extern "C" int m3r_mem_commit_ordered(void* const* arena, const void* const* staged, int32_t depth, int32_t F, int32_t Nt,
                                      int32_t width, int64_t row0, const int32_t* keep, int64_t keep_stride, void* stream) {
  using namespace m3r;
  if (!arena || !staged || !keep) return set_error("mem_commit_ordered: null pointer");
  if (F < 0 || F > M3R_MAX_COMMIT || depth < 1 || depth > M3R_MAX_GROUPS || Nt < 0 || width < 8 || width % 8 || row0 < 0)
    return set_error("mem_commit_ordered: F in [0, %d], depth in [1, %d], Nt >= 0, row0 >= 0 and width a positive multiple of 8",
                     M3R_MAX_COMMIT, M3R_MAX_GROUPS);
  if (reinterpret_cast<uintptr_t>(keep) % 4) return set_error("mem_commit_ordered: keep must be 4-byte aligned");
  CommitArgs a = {};
  for (int l = 0; l < depth; ++l) {
    if (!arena[l] || !staged[l] || reinterpret_cast<uintptr_t>(arena[l]) % 16 || reinterpret_cast<uintptr_t>(staged[l]) % 16)
      return set_error("mem_commit_ordered: arena[%d] / staged[%d] null or not 16-byte aligned", l, l);
    a.dst[l] = reinterpret_cast<uint4*>(arena[l]);
    a.src[l] = reinterpret_cast<const uint4*>(staged[l]);
  }
  if (F == 0 || Nt == 0) return 0;
  const int w16 = width / 8;
  const long long n = (long long)Nt * w16;
  const int threads = 256;
  const int chunks = (int)std::min<long long>((n + threads - 1) / threads, 64);
  cudaError_t e = launch_pdl(mem_commit_ordered_kernel, dim3(chunks, F, depth), dim3(threads), 0,
                             reinterpret_cast<cudaStream_t>(stream), a, keep, (long long)keep_stride, (int)Nt, w16, (long long)row0);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("mem_commit_ordered launch: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

extern "C" int m3r_mem_compact_rows(void* const* arena, int32_t depth, int32_t B, int32_t width, int64_t cap,
                                    const int64_t* base_row, const int32_t* run_offset, const int32_t* runs, void* stream) {
  if (!arena || !base_row || !run_offset || !runs) return set_error("mem_compact_rows: null pointer");
  if (B < 0 || B > M3R_MAX_COMMIT || depth < 1 || depth > M3R_MAX_GROUPS || width < 8 || width % 8 || cap < 1)
    return set_error("mem_compact_rows: B in [0, %d], depth in [1, %d], width a positive multiple of 8 and cap >= 1",
                     M3R_MAX_COMMIT, M3R_MAX_GROUPS);
  CompactArgs a = {};
  for (int l = 0; l < depth; ++l) {
    if (!arena[l] || reinterpret_cast<uintptr_t>(arena[l]) % 16)
      return set_error("mem_compact_rows: arena[%d] null or not 16-byte aligned", l);
    a.buf[l] = reinterpret_cast<uint4*>(arena[l]);
  }
  if (run_offset[0] != 0) return set_error("mem_compact_rows: run_offset[0] = %d, not 0", run_offset[0]);
  for (int b = 0; b < B; ++b) {
    if (run_offset[b + 1] < run_offset[b] || run_offset[b + 1] > M3R_MAX_COMPACT_RUNS)
      return set_error("mem_compact_rows: run_offset must be non-decreasing and end at most at %d", M3R_MAX_COMPACT_RUNS);
    if (base_row[b] < 0 || (b > 0 && base_row[b] < base_row[b - 1] + cap))
      return set_error("mem_compact_rows: base_row[%d] = %lld: base rows must be >= 0, ascending and cap apart", b,
                       (long long)base_row[b]);
    a.base[b] = base_row[b];
    a.run0[b] = run_offset[b];
    for (int k = run_offset[b]; k < run_offset[b + 1]; ++k) {
      const int32_t src = runs[3 * k], dst = runs[3 * k + 1], n = runs[3 * k + 2];
      if (n < 0 || dst < 0 || dst > src || (int64_t)src + n > cap)
        return set_error("mem_compact_rows: scene %d run %d (src %d, dst %d, rows %d) needs 0 <= dst_row <= src_row and "
                         "src_row + rows <= cap (%lld)", b, k - run_offset[b], src, dst, n, (long long)cap);
      if (k > run_offset[b] && (src < runs[3 * k - 3] + runs[3 * k - 1] || dst < runs[3 * k - 2] + runs[3 * k - 1]))
        return set_error("mem_compact_rows: scene %d run %d out of order (runs ascending, each at or past the previous "
                         "run's end)", b, k - run_offset[b]);
      a.runs[k] = make_int3(src, dst, n);
    }
  }
  a.run0[B] = run_offset[B];
  if (B == 0 || run_offset[B] == 0) return 0;
  const int w16 = width / 8;
  const int chunks = (w16 + COMPACT_COLS - 1) / COMPACT_COLS;
  cudaError_t e = launch_pdl(mem_compact_kernel, dim3(chunks, B, depth), dim3(COMPACT_COLS * COMPACT_LANES), 0,
                             reinterpret_cast<cudaStream_t>(stream), a, w16);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("mem_compact_rows launch: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}
