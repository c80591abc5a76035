/*
 * must3r_b200 — C ABI of the H100-native MUSt3R inference hot path (libm3r_b200.so).
 *
 * Plain pointers and sizes only (no torch types).  All pointers are DEVICE pointers unless noted;
 * buffers are borrowed for the duration of the call; work is enqueued on `stream` (the caller's current
 * CUDA stream, as a cudaStream_t cast to void*).  Every entry point returns 0 on success or a non-zero
 * code; m3r_last_error() returns a human-readable message for the calling thread's last failure.
 *
 * Each function names the reference interface it replaces (paths relative to the reference repo).
 * 16-bit operands are fp16 (is_bf16 = 0) or bf16 (is_bf16 = 1); accumulation, LayerNorm, softmax and the
 * residual stream are fp32.  The *_e4m3 entry points add float8 e4m3 operands for the GEMMs whose A operand is an
 * affine-free LayerNorm output (the other operands stay bf16); they leave every existing struct and entry point as it was.
 */
#ifndef MUST3R_B200_H
#define MUST3R_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define M3R_ABI_VERSION 4
#define M3R_MAX_PEERS 8
#define M3R_MAX_GROUPS 16

/* m3r_decoder_call.mem_mode (MEMORY_MODES, must3r/model/blocks/layers.py:9) */
#define M3R_MEM_KV 0
#define M3R_MEM_NORM_Y 1
#define M3R_MEM_RAW 2
/* out_dtype */
#define M3R_OUT_F32 0
#define M3R_OUT_16 1
#define M3R_OUT_E4M3 2   /* float8 e4m3 bytes (round to nearest even; finite values beyond +-448 saturate to +-448) */
/* activation */
#define M3R_ACT_NONE 0
#define M3R_ACT_GELU 1

const char* m3r_last_error(void);
int m3r_abi_version(void);
/* Number of kernels this library has launched in this process (bench.py reports it as gpu_launches). */
long long m3r_launch_count(void);
/* Optional per-kernel device timing for bench.py: CUDA events are recorded on the launch stream around every
 * GEMM / attention / LayerNorm kernel while enabled.  m3r_prof_read synchronises and fills
 * out[cat*4 + {0: ms, 1: launches, 2: algorithmic flops, 3: algorithmic bytes}] for the 7 categories
 * gemm_kernel<256>, gemm_kernel<128>, gemm_kernel<64>, attn_kernel<QT=2>, attn_kernel<QT=1> (key splits merged in-kernel), layernorm,
 * other (28 doubles). */
void m3r_prof_enable(int on);
int m3r_prof_read(double* out);
/* Debug hook (tools/trace_attn.py, tools/trace_gemm.py): device buffer that subsequent attention / GEMM launches fill
 * with %globaltimer stamps (64 / 16 uint64 per CTA: entry, barrier waits, epilogue, exit); NULL = off.  Only builds made
 * with M3R_TRACE=1 carry the stamps; otherwise the call fails with an error. */
int m3r_debug_trace(void* buf);

/* ---------------------------------------------------------------------------------------------------
 * Linear layer y = act(x W^T + b) (+ residual) on wgmma tensor cores.
 * Replaces nn.Linear / croco Mlp call sites: must3r/model/blocks/attention.py:88-89,108-111,
 * dust3r/croco/models/blocks.py:67-70, must3r/model/decoder.py:50, must3r/model/blocks/head.py:67,
 * and, with rope_tab != NULL, the fused qkv projection + curope.rope_2d
 * (dust3r/croco/models/curope/curope.cpp:49) of Attention.forward (attention.py:92-96).
 * ------------------------------------------------------------------------------------------------- */
typedef struct {
  const void* A;          /* [M,K] 16-bit, row-major, leading dim lda (elements) */
  int64_t lda;
  const void* W;          /* [N,K] 16-bit, row-major (nn.Linear.weight layout), leading dim ldw */
  int64_t ldw;
  int32_t M, N, K;        /* N % 64 == 0, K % 64 == 0 */
  int32_t is_bf16;
  const float* bias;      /* [N] fp32 or NULL */
  int32_t act;            /* M3R_ACT_* (applied after bias/rope, before residual) */
  const float* residual;  /* [M,N] fp32 (leading dim ldr) added after the activation, or NULL */
  int64_t ldr;
  const float* rowbias;   /* [N] fp32 added to rows with (row % rb_period) >= rb_first, or NULL
                             (image2_embed, must3r/model/decoder.py:282,287) */
  int32_t rb_period, rb_first;
  const float* rope_tab;  /* [rope_period,64] fp32 = per token (cosY[16], sinY[16], cosX[16], sinX[16]);
                             rotates columns < rope_cols in 64-wide heads; or NULL */
  int32_t rope_cols, rope_period;
  void* out;              /* [M,N] fp32 or 16-bit, leading dim ldc (elements) */
  int64_t ldc;
  int32_t out_dtype;      /* M3R_OUT_* */
  int32_t rows_per_batch; /* output row remap for appending into [B,cap,N] buffers:              */
  int64_t batch_stride_rows; /* out_row = (row / rows_per_batch) * batch_stride_rows + row % rows_per_batch;
                                rows_per_batch <= 0 disables the remap */
  /* Fused "GEMM -> all-gather": when n_peer_out > 0 the 16-bit output tile is ALSO stored, with the same row mapping
   * and ldc, to these device pointers - the same buffer in the other GPUs of the NVSwitch domain, mapped into this
   * process with m3r_ipc_open (peer stores travel over NVLink while the kernel is still computing other tiles). */
  int32_t n_peer_out;
  void* peer_out[M3R_MAX_PEERS];
  /* 1 = W is not written by the launch that precedes this one in the stream (model weights): the kernel then requests
   * its first weight tiles before the programmatic-dependency wait, hiding their HBM latency behind the predecessor's
   * tail.  0 = no assumption. */
  int32_t w_static;
  /* LayerNorm fused into the PRODUCING GEMM (must3r/model/blocks/layers.py:42,46,65,70,71,76 call sites): when norm_out
   * != NULL the output must be the fp32 residual stream x [M,N] with N = the model width (N % 64 == 0, N <= 768) and the
   * epilogue also writes normalised rows (x - mean) * rsqrt(var + norm_eps) as 16-bit to norm_out (leading dim ldn): the
   * A operand of the next GEMM, whose weight / bias carry the LayerNorm affine (W * diag(gamma), b + W beta).  The CTAs
   * holding the column tiles of one 128-row block exchange per-row (mean, M2) partials through device memory and meet
   * at a device-scope counter, so the whole problem must fit in one wave (ceil(M/128) * N/64 <= SM count) and such
   * launches must not run concurrently on two streams of one device.  norm_out rows are not remapped, so norm_out
   * cannot be combined with rows_per_batch > 0 (an argument error).
   * Base pointers: bias, rowbias, rope_tab and residual 8-byte aligned; out, peer_out and norm_out 16-byte aligned. */
  void* norm_out;
  int64_t ldn;
  float norm_eps;
} m3r_gemm_args;

int m3r_gemm(const m3r_gemm_args* args, void* stream);

/* e4m3 options of a GEMM (m3r_gemm_e4m3 / m3r_gemm_grouped_e4m3; a NULL pointer = m3r_gemm / m3r_gemm_grouped):
 * a_e4m3 = 1: A [M,K] and W [N,K] are float8 e4m3 (1 byte per element; lda / ldw multiples of 16, K % 128 == 0, N % 64 ==
 *   0), is_bf16 must be 1 (16-bit outputs are bf16), and accumulator column n is multiplied by w_scale[n] before bias,
 *   RoPE, GELU, residual, norm_out and the stores (grouped form: w_scale is indexed by the row of the stacked W, like W).
 *   w_scale is required (8-byte aligned).  W = round_e4m3(W_true / w_scale) row by row.  Not combinable with norm_out
 *   (the GEMMs that emit a LayerNorm have unbounded 16-bit A operands).
 * norm_e4m3 = 1: norm_out rows are written as e4m3 (ldn in bytes, a multiple of 16; M3R_OUT_E4M3).  The normalised row
 *   (x - mean) * rstd of D values has |y| <= sqrt(D - 1) (<= 32 for D <= 1025), far inside e4m3's range, so no scale
 *   is needed for it. */
typedef struct {
  int32_t a_e4m3;
  const float* w_scale;
  int32_t norm_e4m3;
} m3r_gemm_e4m3_args;

int m3r_gemm_e4m3(const m3r_gemm_args* args, const m3r_gemm_e4m3_args* e8, void* stream);

/* Grouped form: `groups` problems of identical shape [args->M, args->N, args->K] in one launch.  A = [groups*M, K]
 * (group g = rows [g*M, (g+1)*M)), W rows [g*w_group_rows, +N), bias + g*bias_group; args->out / peer_out are ignored,
 * group g writes out[g] (and peer_out[g*M3R_MAX_PEERS + r], r < args->n_peer_out) with args' ldc / row remap.
 * Replaces the per-level K|V projections of the memory append (must3r/model/decoder.py:323-330). */
typedef struct {
  int32_t groups;
  int64_t w_group_rows;
  int64_t bias_group;
  void* out[M3R_MAX_GROUPS];
  void* peer_out[M3R_MAX_GROUPS * M3R_MAX_PEERS];
  int32_t max_ctas;           /* > 0: run on at most this many SMs (persistent tile loop).  The memory append runs on a side
                                 stream next to the last decoder block; its CTAs (slow when they store over NVLink) must not
                                 take the SMs the LayerNorm-emitting GEMMs of the main chain need to be co-resident */
} m3r_gemm_group;

int m3r_gemm_grouped(const m3r_gemm_args* args, const m3r_gemm_group* grp, void* stream);
int m3r_gemm_grouped_e4m3(const m3r_gemm_args* args, const m3r_gemm_group* grp, const m3r_gemm_e4m3_args* e8, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * LayerNorm over the last dim of fp32 rows (optionally of x + add), output 16-bit (GEMM operand) or fp32.
 * Replaces nn.LayerNorm call sites: must3r/model/blocks/layers.py:42,46,65,70,71,76, encoder.py:37,
 * decoder.py:76, feedback_mechanism.py:14 (eps 1e-5), and the `new_mem[l] + offset` add of
 * feedback_mechanism.py:49-51 when add != NULL.
 * ------------------------------------------------------------------------------------------------- */
int m3r_layernorm(const float* x, int64_t ldx, const float* add, int64_t ldadd, const float* gamma,
                  const float* beta, float eps, int32_t M, int32_t D, void* out, int64_t ldo, int32_t out_dtype,
                  int32_t is_bf16, void* stream);

/* Affine-free LayerNorm: out16 = ((x [+ add]) - mean) * rsqrt(var + eps) as 16-bit rows = the A operand of a GEMM whose
 * weights carry the LayerNorm affine (W * diag(gamma), b + W beta).  `add` (may be NULL) is applied to rows < add_rows and
 * repeats with period add_period rows: one launch normalises new_mem[l] + offset of every decoder level
 * (must3r/model/feedback_mechanism.py:49-51, decoder.py:323-330).  Used where the producing GEMM cannot emit the
 * normalised rows itself (m3r_gemm_args.norm_out: multi-wave problems). */
int m3r_normalize16(const float* x, int64_t ldx, const float* add, int64_t ldadd, int32_t add_rows, int32_t add_period,
                    float eps, int32_t M, int32_t D, void* out16, int64_t ldo, int32_t is_bf16, void* stream);
/* The same rows written as e4m3 bytes (M3R_OUT_E4M3; ldo in bytes, a multiple of 4): the A operand of an e4m3 GEMM. */
int m3r_normalize8(const float* x, int64_t ldx, const float* add, int64_t ldadd, int32_t add_rows, int32_t add_period,
                   float eps, int32_t M, int32_t D, void* out8, int64_t ldo, void* stream);

/* fp32 -> 16-bit cast of [M,D] rows (encoder features entering the decoder projector, decoder.py:274). */
int m3r_cast16(const float* x, int64_t ldx, int32_t M, int32_t D, void* out, int64_t ldo, int32_t is_bf16,
               void* stream);

/* LayerNorm of 16-bit rows -> 16-bit rows (memory_mode 'raw': norm_y applied to the stored tokens at use,
 * must3r/model/blocks/layers.py:92), and fp32 (x + add) -> 16-bit (what 'raw' stores, layers.py:82-83 after the feedback
 * offset of decoder.py:323-330). */
int m3r_layernorm16(const void* x16, int64_t ldx, const float* gamma, const float* beta, float eps, int32_t M, int32_t D,
                    void* out16, int64_t ldo, int32_t is_bf16, void* stream);
int m3r_add_cast16(const float* x, int64_t ldx, const float* add, int64_t ldadd, int32_t M, int32_t D, void* out,
                   int64_t ldo, int32_t is_bf16, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * RoPE trig table: tab[t] = (cos, sin)(pos[t,axis] * F0 / base^(d/16)), d<16, for axis y then x.
 * Same arithmetic as dust3r/croco/models/curope/kernels.cu:45-55 (fp32 powf/cosf/sinf).
 * pos: [T,2] int64 (y,x).
 * ------------------------------------------------------------------------------------------------- */
int m3r_rope_table(const int64_t* pos, int32_t T, float base, float f0, float* tab, void* stream);

/* Stand-alone in-place 2-D RoPE with the curope operator contract (curope.cpp:49-69):
 * tokens [B,N,H,D=64] 16-bit or fp32 with strides (sB,sN,sH,1) in elements, pos [B,N,2] int64.
 * B, N, H and D must not be negative (an argument error, even when their product is positive); D % 4 == 0. */
int m3r_rope_2d(void* tokens, int32_t dtype /*0 f32,1 f16,2 bf16*/, int32_t B, int32_t N, int32_t H, int32_t D,
                int64_t sB, int64_t sN, int64_t sH, const int64_t* pos, float base, float fwd, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * FlashAttention-style softmax(Q K^T / 8) V, head_dim 64, on wgmma (S, P and O in registers, online softmax).
 * Replaces CoreAttention.attention (must3r/model/blocks/attention.py:37-79) for both self-attention and
 * the memory cross-attention, including the "drop each image's own new tokens" mask of
 * MUSt3R.make_mem_mask (must3r/model/decoder.py:119-139) and the torch.cat / expand / boolean gather of
 * decoder.py:306-317, which become two key/value segments plus a skip range.
 *
 * Query rows of (batch b, head h): Q + (b*Nq + i)*ldq + h*64.
 * Keys come from up to two segments; segment s of batch b: rows K_s + ((b / kv_group) * kv_bstride_s + j)*ldk_s
 * (+ h*64), j < Nk_s.  kv_group query batches share one K/V batch (the views of one scene).
 * Keys with global index in [skip_lo + (b % kv_group)*skip_step, +skip_len) are not attended (skip_len = 0:
 * no mask); global index = j for segment 0 and Nk_0 + j for segment 1.
 * ------------------------------------------------------------------------------------------------- */
typedef struct {
  const void* Q; int64_t ldq;
  const void* K0; const void* V0; int64_t ldk0; int64_t kv_bstride0; int32_t Nk0;
  const void* K1; const void* V1; int64_t ldk1; int64_t kv_bstride1; int32_t Nk1;
  void* O; int64_t ldo;     /* [B*Nq, H*64] 16-bit */
  int32_t B, H, Nq;
  int32_t kv_group;         /* >= 1 */
  int32_t skip_lo, skip_step, skip_len;
  int32_t is_bf16;
  float scale;              /* 1/sqrt(64) */
  /* Export mode (both non-NULL; O may then be NULL): write the UNNORMALISED attention state of this key set instead of
   * the normalised output - export_o [B*Nq, H*64] fp32 = sum_j 2^(s_ij*c - m_i) v_j, export_ml [B*Nq, H, 2] fp32 =
   * (m_i, l_i) with c = scale*log2(e), m_i the running maximum in log2 units (-inf if the row saw no key) - so that key
   * shards held by different GPUs can be merged exactly (m3r_attn_merge): context-parallel memory cross-attention. */
  float* export_o;
  float* export_ml;
} m3r_attn_args;

int m3r_attention(const m3r_attn_args* args, void* stream);
/* Ragged form: K/V batch k (of B / kv_group) attends to rows j < nk0_b[k] of segment 0 only; nk0_b is an int32 device
 * array [B / kv_group] read by the kernel, its values clamped to [0, Nk0], and Nk0 (>= 1) is the longest batch: the length
 * the tensor maps and the key splits are planned for.  Rows at or past a batch's own length may hold anything (NaN and inf
 * included) and influence no output bit.  Segment 1 and the skip range keep their meaning (segment 1's global index is
 * Nk0 + j for every batch).  Equal lengths give bitwise the result of m3r_attention.  Export mode is an argument error.
 * The lengths are only known on the device, so a batch left with no key at all cannot be refused: its rows come out 0.
 * Used by the decoder call over several SLAM sessions (m3r_decoder_forward_ragged), whose memories differ in length. */
int m3r_attention_ragged(const m3r_attn_args* args, const int32_t* nk0_b, void* stream);

/* Merge `n` exported attention states of the same queries over disjoint key sets:
 * out[r, c] = sum_k o_k[r, c] 2^(m_k[r,h] - m) / sum_k l_k[r,h] 2^(m_k[r,h] - m), m = max_k m_k, h = c / 64.
 * parts_o[k] / parts_ml[k]: device pointers as exported above (rows x H*64 fp32, rows x H x 2 fp32); out: [rows, H*64]
 * 16-bit with leading dim ldo.  m3r_attn_state_fill writes the state of an EMPTY key set (o = 0, m = -inf, l = 0).
 * Base pointers: every parts_o[k], out and export_o 16-byte aligned and every parts_ml[k] and export_ml 8-byte aligned
 * (non-null parts), refused before any CUDA call otherwise. */
int m3r_attn_merge(const float* const* parts_o, const float* const* parts_ml, int32_t n, int64_t rows, int32_t H,
                   void* out, int64_t ldo, int32_t is_bf16, void* stream);
int m3r_attn_state_fill(float* export_o, float* export_ml, int64_t rows, int32_t H, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Patch embedding front end: im2col of [V,3,H,W] fp32 images into [V*N, 768] 16-bit rows
 * (col = c*256 + i*16 + j, the flattened Conv2d(3,D,16,16) weight order, dust3r/croco/models/blocks.py:222),
 * to be followed by m3r_gemm with the [D,768] weight.  Tokens in raster order (patch_embed.py:20-29).
 * Base pointers: img 16-byte aligned (float4 loads), out 8-byte aligned; refused before any CUDA call otherwise.
 * ------------------------------------------------------------------------------------------------- */
int m3r_im2col16(const float* img, int32_t V, int32_t H, int32_t W, void* out, int32_t is_bf16, void* stream);

/* Head unpatchify (must3r/tools/image.py:9-14 + head.py:71): proj [V*N,1792] fp32 ->
 * out[v,16y+i,16x+j,c] = proj[v, y*w+x, c*256+16i+j], out [V,H,W,7] fp32.  C (7 for the model) must be >= 1. */
int m3r_unpatchify(const float* proj, int32_t V, int32_t H, int32_t W, int32_t C, float* out, void* stream);

/* postprocess(compute_cam=False) (must3r/engine/inference.py:16-27, must3r/tools/geometry.py:14-18):
 * pm [P,7] -> pts3d [P,3], pts3d_local [P,3], conf [P]. */
int m3r_postprocess(const float* pm, int64_t P, float* pts3d, float* pts3d_local, float* conf, void* stream);

/* Nearest-neighbour distance of Q query points [Q,3] fp32 to a database [P,3] fp32: out[i] = min_j |q_i - p_j| (inf for an
 * empty database).  Replaces the per-frame scipy KD-tree query of the SLAM keyframe test
 * (must3r/slam/nns.py:57-62, called from must3r/slam/model.py:82). */
int m3r_nn_min_dist(const float* queries, int32_t Q, const float* db, int64_t P, float* out, void* stream);

/* Exact nearest-neighbour grid index over a point map with per-point buckets (the viewing-direction quadrants of
 * must3r/slam/nns.py:65-95 QuandrantSearcher, or one bucket for KDTree_scipy).  Cells are cubes of side h.
 * m3r_pointgrid_keys: keys[i] = 64-bit sort key of pts[i] [P,3] fp32 with bucket[i] (int32 in [0, 512), NULL = all 0):
 * the bucket, then the Morton code of the cell floor(pts * inv_h); points whose cell is out of the key range or non-finite get
 * the bucket's overflow key, which sorts after all its cells.  The caller sorts the points by key and builds
 * pts [P,3] (sorted), cell_keys [C] (the distinct sorted keys), cell_off [C+1] int32 (point range of each cell) and
 * bucket_cells [nb+1] int32 (cell range of each bucket).
 * m3r_pointgrid_query: out[i] = distance from queries[i] to the nearest point of bucket qbucket[i] (NULL = all 0), inf if
 * that bucket is empty; bitwise equal to m3r_nn_min_dist over that bucket's points. */
int m3r_pointgrid_keys(const float* pts, const int32_t* bucket, int64_t P, float inv_h, int64_t* keys, void* stream);
int m3r_pointgrid_query(const float* queries, const int32_t* qbucket, int32_t Q, const float* pts, int64_t P,
                        const int64_t* cell_keys, const int32_t* cell_off, int32_t C, const int32_t* bucket_cells,
                        int32_t nb, float h, float inv_h, float* out, void* stream);

/* One frame's camera and keyframe test in the SLAM front end (must3r/slam/model.py:147-172 get_camera_pose, :62-91
 * get_overlap_score, :231-235 the keyframe decision): a small device record per view, read back once by the host. */
typedef struct {
  float c2w[16];          /* camera-to-world, row-major 4x4 */
  float w2c[16];          /* its rigid inverse */
  float focal;            /* Weiszfeld focal in pixels, clamped below at 0 */
  float conf_mean;        /* mean of conf */
  float conf_median;      /* lower median of conf (torch.median); NaN if any conf is NaN */
  int32_t n_conf;         /* subsampled points with conf > min_conf_keyframe (m3r_slam_keyframe) */
  double score;           /* overlap score (m3r_slam_keyframe) */
  int32_t keyframe;       /* keyframe decision (m3r_slam_keyframe) */
  int32_t reserved;
} m3r_slam_record;
/* overlap modes of m3r_slam_keyframe */
#define M3R_OVERLAP_NN 0
#define M3R_OVERLAP_NN_NORM 1
#define M3R_OVERLAP_MEANCONF 2
#define M3R_OVERLAP_MEDIANCONF 3
/* B views of [H, W]: pts3d [B,H,W,3], pts3d_local [B,H,W,3], conf [B,H,W] fp32 -> rec[B].  focal = the Weiszfeld fit of
 * pixel - (ppx, ppy) ~ focal * (x, y) / z (closed-form L2 start, 10 re-weighted steps).  Unless is_first: when
 * has_seq_focal, pts3d_local's z is scaled IN PLACE by seq_focal / focal (fp32, as the reference); then the rotation and
 * translation minimising sum (conf - 1) |R x_local + t - x_world|^2 (Horn's quaternion, det R = +1).  is_first gives
 * the identity pose.  Each view is one thread-block cluster; one launch. */
int m3r_slam_pose(const float* pts3d, float* pts3d_local, const float* conf, int32_t B, int32_t H, int32_t W, float ppx,
                  float ppy, int32_t has_seq_focal, float seq_focal, int32_t is_first, m3r_slam_record* rec, void* stream);
/* Overlap score and keyframe decision of one view whose record m3r_slam_pose wrote.  The subsampled points are the
 * pixels (s*i, s*j) of [H, W] (s = subsamp); dists [ceil(H/s) * ceil(W/s)] = the nearest-map-point distance of every
 * one of them, conf [H,W] and pts3d_local [H,W,3] the full maps.  NN modes: the `percentile` (np.percentile, linear)
 * of dists (divided by z + 1e-9 for NN_NORM) over the points with conf > min_conf_keyframe, +inf counted as FLT_MAX,
 * NaN if one of them is NaN, 0 if there is none; the conf modes take the record's mean / median.  keyframe = is_first
 * or ((score > thr for NN modes, score < thr otherwise) and conf_median > min_conf_keyframe). */
int m3r_slam_keyframe(const float* dists, const float* conf, const float* pts3d_local, int32_t H, int32_t W, int32_t subsamp,
                      int32_t mode, double percentile, double thr, float min_conf_keyframe, int32_t is_first,
                      m3r_slam_record* rec, void* stream);
/* Several cameras of one SLAM map in one step (must3r_b200/engine/slam_cameras.py): m3r_slam_pose over B views whose
 * has_seq_focal[v], seq_focal[v] and is_first[v] (host arrays [B], B <= 64) are the view's own camera's; each record is
 * bitwise what m3r_slam_pose writes for that view alone with those values.  One cluster per view. */
int m3r_slam_pose_views(const float* pts3d, float* pts3d_local, const float* conf, int32_t B, int32_t H, int32_t W,
                        float ppx, float ppy, const int32_t* has_seq_focal, const float* seq_focal, const int32_t* is_first,
                        m3r_slam_record* rec, void* stream);
/* m3r_slam_keyframe of F frames of one [H, W] shape in one launch, one cluster per frame: frame f reads dists + f * Q
 * (Q = ceil(H/s) * ceil(W/s)), conf + f * H * W, pts3d_local + f * H * W * 3 and writes rec[f], bitwise what
 * m3r_slam_keyframe writes for it alone with is_first[f] (host array [F], 1 <= F <= 64). */
int m3r_slam_keyframe_frames(const float* dists, const float* conf, const float* pts3d_local, int32_t F, int32_t H, int32_t W,
                             int32_t subsamp, int32_t mode, double percentile, double thr, float min_conf_keyframe,
                             const int32_t* is_first, m3r_slam_record* rec, void* stream);

/* Confidence-filtered point cloud of a reconstructed scene at T thresholds (must3r/demo/gradio.py:131-156
 * get_3D_model_from_scene with as_pointcloud, :91-92 the masking).  A device table of V views, each of its own H x W: */
typedef struct {
  const float* pts3d;     /* [H,W,3]: world points, or local points when c2w is set */
  const float* c2w;       /* NULL, or the 4x4 row-major camera-to-world applied to pts3d (geotrf, local_pointmaps) */
  const float* conf;      /* [H,W] */
  const float* img;       /* [3,H,W] ImgNorm image; colour = clip(x * 0.5 + 0.5, 0, 1) (dust3r rgb) */
  int32_t H, W;
  int64_t first_tile;     /* sum over the earlier views of ceil(H * W / M3R_SCENE_TILE) */
} m3r_scene_view;
#define M3R_SCENE_TILE 1024
#define M3R_SCENE_MAX_THR 8
/* Pass 1: tile_counts [T, n_tiles] int32 = pixels of each tile with conf >= thr[t] (thr: T fp32 on the device; NaN conf
 * is never selected), tile_off [T, n_tiles] int64 = their exclusive prefix in tile order, counts [T] int64 = the totals.
 * n_tiles = the first_tile the view after the last one would have. */
int m3r_scene_count(const m3r_scene_view* views, int32_t V, const float* thr, int32_t T, int64_t n_tiles,
                    int32_t* tile_counts, int64_t* tile_off, int64_t* counts, void* stream);
/* Pass 2, one launch for every view and threshold: the points of threshold t go to rows [base_t, base_t + counts[t]) of
 * pts_out / col_out [sum(counts), 3] fp32, base_t = counts[0] + ... + counts[t-1], view-major then in raster order (the
 * order of numpy's boolean masking); nothing else is written.  tile_off and counts come from m3r_scene_count on the same
 * views and thresholds. */
int m3r_scene_points(const m3r_scene_view* views, int32_t V, const float* thr, int32_t T, int64_t n_tiles,
                     const int64_t* tile_off, const int64_t* counts, float* pts_out, float* col_out, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Input preprocessing of V RGB uint8 frames of one size: src [V, src_h, src_w, 3] uint8 (HWC; pixel stride 3 bytes,
 * row pitch src_pitch bytes, frame stride src_vstride bytes - a crop view or a padded frame needs no copy) -> fp32
 * [V, 3, h, w] images in the ImgNorm range (the encoder's input).  Two separable passes, horizontal then vertical;
 * the host computes the coefficient tables (must3r_b200/engine/images.py): bounds [n, 2] int32 = (first source
 * index, tap count <= k) and weights [n, k] per output column (x) / row (y).  `tmp` is device scratch.
 * ------------------------------------------------------------------------------------------------- */
/* Pillow's 8-bit Image.resize (LANCZOS / BICUBIC; dust3r/dust3r/utils/image.py:64-71 _resize_pil_image) bit for bit,
 * then the crop box and ImgNorm of the SLAM front end (must3r/slam/model.py:99-120).  Weights are int32 with 22
 * fractional bits.  The horizontal pass reads source rows [row0, row0 + rows) and writes tmp [V, rows, out_w, 3] uint8;
 * y bounds are relative to row0.  Outputs (either may be NULL, not both): out_u8 [V, out_h, out_w, 3] = the resized
 * image; out [V, 3, crop_h, crop_w] fp32 = ImgNorm of its box (crop_x, crop_y, crop_w, crop_h). */
int m3r_resample_pil_u8(const uint8_t* src, int64_t src_pitch, int64_t src_vstride, int32_t V, int32_t src_h, int32_t src_w,
                        const int32_t* xbounds, const int32_t* xweights, int32_t xk, int32_t out_w,
                        const int32_t* ybounds, const int32_t* yweights, int32_t yk, int32_t out_h, int32_t row0,
                        int32_t rows, uint8_t* tmp, uint8_t* out_u8, int32_t crop_x, int32_t crop_y, int32_t crop_w,
                        int32_t crop_h, float* out, void* stream);
/* Antialiased bilinear resize (aten _upsample_bilinear2d_aa, torchvision Resize) of ImgNorm(src) with fp32 weights:
 * the demo's CenterCrop + Resize (must3r/tools/image.py:53-93, applied by must3r/demo/inference.py:63-76); src points at
 * the crop's first pixel.  tmp: [V, 3, src_h, out_w] fp32; out: [V, 3, out_h, out_w] fp32. */
int m3r_resize_aa_bilinear_u8(const uint8_t* src, int64_t src_pitch, int64_t src_vstride, int32_t V, int32_t src_h,
                              int32_t src_w, const int32_t* xbounds, const float* xweights, int32_t xk, int32_t out_w,
                              const int32_t* ybounds, const float* yweights, int32_t yk, int32_t out_h, float* tmp,
                              float* out, void* stream);

/* ---- Baseline JPEG decoding (jpeg.cu), bit for bit what Pillow (libjpeg-turbo, JDCT_ISLOW, fancy upsampling) gives.
 * Host: m3r_jpeg_parse reads the headers of a file held in memory; m3r_jpeg_prepare makes one pass over the entropy-
 * coded data into a caller buffer (byte unstuffing, restart markers removed) with the Huffman / quantisation tables and
 * the restart-segment table; m3r_jpeg_plan lays out a batch.  Device: m3r_jpeg_decode decodes the batch on `stream`. */
typedef struct m3r_jpeg_info {
  int32_t width, height, ncomp;
  int32_t eligible;            /* 1: the GPU decoder takes the file (baseline / extended 8-bit Huffman, one scan, gray
                                  or YCbCr with luma sampling 1x1, 2x1, 2x2 or 1x2 and chroma 1x1) */
  int32_t orientation;         /* EXIF IFD0 0x0112, else XMP tiff:Orientation (Pillow's getexif); 1 when absent */
  int32_t orientation_exact;   /* 0: the metadata is unusual enough that only Pillow can say what exif_transpose does */
  int32_t restart_interval;    /* MCUs per restart segment, 0 = none */
  int32_t hs[3], vs[3];        /* sampling factors */
  int64_t scan_offset;         /* first byte of the entropy-coded data */
  int64_t prep_bytes;          /* bytes m3r_jpeg_prepare writes at most */
} m3r_jpeg_info;

/* One prepared image of a batch.  Offsets are bytes from the start of the batch's prepared buffer (which is copied to
 * the device as one piece); `out` is the image's device output [H, W, 3] uint8 (W, H swapped for orientations 5..8). */
typedef struct m3r_jpeg_desc {
  int64_t tables_off, segs_off, subs_off, stream_off, stream_bytes;
  uint8_t* out;
  int32_t width, height, ncomp, orientation;   /* orientation: the transpose applied on the store (1 = none) */
  int32_t mcux, mcuy, bpm, restart_interval, nseg, nsub;
  int32_t hs[3], vs[3];
  /* m3r_jpeg_plan: prefix sums over the batch and workspace offsets */
  int64_t sub_base, blk_base, pix_base, coef_off, plane_off[3];
} m3r_jpeg_desc;

/* Parse the headers; returns 0 (info filled, eligible or not) or 1 for a file that is not a JPEG at all. */
int m3r_jpeg_parse(const uint8_t* data, int64_t size, m3r_jpeg_info* info);
/* Fill `dst` (info->prep_bytes, 16-byte aligned) and `desc` (offsets + base_off).  Returns 0, or 2 when the entropy-coded
 * data makes the file ineligible after all (a second scan, misnumbered or missing restart markers, no EOI). */
int m3r_jpeg_prepare(const uint8_t* data, int64_t size, const m3r_jpeg_info* info, int32_t orientation, uint8_t* dst,
                     int64_t base_off, m3r_jpeg_desc* desc);
/* Fill the batch fields of `descs` and return the device workspace bytes m3r_jpeg_decode needs (-1 on error). */
int64_t m3r_jpeg_plan(m3r_jpeg_desc* descs, int32_t n);
/* Decode the batch: `host_descs` (planned) describe it, `dev_blob` is the device copy of the prepared buffer, whose
 * descriptor array sits at byte `descs_off`.  status[n] (device int32) gets 0 or the M3R_JPEG_E* bits of each image. */
int m3r_jpeg_decode(const m3r_jpeg_desc* host_descs, int32_t n, const uint8_t* dev_blob, int64_t descs_off, uint8_t* work,
                    int64_t work_bytes, int32_t* status, void* stream);
#define M3R_JPEG_EHUFF 1       /* a code missing from its table, or a coefficient past the end of a block */
#define M3R_JPEG_ESHORT 2      /* a restart segment ends before its last MCU */
#define M3R_JPEG_ESYNC 4       /* the parallel decoder did not agree with itself within its round budget */

/* ---- PNG decoding (png.cu), bit for bit what Pillow's .convert('RGB') gives for 8-bit, non-interlaced L, RGB, P, LA
 * and RGBA images.  Host: m3r_png_parse walks the chunks of a file held in memory (signature, CRCs of the chunks before
 * the image data, zlib header); m3r_png_prepare copies the palette and the concatenated IDAT payloads into a caller
 * buffer; m3r_png_plan lays out a batch.  Device: m3r_png_decode inflates and unfilters the batch on `stream`. */
typedef struct m3r_png_info {
  int32_t width, height;
  int32_t bit_depth, color_type, interlace;
  int32_t channels;            /* samples per pixel of the colour type: 1 (L, P), 2 (LA), 3 (RGB), 4 (RGBA) */
  int32_t palette_entries;     /* PLTE entries, 0 when there is none */
  int32_t eligible;            /* 1: the GPU decoder takes the file (the caller adds Pillow's size limit and, for the
                                  EXIF transpose, has_exif / has_text) */
  int32_t has_exif;            /* an eXIf chunk */
  int32_t has_text;            /* a tEXt, zTXt or iTXt chunk (Pillow's getexif reads EXIF from these too) */
  int64_t text_bytes;          /* payload bytes of those text chunks */
  int64_t idat_bytes;          /* the zlib stream: the IDAT payloads concatenated */
  int64_t prep_bytes;          /* bytes m3r_png_prepare writes */
} m3r_png_info;

/* One prepared image of a batch; offsets are bytes from the start of the batch's prepared buffer.  `out` is the image's
 * device output [H, W, 3] uint8 (W, H swapped for orientations 5..8). */
typedef struct m3r_png_desc {
  int64_t plte_off;            /* 768 bytes: the palette as RGB triplets */
  int64_t stream_off, stream_bytes;
  uint8_t* out;
  int32_t width, height, channels, color_type, palette_entries, orientation;
  /* m3r_png_plan: the image's scanline workspace (filter byte + W * channels bytes per row) */
  int64_t raw_off, raw_bytes;
} m3r_png_desc;

/* Parse the chunks; returns 0 (info filled, eligible or not) or 1 for a file that is not a PNG at all. */
int m3r_png_parse(const uint8_t* data, int64_t size, m3r_png_info* info);
/* Fill `dst` (info->prep_bytes, 16-byte aligned) and `desc` (offsets + base_off); 0, or set_error when the data is not
 * the eligible PNG that was parsed. */
int m3r_png_prepare(const uint8_t* data, int64_t size, const m3r_png_info* info, int32_t orientation, uint8_t* dst,
                    int64_t base_off, m3r_png_desc* desc);
/* Fill the workspace fields of `descs` and return the device workspace bytes m3r_png_decode needs (-1 on error). */
int64_t m3r_png_plan(m3r_png_desc* descs, int32_t n);
/* Decode the batch: `host_descs` (planned) describe it, `dev_blob` is the device copy of the prepared buffer, whose
 * descriptor array sits at byte `descs_off`.  status[n] (device int32) gets 0 or the M3R_PNG_E* bits of each image. */
int m3r_png_decode(const m3r_png_desc* host_descs, int32_t n, const uint8_t* dev_blob, int64_t descs_off, uint8_t* work,
                   int64_t work_bytes, int32_t* status, void* stream);
#define M3R_PNG_EBTYPE 1       /* a deflate block of type 3 */
#define M3R_PNG_ESTORED 2      /* a stored block whose LEN is not the complement of NLEN */
#define M3R_PNG_ECODES 4       /* more than 286 length or 30 distance codes, or code lengths over-subscribed or
                                  incomplete (zlib allows an incomplete code only for a single code of length 1) */
#define M3R_PNG_EREPEAT 8      /* a repeat code with no previous length, or one that runs past HLIT + HDIST */
#define M3R_PNG_ENOEOB 16      /* a dynamic block without an end-of-block code */
#define M3R_PNG_ESYMBOL 32     /* a code absent from its table, length symbol 286/287 or distance symbol 30/31 */
#define M3R_PNG_EDIST 64       /* a distance before the start of the output */
#define M3R_PNG_ELENGTH 128    /* the stream ends early, or its output is not H * (1 + W * channels) bytes */
#define M3R_PNG_EFILTER 256    /* a scanline filter type above 4 */
#define M3R_PNG_EPALETTE 512   /* a palette index past the PLTE entries */
#define M3R_PNG_EADLER 1024    /* the Adler-32 of the output is not the stream's */

/* ===================================================================================================
 * Whole-model entry points: one call enqueues every kernel of a forward pass from C++ (no per-layer
 * Python/ctypes overhead).  Weight structs hold DEVICE pointers (16-bit matrices in nn.Linear layout,
 * fp32 biases / LayerNorm affines); the `blocks` arrays themselves live in HOST memory.
 * ================================================================================================= */

/* Block (must3r/model/blocks/layers.py:36-54): norm1, attn.{qkv,proj}, norm2, mlp.{fc1,fc2} */
typedef struct {
  const float* norm1_w; const float* norm1_b;
  const void* qkv_w; const float* qkv_b;       /* [3D,D] */
  const void* proj_w; const float* proj_b;     /* [D,D]  */
  const float* norm2_w; const float* norm2_b;
  const void* fc1_w; const float* fc1_b;       /* [4D,D] */
  const void* fc2_w; const float* fc2_b;       /* [D,4D] */
} m3r_enc_block;

/* Dust3rEncoder (must3r/model/encoder.py:13-52) */
typedef struct {
  int32_t embed_dim, depth, num_heads, mlp_hidden;
  float ln_eps, rope_base, rope_f0;
  int32_t is_bf16;
  const void* patch_w; const float* patch_b;   /* [D,768] = patch_embed.proj.weight.view(D,-1) */
  const m3r_enc_block* blocks;                 /* host array [depth] */
  const float* norm_w; const float* norm_b;    /* norm_enc */
} m3r_encoder_weights;

int64_t m3r_encoder_workspace_bytes(const m3r_encoder_weights* w, int32_t V, int32_t H, int32_t W);

/* Dust3rEncoder.forward (encoder.py:46-52): img [V,3,H,W] fp32 -> x [V*N, D] fp32.
 * pos: [N,2] int64 (y,x) positions of ONE view's tokens (all views of a call share the grid). */
int m3r_encoder_forward(const m3r_encoder_weights* w, const float* img, int32_t V, int32_t H, int32_t W,
                        const int64_t* pos, float* out_x, void* workspace, int64_t workspace_bytes, void* stream);

/* FP8 encoder (same workspace): w->is_bf16 = 1 and, per block, qkv_w / fc1_w are e4m3 [3D,D] / [4D,D] with norm1 / norm2
 * folded in (W * diag(gamma), b + W beta, then quantised row by row; norm1_w .. norm2_b unused); blocks8[l] holds their
 * per-row scales.  Each LayerNorm before qkv / fc1 becomes an affine-free m3r_normalize8; patch embedding, proj, fc2,
 * attention and the residual stream run as in bf16. */
typedef struct {
  const float* qkv_s;     /* [3D] */
  const float* fc1_s;     /* [4D] */
} m3r_enc_block_e4m3;
int m3r_encoder_forward_e4m3(const m3r_encoder_weights* w, const m3r_enc_block_e4m3* blocks8, const float* img, int32_t V,
                             int32_t H, int32_t W, const int64_t* pos, float* out_x, void* workspace,
                             int64_t workspace_bytes, void* stream);

/* CachedDecoderBlock (must3r/model/blocks/layers.py:57-99).  Every LayerNorm of the block is applied WITHOUT its affine
 * (by the epilogue of the GEMM that produced the rows, m3r_gemm_args.norm_out, or by m3r_normalize16); the affine lives in the
 * consuming Linear: W' = W * diag(gamma), b' = b + W beta (exact in real arithmetic; rounded to 16 bits once, like W).
 * Because norm1 and norm_y normalise the same block input, the self-attention qkv projection and the K|V projection of
 * the new memory tokens (layers.py:81-88,91) become ONE GEMM with the stacked weight a_w. */
typedef struct {
  const void* a_w; const float* a_b;           /* [5D,D]: rows [0,3D) attn.qkv (norm1 folded), rows [3D,5D) cross_attn.projk ;
                                                  projv (norm_y folded).  blocks[l].a_w == blocks[0].a_w + l*5D*D and
                                                  blocks[l].a_b == blocks[0].a_b + l*5D let the memory append run as one
                                                  grouped GEMM; otherwise it falls back to one GEMM per level */
  const void* proj_w; const float* proj_b;     /* attn.proj [D,D] */
  const void* q_w; const float* q_b;           /* cross_attn.projq [D,D], norm2 folded */
  const void* cproj_w; const float* cproj_b;   /* cross_attn.proj [D,D] */
  const void* fc1_w; const float* fc1_b;       /* mlp.fc1 [4D,D], norm3 folded */
  const void* fc2_w; const float* fc2_b;       /* mlp.fc2 [D,4D] */
  const float* normy_w; const float* normy_b;  /* norm_y affine: memory_mode norm_y / raw only (rows stored / normalised at use) */
  const void* kv_w; const float* kv_b;         /* UNFOLDED [projk ; projv] [2D,D]: memory_mode norm_y / raw (K|V of stored rows
                                                  projected at use, layers.py:92-96); may be NULL for memory_mode kv */
} m3r_dec_block;

/* MUSt3R (must3r/model/decoder.py:14-156) */
typedef struct {
  int32_t enc_dim, embed_dim, depth, num_heads, mlp_hidden, out_dim;
  float ln_eps, fb_ln_eps, rope_base, rope_f0;
  int32_t is_bf16;
  int32_t feedback;                            /* 0 none, 1 single_mlp, 2 single_linear */
  const void* embed_w; const float* embed_b;   /* feat_embed_enc_to_dec [D,enc_dim] */
  const float* image2_embed;                   /* [D] */
  const m3r_dec_block* blocks;                 /* host array [depth] */
  const void* fb1_w; const float* fb1_b;       /* feedback_layer.fc1 [4D,D] (or the single linear [D,D]), feedback_norm folded */
  const void* fb2_w; const float* fb2_b;       /* feedback_layer.fc2 [D,4D] */
  const void* head_w; const float* head_b;     /* head_dec.proj [out_dim,D], norm_dec folded */
} m3r_decoder_weights;

/* One aspect-ratio group of a decoder call (MUSt3R.forward_list, decoder.py:158): B scenes x n_views views */
typedef struct {
  int32_t n_views, N, H, W;
  const float* x_enc;      /* [B*n_views*N, enc_dim] fp32 encoder features */
  const int64_t* pos;      /* [B*n_views*N, 2] int64 */
  float* pointmaps;        /* out: [B*n_views, H, W, out_dim/256] fp32 */
} m3r_dec_group;

typedef struct {
  int32_t B, G;
  const m3r_dec_group* groups;     /* host array [G] */
  int32_t Nm;                      /* memory tokens per scene before this call */
  const void* const* mem;          /* host array [depth] of device ptrs: [B, >=Nm, 2D] 16-bit (NULL if Nm==0) */
  int64_t mem_bstride_rows;        /* rows between consecutive scenes in mem[l] */
  int32_t render;                  /* 1: read-only pass (decoder.py:307); 0: memory update */
  int32_t is_init;                 /* current_mem is None: view 0 of group 0 gets no image2_embed (decoder.py:176,280) */
  void* const* mem_out;            /* update only: host array [depth] of device ptrs [B, >=Nm+Nt, 2D]; rows [0,Nm) are
                                      copied from mem[l] unless mem_out[l]==mem[l]; the new rows follow */
  int64_t mem_out_bstride_rows;
  int32_t new_only;                /* update only: 1 = mem_out[l] is [B, Nt, 2D] and receives ONLY the new post-feedback
                                      K|V rows (no copy of the old memory) - used by the sharded schedule, where the new
                                      tokens of all ranks are all-gathered into a pre-allocated memory buffer */
  int32_t n_peers;                 /* > 0 (with new_only): the post-feedback K|V GEMM epilogue stores the new rows straight
                                      into every rank's memory buffer (fused GEMM -> all-gather over NVLink peer memory) */
  void* const* peer_mem;           /* host array [n_peers * depth]: peer_mem[r * depth + l] = rank r's memory buffer of
                                      level l ([1, cap, 2D] 16-bit), already offset to the row where THIS rank's tokens go */
  int32_t mem_mode;                /* M3R_MEM_KV: memory rows are K|V (2D wide); M3R_MEM_NORM_Y: rows are norm_y(x) (D wide) and
                                      K|V are projected at use; M3R_MEM_RAW: rows are x (D wide), norm_y + projection at use
                                      (must3r/model/blocks/layers.py:81-96).  All widths "2D" above become D for the last two.
                                      peer output (n_peers > 0) needs M3R_MEM_KV. */
  /* ---- context-parallel memory cross-attention (SURVEY.md 8f rank 2; no reference counterpart): cp_world > 1 means the
   * memory tokens of the ONE scene (B == 1, mem_mode kv) are SHARDED over cp_world GPUs, each running this same call on the
   * same views.  mem[] / Nm describe only THIS rank's rows (Nm may be 0); every rank computes the attention state of the
   * queries over its shard (m3r_attn_args.export_o), copies it into slot cp_rank of every rank's staging buffer
   * (m3r_peer_bcast over NVLink), the ranks meet at a device-side flag barrier (m3r_peer_signal / m3r_peer_wait, epoch
   * cp_epoch0 + layer + 1) and merge the cp_world states (m3r_attn_merge): exactly the softmax over the union of the
   * shards.  New tokens attend to each other (calls with several views) on rank 0.  Only the rank with cp_owner = 1
   * appends the call's new rows (mem_out); the others skip the feedback MLP and the append.  The caller guarantees that
   * the scene's memory is non-empty globally (the very first call of a scene runs without cp). */
  int32_t cp_world, cp_rank, cp_owner;
  void* const* cp_stage;           /* host array [cp_world]: rank q's staging buffer as mapped here: 2 * cp_world slots */
  int64_t cp_slot_bytes;           /* bytes per slot, >= m3r_decoder_cp_slot_bytes() */
  void* const* cp_flag_slots;      /* host array [cp_world]: this rank's uint32 slot in rank q's flag array */
  const void* cp_flags_local;      /* this rank's own flag array */
  uint32_t cp_epoch0;              /* the call consumes epochs cp_epoch0 + 1 .. cp_epoch0 + depth */
} m3r_decoder_call;

/* bytes of one staging slot for a call with M token rows: M * H * (64 * 4 + 8), rounded up to 256 */
int64_t m3r_decoder_cp_slot_bytes(const m3r_decoder_weights* w, int64_t M);

int64_t m3r_decoder_workspace_bytes(const m3r_decoder_weights* w, const m3r_decoder_call* call);

/* ---------------------------------------------------------------------------------------------------
 * Peer memory for the multi-GPU schedule (one process per GPU): buffers allocated with m3r_peer_alloc can be exported
 * as a 64-byte CUDA IPC handle, exchanged through torch.distributed, and mapped by the other ranks of the node.
 * ------------------------------------------------------------------------------------------------- */
int m3r_peer_alloc(int64_t bytes, void** ptr);
int m3r_peer_free(void* ptr);
int m3r_ipc_export(void* ptr, void* handle64);
int m3r_ipc_open(const void* handle64, void** ptr);
int m3r_ipc_close(void* ptr);
/* Device-side barrier of the multi-GPU schedule (no reference counterpart; replaces a host-blocking collective per update
 * round).  Each rank owns slot `rank` of a uint32[world] flag array that lives in every rank's peer-visible memory.
 * m3r_peer_signal(flag_slots = address of MY slot in each of the n ranks' arrays, value): enqueued after the kernels whose
 * peer stores must be visible; writes `value` (a monotonically increasing epoch) with system-scope release semantics.
 * m3r_peer_wait(local_flags = this rank's own array, rank_mask, value): a kernel that spins on the GPU until every slot r
 * with bit r of rank_mask set has reached `value`; work enqueued after it sees the rows those ranks stored. */
/* Copy `bytes` (multiple of 16) from src to the same-sized block dsts[k], k < n: this GPU's staging buffer and its peers'
 * (NVLink stores): the exchange step of the context-parallel cross-attention.  src and every dsts[k] must be non-null and
 * 16-byte aligned (uint4 loads and stores), refused before any CUDA call otherwise. */
int m3r_peer_bcast(const void* src, void* const* dsts, int32_t n, int64_t bytes, void* stream);
int m3r_peer_signal(void* const* flag_slots, int32_t n, uint32_t value, void* stream);
int m3r_peer_wait(const void* local_flags, uint32_t rank_mask, uint32_t value, void* stream);

/* MUSt3R.forward / forward_list (decoder.py:158-350) for memory_mode 'kv'. */
int m3r_decoder_forward(const m3r_decoder_weights* w, const m3r_decoder_call* call, void* workspace,
                        int64_t workspace_bytes, void* stream);

/* The same memory update over B scenes whose memories hold different numbers of tokens (several SLAM sessions stepped
 * together, must3r_b200/engine/slam_sessions.py): scene b attends to rows [0, nm_scene[b]) of its memory, nm_scene an
 * int32 device array [B] (values clamped to [0, call->Nm]); call->Nm is the longest memory and must be >= 1, and each
 * scene's memory rows begin at b * mem_bstride_rows.  Every layer's memory cross-attention runs as m3r_attention_ragged.
 * Only memory_mode kv with new_only = 1 (no render, no peers, no context parallel): the new post-feedback K|V rows of
 * every scene go to mem_out[l] [B, Nt, 2D] and nothing is written into the memory; m3r_mem_commit appends them.  The
 * workspace is m3r_decoder_workspace_bytes(w, call). */
int m3r_decoder_forward_ragged(const m3r_decoder_weights* w, const m3r_decoder_call* call, const int32_t* nm_scene,
                               void* workspace, int64_t workspace_bytes, void* stream);

/* FP8 decoder: w->is_bf16 = 1, and the GEMMs fed by an affine-free LayerNorm take e4m3 operands: a_w (qkv | projk;projv,
 * [depth, 5D, D] e4m3, one byte per element), q_w, fc1_w and (feedback) fb1_w hold e4m3 weights with per-row scales in w8.
 * Everything else (proj, cproj, fc2, embed, head, the K|V memory, attention) stays bf16.  nm_scene = NULL runs
 * m3r_decoder_forward, otherwise m3r_decoder_forward_ragged; same workspace. */
typedef struct {
  const float* a_s;       /* [5D]; blocks[l].a_s == blocks[0].a_s + l*5D for the grouped memory append */
  const float* q_s;       /* [D] */
  const float* fc1_s;     /* [4D] */
} m3r_dec_block_e4m3;
typedef struct {
  const m3r_dec_block_e4m3* blocks;  /* host array [depth] */
  const float* fb1_s;                /* [4D] (single_mlp) or [D] (single_linear); NULL without feedback */
} m3r_decoder_e4m3;
int m3r_decoder_forward_e4m3(const m3r_decoder_weights* w, const m3r_decoder_e4m3* w8, const m3r_decoder_call* call,
                             const int32_t* nm_scene, void* workspace, int64_t workspace_bytes, void* stream);

/* The render pass (call->render = 1, decoder.py:307) over B scenes whose memories hold different numbers of tokens
 * (several offline reconstructions stepped together, must3r_b200/engine/scenes.py): the n_views views of scene b in every
 * group attend to rows [0, nm_scene[b]) of that scene's memory, nm_scene an int32 device array [B] (values clamped to
 * [0, call->Nm]); call->Nm is the longest memory and must be >= 1, and scene b's memory rows begin at
 * b * mem_bstride_rows.  Every layer's memory cross-attention runs as m3r_attention_ragged with kv_group = n_views.
 * Nothing is written into the memory.  w8 = NULL runs the 16-bit decoder, otherwise the FP8 decoder of
 * m3r_decoder_forward_e4m3.  Only memory_mode kv, no peers, no context parallel and is_init = 0; anything else is an
 * argument error.  The workspace is m3r_decoder_workspace_bytes(w, call). */
int m3r_decoder_render_ragged(const m3r_decoder_weights* w, const m3r_decoder_e4m3* w8, const m3r_decoder_call* call,
                              const int32_t* nm_scene, void* workspace, int64_t workspace_bytes, void* stream);

/* Keyframe commit of several SLAM sessions in one launch: for each scene b < B whose flag keep[b * keep_stride] (int32,
 * device; e.g. the keyframe field of its m3r_slam_record) is non-zero, copy rows [0, Nt) of staged[l] + b * Nt * width
 * (the [B, Nt, width] 16-bit new_only output of m3r_decoder_forward_ragged) to rows dst_row[b] .. dst_row[b] + Nt - 1 of
 * arena[l] (rows of `width` 16-bit elements), for every level l < depth.  A scene whose flag is zero writes nothing.
 * arena, staged: host arrays [depth] of device pointers; dst_row: host array [B].  B <= M3R_MAX_COMMIT,
 * depth <= M3R_MAX_GROUPS, width % 8 == 0, every arena / staged pointer 16-byte aligned and keep 4-byte aligned. */
#define M3R_MAX_COMMIT 64
int m3r_mem_commit(void* const* arena, const void* const* staged, int32_t depth, int32_t B, int32_t Nt, int32_t width,
                   const int64_t* dst_row, const int32_t* keep, int64_t keep_stride, void* stream);
/* m3r_mem_commit of part of each staged block: rows [row0, row0 + rows) of staged[l] + b * src_stride_rows * width go to
 * rows dst_row[b] .. dst_row[b] + rows - 1 of arena[l].  m3r_mem_commit is the case row0 = 0, rows = src_stride_rows = Nt.
 * Used where a refinement pass overwrites a step's rows in place except those of the reference view.  Same conditions,
 * and 0 <= row0, row0 + rows <= src_stride_rows. */
int m3r_mem_commit_rows(void* const* arena, const void* const* staged, int32_t depth, int32_t B, int32_t row0, int32_t rows,
                        int32_t src_stride_rows, int32_t width, const int64_t* dst_row, const int32_t* keep,
                        int64_t keep_stride, void* stream);
/* Keyframe commit of the F frames of one step of a multi-camera SLAM run, whose frames were decoded together against one
 * shared memory (must3r_b200/engine/slam_cameras.py): frame k < F whose flag keep[k * keep_stride] (int32, device; the
 * keyframe field of its m3r_slam_record) is non-zero copies rows [0, Nt) of staged[l] + k * Nt * width (the [F, Nt, width]
 * 16-bit new_only output of the decoder) to rows row0 + Nt * j .. row0 + Nt * (j + 1) - 1 of arena[l], j being the number
 * of frames before k whose flag is set, for every level l < depth.  The result is bitwise that of m3r_mem_commit called
 * frame after frame with the rows counted on the host; rows past row0 + Nt * (flags set) are not written.  The flags are
 * read on the device.  arena, staged: host arrays [depth] of device pointers.  F <= M3R_MAX_COMMIT,
 * depth <= M3R_MAX_GROUPS, width % 8 == 0, row0 >= 0, every arena / staged pointer 16-byte aligned, keep 4-byte aligned. */
int m3r_mem_commit_ordered(void* const* arena, const void* const* staged, int32_t depth, int32_t F, int32_t Nt, int32_t width,
                           int64_t row0, const int32_t* keep, int64_t keep_stride, void* stream);
/* Order-preserving compaction, in place, of the memories of B scenes at every level in one launch (several videos
 * reconstructed together, must3r_b200/engine/videos.py: the rows of frames that left the rolling window).  Scene b owns
 * rows base_row[b] .. base_row[b] + cap - 1 of arena[l] (rows of `width` 16-bit elements; slot s of a [S, cap, width]
 * arena has base row s * cap).  Its kept runs are runs[3k .. 3k + 2] = (src_row, dst_row, rows), int32 relative to its
 * base, for k in [run_offset[b], run_offset[b + 1]): rows src_row .. src_row + rows - 1 move to dst_row .. dst_row + rows
 * - 1.  The result is bitwise that of the runs applied one after another, each as buf[dst:dst+rows] =
 * buf[src:src+rows].clone(), also where a run's source and destination overlap; only the runs' destination rows are
 * written, and no scratch buffer is used.  Conditions (argument errors otherwise): 0 <= dst_row <= src_row,
 * src_row + rows <= cap, each run's src_row and dst_row at or past the end of the previous run's; run_offset[0] = 0,
 * non-decreasing, run_offset[B] <= M3R_MAX_COMPACT_RUNS; base rows >= 0, ascending and at least cap apart;
 * B <= M3R_MAX_COMMIT, depth <= M3R_MAX_GROUPS, width % 8 == 0, every arena pointer 16-byte aligned.  arena, base_row,
 * run_offset and runs are host arrays. */
#define M3R_MAX_COMPACT_RUNS 128
int m3r_mem_compact_rows(void* const* arena, int32_t depth, int32_t B, int32_t width, int64_t cap, const int64_t* base_row,
                         const int32_t* run_offset, const int32_t* runs, void* stream);


#ifdef __cplusplus
}
#endif
#endif /* MUST3R_B200_H */
