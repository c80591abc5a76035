// HBM-bound kernels of the hot path: LayerNorm (fp32 rows -> 16-bit GEMM operand), casts, RoPE table,
// stand-alone curope-compatible RoPE, im2col for the patch embedding, head unpatchify, postprocess.
// All are coalesced / 16-byte vectorised; one warp per row for the row-wise ones.
#include "ptx.cuh"
#include "m3r_internal.h"

namespace m3r {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------- LayerNorm
// One warp per row; the row lives in registers (D <= 32 * 4 * MAXV). Two-pass mean / variance like torch.
template <int MAXV, bool IN16, bool PRE>
__global__ void __launch_bounds__(256) layernorm_kernel(const void* __restrict__ xv, long long ldx,
                                                        const float* __restrict__ add, long long ldadd,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        float eps, int M, int D, void* __restrict__ out, long long ldo,
                                                        int out_dtype, int is_bf16, int add_rows, int add_period) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int nv = D >> 2;  // float4 per row
  // PRE (small, latency-bound launches of the one-view chain): gamma / beta are weights, so they are fetched before the
  // programmatic-dependency wait, under the previous kernel's tail.  Large launches keep their registers for occupancy.
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  float4 gv[PRE ? MAXV : 1], bv[PRE ? MAXV : 1];
  const bool affine = gamma != nullptr;          // nullptr: plain normalisation (the consumer GEMM's weights carry the affine)
  if (PRE && affine) {
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int idx = lane + i * 32;
      if (idx < nv) { gv[i] = __ldg(g4 + idx); bv[i] = __ldg(b4 + idx); }
    }
  }
  griddep_wait();
  griddep_launch();
  if (row >= M) return;
  const float4* xr = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(xv) + (IN16 ? 0 : (long long)row * ldx));
  const uint2* xh = reinterpret_cast<const uint2*>(reinterpret_cast<const uint16_t*>(xv) + (IN16 ? (long long)row * ldx : 0));
  // `add` covers rows < add_rows and repeats with period add_period (one feedback offset for every decoder level)
  const float4* ar = (add && row < add_rows) ? reinterpret_cast<const float4*>(add + (long long)(row % add_period) * ldadd) : nullptr;
  float4 v[MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + i * 32;
    if (idx < nv) {
      float4 t;
      if (IN16) {
        const uint2 h = xh[idx];
        t = make_float4(unpack16_lo(h.x, is_bf16), unpack16_hi(h.x, is_bf16), unpack16_lo(h.y, is_bf16), unpack16_hi(h.y, is_bf16));
      } else {
        t = xr[idx];
      }
      if (ar) { const float4 a = ar[idx]; t.x += a.x; t.y += a.y; t.z += a.z; t.w += a.w; }
      v[i] = t;
      s += (t.x + t.y) + (t.z + t.w);
    } else {
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  const float mean = warp_sum(s) / D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + i * 32;
    if (idx < nv) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / D + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int idx = lane + i * 32;
    if (idx < nv) {
      float4 y;
      y.x = (v[i].x - mean) * rstd; y.y = (v[i].y - mean) * rstd; y.z = (v[i].z - mean) * rstd; y.w = (v[i].w - mean) * rstd;
      if (affine) {
        const float4 g = PRE ? gv[PRE ? i : 0] : __ldg(g4 + idx), b = PRE ? bv[PRE ? i : 0] : __ldg(b4 + idx);
        y.x = y.x * g.x + b.x; y.y = y.y * g.y + b.y; y.z = y.z * g.z + b.z; y.w = y.w * g.w + b.w;
      }
      if (out_dtype == M3R_OUT_F32) {
        reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + (long long)row * ldo)[idx] = y;
      } else if (out_dtype == M3R_OUT_E4M3) {
        reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(out) + (long long)row * ldo)[idx] = pack_e4m3x4(y.x, y.y, y.z, y.w);
      } else {
        uint2 w;
        w.x = pack16(y.x, y.y, is_bf16);
        w.y = pack16(y.z, y.w, is_bf16);
        reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(out) + (long long)row * ldo)[idx] = w;
      }
    }
  }
}

__global__ void __launch_bounds__(256) cast16_kernel(const float* __restrict__ x, long long ldx,
                                                     const float* __restrict__ add, long long ldadd, int M, int D,
                                                     uint16_t* __restrict__ out, long long ldo, int is_bf16) {
  const int nv = D >> 2;
  const long long total = (long long)M * nv;
  griddep_wait();
  griddep_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int row = int(i / nv), c = int(i % nv);
    float4 t = reinterpret_cast<const float4*>(x + (long long)row * ldx)[c];
    if (add) {
      const float4 a = reinterpret_cast<const float4*>(add + (long long)row * ldadd)[c];
      t.x += a.x; t.y += a.y; t.z += a.z; t.w += a.w;
    }
    uint2 w;
    w.x = pack16(t.x, t.y, is_bf16);
    w.y = pack16(t.z, t.w, is_bf16);
    reinterpret_cast<uint2*>(out + (long long)row * ldo)[c] = w;
  }
}

// ---------------------------------------------------------------------------------------------- RoPE
// tab[t][0..15]=cos(y*w_d) [16..31]=sin(y*w_d) [32..47]=cos(x*w_d) [48..63]=sin(x*w_d), w_d = f0 / base^(d/16)
__global__ void rope_table_kernel(const long long* __restrict__ pos, int T, float base, float f0, float* __restrict__ tab) {
  griddep_wait();
  griddep_launch();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T * 32) return;
  const int t = i >> 5, axis = (i >> 4) & 1, d = i & 15;
  const float inv_freq = f0 / powf(base, d / 16.0f);
  const float ang = float(pos[2 * t + axis]) * inv_freq;
  tab[t * 64 + axis * 32 + d] = cosf(ang);
  tab[t * 64 + axis * 32 + 16 + d] = sinf(ang);
}

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// curope contract: one thread per (token, head, pair index); fp32 trig, rounding only at the store.
template <typename T>
__global__ void rope2d_kernel(T* __restrict__ tok, int B, int N, int H, int D, long long sB, long long sN, long long sH,
                              const long long* __restrict__ pos, float base, float fwd) {
  const int Q = D >> 2;
  const long long total = (long long)B * N * H * 2 * Q;
  griddep_wait();
  griddep_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int d = int(i % Q);
    const int axis = int((i / Q) % 2);
    const int h = int((i / (2 * Q)) % H);
    const long long bn = i / (2LL * Q * H);
    const int n = int(bn % N), b = int(bn / N);
    const float inv_freq = fwd / powf(base, d / float(Q));
    const float ang = float(pos[(b * (long long)N + n) * 2 + axis]) * inv_freq;
    const float c = cosf(ang), s = sinf(ang);
    T* p = tok + b * sB + n * sN + h * sH + axis * 2 * Q + d;
    const float u = to_f<T>(p[0]), v = to_f<T>(p[Q]);
    p[0] = from_f<T>(u * c - v * s);
    p[Q] = from_f<T>(v * c + u * s);
  }
}

// ---------------------------------------------------------------------------------------------- patch embed
// out[(v*gh+py)*gw+px][c*256+i*16+j] = img[v][c][py*16+i][px*16+j]; each thread converts 4 consecutive j.
__global__ void __launch_bounds__(256) im2col16_kernel(const float* __restrict__ img, int V, int H, int W,
                                                       uint16_t* __restrict__ out, int is_bf16) {
  const int gw = W >> 4, gh = H >> 4;
  const long long total = (long long)V * 3 * H * (W >> 2);
  griddep_wait();
  griddep_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xq = int(i % (W >> 2));          // float4 index along the image row
    long long r = i / (W >> 2);
    const int y = int(r % H); r /= H;
    const int c = int(r % 3);
    const int v = int(r / 3);
    const float4 t = reinterpret_cast<const float4*>(img + (((long long)v * 3 + c) * H + y) * W)[xq];
    const int px = xq >> 2, j = (xq & 3) << 2, py = y >> 4, ii = y & 15;
    const long long row = ((long long)v * gh + py) * gw + px;
    uint2 w;
    w.x = pack16(t.x, t.y, is_bf16);
    w.y = pack16(t.z, t.w, is_bf16);
    *reinterpret_cast<uint2*>(out + row * 768 + c * 256 + ii * 16 + j) = w;
  }
}

// ---------------------------------------------------------------------------------------------- head
// out[v][16y+i][16x+j][c] = proj[v*N + y*gw + x][c*256 + 16i + j].  One thread per output pixel (C floats).
__global__ void __launch_bounds__(256) unpatchify_kernel(const float* __restrict__ proj, int V, int H, int W, int C,
                                                         float* __restrict__ out) {
  const int gw = W >> 4, gh = H >> 4;
  const long long total = (long long)V * H * W;
  griddep_wait();
  griddep_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int X = int(i % W);
    const int Y = int((i / W) % H);
    const int v = int(i / ((long long)W * H));
    const long long row = ((long long)v * gh + (Y >> 4)) * gw + (X >> 4);
    const float* src = proj + row * (long long)(C * 256) + (Y & 15) * 16 + (X & 15);
    float* dst = out + i * C;
    for (int c = 0; c < C; ++c) dst[c] = src[c * 256];
  }
}

// pts = v / max(|v|,1e-8) * expm1(|v|) for channels 0:3 and 3:6; conf = 1 + exp(ch6)
__global__ void __launch_bounds__(256) postprocess_kernel(const float* __restrict__ pm, long long P,
                                                          float* __restrict__ pts3d, float* __restrict__ local,
                                                          float* __restrict__ conf) {
  griddep_wait();
  griddep_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x) {
    const float* s = pm + i * 7;
    float a[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) a[k] = s[k];
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      const float x = a[3 * g], y = a[3 * g + 1], z = a[3 * g + 2];
      const float d = sqrtf(x * x + y * y + z * z);
      const float f = expm1f(d) / fmaxf(d, 1e-8f);
      float* o = (g == 0 ? pts3d : local) + i * 3;
      o[0] = x * f; o[1] = y * f; o[2] = z * f;
    }
    conf[i] = 1.0f + expf(a[6]);
  }
}

// ---------------------------------------------------------------------------------------------- attention state merge
// Context-parallel cross-attention: every GPU exports the unnormalised (O, m, l) of ITS shard of the memory tokens; the
// states of all shards are merged exactly (same formula as the in-kernel merge of key splits, attention.cu).
struct PartList { const float* o[M3R_MAX_PEERS]; const float2* ml[M3R_MAX_PEERS]; };
__global__ void __launch_bounds__(256) attn_merge_kernel(PartList pl, int n, long long rows, int H, uint16_t* __restrict__ out,
                                                         long long ldo, int is_bf16) {
  griddep_wait();
  griddep_launch();
  const long long total = rows * H * 8;                 // one thread = 8 consecutive output columns of one head
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = int(i & 7);
    const long long rh = i >> 3;                        // row * H + h
    float mk[M3R_MAX_PEERS], lk[M3R_MAX_PEERS];
    float m = -INFINITY;
#pragma unroll
    for (int k = 0; k < M3R_MAX_PEERS; ++k) if (k < n) { const float2 v = __ldcg(pl.ml[k] + rh); mk[k] = v.x; lk[k] = v.y; m = fmaxf(m, v.x); }
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float l = 0.f;
#pragma unroll
    for (int k = 0; k < M3R_MAX_PEERS; ++k) if (k < n) {
      const float w = (mk[k] == -INFINITY) ? 0.f : exp2f(mk[k] - m);
      l = fmaf(lk[k], w, l);
      const float4* o4 = reinterpret_cast<const float4*>(pl.o[k] + rh * 64 + c8 * 8);
      const float4 a = __ldcg(o4), b = __ldcg(o4 + 1);
      acc[0] = fmaf(a.x, w, acc[0]); acc[1] = fmaf(a.y, w, acc[1]); acc[2] = fmaf(a.z, w, acc[2]); acc[3] = fmaf(a.w, w, acc[3]);
      acc[4] = fmaf(b.x, w, acc[4]); acc[5] = fmaf(b.y, w, acc[5]); acc[6] = fmaf(b.z, w, acc[6]); acc[7] = fmaf(b.w, w, acc[7]);
    }
    const float inv = l > 0.f ? 1.0f / l : 0.f;
    const long long row = rh / H;
    const int h = int(rh % H);
    uint4 w4;
    w4.x = pack16(acc[0] * inv, acc[1] * inv, is_bf16); w4.y = pack16(acc[2] * inv, acc[3] * inv, is_bf16);
    w4.z = pack16(acc[4] * inv, acc[5] * inv, is_bf16); w4.w = pack16(acc[6] * inv, acc[7] * inv, is_bf16);
    *reinterpret_cast<uint4*>(out + row * ldo + h * 64 + c8 * 8) = w4;
  }
}

__global__ void __launch_bounds__(256) attn_state_fill_kernel(float4* __restrict__ o, long long n_o4, float2* __restrict__ ml, long long n_ml) {
  griddep_wait();
  griddep_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_o4; i += (long long)gridDim.x * blockDim.x) o[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_ml; i += (long long)gridDim.x * blockDim.x) ml[i] = make_float2(-INFINITY, 0.f);
}

// one source block -> the same offset in n destination buffers (this GPU's and its peers', NVLink stores), 16 B per thread
struct DstList { uint4* p[M3R_MAX_PEERS]; };
__global__ void __launch_bounds__(256) peer_bcast_kernel(const uint4* __restrict__ src, DstList dst, int n, long long n_vec) {
  griddep_wait();
  griddep_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = src[i];
#pragma unroll
    for (int k = 0; k < M3R_MAX_PEERS; ++k) if (k < n) dst.p[k][i] = v;
  }
}

// ---------------------------------------------------------------------------------------------- nearest-neighbour distance
// out[i] = min_j |q_i - p_j| (inf when the database is empty): the keyframe overlap score of the SLAM front end
// (must3r/slam/model.py:62-91) queries a scipy KD-tree on the CPU per frame (must3r/slam/nns.py:57-62); here the database
// points of one viewing-direction quadrant stay on the GPU and are scanned in shared-memory tiles (one query per thread).
__global__ void __launch_bounds__(256) nn_min_dist_kernel(const float* __restrict__ q, int Q, const float* __restrict__ pdb, long long P,
                                                          float* __restrict__ out) {
  __shared__ float sp[1024 * 3];
  griddep_wait();
  griddep_launch();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (i < Q) { qx = q[3 * i]; qy = q[3 * i + 1]; qz = q[3 * i + 2]; }
  float best = INFINITY;
  for (long long base = 0; base < P; base += 1024) {
    const int n = (int)((P - base) < 1024 ? (P - base) : 1024);
    __syncthreads();
    for (int t = threadIdx.x; t < n * 3; t += blockDim.x) sp[t] = pdb[base * 3 + t];
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < n; ++j) {
      const float dx = qx - sp[3 * j], dy = qy - sp[3 * j + 1], dz = qz - sp[3 * j + 2];
      best = fminf(best, fmaf(dx, dx, fmaf(dy, dy, dz * dz)));
    }
  }
  if (i < Q) out[i] = sqrtf(best);
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("%s launch: %s", what, cudaGetErrorString(e));
  count_launch();
  return 0;
}

static int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = (long long)num_sms() * 16;
  return int(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace m3r

using namespace m3r;

// The row kernels move float4 (fp32) and uint2 (16-bit) units: base pointers off that grid are refused before any launch.
static bool misaligned(const void* ptr, unsigned bytes) { return ptr && (reinterpret_cast<uintptr_t>(ptr) % bytes) != 0; }

static int layernorm_impl(const float* x, int64_t ldx, const float* add, int64_t ldadd, int add_rows, int add_period, const float* gamma,
                          const float* beta, float eps, int32_t M, int32_t D, void* out, int64_t ldo,
                          int32_t out_dtype, int32_t is_bf16, void* stream) {
  if (!x || !out) return set_error("layernorm: null pointer");
  if (M <= 0) return 0;
  if (D % 4 || D > 2048 || ldx % 4 || (add && ldadd % 4) || ldo % 4) return set_error("layernorm: D=%d must be a multiple of 4, <= 2048, 16B-aligned rows", D);
  if (misaligned(x, 16) || misaligned(add, 16) || misaligned(gamma, 16) || misaligned(beta, 16))
    return set_error("layernorm: x, add, gamma and beta must be 16-byte aligned (float4 loads)");
  const int out_align = out_dtype == M3R_OUT_F32 ? 16 : out_dtype == M3R_OUT_E4M3 ? 4 : 8;
  if (misaligned(out, out_align)) return set_error("layernorm: out must be %d-byte aligned", out_align);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int wpb = M <= 4096 ? 4 : 8;          // small row counts: more, smaller blocks cover more SMs
  const int grid = (M + wpb - 1) / wpb;
  ProfScope prof(PROF_LN, 0.0, (double)M * D * (4.0 + (add ? 4.0 : 0.0) + (out_dtype == M3R_OUT_E4M3 ? 1.0 : out_dtype ? 2.0 : 4.0)), s);
  if (D <= 1024 && M <= 4096)
    launch_pdl(layernorm_kernel<8, false, true>, dim3(grid), dim3(wpb * 32), 0, s, (const void*)x, (long long)ldx, add, (long long)ldadd, gamma, beta, eps, (int)M, (int)D, out, (long long)ldo, (int)out_dtype, (int)is_bf16, add_rows, add_period);
  else if (D <= 1024)
    launch_pdl(layernorm_kernel<8, false, false>, dim3(grid), dim3(wpb * 32), 0, s, (const void*)x, (long long)ldx, add, (long long)ldadd, gamma, beta, eps, (int)M, (int)D, out, (long long)ldo, (int)out_dtype, (int)is_bf16, add_rows, add_period);
  else
    launch_pdl(layernorm_kernel<16, false, false>, dim3(grid), dim3(wpb * 32), 0, s, (const void*)x, (long long)ldx, add, (long long)ldadd, gamma, beta, eps, (int)M, (int)D, out, (long long)ldo, (int)out_dtype, (int)is_bf16, add_rows, add_period);
  return check_launch("layernorm");
}

extern "C" int m3r_layernorm(const float* x, int64_t ldx, const float* add, int64_t ldadd, const float* gamma,
                             const float* beta, float eps, int32_t M, int32_t D, void* out, int64_t ldo,
                             int32_t out_dtype, int32_t is_bf16, void* stream) {
  if (!gamma || !beta) return set_error("layernorm: null pointer");
  return layernorm_impl(x, ldx, add, ldadd, M, 1 << 30, gamma, beta, eps, M, D, out, ldo, out_dtype, is_bf16, stream);
}

extern "C" int m3r_normalize16(const float* x, int64_t ldx, const float* add, int64_t ldadd, int32_t add_rows, int32_t add_period,
                               float eps, int32_t M, int32_t D, void* out16, int64_t ldo, int32_t is_bf16, void* stream) {
  if (add && (add_rows < 0 || add_period <= 0)) return set_error("normalize16: bad add_rows / add_period");
  return layernorm_impl(x, ldx, add, ldadd, add ? add_rows : 0, add ? add_period : 1, nullptr, nullptr, eps, M, D, out16, ldo, M3R_OUT_16, is_bf16, stream);
}

// Affine-free rows as e4m3: |(x - mean) * rstd| <= sqrt(D - 1) for a row of D values (equality when one value differs
// from all the others), i.e. <= 45 for D <= 2048, well inside e4m3's +-448; the A operand of an e4m3 GEMM needs no scale.
extern "C" int m3r_normalize8(const float* x, int64_t ldx, const float* add, int64_t ldadd, int32_t add_rows, int32_t add_period,
                              float eps, int32_t M, int32_t D, void* out8, int64_t ldo, void* stream) {
  if (add && (add_rows < 0 || add_period <= 0)) return set_error("normalize8: bad add_rows / add_period");
  return layernorm_impl(x, ldx, add, ldadd, add ? add_rows : 0, add ? add_period : 1, nullptr, nullptr, eps, M, D, out8, ldo, M3R_OUT_E4M3, 0, stream);
}

extern "C" int m3r_layernorm16(const void* x16, int64_t ldx, const float* gamma, const float* beta, float eps, int32_t M,
                               int32_t D, void* out16, int64_t ldo, int32_t is_bf16, void* stream) {
  if (!x16 || !gamma || !beta || !out16) return set_error("layernorm16: null pointer");
  if (M <= 0) return 0;
  if (D % 4 || D > 2048 || ldx % 4 || ldo % 4) return set_error("layernorm16: D=%d must be a multiple of 4, <= 2048, 8B-aligned rows", D);
  if (misaligned(x16, 8) || misaligned(out16, 8)) return set_error("layernorm16: x16 and out16 must be 8-byte aligned");
  if (misaligned(gamma, 16) || misaligned(beta, 16)) return set_error("layernorm16: gamma and beta must be 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int wpb = M <= 4096 ? 4 : 8;
  const int grid = (M + wpb - 1) / wpb;
  ProfScope prof(PROF_LN, 0.0, (double)M * D * 4.0, s);
  const float* none = nullptr;
  if (D <= 1024)
    launch_pdl(layernorm_kernel<8, true, false>, dim3(grid), dim3(wpb * 32), 0, s, x16, (long long)ldx, none, 0LL, gamma, beta, eps, (int)M, (int)D, out16, (long long)ldo, 1, (int)is_bf16, 0, 1);
  else
    launch_pdl(layernorm_kernel<16, true, false>, dim3(grid), dim3(wpb * 32), 0, s, x16, (long long)ldx, none, 0LL, gamma, beta, eps, (int)M, (int)D, out16, (long long)ldo, 1, (int)is_bf16, 0, 1);
  return check_launch("layernorm16");
}

static int cast16_impl(const float* x, int64_t ldx, const float* add, int64_t ldadd, int32_t M, int32_t D, void* out, int64_t ldo,
                       int32_t is_bf16, void* stream) {
  if (!x || !out) return set_error("cast16: null pointer");
  if (M <= 0) return 0;
  if (D % 4 || ldx % 4 || ldo % 4 || (add && ldadd % 4)) return set_error("cast16: alignment");
  if (misaligned(x, 16) || misaligned(add, 16)) return set_error("cast16: x and add must be 16-byte aligned (float4 loads)");
  if (misaligned(out, 8)) return set_error("cast16: out must be 8-byte aligned");
  launch_pdl(cast16_kernel, dim3(grid_for((long long)M * (D / 4), 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
             x, (long long)ldx, add, (long long)ldadd, (int)M, (int)D, reinterpret_cast<uint16_t*>(out), (long long)ldo, (int)is_bf16);
  return check_launch("cast16");
}

extern "C" int m3r_cast16(const float* x, int64_t ldx, int32_t M, int32_t D, void* out, int64_t ldo, int32_t is_bf16,
                          void* stream) {
  return cast16_impl(x, ldx, nullptr, 0, M, D, out, ldo, is_bf16, stream);
}

extern "C" int m3r_add_cast16(const float* x, int64_t ldx, const float* add, int64_t ldadd, int32_t M, int32_t D, void* out,
                              int64_t ldo, int32_t is_bf16, void* stream) {
  return cast16_impl(x, ldx, add, ldadd, M, D, out, ldo, is_bf16, stream);
}

extern "C" int m3r_rope_table(const int64_t* pos, int32_t T, float base, float f0, float* tab, void* stream) {
  if (!pos || !tab) return set_error("rope_table: null pointer");
  if (T <= 0) return 0;
  launch_pdl(rope_table_kernel, dim3((T * 32 + 255) / 256), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
             reinterpret_cast<const long long*>(pos), (int)T, base, f0, tab);
  return check_launch("rope_table");
}

extern "C" int m3r_rope_2d(void* tokens, int32_t dtype, int32_t B, int32_t N, int32_t H, int32_t D, int64_t sB,
                           int64_t sN, int64_t sH, const int64_t* pos, float base, float fwd, void* stream) {
  if (!tokens || !pos) return set_error("rope_2d: null pointer");
  if (B < 0 || N < 0 || H < 0 || D < 0) return set_error("rope_2d: negative dimension (B=%d, N=%d, H=%d, D=%d)", B, N, H, D);
  if (D % 4) return set_error("rope_2d: token dim must be multiple of 4");   // kernels.cu:94
  const long long total = (long long)B * N * H * (D / 2);
  if (total <= 0) return 0;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int grid = grid_for(total, 256);
  const long long* p = reinterpret_cast<const long long*>(pos);
  if (dtype == 0) launch_pdl(rope2d_kernel<float>, dim3(grid), dim3(256), 0, s, reinterpret_cast<float*>(tokens), (int)B, (int)N, (int)H, (int)D, (long long)sB, (long long)sN, (long long)sH, p, base, fwd);
  else if (dtype == 1) launch_pdl(rope2d_kernel<__half>, dim3(grid), dim3(256), 0, s, reinterpret_cast<__half*>(tokens), (int)B, (int)N, (int)H, (int)D, (long long)sB, (long long)sN, (long long)sH, p, base, fwd);
  else if (dtype == 2) launch_pdl(rope2d_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, s, reinterpret_cast<__nv_bfloat16*>(tokens), (int)B, (int)N, (int)H, (int)D, (long long)sB, (long long)sN, (long long)sH, p, base, fwd);
  else return set_error("rope_2d: bad dtype %d", dtype);
  return check_launch("rope_2d");
}

extern "C" int m3r_im2col16(const float* img, int32_t V, int32_t H, int32_t W, void* out, int32_t is_bf16, void* stream) {
  if (!img || !out) return set_error("im2col16: null pointer");
  if (H % 16 || W % 16) return set_error("im2col16: image size (%d,%d) is not a multiple of the patch size 16", H, W);
  if (misaligned(img, 16)) return set_error("im2col16: img must be 16-byte aligned (float4 loads)");
  if (misaligned(out, 8)) return set_error("im2col16: out must be 8-byte aligned");
  if (V <= 0) return 0;
  launch_pdl(im2col16_kernel, dim3(grid_for((long long)V * 3 * H * (W / 4), 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
             img, (int)V, (int)H, (int)W, reinterpret_cast<uint16_t*>(out), (int)is_bf16);
  return check_launch("im2col16");
}

extern "C" int m3r_unpatchify(const float* proj, int32_t V, int32_t H, int32_t W, int32_t C, float* out, void* stream) {
  if (!proj || !out) return set_error("unpatchify: null pointer");
  if (H % 16 || W % 16) return set_error("unpatchify: bad image size");
  if (C < 1) return set_error("unpatchify: C=%d channels, must be >= 1", C);
  if (V <= 0) return 0;
  launch_pdl(unpatchify_kernel, dim3(grid_for((long long)V * H * W, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), proj, (int)V, (int)H, (int)W, (int)C, out);
  return check_launch("unpatchify");
}

extern "C" int m3r_postprocess(const float* pm, int64_t P, float* pts3d, float* pts3d_local, float* conf, void* stream) {
  if (!pm || !pts3d || !pts3d_local || !conf) return set_error("postprocess: null pointer");
  if (P <= 0) return 0;
  launch_pdl(postprocess_kernel, dim3(grid_for(P, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), pm, (long long)P, pts3d, pts3d_local, conf);
  return check_launch("postprocess");
}

extern "C" int m3r_attn_merge(const float* const* parts_o, const float* const* parts_ml, int32_t n, int64_t rows, int32_t H,
                              void* out, int64_t ldo, int32_t is_bf16, void* stream) {
  if (!parts_o || !parts_ml || !out || n < 1 || n > M3R_MAX_PEERS) return set_error("attn_merge: 1..%d states", M3R_MAX_PEERS);
  if (rows <= 0) return 0;
  if (ldo % 8) return set_error("attn_merge: ldo must be a multiple of 8");
  for (int k = 0; k < n; ++k) {
    if (!parts_o[k] || misaligned(parts_o[k], 16)) return set_error("attn_merge: parts_o[%d] must be a 16-byte aligned pointer", k);
    if (!parts_ml[k] || misaligned(parts_ml[k], 8)) return set_error("attn_merge: parts_ml[%d] must be an 8-byte aligned pointer", k);
  }
  if (misaligned(out, 16)) return set_error("attn_merge: out must be 16-byte aligned");
  PartList pl;
  for (int k = 0; k < M3R_MAX_PEERS; ++k) { pl.o[k] = k < n ? parts_o[k] : nullptr; pl.ml[k] = k < n ? reinterpret_cast<const float2*>(parts_ml[k]) : nullptr; }
  launch_pdl(attn_merge_kernel, dim3(grid_for(rows * H * 8, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), pl, (int)n,
             (long long)rows, (int)H, reinterpret_cast<uint16_t*>(out), (long long)ldo, (int)is_bf16);
  return check_launch("attn_merge");
}

extern "C" int m3r_attn_state_fill(float* export_o, float* export_ml, int64_t rows, int32_t H, void* stream) {
  if (!export_o || !export_ml) return set_error("attn_state_fill: null pointer");
  if (misaligned(export_o, 16)) return set_error("attn_state_fill: export_o must be 16-byte aligned (float4 stores)");
  if (misaligned(export_ml, 8)) return set_error("attn_state_fill: export_ml must be 8-byte aligned (float2 stores)");
  if (rows <= 0) return 0;
  launch_pdl(attn_state_fill_kernel, dim3(grid_for(rows * H * 16, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
             reinterpret_cast<float4*>(export_o), (long long)(rows * H * 16), reinterpret_cast<float2*>(export_ml), (long long)(rows * H));
  return check_launch("attn_state_fill");
}

extern "C" int m3r_peer_bcast(const void* src, void* const* dsts, int32_t n, int64_t bytes, void* stream) {
  if (!src || !dsts || n < 1 || n > M3R_MAX_PEERS || bytes % 16) return set_error("peer_bcast: 1..%d destinations, bytes %% 16 == 0", M3R_MAX_PEERS);
  if (misaligned(src, 16)) return set_error("peer_bcast: src must be 16-byte aligned (uint4 loads)");
  for (int k = 0; k < n; ++k)
    if (!dsts[k] || misaligned(dsts[k], 16)) return set_error("peer_bcast: dsts[%d] must be a non-null, 16-byte aligned pointer", k);
  if (bytes <= 0) return 0;
  DstList dl;
  for (int k = 0; k < M3R_MAX_PEERS; ++k) dl.p[k] = k < n ? reinterpret_cast<uint4*>(dsts[k]) : nullptr;
  launch_pdl(peer_bcast_kernel, dim3(grid_for(bytes / 16, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
             reinterpret_cast<const uint4*>(src), dl, (int)n, (long long)(bytes / 16));
  return check_launch("peer_bcast");
}

extern "C" int m3r_nn_min_dist(const float* queries, int32_t Q, const float* db, int64_t P, float* out, void* stream) {
  if (!queries || !out || (P > 0 && !db)) return set_error("nn_min_dist: null pointer");
  if (Q <= 0) return 0;
  launch_pdl(nn_min_dist_kernel, dim3((Q + 255) / 256), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), queries, (int)Q, db, (long long)P, out);
  return check_launch("nn_min_dist");
}
