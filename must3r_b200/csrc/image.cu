// Input preprocessing: RGB uint8 frames (HWC, arbitrary row pitch) -> the encoder's fp32 [V,3,h,w] images, in two
// separable passes (horizontal, then vertical) whose per-column / per-row coefficient tables are computed on the host
// (must3r_b200/engine/images.py).  One thread per output pixel (all three channels); a launch covers V frames.
//
//  * m3r_resample_pil_u8: Pillow's 8-bit resampler (Image.resize with LANCZOS / BICUBIC) bit for bit.  The weights are
//    int32 with 22 fractional bits; each pass starts its accumulator at 0.5 (1 << 21), shifts right by 22 and clamps
//    to 0..255, and the horizontal pass stores an 8-bit intermediate, as Pillow does.  The vertical pass fuses the
//    crop box and ImgNorm.
//  * m3r_resize_aa_bilinear_u8: aten's antialiased bilinear resize (_upsample_bilinear2d_aa) of the ImgNorm'ed image,
//    fp32 weights and accumulation, normalising the uint8 input inline.
#include "ptx.cuh"
#include "m3r_internal.h"

namespace m3r {

// ImgNorm = ToTensor then Normalize(0.5, 0.5): (x / 255 - 0.5) / 0.5 in fp32, in that order, with IEEE divisions
// (torchvision's arithmetic; the result is bitwise the host transform's).
__device__ __forceinline__ float img_norm(int v) {
  return __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.f), 0.5f), 0.5f);
}

__device__ __forceinline__ int clip8(int acc) {
  const int v = acc >> 22;                       // arithmetic shift: floor, as Pillow's clip8 lookup
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// tmp[v, r, x, c] = clip8(0.5 + sum_k src[v, row0 + r, b0(x) + k, c] * w[x, k])
__global__ void __launch_bounds__(128) pil_horiz_kernel(const uint8_t* __restrict__ src, long long pitch, long long vstride,
                                                        int row0, int rows, int out_w, const int* __restrict__ xb,
                                                        const int* __restrict__ xw, int xk, uint8_t* __restrict__ tmp) {
  griddep_wait();
  griddep_launch();
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= out_w) return;
  const int r = blockIdx.y, v = blockIdx.z;
  const uint8_t* s = src + v * vstride + (long long)(row0 + r) * pitch + 3 * __ldg(xb + 2 * x);
  const int n = __ldg(xb + 2 * x + 1);
  const int* w = xw + (long long)x * xk;
  int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
  for (int k = 0; k < n; ++k) {
    const int c = __ldg(w + k);
    a0 += (int)s[3 * k] * c;
    a1 += (int)s[3 * k + 1] * c;
    a2 += (int)s[3 * k + 2] * c;
  }
  uint8_t* o = tmp + (((long long)v * rows + r) * out_w + x) * 3;
  o[0] = (uint8_t)clip8(a0);
  o[1] = (uint8_t)clip8(a1);
  o[2] = (uint8_t)clip8(a2);
}

// p = clip8(0.5 + sum_k tmp[v, b0(y) + k, x, c] * w[y, k]); out_u8[v, y, x, c] = p (optional) and, inside the crop box,
// out[v, c, y - cy, x - cx] = ImgNorm(p) (optional)
__global__ void __launch_bounds__(128) pil_vert_kernel(const uint8_t* __restrict__ tmp, int rows, int out_w, int out_h,
                                                       const int* __restrict__ yb, const int* __restrict__ yw, int yk,
                                                       uint8_t* __restrict__ out_u8, int cx, int cy, int cw, int ch,
                                                       float* __restrict__ out) {
  griddep_wait();
  griddep_launch();
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= out_w) return;
  const int y = blockIdx.y, v = blockIdx.z;
  const long long rstride = (long long)out_w * 3;
  const uint8_t* t = tmp + (long long)v * rows * rstride + (long long)__ldg(yb + 2 * y) * rstride + 3 * x;
  const int n = __ldg(yb + 2 * y + 1);
  const int* w = yw + (long long)y * yk;
  int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
  for (int k = 0; k < n; ++k) {
    const int c = __ldg(w + k);
    a0 += (int)t[k * rstride] * c;
    a1 += (int)t[k * rstride + 1] * c;
    a2 += (int)t[k * rstride + 2] * c;
  }
  const int p0 = clip8(a0), p1 = clip8(a1), p2 = clip8(a2);
  if (out_u8) {
    uint8_t* o = out_u8 + (((long long)v * out_h + y) * out_w + x) * 3;
    o[0] = (uint8_t)p0; o[1] = (uint8_t)p1; o[2] = (uint8_t)p2;
  }
  const int yy = y - cy, xx = x - cx;
  if (out && yy >= 0 && yy < ch && xx >= 0 && xx < cw) {
    const long long plane = (long long)ch * cw;
    float* o = out + (long long)v * 3 * plane + (long long)yy * cw + xx;
    o[0] = img_norm(p0);
    o[plane] = img_norm(p1);
    o[2 * plane] = img_norm(p2);
  }
}

// tmp[v, c, r, x] = sum_k ImgNorm(src[v, r, b0(x) + k, c]) * w[x, k]   (fp32, planar)
__global__ void __launch_bounds__(128) aa_horiz_kernel(const uint8_t* __restrict__ src, long long pitch, long long vstride,
                                                       int rows, int out_w, const int* __restrict__ xb,
                                                       const float* __restrict__ xw, int xk, float* __restrict__ tmp) {
  griddep_wait();
  griddep_launch();
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= out_w) return;
  const int r = blockIdx.y, v = blockIdx.z;
  const uint8_t* s = src + v * vstride + (long long)r * pitch + 3 * __ldg(xb + 2 * x);
  const int n = __ldg(xb + 2 * x + 1);
  const float* w = xw + (long long)x * xk;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int k = 0; k < n; ++k) {
    const float c = __ldg(w + k);
    a0 += img_norm(s[3 * k]) * c;
    a1 += img_norm(s[3 * k + 1]) * c;
    a2 += img_norm(s[3 * k + 2]) * c;
  }
  const long long plane = (long long)rows * out_w;
  float* o = tmp + (long long)v * 3 * plane + (long long)r * out_w + x;
  o[0] = a0;
  o[plane] = a1;
  o[2 * plane] = a2;
}

// out[v, c, y, x] = sum_k tmp[v, c, b0(y) + k, x] * w[y, k]
__global__ void __launch_bounds__(128) aa_vert_kernel(const float* __restrict__ tmp, int rows, int out_w, int out_h,
                                                      const int* __restrict__ yb, const float* __restrict__ yw, int yk,
                                                      float* __restrict__ out) {
  griddep_wait();
  griddep_launch();
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= out_w) return;
  const int y = blockIdx.y, v = blockIdx.z;
  const long long tplane = (long long)rows * out_w, oplane = (long long)out_h * out_w;
  const float* t = tmp + (long long)v * 3 * tplane + (long long)__ldg(yb + 2 * y) * out_w + x;
  const int n = __ldg(yb + 2 * y + 1);
  const float* w = yw + (long long)y * yk;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int k = 0; k < n; ++k) {
    const float c = __ldg(w + k);
    a0 += t[(long long)k * out_w] * c;
    a1 += t[tplane + (long long)k * out_w] * c;
    a2 += t[2 * tplane + (long long)k * out_w] * c;
  }
  float* o = out + (long long)v * 3 * oplane + (long long)y * out_w + x;
  o[0] = a0;
  o[oplane] = a1;
  o[2 * oplane] = a2;
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("%s launch: %s", what, cudaGetErrorString(e));
  count_launch();
  return 0;
}

static int check_frames(const char* what, const void* src, int64_t pitch, int64_t vstride, int32_t V, int32_t h, int32_t w) {
  if (!src) return set_error("%s: null source", what);
  if (V > 65535) return set_error("%s: %d frames in one call (at most 65535)", what, V);
  if (h <= 0 || w <= 0 || h > 65535) return set_error("%s: bad source size %dx%d", what, w, h);
  if (pitch < 3LL * w) return set_error("%s: row pitch %lld is less than 3 * width %d", what, (long long)pitch, w);
  if (V > 1 && vstride < pitch * h && vstride > -pitch * h) return set_error("%s: frames overlap (frame stride %lld)", what, (long long)vstride);
  return 0;
}

}  // namespace m3r

using namespace m3r;

extern "C" int m3r_resample_pil_u8(const uint8_t* src, int64_t src_pitch, int64_t src_vstride, int32_t V, int32_t src_h,
                                   int32_t src_w, const int32_t* xbounds, const int32_t* xweights, int32_t xk, int32_t out_w,
                                   const int32_t* ybounds, const int32_t* yweights, int32_t yk, int32_t out_h, int32_t row0,
                                   int32_t rows, uint8_t* tmp, uint8_t* out_u8, int32_t crop_x, int32_t crop_y,
                                   int32_t crop_w, int32_t crop_h, float* out, void* stream) {
  if (V <= 0) return 0;
  if (int rc = check_frames("resample_pil_u8", src, src_pitch, src_vstride, V, src_h, src_w)) return rc;
  if (!xbounds || !xweights || !ybounds || !yweights || !tmp) return set_error("resample_pil_u8: null pointer");
  if (!out_u8 && !out) return set_error("resample_pil_u8: no output");
  if (xk <= 0 || yk <= 0 || out_w <= 0 || out_h <= 0 || out_h > 65535) return set_error("resample_pil_u8: bad output size %dx%d", out_w, out_h);
  if (row0 < 0 || rows <= 0 || row0 + rows > src_h) return set_error("resample_pil_u8: source rows [%d,%d) outside [0,%d)", row0, row0 + rows, src_h);
  if (rows > 65535) return set_error("resample_pil_u8: %d source rows", rows);
  if (out && (crop_x < 0 || crop_y < 0 || crop_w <= 0 || crop_h <= 0 || crop_x + crop_w > out_w || crop_y + crop_h > out_h))
    return set_error("resample_pil_u8: crop box (%d,%d,%d,%d) outside the %dx%d resized image", crop_x, crop_y, crop_x + crop_w,
                     crop_y + crop_h, out_w, out_h);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  ProfScope prof(PROF_OTHER, 0.0, (double)V * ((double)rows * src_pitch + (double)out_h * out_w * 3 * 2 + (out ? 12.0 * crop_w * crop_h : 0.0)), s);
  const int bx = (out_w + 127) / 128;
  launch_pdl(pil_horiz_kernel, dim3(bx, rows, V), dim3(128), 0, s, src, (long long)src_pitch, (long long)src_vstride, (int)row0,
             (int)rows, (int)out_w, (const int*)xbounds, (const int*)xweights, (int)xk, tmp);
  if (int rc = check_launch("resample_pil_u8 (horizontal pass)")) return rc;
  launch_pdl(pil_vert_kernel, dim3(bx, out_h, V), dim3(128), 0, s, (const uint8_t*)tmp, (int)rows, (int)out_w, (int)out_h,
             (const int*)ybounds, (const int*)yweights, (int)yk, out_u8, (int)crop_x, (int)crop_y, (int)crop_w, (int)crop_h, out);
  return check_launch("resample_pil_u8 (vertical pass)");
}

extern "C" int m3r_resize_aa_bilinear_u8(const uint8_t* src, int64_t src_pitch, int64_t src_vstride, int32_t V, int32_t src_h,
                                         int32_t src_w, const int32_t* xbounds, const float* xweights, int32_t xk,
                                         int32_t out_w, const int32_t* ybounds, const float* yweights, int32_t yk,
                                         int32_t out_h, float* tmp, float* out, void* stream) {
  if (V <= 0) return 0;
  if (int rc = check_frames("resize_aa_bilinear_u8", src, src_pitch, src_vstride, V, src_h, src_w)) return rc;
  if (!xbounds || !xweights || !ybounds || !yweights || !tmp || !out) return set_error("resize_aa_bilinear_u8: null pointer");
  if (xk <= 0 || yk <= 0 || out_w <= 0 || out_h <= 0 || out_h > 65535)
    return set_error("resize_aa_bilinear_u8: bad output size %dx%d", out_w, out_h);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  ProfScope prof(PROF_OTHER, 0.0, (double)V * ((double)src_h * src_pitch + 24.0 * src_h * out_w + 12.0 * out_h * out_w), s);
  const int bx = (out_w + 127) / 128;
  launch_pdl(aa_horiz_kernel, dim3(bx, src_h, V), dim3(128), 0, s, src, (long long)src_pitch, (long long)src_vstride,
             (int)src_h, (int)out_w, (const int*)xbounds, xweights, (int)xk, tmp);
  if (int rc = check_launch("resize_aa_bilinear_u8 (horizontal pass)")) return rc;
  launch_pdl(aa_vert_kernel, dim3(bx, out_h, V), dim3(128), 0, s, (const float*)tmp, (int)src_h, (int)out_w, (int)out_h,
             (const int*)ybounds, yweights, (int)yk, out);
  return check_launch("resize_aa_bilinear_u8 (vertical pass)");
}
