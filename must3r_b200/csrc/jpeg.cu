// Baseline JPEG decoding, bit for bit what Pillow gives (libjpeg-turbo with JDCT_ISLOW and fancy upsampling).
//
// Host (plain C++, called through ctypes with the GIL released): the header parser (markers, colour space as libjpeg's
// default_decompress_parms, orientation as Pillow's getexif, eligibility) and one linear pass over the entropy-coded
// data that unstuffs it (FF 00 -> FF), drops the restart markers and records where each restart segment starts.
//
// Device, one launch sequence per batch of images of any sizes and samplings:
//  1. Huffman decoding by self-synchronisation (Weissenberger & Schmidt, ICPP 2018 / HiPC 2021).  Each restart segment
//     is cut into SUB_BITS-bit subsequences, one thread each.  The decoder state is (bit offset, block within the MCU,
//     zig-zag index).  jpeg_spec_kernel decodes every subsequence from an assumed state (the segment's first one from
//     its known start); jpeg_sync_kernel rounds re-decode from a predecessor's exit state, walking on into the next
//     subsequences until the states meet, until no entry state changes (every round fixes at least the first wrong
//     subsequence of each segment for good; a batch that needs more
//     than SYNC_ROUNDS rounds is reported with M3R_JPEG_ESYNC and decoded by Pillow); 
//     jpeg_recount_kernel checks the chain without races and counts each subsequence's blocks; a segmented scan of the
//     blocks each subsequence completes gives its first block; jpeg_write_kernel stores de-zigzagged coefficients and DC
//     differences; jpeg_dc_kernel turns the differences into values with a per-component scan that restarts at every
//     restart segment.
//  2. jpeg_idct_kernel: dequantisation and jidctint.c's jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2, 64-bit JLONG
//     arithmetic, DESCALE rounding, range_limit[x & RANGE_MASK]), one thread per block.
//  3. jpeg_color_kernel: jdsample.c's fancy upsampling (h2v1, h1v2, h2v2; box when the downsampled width is <= 2 for
//     the h2 cases) with edge replication at the downsampled size, jdcolor.c's YCbCr->RGB tables (ONE_HALF rounding),
//     gray replicated to RGB, and the EXIF transpose applied on the store.
// No kernel reads outside its image's prepared buffer or writes outside its image's output and workspace; a malformed
// stream sets that image's status word.
#include <string.h>
#include <algorithm>
#include "m3r_internal.h"

namespace m3r {

constexpr int SUB_BITS = 2048;       // subsequence length of the parallel Huffman decoder
constexpr int SYNC_ROUNDS = 32;      // synchronisation rounds before an image is handed back as M3R_JPEG_ESYNC
constexpr int SLACK = 8;             // zero bytes after each stream: the bit reader may look 40 bits ahead

struct JHuff {
  uint16_t lut[512];                 // 9-bit lookahead: (length << 8) | symbol, 0 = longer code
  int32_t maxcode[18];               // largest code of each length, -1 if none
  int32_t valoff[18];                // vals index of a code of that length = code + valoff
  uint8_t vals[256];
};

struct JTables {
  uint16_t qt[3][64];                // per component, natural order
  JHuff dc[3], ac[3];                // per component
  uint8_t blk_comp[10], blk_x[10], blk_y[10];
  uint8_t pad[2];
};

struct JSeg { uint32_t start, end; };             // bits of the unstuffed stream
struct JSub { uint32_t start, end, seg, pad; };

__constant__ uint8_t c_natural[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
static const uint8_t h_natural[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ============================================================================================ host: headers
struct RawHuff { bool defined = false; uint8_t bits[17] = {}; uint8_t vals[256] = {}; };
struct Header {
  m3r_jpeg_info info;
  uint16_t qt[4][64];
  bool qt_defined[4] = {};
  RawHuff dc[4], ac[4];
  int comp_id[3], comp_tq[3], comp_td[3], comp_ta[3];
};

static int rd16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// EXIF IFD0 orientation: 0 when absent; -1 when the TIFF data or the tag is not the plain SHORT Pillow certainly reads.
static int exif_orientation(const uint8_t* d, int64_t n) {
  if (n < 8) return -1;
  bool le;
  if (d[0] == 'I' && d[1] == 'I') le = true;
  else if (d[0] == 'M' && d[1] == 'M') le = false;
  else return -1;
  auto u16 = [&](int64_t o) -> int { return le ? (d[o] | (d[o + 1] << 8)) : ((d[o] << 8) | d[o + 1]); };
  auto u32 = [&](int64_t o) -> int64_t {
    return le ? ((int64_t)d[o] | ((int64_t)d[o + 1] << 8) | ((int64_t)d[o + 2] << 16) | ((int64_t)d[o + 3] << 24))
              : (((int64_t)d[o] << 24) | ((int64_t)d[o + 1] << 16) | ((int64_t)d[o + 2] << 8) | (int64_t)d[o + 3]);
  };
  if (u16(2) != 42) return -1;
  const int64_t ifd = u32(4);
  if (ifd < 8 || ifd + 2 > n) return -1;
  const int cnt = u16(ifd);
  if (ifd + 2 + 12LL * cnt > n) return -1;
  int found = 0;
  for (int k = 0; k < cnt; ++k) {
    const int64_t e = ifd + 2 + 12LL * k;
    if (u16(e) != 0x0112) continue;
    if (found || u16(e + 2) != 3 || u32(e + 4) != 1) return -1;
    found = u16(e + 8);
    if (found == 0) return -1;
  }
  return found;
}

// Pillow's XMP fallback: the first match of rb'tiff:Orientation(="|>)([0-9])'; 0 when there is none.
static int xmp_orientation(const uint8_t* d, int64_t n) {
  static const char key[] = "tiff:Orientation";
  const int64_t kl = sizeof(key) - 1;
  for (int64_t i = 0; i + kl < n; ++i) {
    if (memcmp(d + i, key, kl) != 0) continue;
    const int64_t j = i + kl;
    if (j + 2 < n && d[j] == '=' && d[j + 1] == '"' && d[j + 2] >= '0' && d[j + 2] <= '9') return d[j + 2] - '0' ? d[j + 2] - '0' : 10;
    if (j + 1 < n && d[j] == '>' && d[j + 1] >= '0' && d[j + 1] <= '9') return d[j + 1] - '0' ? d[j + 1] - '0' : 10;
  }
  return 0;
}

// libjpeg's jpeg_make_d_derived_tbl checks, then the decoder's tables; false for a table libjpeg rejects
static bool build_huff(const RawHuff& r, bool dc, JHuff& t) {
  memset(&t, 0, sizeof(t));
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    t.maxcode[l] = -1;
    if (code + r.bits[l] >= (1 << l)) return false;   // JERR_BAD_HUFF_TABLE: no code may be all ones (checked
                                                       // before the lookahead table is filled)
    if (r.bits[l]) {
      t.valoff[l] = k - code;
      for (int j = 0; j < r.bits[l]; ++j, ++k, ++code) {
        if (l <= 9)
          for (int s = 0; s < (1 << (9 - l)); ++s) t.lut[(code << (9 - l)) | s] = (uint16_t)((l << 8) | r.vals[k]);
      }
      t.maxcode[l] = code - 1;
    }
    code <<= 1;
  }
  if (dc)
    for (int j = 0; j < k; ++j)
      if (r.vals[j] > 15) return false;
  memcpy(t.vals, r.vals, 256);
  return true;
}

static int parse_header(const uint8_t* data, int64_t size, Header& h) {
  memset(&h.info, 0, sizeof(h.info));
  m3r_jpeg_info& info = h.info;
  info.orientation = 1;
  info.orientation_exact = 1;
  if (!data || size < 4 || data[0] != 0xFF || data[1] != 0xD8) return 1;
  bool jfif = false, adobe = false, sof = false, ok = true;
  int adobe_transform = -1, exif_o = 0, exif_segments = 0, xmp_o = 0, nxmp = 0;
  int64_t i = 2;
  for (;;) {
    if (i >= size || data[i] != 0xFF) { ok = false; break; }
    while (i < size && data[i] == 0xFF) ++i;
    if (i >= size) { ok = false; break; }
    const int m = data[i++];
    if (m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01 || m == 0xD8) { ok = false; break; }   // no scan
    if (i + 2 > size) { ok = false; break; }
    const int len = rd16(data + i);
    if (len < 2 || i + len > size) { ok = false; break; }
    const uint8_t* p = data + i + 2;
    const int n = len - 2;
    i += len;
    if (m == 0xE0) {
      if (n >= 14 && memcmp(p, "JFIF\0", 5) == 0) jfif = true;
    } else if (m == 0xEE) {
      if (n >= 12 && memcmp(p, "Adobe", 5) == 0) { adobe = true; adobe_transform = p[11]; }
    } else if (m == 0xE1) {
      if (n >= 6 && memcmp(p, "Exif\0\0", 6) == 0) {
        if (++exif_segments == 1) exif_o = exif_orientation(p + 6, n - 6);
      } else {
        static const char ns[] = "http://ns.adobe.com/xap/1.0/";
        if (n >= (int)sizeof(ns) && memcmp(p, ns, sizeof(ns)) == 0) {   // the prefix and its NUL
          ++nxmp;
          xmp_o = xmp_orientation(p + sizeof(ns), n - (int)sizeof(ns));
        }
      }
    } else if (m == 0xDB) {
      int o = 0;
      while (o < n) {
        const int pq = p[o] >> 4, tq = p[o] & 15;
        ++o;
        if (pq > 1 || tq > 3 || o + 64 * (pq + 1) > n) { ok = false; break; }
        for (int k = 0; k < 64; ++k) h.qt[tq][h_natural[k]] = pq ? (uint16_t)rd16(p + o + 2 * k) : p[o + k];
        h.qt_defined[tq] = true;
        o += 64 * (pq + 1);
      }
      if (!ok) break;
    } else if (m == 0xC4) {
      int o = 0;
      while (o < n) {
        const int tc = p[o] >> 4, th = p[o] & 15;
        if (tc > 1 || th > 3 || o + 17 > n) { ok = false; break; }
        RawHuff& t = tc ? h.ac[th] : h.dc[th];
        int total = 0;
        for (int l = 1; l <= 16; ++l) total += (t.bits[l] = p[o + l]);
        o += 17;
        if (total > 256 || o + total > n) { ok = false; break; }
        memset(t.vals, 0, sizeof(t.vals));
        memcpy(t.vals, p + o, total);
        t.defined = true;
        o += total;
      }
      if (!ok) break;
    } else if (m == 0xDD) {
      if (n < 2) { ok = false; break; }
      info.restart_interval = rd16(p);
    } else if (m == 0xC0 || m == 0xC1) {
      if (sof || n < 6) { ok = false; break; }
      sof = true;
      if (p[0] != 8) ok = false;
      info.height = rd16(p + 1);
      info.width = rd16(p + 3);
      info.ncomp = p[5];
      if (info.ncomp != 1 && info.ncomp != 3) { ok = false; break; }
      if (n < 6 + 3 * info.ncomp) { ok = false; break; }
      for (int c = 0; c < info.ncomp; ++c) {
        h.comp_id[c] = p[6 + 3 * c];
        info.hs[c] = p[7 + 3 * c] >> 4;
        info.vs[c] = p[7 + 3 * c] & 15;
        h.comp_tq[c] = p[8 + 3 * c];
        if (info.hs[c] < 1 || info.hs[c] > 4 || info.vs[c] < 1 || info.vs[c] > 4 || h.comp_tq[c] > 3) ok = false;
      }
    } else if ((m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8) || m == 0xCC) {
      ok = false;     // progressive, lossless, hierarchical or arithmetic-coded
      break;
    } else if (m == 0xDA) {
      if (!sof || n < 1) { ok = false; break; }
      const int ns = p[0];
      if (ns != info.ncomp || n < 4 + 2 * ns) { ok = false; break; }
      for (int c = 0; c < ns; ++c) {
        if (p[1 + 2 * c] != h.comp_id[c]) ok = false;      // the scan's component order is the frame's
        h.comp_td[c] = p[2 + 2 * c] >> 4;
        h.comp_ta[c] = p[2 + 2 * c] & 15;
        if (h.comp_td[c] > 3 || h.comp_ta[c] > 3) ok = false;
      }
      const uint8_t* q = p + 1 + 2 * ns;
      if (q[0] != 0 || q[1] != 63 || q[2] != 0) ok = false;
      info.scan_offset = i;
      break;
    }
  }
  // orientation, as Pillow's getexif: the first Exif segment's IFD0 tag, else the last XMP packet's tiff:Orientation
  if (exif_segments > 1 || exif_o < 0 || nxmp > 1) info.orientation_exact = 0;
  const int o = exif_o > 0 ? exif_o : xmp_o;
  info.orientation = (o >= 1 && o <= 8) ? o : 1;
  if (!ok || !sof || info.scan_offset == 0 || info.width <= 0 || info.height <= 0) return 0;
  if (size - info.scan_offset >= (1LL << 28)) return 0;
  for (int c = 0; c < info.ncomp; ++c) {
    if (!h.qt_defined[h.comp_tq[c]] || !h.dc[h.comp_td[c]].defined || !h.ac[h.comp_ta[c]].defined) return 0;
    JHuff t;                                           // a table libjpeg rejects makes Pillow raise: not eligible
    if (!build_huff(h.dc[h.comp_td[c]], true, t) || !build_huff(h.ac[h.comp_ta[c]], false, t)) return 0;
  }
  if (info.ncomp == 3) {
    bool rgb;
    if (jfif) rgb = false;
    else if (adobe) rgb = adobe_transform == 0;
    else rgb = h.comp_id[0] == 'R' && h.comp_id[1] == 'G' && h.comp_id[2] == 'B';
    if (rgb) return 0;
    const int hs = info.hs[0], vs = info.vs[0];
    if (!((hs == 1 || hs == 2) && (vs == 1 || vs == 2))) return 0;
    for (int c = 1; c < 3; ++c)
      if (info.hs[c] != 1 || info.vs[c] != 1) return 0;
  } else {
    info.hs[0] = info.vs[0] = 1;                       // a one-component scan is not interleaved: MCU = one block
  }
  info.eligible = 1;
  const int64_t mcux = (info.width + 8 * info.hs[0] - 1) / (8 * info.hs[0]);
  const int64_t mcuy = (info.height + 8 * info.vs[0] - 1) / (8 * info.vs[0]);
  const int64_t nseg = info.restart_interval ? (mcux * mcuy + info.restart_interval - 1) / info.restart_interval : 1;
  const int64_t bytes = size - info.scan_offset;
  const int64_t nsub = bytes * 8 / SUB_BITS + nseg + 1;
  info.prep_bytes = (int64_t)sizeof(JTables) + 16 * ((nseg * (int64_t)sizeof(JSeg) + 15) / 16) + nsub * (int64_t)sizeof(JSub) +
                    ((bytes + SLACK + 15) / 16) * 16;
  return 0;
}

// ============================================================================================ device: Huffman
struct Bits {
  const uint8_t* p;
  int64_t n;                          // readable bytes (stream + slack)
  __device__ __forceinline__ uint32_t peek32(uint32_t bit) const {
    const int64_t b = bit >> 3;
    uint64_t v = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) v = (v << 8) | (b + k < n ? __ldg(p + b + k) : 0u);
    return (uint32_t)(v >> (8 - (bit & 7)));
  }
};

__device__ __forceinline__ int huff_decode(const JHuff* __restrict__ h, uint32_t w, int& len) {
  const int top = w >> 16;
  const int e = __ldg(&h->lut[top >> 7]);
  if (e) { len = e >> 8; return e & 255; }
  for (int l = 10; l <= 16; ++l) {
    const int code = top >> (16 - l);
    if (code <= __ldg(&h->maxcode[l])) { len = l; return __ldg(&h->vals[(__ldg(&h->valoff[l]) + code) & 255]); }
  }
  len = 0;
  return -1;
}

__device__ __forceinline__ int extend(uint32_t w, int len, int s) {
  if (s == 0) return 0;
  const int v = (int)((w << len) >> (32 - s));
  return v < (1 << (s - 1)) ? v + (int)(~0u << s) + 1 : v;
}

// State: (bit << 16) | (block within MCU << 8) | zig-zag index.  Decodes symbols while the bit offset is below `end`;
// returns the blocks completed.  WRITE: stores the coefficients of blocks [blk, blk_end) and reports errors in them.
template <bool WRITE>
__device__ uint32_t decode_run(const JTables* __restrict__ T, Bits bits, int bpm, uint64_t& st, uint32_t end,
                               int16_t* __restrict__ coef, int64_t blk, int64_t blk_end, uint32_t seg_end, int& err) {
  uint32_t p = (uint32_t)(st >> 16);
  int c = (int)((st >> 8) & 255), z = (int)(st & 255);
  uint32_t done = 0;
  while (p < end) {
    if (WRITE && blk >= blk_end) break;
    const int comp = __ldg(&T->blk_comp[c]);
    const uint32_t w = bits.peek32(p);
    int len, bad = 0;
    if (z == 0) {
      const int s = huff_decode(&T->dc[comp], w, len);
      if (len == 0 || s > 11) { bad = 1; p += len ? len : 1; z = 64; }
      else {
        if (WRITE) coef[blk * 64] = (int16_t)extend(w, len, s);
        p += len + s;
        z = 1;
      }
    } else {
      const int s = huff_decode(&T->ac[comp], w, len);
      if (len == 0) { bad = 1; p += 1; z = 64; }
      else {
        const int r = s >> 4, sz = s & 15;
        if (sz == 0) {
          z = r == 15 ? min(z + 16, 64) : 64;
          p += len;
        } else if (sz > 10 || z + r > 63) { bad = 1; p += len + sz; z = 64; }
        else {
          z += r;
          if (WRITE) coef[blk * 64 + c_natural[z]] = (int16_t)extend(w, len, sz);
          p += len + sz;
          ++z;
        }
      }
    }
    if (WRITE) {
      if (bad) err |= M3R_JPEG_EHUFF;
      if (p > seg_end) err |= M3R_JPEG_ESHORT;
    }
    if (z >= 64) {
      z = 0;
      c = c + 1 == bpm ? 0 : c + 1;
      ++done;
      if (WRITE) ++blk;
    }
  }
  st = ((uint64_t)p << 16) | ((uint64_t)c << 8) | (uint64_t)z;
  return done;
}

// A subsequence's entry state and the exit state decoded from it, written and read as one 16-byte atomic so that the
// racing synchronisation rounds never see the entry of one decode with the exit of another.
struct __align__(16) JRec { unsigned long long entry, exit; };

__device__ __forceinline__ JRec load_rec(JRec* r) { const JRec z{~0ull, ~0ull}; return atomicCAS(r, z, z); }

struct JWork {                      // batch-wide arrays at the front of the workspace, indexed by global subsequence
  JRec* rec; uint32_t* count; uint32_t* first; uint32_t* changed;
};

__device__ __forceinline__ int find_image(const m3r_jpeg_desc* __restrict__ d, int n, int64_t g, int field) {
  int lo = 0, hi = n - 1;            // last image whose base <= g
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const int64_t b = field == 0 ? d[mid].sub_base : field == 1 ? d[mid].blk_base : d[mid].pix_base;
    if (b <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

struct SubCtx {
  const JTables* T; Bits bits; JSub sub; JSeg seg; int bpm; bool first;
};

__device__ __forceinline__ SubCtx sub_ctx(const uint8_t* blob, const m3r_jpeg_desc& d, int64_t j) {
  SubCtx s;
  s.T = reinterpret_cast<const JTables*>(blob + d.tables_off);
  s.bits.p = blob + d.stream_off;
  s.bits.n = d.stream_bytes + SLACK;
  s.sub = reinterpret_cast<const JSub*>(blob + d.subs_off)[j];
  s.seg = reinterpret_cast<const JSeg*>(blob + d.segs_off)[s.sub.seg];
  s.bpm = d.bpm;
  s.first = s.sub.start == s.seg.start;
  return s;
}

__global__ void __launch_bounds__(128) jpeg_spec_kernel(const uint8_t* __restrict__ blob, const m3r_jpeg_desc* __restrict__ descs,
                                                        int n, int64_t nsub, JWork w) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nsub) return;
  const int i = find_image(descs, n, g, 0);
  const SubCtx s = sub_ctx(blob, descs[i], g - descs[i].sub_base);
  const uint64_t e = (uint64_t)s.sub.start << 16;
  uint64_t st = e;
  int err = 0;
  w.count[g] = decode_run<false>(s.T, s.bits, s.bpm, st, s.sub.end, nullptr, 0, 0, 0, err);
  w.rec[g] = JRec{e, st};
}

// One synchronisation round.  A subsequence whose entry state differs from its predecessor's exit state is decoded
// again from that exit, and the thread carries on into the following subsequences of the segment until it exits in the
// state the next one was decoded from (two decoders that meet in one state agree from there on).  Walking on matters:
// a decoder whose block-within-MCU phase is off by blocks that share Huffman tables never falls back into step by
// itself, so only propagation fixes it.  Threads of one round may overwrite each other's results; the round flag
// makes another round run, and every round fixes at least the first wrong subsequence of each segment for good.  The
// blocks counted here are not kept: jpeg_recount_kernel counts them once the chain has settled.
__global__ void __launch_bounds__(128) jpeg_sync_kernel(const uint8_t* __restrict__ blob, const m3r_jpeg_desc* __restrict__ descs,
                                                        int n, int64_t nsub, JWork w, int round) {
  if (round > 0 && *(volatile uint32_t*)&w.changed[round - 1] == 0) return;
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nsub) return;
  const int i = find_image(descs, n, g, 0);
  const m3r_jpeg_desc& d = descs[i];
  SubCtx s = sub_ctx(blob, d, g - d.sub_base);
  if (s.first) return;
  uint64_t st = load_rec(w.rec + g - 1).exit;
  if (st == load_rec(w.rec + g).entry) return;
  const int64_t end = d.sub_base + d.nsub;
  for (int64_t k = g;;) {
    const uint64_t e = st;
    int err = 0;
    decode_run<false>(s.T, s.bits, s.bpm, st, s.sub.end, nullptr, 0, 0, 0, err);
    atomicExch(w.rec + k, JRec{e, st});
    if (++k == end) break;
    const JSub nx = reinterpret_cast<const JSub*>(blob + d.subs_off)[k - d.sub_base];
    if (nx.start == reinterpret_cast<const JSeg*>(blob + d.segs_off)[nx.seg].start) break;   // the next segment
    if (st == load_rec(w.rec + k).entry) break;
    s.sub = nx;
  }
  w.changed[round] = 1;
}

// After the rounds, every subsequence is decoded once more from its predecessor's exit state, with no other writer:
// the blocks it completes are exact, and an exit that differs from the recorded one (the rounds ran out, or two
// threads of a round interleaved their writes) marks the image M3R_JPEG_ESYNC.
__global__ void __launch_bounds__(128) jpeg_recount_kernel(const uint8_t* __restrict__ blob, const m3r_jpeg_desc* __restrict__ descs,
                                                           int n, int64_t nsub, JWork w, int32_t* __restrict__ status) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nsub) return;
  const int i = find_image(descs, n, g, 0);
  const SubCtx s = sub_ctx(blob, descs[i], g - descs[i].sub_base);
  uint64_t st = s.first ? (uint64_t)s.sub.start << 16 : w.rec[g - 1].exit;
  int err = 0;
  w.count[g] = decode_run<false>(s.T, s.bits, s.bpm, st, s.sub.end, nullptr, 0, 0, 0, err);
  if (st != w.rec[g].exit) atomicOr(status + i, M3R_JPEG_ESYNC);
}

// Inclusive segmented sum over a CTA of blockDim.x (a multiple of 32) threads, `n` elements in chunks; load(k, flag,
// value) gives element k (flag = a segment starts here), store(k, sum).
template <class Load, class Store>
__device__ void seg_scan(int64_t n, Load load, Store store) {
  __shared__ int s_val[32], s_flag[32];
  __shared__ int s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < n; base += blockDim.x) {
    const int64_t k = base + threadIdx.x;
    int f = 1, v = 0;
    if (k < n) load(k, f, v);
    for (int d = 1; d < 32; d <<= 1) {
      const int ov = __shfl_up_sync(~0u, v, d), of = __shfl_up_sync(~0u, f, d);
      if (lane >= d && !f) { v += ov; f = of; }
    }
    if (lane == 31) { s_val[warp] = v; s_flag[warp] = f; }
    __syncthreads();
    if (warp == 0) {                  // exclusive prefix of the warp totals, starting from the previous chunk's carry
      int wv = lane < nw ? s_val[lane] : 0, wf = lane < nw ? s_flag[lane] : 0;
      for (int d = 1; d < 32; d <<= 1) {
        const int ov = __shfl_up_sync(~0u, wv, d), of = __shfl_up_sync(~0u, wf, d);
        if (lane >= d && !wf) { wv += ov; wf = of; }
      }
      const int carry = s_carry;
      const int incl = wf ? wv : wv + carry;
      const int excl = __shfl_up_sync(~0u, incl, 1);
      __syncwarp();
      if (lane < nw) s_val[lane] = lane == 0 ? carry : excl;
      if (lane == nw - 1) s_flag[0] = incl;       // the chunk's total, the next chunk's carry
    }
    __syncthreads();
    const int prefix = s_val[warp];
    if (!f) v += prefix;
    if (k < n) store(k, v);
    __syncthreads();
    if (threadIdx.x == 0) s_carry = s_flag[0];
    __syncthreads();
  }
}

// first[g] = the block a subsequence's entry state is in: the segment's first block plus the blocks completed before it
__global__ void __launch_bounds__(1024) jpeg_first_kernel(const uint8_t* __restrict__ blob, const m3r_jpeg_desc* __restrict__ descs,
                                                          JWork w) {
  const m3r_jpeg_desc& d = descs[blockIdx.x];
  const JSub* subs = reinterpret_cast<const JSub*>(blob + d.subs_off);
  const JSeg* segs = reinterpret_cast<const JSeg*>(blob + d.segs_off);
  const int64_t seg_blocks = (int64_t)(d.restart_interval ? d.restart_interval : d.mcux * d.mcuy) * d.bpm;
  const int64_t g0 = d.sub_base;
  seg_scan(d.nsub,
           [&](int64_t k, int& f, int& v) {
             const JSub s = subs[k];
             f = s.start == segs[s.seg].start;
             v = (int)w.count[g0 + k] + (f ? (int)(s.seg * seg_blocks) : 0);
           },
           [&](int64_t k, int v) { w.first[g0 + k] = (uint32_t)(v - (int)w.count[g0 + k]); });
}

__global__ void __launch_bounds__(128) jpeg_write_kernel(const uint8_t* __restrict__ blob, const m3r_jpeg_desc* __restrict__ descs,
                                                         int n, int64_t nsub, JWork w, uint8_t* __restrict__ work,
                                                         int32_t* __restrict__ status) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nsub) return;
  const int i = find_image(descs, n, g, 0);
  const m3r_jpeg_desc& d = descs[i];
  const SubCtx s = sub_ctx(blob, d, g - d.sub_base);
  const int64_t total = (int64_t)d.mcux * d.mcuy * d.bpm;
  const int64_t seg_blocks = (int64_t)(d.restart_interval ? d.restart_interval : d.mcux * d.mcuy) * d.bpm;
  const int64_t blk_end = min(total, (int64_t)(s.sub.seg + 1) * seg_blocks);
  int err = 0;
  uint64_t st = s.first ? (uint64_t)s.sub.start << 16 : w.rec[g - 1].exit;
  const int64_t blk = w.first[g];
  if (blk < blk_end && (int64_t)(blk % d.bpm) != (int64_t)((st >> 8) & 255)) err |= M3R_JPEG_ESYNC;
  const bool last = g + 1 == d.sub_base + d.nsub || s.sub.end == s.seg.end;
  if (last && blk + w.count[g] < blk_end) err |= M3R_JPEG_ESHORT;
  if (!err && blk < blk_end)
    decode_run<true>(s.T, s.bits, s.bpm, st, s.sub.end, reinterpret_cast<int16_t*>(work + d.coef_off), blk, blk_end,
                     s.seg.end, err);
  if (err) atomicOr(status + i, err);
}

// DC prediction: per image and component, the differences summed over the component's blocks in decode order,
// restarting at every restart segment; the value is stored as libjpeg's JCOEF (int16).
__global__ void __launch_bounds__(1024) jpeg_dc_kernel(const uint8_t* __restrict__ blob, const m3r_jpeg_desc* __restrict__ descs,
                                                       uint8_t* __restrict__ work) {
  const m3r_jpeg_desc& d = descs[blockIdx.x];
  const int comp = blockIdx.y;
  if (comp >= d.ncomp) return;
  const int hv = d.hs[comp] * d.vs[comp];
  int off = 0;
  for (int c = 0; c < comp; ++c) off += d.hs[c] * d.vs[c];
  int16_t* coef = reinterpret_cast<int16_t*>(work + d.coef_off);
  const int64_t per_seg = (int64_t)(d.restart_interval ? d.restart_interval : d.mcux * d.mcuy) * hv;
  const int bpm = d.bpm;
  auto blk = [=](int64_t k) { return (k / hv) * bpm + off + k % hv; };
  seg_scan((int64_t)d.mcux * d.mcuy * hv,
           [&](int64_t k, int& f, int& v) { f = k % per_seg == 0; v = coef[blk(k) * 64]; },
           [&](int64_t k, int v) { coef[blk(k) * 64] = (int16_t)v; });
}

// ============================================================================================ device: IDCT
#define FIX_0_298631336 ((long long)2446)
#define FIX_0_390180644 ((long long)3196)
#define FIX_0_541196100 ((long long)4433)
#define FIX_0_765366865 ((long long)6270)
#define FIX_0_899976223 ((long long)7373)
#define FIX_1_175875602 ((long long)9633)
#define FIX_1_501321110 ((long long)12299)
#define FIX_1_847759065 ((long long)15137)
#define FIX_1_961570560 ((long long)16069)
#define FIX_2_053119869 ((long long)16819)
#define FIX_2_562915447 ((long long)20995)
#define FIX_3_072711026 ((long long)25172)

// One 8-point pass of jpeg_idct_islow over in[0], in[s], .., in[7s]; `shift` is the DESCALE amount.
__device__ __forceinline__ void idct8(const long long* in, int s, long long* out, int shift) {
  long long z2 = in[2 * s], z3 = in[6 * s];
  long long z1 = (z2 + z3) * FIX_0_541196100;
  long long tmp2 = z1 + z3 * (-FIX_1_847759065);
  long long tmp3 = z1 + z2 * FIX_0_765366865;
  z2 = in[0];
  z3 = in[4 * s];
  long long tmp0 = (z2 + z3) * 8192, tmp1 = (z2 - z3) * 8192;
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in[7 * s]; tmp1 = in[5 * s]; tmp2 = in[3 * s]; tmp3 = in[s];
  z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * FIX_1_175875602;
  tmp0 *= FIX_0_298631336; tmp1 *= FIX_2_053119869; tmp2 *= FIX_3_072711026; tmp3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447; z3 *= -FIX_1_961570560; z4 *= -FIX_0_390180644;
  z3 += z5; z4 += z5;
  tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
  const long long r = 1LL << (shift - 1);
  out[0] = (tmp10 + tmp3 + r) >> shift; out[7] = (tmp10 - tmp3 + r) >> shift;
  out[1] = (tmp11 + tmp2 + r) >> shift; out[6] = (tmp11 - tmp2 + r) >> shift;
  out[2] = (tmp12 + tmp1 + r) >> shift; out[5] = (tmp12 - tmp1 + r) >> shift;
  out[3] = (tmp13 + tmp0 + r) >> shift; out[4] = (tmp13 - tmp0 + r) >> shift;
}

// range_limit[x & RANGE_MASK] of the post-IDCT table: x as a 10-bit two's-complement number, plus CENTERJSAMPLE, clamped
__device__ __forceinline__ uint8_t range_limit_idct(long long x) {
  const int v = ((int)(x & 1023) ^ 512) - 512;
  return (uint8_t)min(max(v + 128, 0), 255);
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(const uint8_t* __restrict__ blob, const m3r_jpeg_desc* __restrict__ descs,
                                                        int n, int64_t nblk, uint8_t* __restrict__ work) {
  const int64_t gb = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gb >= nblk) return;
  const int i = find_image(descs, n, gb, 1);
  const m3r_jpeg_desc& d = descs[i];
  const JTables* T = reinterpret_cast<const JTables*>(blob + d.tables_off);
  const int64_t b = gb - d.blk_base;
  const int64_t mcu = b / d.bpm;
  const int k = (int)(b % d.bpm);
  const int comp = T->blk_comp[k];
  const int mx = (int)(mcu % d.mcux), my = (int)(mcu / d.mcux);
  const int pw = d.mcux * d.hs[comp] * 8;
  const int px = (mx * d.hs[comp] + T->blk_x[k]) * 8, py = (my * d.vs[comp] + T->blk_y[k]) * 8;
  const int16_t* cf = reinterpret_cast<const int16_t*>(work + d.coef_off) + b * 64;
  const uint16_t* q = T->qt[comp];
  long long ws[64];
#pragma unroll
  for (int col = 0; col < 8; ++col) {
    long long v[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) v[r] = (long long)cf[r * 8 + col] * (long long)__ldg(q + r * 8 + col);
    long long o[8];
    idct8(v, 1, o, 11);                               // CONST_BITS - PASS1_BITS
#pragma unroll
    for (int r = 0; r < 8; ++r) ws[r * 8 + col] = (int)o[r];
  }
  uint8_t* plane = work + d.plane_off[comp];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    long long o[8];
    idct8(ws + r * 8, 1, o, 18);                      // CONST_BITS + PASS1_BITS + 3
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      lo |= (uint32_t)range_limit_idct(o[c]) << (8 * c);
      hi |= (uint32_t)range_limit_idct(o[c + 4]) << (8 * c);
    }
    uint2* dst = reinterpret_cast<uint2*>(plane + (int64_t)(py + r) * pw + px);
    *dst = make_uint2(lo, hi);
  }
}

// ============================================================================================ device: colour
__device__ __forceinline__ int chroma(const uint8_t* __restrict__ pl, int pw, int dw, int dh, int h2, int v2, int x, int y) {
  if (!h2 && !v2) return pl[(int64_t)y * pw + x];
  if (h2 && dw <= 2) {                                // jdsample.c's box upsampling
    return pl[(int64_t)(v2 ? y >> 1 : y) * pw + (x >> 1)];
  }
  if (!v2) {                                          // h2v1
    const int i = x >> 1;
    const uint8_t* r = pl + (int64_t)y * pw;
    return (x & 1) ? (3 * r[i] + r[min(i + 1, dw - 1)] + 2) >> 2 : (3 * r[i] + r[max(i - 1, 0)] + 1) >> 2;
  }
  const int row = y >> 1;
  const int nb = (y & 1) ? min(row + 1, dh - 1) : max(row - 1, 0);
  const uint8_t* r0 = pl + (int64_t)row * pw;
  const uint8_t* r1 = pl + (int64_t)nb * pw;
  if (!h2) return (3 * r0[x] + r1[x] + ((y & 1) ? 2 : 1)) >> 2;    // h1v2
  const int i = x >> 1;                               // h2v2: column sums of the two nearest rows
  const int j = (x & 1) ? min(i + 1, dw - 1) : max(i - 1, 0);
  const int ci = 3 * r0[i] + r1[i], cj = 3 * r0[j] + r1[j];
  return (x & 1) ? (3 * ci + cj + 7) >> 4 : (3 * ci + cj + 8) >> 4;
}

__global__ void __launch_bounds__(256) jpeg_color_kernel(const m3r_jpeg_desc* __restrict__ descs, int n, int64_t npix,
                                                         const uint8_t* __restrict__ work) {
  const int64_t gp = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gp >= npix) return;
  const int i = find_image(descs, n, gp, 2);
  const m3r_jpeg_desc& d = descs[i];
  const int64_t pix = gp - d.pix_base;
  const int W = d.width, H = d.height;
  const int x = (int)(pix % W), y = (int)(pix / W);
  const int pw0 = d.mcux * d.hs[0] * 8;
  const int Y = work[d.plane_off[0] + (int64_t)y * pw0 + x];
  int R = Y, G = Y, B = Y;
  if (d.ncomp == 3) {
    const int h2 = d.hs[0] == 2, v2 = d.vs[0] == 2;
    const int pwc = d.mcux * 8, dw = (W + h2) >> h2, dh = (H + v2) >> v2;
    const int cb = chroma(work + d.plane_off[1], pwc, dw, dh, h2, v2, x, y) - 128;
    const int cr = chroma(work + d.plane_off[2], pwc, dw, dh, h2, v2, x, y) - 128;
    R = Y + ((91881 * cr + 32768) >> 16);
    G = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
    B = Y + ((116130 * cb + 32768) >> 16);
    R = min(max(R, 0), 255); G = min(max(G, 0), 255); B = min(max(B, 0), 255);
  }
  int dx = x, dy = y, OW = W;                         // Pillow's exif_transpose methods
  switch (d.orientation) {
    case 2: dx = W - 1 - x; break;
    case 3: dx = W - 1 - x; dy = H - 1 - y; break;
    case 4: dy = H - 1 - y; break;
    case 5: dx = y; dy = x; OW = H; break;
    case 6: dx = H - 1 - y; dy = x; OW = H; break;
    case 7: dx = H - 1 - y; dy = W - 1 - x; OW = H; break;
    case 8: dx = y; dy = W - 1 - x; OW = H; break;
    default: break;
  }
  uint8_t* o = d.out + ((int64_t)dy * OW + dx) * 3;
  o[0] = (uint8_t)R; o[1] = (uint8_t)G; o[2] = (uint8_t)B;
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("jpeg_decode (%s) launch: %s", what, cudaGetErrorString(e));
  count_launch();
  return 0;
}

static int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

}  // namespace m3r

using namespace m3r;

extern "C" int m3r_jpeg_parse(const uint8_t* data, int64_t size, m3r_jpeg_info* info) {
  if (!info) return set_error("jpeg_parse: null info");
  Header h;
  const int rc = parse_header(data, size, h);
  *info = h.info;
  return rc;
}

extern "C" int m3r_jpeg_prepare(const uint8_t* data, int64_t size, const m3r_jpeg_info* info_in, int32_t orientation,
                                uint8_t* dst, int64_t base_off, m3r_jpeg_desc* desc) {
  if (!data || !info_in || !dst || !desc) return set_error("jpeg_prepare: null pointer");
  Header h;
  if (parse_header(data, size, h) != 0 || !h.info.eligible || h.info.prep_bytes != info_in->prep_bytes)
    return set_error("jpeg_prepare: the data is not the eligible JPEG that was parsed");
  if (orientation < 1 || orientation > 8) return set_error("jpeg_prepare: orientation %d", orientation);
  const m3r_jpeg_info& info = h.info;
  memset(desc, 0, sizeof(*desc));
  JTables* T = reinterpret_cast<JTables*>(dst);
  memset(T, 0, sizeof(JTables));
  int bpm = 0;
  for (int c = 0; c < info.ncomp; ++c) {
    memcpy(T->qt[c], h.qt[h.comp_tq[c]], sizeof(T->qt[c]));
    if (!build_huff(h.dc[h.comp_td[c]], true, T->dc[c]) || !build_huff(h.ac[h.comp_ta[c]], false, T->ac[c])) return 2;
    for (int by = 0; by < info.vs[c]; ++by)
      for (int bx = 0; bx < info.hs[c]; ++bx, ++bpm) {
        T->blk_comp[bpm] = (uint8_t)c; T->blk_x[bpm] = (uint8_t)bx; T->blk_y[bpm] = (uint8_t)by;
      }
  }
  const int64_t mcux = (info.width + 8 * info.hs[0] - 1) / (8 * info.hs[0]);
  const int64_t mcuy = (info.height + 8 * info.vs[0] - 1) / (8 * info.vs[0]);
  const int Ri = info.restart_interval;
  const int64_t nseg = Ri ? (mcux * mcuy + Ri - 1) / Ri : 1;
  const int64_t segs_off = sizeof(JTables);
  const int64_t subs_off = segs_off + 16 * ((nseg * (int64_t)sizeof(JSeg) + 15) / 16);
  const int64_t bytes = size - info.scan_offset;
  const int64_t max_subs = bytes * 8 / SUB_BITS + nseg + 1;
  const int64_t stream_off = subs_off + max_subs * (int64_t)sizeof(JSub);
  JSeg* segs = reinterpret_cast<JSeg*>(dst + segs_off);
  uint8_t* out = dst + stream_off;
  // the one pass over the entropy-coded data: unstuff, split at the restart markers, stop at EOI
  int64_t o = 0, seg = 0, i = info.scan_offset;
  int expect = 0;
  bool eoi = false;
  segs[0].start = 0;
  while (i < size) {
    const uint8_t b = data[i];
    if (b != 0xFF) { out[o++] = b; ++i; continue; }
    int64_t j = i + 1;
    while (j < size && data[j] == 0xFF) ++j;
    if (j >= size) break;
    const int m = data[j];
    i = j + 1;
    if (m == 0x00) { out[o++] = 0xFF; continue; }
    if (m >= 0xD0 && m <= 0xD7) {
      if (!Ri || (m & 7) != expect || seg + 1 >= nseg) return 2;
      expect = (expect + 1) & 7;
      segs[seg].end = (uint32_t)(o * 8);
      segs[++seg].start = (uint32_t)(o * 8);
      continue;
    }
    if (m == 0xD9) { eoi = true; break; }
    return 2;                                          // another scan, a table, DNL: not a one-scan baseline image
  }
  if (!eoi || seg + 1 != nseg) return 2;
  segs[seg].end = (uint32_t)(o * 8);
  memset(out + o, 0, SLACK);
  JSub* subs = reinterpret_cast<JSub*>(dst + subs_off);
  int64_t ns = 0;
  for (int64_t s = 0; s < nseg; ++s) {
    if (segs[s].end <= segs[s].start) return 2;        // an empty restart segment
    for (uint32_t a = segs[s].start; a < segs[s].end; a += SUB_BITS) {
      if (ns >= max_subs) return set_error("jpeg_prepare: subsequence table overflow");
      subs[ns++] = JSub{a, (uint32_t)std::min<int64_t>((int64_t)a + SUB_BITS, segs[s].end), (uint32_t)s, 0};
    }
  }
  desc->tables_off = base_off;
  desc->segs_off = base_off + segs_off;
  desc->subs_off = base_off + subs_off;
  desc->stream_off = base_off + stream_off;
  desc->stream_bytes = o;
  desc->width = info.width;
  desc->height = info.height;
  desc->ncomp = info.ncomp;
  desc->orientation = orientation;
  desc->mcux = (int32_t)mcux;
  desc->mcuy = (int32_t)mcuy;
  desc->bpm = bpm;
  desc->restart_interval = Ri;
  desc->nseg = (int32_t)nseg;
  desc->nsub = (int32_t)ns;
  for (int c = 0; c < 3; ++c) { desc->hs[c] = c < info.ncomp ? info.hs[c] : 0; desc->vs[c] = c < info.ncomp ? info.vs[c] : 0; }
  return 0;
}

// Workspace: [entry u64, exit u64 | count u32 | first u32] per subsequence of the batch, the round flags, then per
// image its coefficients (int16 [blocks][64], all images' back to back so one memset clears them) and its planes.
extern "C" int64_t m3r_jpeg_plan(m3r_jpeg_desc* d, int32_t n) {
  if (!d || n <= 0) { set_error("jpeg_plan: empty batch"); return -1; }
  int64_t subs = 0, blks = 0, pix = 0;
  for (int i = 0; i < n; ++i) {
    d[i].sub_base = subs; d[i].blk_base = blks; d[i].pix_base = pix;
    subs += d[i].nsub;
    blks += (int64_t)d[i].mcux * d[i].mcuy * d[i].bpm;
    pix += (int64_t)d[i].width * d[i].height;
  }
  int64_t off = align256(subs * 24) + align256(4 * SYNC_ROUNDS);
  for (int i = 0; i < n; ++i) {
    d[i].coef_off = off;
    off += (int64_t)d[i].mcux * d[i].mcuy * d[i].bpm * 128;
  }
  off = align256(off);
  for (int i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) {
      d[i].plane_off[c] = off;
      if (c < d[i].ncomp) off += align256((int64_t)d[i].mcux * d[i].hs[c] * 8 * d[i].mcuy * d[i].vs[c] * 8);
    }
  return off;
}

extern "C" int m3r_jpeg_decode(const m3r_jpeg_desc* hd, int32_t n, const uint8_t* blob, int64_t descs_off, uint8_t* work,
                               int64_t work_bytes, int32_t* status, void* stream) {
  if (n <= 0) return 0;
  if (!hd || !blob || !work || !status) return set_error("jpeg_decode: null pointer");
  if (n > 65535) return set_error("jpeg_decode: %d images in one call", n);
  int64_t subs = 0, blks = 0, pix = 0;
  for (int i = 0; i < n; ++i) {
    if (hd[i].sub_base != subs || hd[i].blk_base != blks || hd[i].pix_base != pix) return set_error("jpeg_decode: batch not planned");
    if (!hd[i].out) return set_error("jpeg_decode: image %d has no output", i);
    subs += hd[i].nsub;
    blks += (int64_t)hd[i].mcux * hd[i].mcuy * hd[i].bpm;
    pix += (int64_t)hd[i].width * hd[i].height;
  }
  const int64_t last = hd[n - 1].ncomp == 3 ? hd[n - 1].plane_off[2] + (int64_t)hd[n - 1].mcux * 8 * hd[n - 1].mcuy * 8
                                             : hd[n - 1].plane_off[0] + (int64_t)hd[n - 1].mcux * 8 * hd[n - 1].mcuy * 8;
  if (last > work_bytes) return set_error("jpeg_decode: workspace of %lld bytes, %lld needed", (long long)work_bytes, (long long)last);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const m3r_jpeg_desc* dd = reinterpret_cast<const m3r_jpeg_desc*>(blob + descs_off);
  JWork w;
  w.rec = reinterpret_cast<JRec*>(work);
  w.count = reinterpret_cast<uint32_t*>(w.rec + subs);
  w.first = w.count + subs;
  w.changed = reinterpret_cast<uint32_t*>(work + align256(subs * 24));
  ProfScope prof(PROF_OTHER, 0.0, (double)(subs * SUB_BITS / 8 + blks * 128 * 2 + pix * 3), s);
  cudaMemsetAsync(status, 0, sizeof(int32_t) * n, s);
  cudaMemsetAsync(w.changed, 0, 4 * SYNC_ROUNDS, s);
  cudaMemsetAsync(work + hd[0].coef_off, 0, blks * 128, s);
  const int sb = (int)((subs + 127) / 128);
  jpeg_spec_kernel<<<sb, 128, 0, s>>>(blob, dd, n, subs, w);
  if (int rc = check_launch("speculative pass")) return rc;
  for (int r = 0; r < SYNC_ROUNDS; ++r) {
    jpeg_sync_kernel<<<sb, 128, 0, s>>>(blob, dd, n, subs, w, r);
    if (int rc = check_launch("synchronisation pass")) return rc;
  }
  jpeg_recount_kernel<<<sb, 128, 0, s>>>(blob, dd, n, subs, w, status);
  if (int rc = check_launch("recount")) return rc;
  jpeg_first_kernel<<<n, 1024, 0, s>>>(blob, dd, w);
  if (int rc = check_launch("block scan")) return rc;
  jpeg_write_kernel<<<sb, 128, 0, s>>>(blob, dd, n, subs, w, work, status);
  if (int rc = check_launch("writing pass")) return rc;
  jpeg_dc_kernel<<<dim3(n, 3), 1024, 0, s>>>(blob, dd, work);
  if (int rc = check_launch("DC prediction")) return rc;
  jpeg_idct_kernel<<<(unsigned)((blks + 127) / 128), 128, 0, s>>>(blob, dd, n, blks, work);
  if (int rc = check_launch("IDCT")) return rc;
  jpeg_color_kernel<<<(unsigned)((pix + 255) / 256), 256, 0, s>>>(dd, n, pix, work);
  return check_launch("colour conversion");
}
