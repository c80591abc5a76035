// PNG decoding, bit for bit what Pillow's .convert('RGB') gives for 8-bit, non-interlaced L, RGB, P, LA and RGBA images.
//
// Host (plain C++, called through ctypes with the GIL released): the chunk walk (signature, every chunk up to IEND,
// the CRC of each chunk before the image data as Pillow checks them, the zlib header as zlib's inflate checks it,
// eligibility) and one pass that copies the palette and the concatenated IDAT payloads into the staging buffer.
//
// Device, one launch sequence per batch of images of any sizes and colour types:
//  1. png_inflate_kernel, one warp per image.  Symbol decoding is serial within a deflate stream, so every lane of the
//     warp runs the same decoder in step (uniform control flow, broadcast loads); lane k keeps the k-th symbol of each
//     run of 32, then the lanes store the run's literals at once and copy its matches one after another, 32 bytes per
//     step, reading the bytes already written to the image's scanline workspace (which holds the whole image, so no
//     position is reused).  A match at p reads only below p, and a literal that follows it in the run lies at or above
//     its end, so this order writes exactly what decoding symbol by symbol writes.  The Huffman tables of each
//     block are built in shared memory by the warp (10-bit lookup, canonical decoding for longer codes).  zlib's checks are repeated and set the image's status bits; the Adler-32 of the output is
//     computed by the warp and compared with the stream's.
//  2. png_unfilter_kernel, one warp per image: rows in groups of 32, one row per lane, as a wavefront (lane r works on
//     column t - r at step t and takes the pixel above from lane r - 1 by a shuffle), so Sub / Avg / Paeth, which chain
//     along a row, and Up / Avg / Paeth, which chain down the columns, stay exact.  Gray is replicated, alpha dropped,
//     palette indices looked up, and the EXIF transpose applied on the store.
// No kernel reads outside its image's staged bytes or writes outside its image's output and scanline workspace.
#include <string.h>
#include "m3r_internal.h"

namespace m3r {

constexpr int PNG_SLACK = 8;          // zero bytes after each stream
constexpr int PLTE_BYTES = 1024;      // the staged palette (768 bytes, padded)
constexpr int LUT_BITS = 10;

// ============================================================================================ host: chunks
static uint32_t crc_table[256];
static bool crc_ready = [] {
  for (uint32_t n = 0; n < 256; ++n) {
    uint32_t c = n;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    crc_table[n] = c;
  }
  return true;
}();

static uint32_t crc32(const uint8_t* p, int64_t n) {
  uint32_t c = 0xFFFFFFFFu;
  for (int64_t i = 0; i < n; ++i) c = crc_table[(c ^ p[i]) & 255] ^ (c >> 8);
  return c ^ 0xFFFFFFFFu;
}

static uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
static bool is_type(const uint8_t* t, const char* s) { return memcmp(t, s, 4) == 0; }

static const uint8_t PNG_SIG[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};

// Walks the chunks and fills `info`.  With `dst`, also stages the palette and the IDAT payloads (m3r_png_prepare).
static int walk(const uint8_t* data, int64_t size, m3r_png_info& info, uint8_t* dst) {
  memset(&info, 0, sizeof(info));
  if (!data || size < 8 || memcmp(data, PNG_SIG, 8) != 0) return 1;
  bool ok = true, ihdr = false, iend = false, plte = false, idat_run = false, idat_done = false;
  int comp = 0, filt = 0;
  uint8_t zhead[2] = {0, 0};
  int64_t pos = 8;
  while (ok) {
    if (pos + 12 > size) { ok = false; break; }       // no IEND
    const uint32_t len = be32(data + pos);
    const uint8_t* type = data + pos + 4;
    const uint8_t* p = data + pos + 8;
    if (len > 0x7FFFFFFFu || pos + 12 + (int64_t)len > size) { ok = false; break; }
    const bool is_idat = is_type(type, "IDAT");
    if (!ihdr && !is_type(type, "IHDR")) { ok = false; break; }
    if (idat_run && !is_idat) { idat_run = false; idat_done = true; }
    // Pillow checks the CRC of every chunk it reads before the image data (and none after it)
    if (!idat_run && !idat_done && !is_idat && crc32(type, 4 + (int64_t)len) != be32(p + len)) { ok = false; break; }
    if (is_type(type, "IHDR")) {
      if (ihdr || len != 13) { ok = false; break; }
      ihdr = true;
      const uint32_t w = be32(p), h = be32(p + 4);
      if (w == 0 || h == 0 || w > 0x7FFFFFFFu || h > 0x7FFFFFFFu) { ok = false; break; }
      info.width = (int32_t)w; info.height = (int32_t)h;
      info.bit_depth = p[8]; info.color_type = p[9]; comp = p[10]; filt = p[11]; info.interlace = p[12];
    } else if (is_type(type, "PLTE")) {
      if (plte || idat_run || idat_done || len % 3 != 0 || len > 768 || len == 0) { ok = false; break; }
      plte = true;
      info.palette_entries = (int32_t)(len / 3);
      if (dst) memcpy(dst, p, len);
    } else if (is_idat) {
      if (idat_done) { ok = false; break; }            // a second run of IDAT chunks
      idat_run = true;
      for (uint32_t k = 0; k < len && info.idat_bytes + k < 2; ++k) zhead[info.idat_bytes + k] = p[k];
      if (dst) memcpy(dst + PLTE_BYTES + info.idat_bytes, p, len);
      info.idat_bytes += len;
    } else if (is_type(type, "IEND")) {
      iend = true;
      break;
    } else if (is_type(type, "eXIf")) {
      info.has_exif = 1;
    } else if (is_type(type, "tEXt") || is_type(type, "zTXt") || is_type(type, "iTXt")) {
      info.has_text = 1;
      info.text_bytes += len;
      // after the image data Pillow decompresses and decodes zTXt / iTXt while loading, and may raise there
      if (idat_done && !is_type(type, "tEXt")) ok = false;
    } else if (is_type(type, "acTL") || is_type(type, "fcTL") || is_type(type, "fdAT")) {
      ok = false;                                      // animated PNG
    } else if (idat_done && !is_type(type, "tIME")) {
      ok = false;                                      // Pillow runs its chunk handlers while loading
    }
    pos += 12 + (int64_t)len;
  }
  const int ct = info.color_type;
  info.channels = ct == 0 || ct == 3 ? 1 : ct == 4 ? 2 : ct == 2 ? 3 : ct == 6 ? 4 : 0;
  if (!ok || !iend || !ihdr || info.idat_bytes < 2 || info.bit_depth != 8 || info.interlace != 0 || comp != 0 || filt != 0 ||
      info.channels == 0 || (ct == 3 && !plte))
    return 0;
  // zlib's header checks (inflateInit: a window of at most 32K, no preset dictionary)
  if ((zhead[0] & 15) != 8 || (zhead[0] >> 4) > 7 || ((zhead[0] << 8) | zhead[1]) % 31 != 0 || (zhead[1] & 0x20)) return 0;
  const int64_t raw = (int64_t)info.height * (1 + (int64_t)info.width * info.channels);
  if (raw >= (1LL << 31) || info.idat_bytes >= (1LL << 31)) return 0;
  info.eligible = 1;
  info.prep_bytes = PLTE_BYTES + (info.idat_bytes + PNG_SLACK + 15) / 16 * 16;
  return 0;
}

// ============================================================================================ device: inflate
struct Huff {
  uint16_t lut[1 << LUT_BITS];        // next LUT_BITS stream bits -> (length << 9) | symbol; 0: a longer code or none
  uint16_t count[16];                 // codes of each length
  uint16_t sym[288];                  // symbols in canonical order (by length, then value)
};

struct InflateSmem {
  Huff lit, dist, cl;
  uint8_t lens[352];                  // code-length code at [0, 19), then HLIT + HDIST lengths at [19, 335)
  uint16_t next[16];                  // table construction, per length: symbols placed so far,
  uint16_t offs[16], first[16];       // first canonical position and first code
};

__constant__ uint16_t c_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// Bit reader, replicated in every lane (all lanes read the same bytes).
struct BitIn {
  const uint8_t* p;
  int64_t n, pos;                     // stream bytes, next byte to load
  uint64_t bb;
  int cnt;
  __device__ __forceinline__ void refill() {
    if (cnt > 56) return;
    const int nb = (64 - cnt) >> 3;                  // whole bytes that fit: cnt ends in [57, 64]
    if (pos >= 0 && pos + 16 <= n) {                 // two aligned 8-byte loads (the stream starts 16-byte aligned)
      const int64_t a = pos & ~7LL;
      const int sh = (int)(pos & 7) * 8;
      const uint64_t w0 = __ldg(reinterpret_cast<const unsigned long long*>(p + a));
      const uint64_t w1 = __ldg(reinterpret_cast<const unsigned long long*>(p + a + 8));
      const uint64_t v = sh ? (w0 >> sh) | (w1 << (64 - sh)) : w0;
      bb |= (nb == 8 ? v : v & ((1ull << (8 * nb)) - 1)) << cnt;
      cnt += 8 * nb;
      pos += nb;
      return;
    }
    while (cnt <= 56) {                              // near the end: bytes past it read as zeros
      const uint64_t b = pos < n ? __ldg(p + pos) : 0u;
      bb |= b << cnt;
      cnt += 8;
      ++pos;
    }
  }
  __device__ __forceinline__ uint32_t get(int k) {   // k <= 32, after a refill that left enough bits
    const uint32_t v = (uint32_t)(bb & ((1ull << k) - 1));
    bb >>= k;
    cnt -= k;
    return v;
  }
  __device__ __forceinline__ bool overrun() const { return pos * 8 - cnt > n * 8; }
};

// Builds `h` from lens[0, n) with the whole warp; returns the M3R_PNG_ECODES bit or 0 (uniform).  zlib's rules:
// over-subscribed lengths are an error; incomplete ones too, unless the longest code has length 1 (one code) and this
// is not the code-length code; no code at all is allowed except for the code-length code.
__device__ int build_huff(Huff& h, const uint8_t* lens, int n, bool codelen, InflateSmem& sm, int lane) {
  uint16_t* next = sm.next;
  if (lane < 16) { h.count[lane] = 0; next[lane] = 0; }
  for (int i = lane; i < (1 << LUT_BITS); i += 32) h.lut[i] = 0;
  __syncwarp();
  for (int s0 = 0; s0 < n; s0 += 32) {                // counts: one leader per group of lanes with the same length
    const int s = s0 + lane;
    const int l = s < n ? lens[s] : 0;
    const unsigned grp = __match_any_sync(~0u, l);
    if (l && lane == __ffs(grp) - 1) h.count[l] += __popc(grp);
    __syncwarp();
  }
  int left = 1, maxl = 0;
  for (int l = 1; l <= 15; ++l) {
    left = (left << 1) - h.count[l];
    if (left < 0) return M3R_PNG_ECODES;
    if (h.count[l]) maxl = l;
  }
  if (maxl == 0) return codelen ? M3R_PNG_ECODES : 0;
  if (left > 0 && (codelen || maxl != 1)) return M3R_PNG_ECODES;
  if (lane == 0) {
    sm.offs[1] = 0; sm.first[1] = 0;
    for (int l = 1; l < 15; ++l) {
      sm.offs[l + 1] = sm.offs[l] + h.count[l];
      sm.first[l + 1] = (sm.first[l] + h.count[l]) << 1;
    }
  }
  __syncwarp();
  for (int s0 = 0; s0 < n; s0 += 32) {
    const int s = s0 + lane;
    const int l = s < n ? lens[s] : 0;
    const unsigned grp = __match_any_sync(~0u, l);
    const int rank = __popc(grp & ((1u << lane) - 1));
    if (l) {
      const int k = next[l] + rank;                    // position among the codes of length l
      h.sym[sm.offs[l] + k] = (uint16_t)s;
      if (l <= LUT_BITS) {
        const uint32_t rev = __brev((uint32_t)(sm.first[l] + k)) >> (32 - l);
        const uint16_t e = (uint16_t)((l << 9) | s);
        for (uint32_t f = 0; f < (1u << (LUT_BITS - l)); ++f) h.lut[rev | (f << l)] = e;
      }
    }
    __syncwarp();
    if (l && lane == __ffs(grp) - 1) next[l] += __popc(grp);
    __syncwarp();
  }
  return 0;
}

// One symbol at the reader's position (lengths up to 15, so one refill covers it); len = 0 when no code matches.
__device__ __forceinline__ int decode_sym(const Huff& h, uint64_t bb, int& len) {
  const uint32_t e = h.lut[bb & ((1u << LUT_BITS) - 1)];
  if (e) { len = e >> 9; return e & 511; }
  int code = 0, first = 0, index = 0;                 // canonical decoding, one bit at a time
  for (int l = 1; l <= 15; ++l) {
    code |= (int)((bb >> (l - 1)) & 1);
    const int c = h.count[l];
    if (code - c < first) { len = l; return h.sym[index + code - first]; }
    index += c;
    first = (first + c) << 1;
    code <<= 1;
  }
  len = 0;
  return -1;
}

// Literals of the run go out together; then its matches in order.  A match at p reads only [p - dist, p): bytes of
// earlier symbols (literals of this run included, stored above) and never a position a later literal of the run takes,
// since those lie at or above p + len.  The output holds the whole image, so no position is ever reused.
__device__ __forceinline__ void flush_run(uint8_t* out, int lane, int nrun, bool is_match, uint32_t at, uint32_t a,
                                          uint32_t b) {
  if (lane < nrun && !is_match) out[at] = (uint8_t)a;
  __syncwarp();
  unsigned m = __ballot_sync(~0u, lane < nrun && is_match);
  while (m) {
    const int k = __ffs(m) - 1;
    m &= m - 1;
    const uint32_t p = __shfl_sync(~0u, at, k), len = __shfl_sync(~0u, a, k), dist = __shfl_sync(~0u, b, k);
    const uint8_t* src = out + p - dist;
    for (uint32_t i = lane; i < len; i += 32) out[p + i] = src[dist >= len ? i : i % dist];
    __syncwarp();
  }
}

__global__ void __launch_bounds__(32) png_inflate_kernel(const uint8_t* __restrict__ blob, const m3r_png_desc* __restrict__ descs,
                                                         uint8_t* __restrict__ work, int32_t* __restrict__ status) {
  __shared__ InflateSmem sm;
  const int lane = threadIdx.x;
  const m3r_png_desc& d = descs[blockIdx.x];
  uint8_t* out = work + d.raw_off;
  const uint32_t expect = (uint32_t)d.raw_bytes;
  BitIn in{blob + d.stream_off, d.stream_bytes, 2, 0, 0};   // the two header bytes were checked on the host
  uint32_t pos = 0;
  int err = 0;
  bool last = false;
#define PNG_FAIL(bit) { err |= (bit); break; }
#define PNG_CHECK_INPUT() if (in.overrun()) PNG_FAIL(M3R_PNG_ELENGTH)
  while (!last && !err) {
    in.refill();
    last = in.get(1);
    const int type = (int)in.get(2);
    PNG_CHECK_INPUT();
    if (type == 3) PNG_FAIL(M3R_PNG_EBTYPE);
    if (type == 0) {                                   // stored: byte-aligned LEN, NLEN, then LEN bytes
      in.get(in.cnt & 7);
      const int64_t bp = in.pos - in.cnt / 8;
      if (bp + 4 > in.n) PNG_FAIL(M3R_PNG_ELENGTH);
      const uint32_t len = __ldg(in.p + bp) | (__ldg(in.p + bp + 1) << 8);
      const uint32_t nlen = __ldg(in.p + bp + 2) | (__ldg(in.p + bp + 3) << 8);
      if (len != (~nlen & 0xFFFFu)) PNG_FAIL(M3R_PNG_ESTORED);
      if (bp + 4 + len > in.n || pos + len > expect) PNG_FAIL(M3R_PNG_ELENGTH);
      for (uint32_t i = lane; i < len; i += 32) out[pos + i] = __ldg(in.p + bp + 4 + i);
      __syncwarp();
      pos += len;
      in.pos = bp + 4 + len; in.bb = 0; in.cnt = 0;
      continue;
    }
    if (type == 1) {                                   // fixed codes
      for (int i = lane; i < 320; i += 32) sm.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : i < 288 ? 8 : 5;
      __syncwarp();
      build_huff(sm.lit, sm.lens, 288, false, sm, lane);
      __syncwarp();
      build_huff(sm.dist, sm.lens + 288, 32, false, sm, lane);
      __syncwarp();
    } else {                                           // dynamic codes
      const int hlit = (int)in.get(5) + 257, hdist = (int)in.get(5) + 1, hclen = (int)in.get(4) + 4;
      PNG_CHECK_INPUT();
      if (hlit > 286 || hdist > 30) PNG_FAIL(M3R_PNG_ECODES);
      in.refill();
      for (int i = lane; i < 19; i += 32) sm.lens[i] = 0;
      __syncwarp();
      for (int i = 0; i < hclen; ++i) {
        const int v = (int)in.get(3);
        if (lane == 0) sm.lens[c_clorder[i]] = (uint8_t)v;
      }
      PNG_CHECK_INPUT();
      __syncwarp();
      if (int e = build_huff(sm.cl, sm.lens, 19, true, sm, lane)) PNG_FAIL(e);
      __syncwarp();
      int idx = 0, prev = -1;                          // prev: the last length read (every lane holds it)
      while (idx < hlit + hdist) {
        in.refill();
        int l;
        const int s = decode_sym(sm.cl, in.bb, l);
        if (l == 0) { err |= M3R_PNG_ESYMBOL; break; }
        in.get(l);
        if (in.overrun()) { err |= M3R_PNG_ELENGTH; break; }
        if (s < 16) {
          if (lane == 0) sm.lens[19 + idx] = (uint8_t)s;
          prev = s;
          ++idx;
          continue;
        }
        int val = 0, rep;
        if (s == 16) {
          if (prev < 0) { err |= M3R_PNG_EREPEAT; break; }
          val = prev;
          rep = 3 + (int)in.get(2);
        } else if (s == 17) {
          rep = 3 + (int)in.get(3);
        } else {
          rep = 11 + (int)in.get(7);
        }
        if (in.overrun()) { err |= M3R_PNG_ELENGTH; break; }
        if (idx + rep > hlit + hdist) { err |= M3R_PNG_EREPEAT; break; }
        prev = val;
        __syncwarp();
        if (lane < rep) sm.lens[19 + idx + lane] = (uint8_t)val;
        for (int i = 32 + lane; i < rep; i += 32) sm.lens[19 + idx + i] = (uint8_t)val;
        __syncwarp();
        idx += rep;
      }
      if (err) break;
      __syncwarp();
      if (sm.lens[19 + 256] == 0) PNG_FAIL(M3R_PNG_ENOEOB);
      if (int e = build_huff(sm.lit, sm.lens + 19, hlit, false, sm, lane)) PNG_FAIL(e);
      __syncwarp();
      if (int e = build_huff(sm.dist, sm.lens + 19 + hlit, hdist, false, sm, lane)) PNG_FAIL(e);
      __syncwarp();
    }
    // symbols, in runs of 32
    bool eob = false;
    while (!eob && !err) {
      int nrun = 0;
      bool is_match = false;
      uint32_t at = 0, a = 0, b = 0;
      while (nrun < 32) {
        in.refill();
        int l;
        const int s = decode_sym(sm.lit, in.bb, l);
        if (l == 0) { err |= M3R_PNG_ESYMBOL; break; }
        in.get(l);
        if (in.overrun()) { err |= M3R_PNG_ELENGTH; break; }
        if (s < 256) {
          if (pos >= expect) { err |= M3R_PNG_ELENGTH; break; }
          if (lane == nrun) { is_match = false; at = pos; a = (uint32_t)s; }
          ++pos; ++nrun;
          continue;
        }
        if (s == 256) { eob = true; break; }
        if (s > 285) { err |= M3R_PNG_ESYMBOL; break; }
        const uint32_t len = c_lbase[s - 257] + in.get(c_lext[s - 257]);
        const int ds = decode_sym(sm.dist, in.bb, l);
        if (l == 0) { err |= M3R_PNG_ESYMBOL; break; }
        in.get(l);
        if (in.overrun()) { err |= M3R_PNG_ELENGTH; break; }
        if (ds > 29) { err |= M3R_PNG_ESYMBOL; break; }
        const uint32_t dist = c_dbase[ds] + in.get(c_dext[ds]);
        if (in.overrun()) { err |= M3R_PNG_ELENGTH; break; }
        if (dist > pos) { err |= M3R_PNG_EDIST; break; }
        if (pos + len > expect) { err |= M3R_PNG_ELENGTH; break; }
        if (lane == nrun) { is_match = true; at = pos; a = len; b = dist; }
        pos += len; ++nrun;
      }
      flush_run(out, lane, nrun, is_match, at, a, b);
    }
  }
#undef PNG_CHECK_INPUT
#undef PNG_FAIL
  if (!err) {                                          // the Adler-32 trailer, byte-aligned after the last block
    in.get(in.cnt & 7);
    const int64_t bp = in.pos - in.cnt / 8;
    if (bp + 4 > in.n) {
      err = M3R_PNG_ELENGTH;
    } else {
      const uint32_t want = ((uint32_t)__ldg(in.p + bp) << 24) | ((uint32_t)__ldg(in.p + bp + 1) << 16) |
                            ((uint32_t)__ldg(in.p + bp + 2) << 8) | __ldg(in.p + bp + 3);
      if (pos != expect) err = M3R_PNG_ELENGTH;
      // a = 1 + sum d_i, b = n + sum (n - i) d_i (mod 65521): per lane sum d_i and sum i d_i, then combined
      constexpr uint32_t MOD = 65521;
      uint64_t s1 = 0, s2 = 0;
      int k = 0;
      const uint32_t* w = reinterpret_cast<const uint32_t*>(out);   // 256-byte aligned
      for (uint32_t j = lane; j < pos / 4; j += 32) {
        const uint32_t v = w[j];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const uint32_t x = (v >> (8 * c)) & 255;
          s1 += x;
          s2 += (uint64_t)(4 * j + c) * x;
        }
        if (++k == 256) { s1 %= MOD; s2 %= MOD; k = 0; }
      }
      for (uint32_t i = pos / 4 * 4 + lane; i < pos; i += 32) {
        s1 += out[i];
        s2 += (uint64_t)i * out[i];
      }
      s1 %= MOD; s2 %= MOD;
      for (int o = 16; o; o >>= 1) {
        s1 += __shfl_xor_sync(~0u, s1, o);
        s2 += __shfl_xor_sync(~0u, s2, o);
      }
      s1 %= MOD; s2 %= MOD;
      const uint64_t n = pos % MOD;
      const uint32_t A = (uint32_t)((1 + s1) % MOD);
      const uint32_t B = (uint32_t)((n + n * s1 + MOD - s2) % MOD);
      if (((B << 16) | A) != want) err |= M3R_PNG_EADLER;
    }
  }
  if (lane == 0) status[blockIdx.x] = err;
}

// ============================================================================================ device: unfilter
__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int p = a + b - c;
  const int pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (pa <= pb && pa <= pc) ? a : pb <= pc ? b : c;
}

__global__ void __launch_bounds__(32) png_unfilter_kernel(const uint8_t* __restrict__ blob, const m3r_png_desc* __restrict__ descs,
                                                          uint8_t* __restrict__ work, int32_t* __restrict__ status) {
  __shared__ uint8_t plte[768];
  const int lane = threadIdx.x;
  const m3r_png_desc& d = descs[blockIdx.x];
  if (status[blockIdx.x]) return;                      // the stream did not inflate cleanly
  const int W = d.width, H = d.height, bpp = d.channels, ct = d.color_type, npal = d.palette_entries;
  const int64_t stride = 1 + (int64_t)W * bpp;
  uint8_t* raw = work + d.raw_off;
  int bad = 0;
  for (int y = lane; y < H; y += 32) bad |= raw[(int64_t)y * stride] > 4;
  if (__any_sync(~0u, bad)) {
    if (lane == 0) status[blockIdx.x] = M3R_PNG_EFILTER;
    return;
  }
  if (ct == 3)
    for (int i = lane; i < 768; i += 32) plte[i] = __ldg(blob + d.plte_off + i);
  __syncwarp();
  const int orient = d.orientation;
  const int OW = orient >= 5 ? H : W;
  for (int y0 = 0; y0 < H; y0 += 32) {
    const int y = y0 + lane;
    const bool act = y < H;
    uint8_t* row = raw + (int64_t)(act ? y : 0) * stride;
    const int ft = act ? row[0] : 0;
    uint32_t cur = 0, prev_above = 0;
    for (int t = 0; t < W + 31; ++t) {
      const int x = t - lane;
      uint32_t above = __shfl_up_sync(~0u, cur, 1);  // lane - 1's pixel at column x, finished at step t - 1
      const bool in_row = act && x >= 0 && x < W;
      if (lane == 0) {                                 // the row above is the last group's last row, unfiltered in place
        above = 0;
        if (in_row && y > 0) {
          const uint8_t* r = raw + (int64_t)(y - 1) * stride + 1 + (int64_t)x * bpp;
          for (int c = 0; c < bpp; ++c) above |= (uint32_t)r[c] << (8 * c);
        }
      }
      if (in_row) {
        uint8_t* f = row + 1 + (int64_t)x * bpp;
        const uint32_t left = x > 0 ? cur : 0u, ul = x > 0 ? prev_above : 0u;
        uint32_t v = 0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          if (c < bpp) {
            const int A = (left >> (8 * c)) & 255, B = (above >> (8 * c)) & 255, Cc = (ul >> (8 * c)) & 255;
            const int pred = ft == 0 ? 0 : ft == 1 ? A : ft == 2 ? B : ft == 3 ? (A + B) >> 1 : paeth(A, B, Cc);
            v |= (uint32_t)((f[c] + pred) & 255) << (8 * c);
          }
        }
        cur = v;
        if (lane == 31)
          for (int c = 0; c < bpp; ++c) f[c] = (uint8_t)(v >> (8 * c));
        uint32_t r, g, b;
        if (ct == 2 || ct == 6) { r = v & 255; g = (v >> 8) & 255; b = (v >> 16) & 255; }
        else if (ct == 3) {
          const int i = v & 255;
          bad |= i >= npal;
          r = plte[3 * i]; g = plte[3 * i + 1]; b = plte[3 * i + 2];
        } else { r = g = b = v & 255; }
        int dx = x, dy = y;                            // Pillow's exif_transpose methods
        switch (orient) {
          case 2: dx = W - 1 - x; break;
          case 3: dx = W - 1 - x; dy = H - 1 - y; break;
          case 4: dy = H - 1 - y; break;
          case 5: dx = y; dy = x; break;
          case 6: dx = H - 1 - y; dy = x; break;
          case 7: dx = H - 1 - y; dy = W - 1 - x; break;
          case 8: dx = y; dy = W - 1 - x; break;
          default: break;
        }
        uint8_t* o = d.out + ((int64_t)dy * OW + dx) * 3;
        o[0] = (uint8_t)r; o[1] = (uint8_t)g; o[2] = (uint8_t)b;
      }
      prev_above = above;
    }
    __syncwarp();
  }
  if (__any_sync(~0u, bad) && lane == 0) status[blockIdx.x] = M3R_PNG_EPALETTE;
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("png_decode (%s) launch: %s", what, cudaGetErrorString(e));
  count_launch();
  return 0;
}

static int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

}  // namespace m3r

using namespace m3r;

extern "C" int m3r_png_parse(const uint8_t* data, int64_t size, m3r_png_info* info) {
  if (!info) return set_error("png_parse: null info");
  return walk(data, size, *info, nullptr);
}

extern "C" int m3r_png_prepare(const uint8_t* data, int64_t size, const m3r_png_info* info_in, int32_t orientation,
                               uint8_t* dst, int64_t base_off, m3r_png_desc* desc) {
  if (!data || !info_in || !dst || !desc) return set_error("png_prepare: null pointer");
  if (orientation < 1 || orientation > 8) return set_error("png_prepare: orientation %d", orientation);
  if (!info_in->eligible || info_in->prep_bytes <= 0) return set_error("png_prepare: the file is not eligible");
  memset(dst, 0, PLTE_BYTES);
  m3r_png_info info;
  if (walk(data, size, info, dst) != 0 || !info.eligible || info.prep_bytes != info_in->prep_bytes)
    return set_error("png_prepare: the data is not the eligible PNG that was parsed");
  memset(dst + PLTE_BYTES + info.idat_bytes, 0, info.prep_bytes - PLTE_BYTES - info.idat_bytes);
  memset(desc, 0, sizeof(*desc));
  desc->plte_off = base_off;
  desc->stream_off = base_off + PLTE_BYTES;
  desc->stream_bytes = info.idat_bytes;
  desc->width = info.width;
  desc->height = info.height;
  desc->channels = info.channels;
  desc->color_type = info.color_type;
  desc->palette_entries = info.palette_entries;
  desc->orientation = orientation;
  return 0;
}

// Workspace: each image's scanlines (filter byte + W * channels bytes per row), 256-byte aligned.
extern "C" int64_t m3r_png_plan(m3r_png_desc* d, int32_t n) {
  if (!d || n <= 0) { set_error("png_plan: empty batch"); return -1; }
  int64_t off = 0;
  for (int i = 0; i < n; ++i) {
    d[i].raw_off = off;
    d[i].raw_bytes = (int64_t)d[i].height * (1 + (int64_t)d[i].width * d[i].channels);
    off += align256(d[i].raw_bytes);
  }
  return off;
}

extern "C" int m3r_png_decode(const m3r_png_desc* hd, int32_t n, const uint8_t* blob, int64_t descs_off, uint8_t* work,
                              int64_t work_bytes, int32_t* status, void* stream) {
  if (n <= 0) return 0;
  if (!hd || !blob || !work || !status) return set_error("png_decode: null pointer");
  if (n > 65535) return set_error("png_decode: %d images in one call", n);
  int64_t off = 0, raw = 0, in = 0;
  for (int i = 0; i < n; ++i) {
    if (hd[i].raw_off != off || hd[i].raw_bytes != (int64_t)hd[i].height * (1 + (int64_t)hd[i].width * hd[i].channels))
      return set_error("png_decode: batch not planned");
    if (!hd[i].out) return set_error("png_decode: image %d has no output", i);
    off += align256(hd[i].raw_bytes);
    raw += hd[i].raw_bytes;
    in += hd[i].stream_bytes;
  }
  if (off > work_bytes) return set_error("png_decode: workspace of %lld bytes, %lld needed", (long long)work_bytes, (long long)off);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const m3r_png_desc* dd = reinterpret_cast<const m3r_png_desc*>(blob + descs_off);
  ProfScope prof(PROF_OTHER, 0.0, (double)(in + 2 * raw), s);
  cudaMemsetAsync(status, 0, sizeof(int32_t) * n, s);
  png_inflate_kernel<<<n, 32, 0, s>>>(blob, dd, work, status);
  if (int rc = check_launch("inflate")) return rc;
  png_unfilter_kernel<<<n, 32, 0, s>>>(blob, dd, work, status);
  return check_launch("unfilter");
}
