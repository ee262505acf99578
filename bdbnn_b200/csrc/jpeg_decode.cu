// Baseline JPEG decode on the device, bit-identical to libjpeg-turbo (jdhuff.c, jidctint.c, jdsample.c, jdcolor.c).
// See include/bdbnn.h for the contract and DESIGN.md §4m for the algorithm; oracle/jpeg_ref.py restates it on the CPU.
//
// Host: bdbnn_jpeg_parse reads one file's markers up to SOS, fills a fixed-size descriptor (geometry, quantisation
// tables, Huffman tables as a 9-bit lookahead plus maxcode / valoff) and copies the entropy-coded data, unstuffed and
// split at the RST markers, into the caller's buffer.  Thread-safe, allocates nothing.
//
// Device, per batch (bdbnn_jpeg_decode_batch), every segment (the data between restart markers, or the whole scan)
// cut into subsequences of S bits, one thread each:
//   phase 1  decode from a guessed start state (the subsequence's first bit, block 0 of the MCU, DC) up to the first
//            codeword boundary at or past the subsequence's end: the exit state (bit, block in MCU, zig-zag index);
//   phase 2  adopt the predecessor's exit as the start and decode again until no start changes: barrier rounds
//            inside a CUDA block, and across blocks one wait per block for the previous block's published exit
//            (decoupled look-back, blocks take their tiles from an atomic counter).  A segment's first subsequence
//            starts at the true state, so every round makes at least one more subsequence exact and the fixed
//            point is the sequential decode;
//   phase 3  exclusive scan of the blocks each subsequence completes, per segment (one warp per segment);
//   phase 4  decode again and write the int16 coefficients of each block into its slot (blocks in MCU order);
//   DC       per-component running sums of the DC differences within each segment (one CUDA block per segment);
//   IDCT     jpeg_idct_islow per block, 8 threads per block, into per-component sample planes;
//   colour   fancy upsampling + ycc_rgb_convert (or gray replication) per output pixel, uint8 HWC RGB.
// Every bit read, table index and coefficient index is bounds-checked; an image whose stream is malformed, or whose
// values leave the range where libjpeg-turbo's SIMD and C arithmetic agree, gets a nonzero status word.
#include <limits.h>
#include <stddef.h>
#include <stdarg.h>

#include <algorithm>
#include <atomic>
#include <utility>

#include "common.cuh"

namespace bdbnn {

constexpr int kJpSubBits = 1024;                  // subsequence length in bits
constexpr int kJpMaxSide = 8192;
constexpr int kJpThreads = 256;
static std::atomic<int> g_jp_sub_bits{0};         // bdbnn_debug_jpeg_subseq_bits override, 0 = kJpSubBits

static int jp_sub_bits() {
  const int v = g_jp_sub_bits.load();
  return v > 0 ? v : kJpSubBits;
}

// jpeg_natural_order: zig-zag index -> natural (row-major) index
#define JP_ZIGZAG                                                                                                     \
  {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,    \
   7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46,   \
   53, 60, 61, 54, 47, 55, 62, 63}
static const uint8_t kZigzag[64] = JP_ZIGZAG;
__constant__ uint8_t c_zigzag[64] = JP_ZIGZAG;

// ---- header parse, on the host (jp_parse) and on the device (jpeg_parse_kernel) ---------------------------------
// Why jp_parse_head refused a file: the host reports kJpWhy[why], the device sets BDBNN_JPEG_RECORD.
enum {
  kJpOk, kJpNotJpeg, kJpBadMarker, kJpTruncated, kJpMarkerBeforeScan, kJpFrameHeader, kJpFrameParams, kJpSof, kJpDht,
  kJpDqt, kJpDri, kJpShortJfif, kJpShortAdobe, kJpMarker, kJpNoFrame, kJpScanHeader, kJpScanOrder, kJpUndefTable,
  kJpSpectral, kJpSampling, kJpAdobeTransform, kJpComponentIds, kJpDcTables, kJpAcTables, kJpHuffOverflow, kJpDcSymbol
};
static const char* const kJpWhy[] = {
    "ok", "not a JPEG", "bad marker", "truncated", "marker before the scan", "frame header", "frame parameters",
    "SOF other than 0 / 1", "DHT", "DQT", "DRI", "short JFIF marker", "short Adobe marker", "unknown marker",
    "no frame header", "scan header", "scan component order", "a component uses an undefined table",
    "spectral selection", "sampling", "Adobe transform", "component ids", "more than two DC tables",
    "more than two AC tables", "Huffman code overflow", "DC symbol > 15"};

// What the header fixes besides the descriptor's tables; scan: offset of the entropy-coded data (after SOS).
struct JpHead {
  int32_t H, W, ncomp, hmax, vmax, mcux, mcuy, bpm, restart;
  int64_t scan;
};

__host__ __device__ __forceinline__ bool jp_same(const uint8_t* s, const char* lit, int n) {
  for (int i = 0; i < n; ++i)
    if (s[i] != uint8_t(lit[i])) return false;
  return true;
}

// Canonical code assignment as jpeg_make_d_derived_tbl (which rejects the same tables); bits: the 16 code counts of
// a DHT table, vals: its symbols.
__host__ __device__ int jp_build_huff(const uint8_t* bits, const uint8_t* vals, bool is_dc, bdbnn_jpeg_huff* h) {
  memset(h, 0, sizeof(*h));
  int code = 0, i = 0;
  for (int L = 1; L <= 16; ++L) {
    const int cnt = bits[L - 1];
    if (cnt) {
      h->valoff[L] = i - code;
      h->maxcode[L] = code + cnt - 1;
    } else {
      h->maxcode[L] = -1;
    }
    for (int c = 0; c < cnt; ++c, ++code, ++i) {
      if (L <= 9) {
        const int lo = code << (9 - L), span = 1 << (9 - L);
        for (int x = 0; x < span; ++x) h->lut[lo + x] = uint16_t((L << 8) | vals[i]);
      }
    }
    if (code >= (1 << L)) return kJpHuffOverflow;
    code <<= 1;
  }
  h->maxcode[0] = -1;
  h->maxcode[17] = INT_MAX;
  for (int k = 0; k < i; ++k) {
    if (is_dc && vals[k] > 15) return kJpDcSymbol;
    h->vals[k] = vals[k];
  }
  return kJpOk;
}

// The markers of file d[0, n) up to SOS: *g and the descriptor's tables (blk_comp onwards; the fields before them are
// not touched).  Returns kJpOk or why the file is refused.  Every read stays inside [0, n).
__host__ __device__ int jp_parse_head(const uint8_t* d, int64_t n, JpHead* g, bdbnn_jpeg_desc* o) {
  if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return kJpNotJpeg;
  int64_t p = 2;
  int32_t q_at[4] = {-1, -1, -1, -1};            // offset of each quantisation table's values, -1 = undefined
  int q_prec[4] = {0, 0, 0, 0};
  int32_t h_at[2][4] = {{-1, -1, -1, -1}, {-1, -1, -1, -1}};   // [DC / AC][slot]: offset of the 16 code counts
  bool have_frame = false, jfif = false;
  int adobe = -1, restart = 0, H = 0, W = 0, nf = 0;
  int cid[3] = {0, 0, 0}, ch[3] = {0, 0, 0}, cv[3] = {0, 0, 0}, cq[3] = {0, 0, 0};
  const uint8_t* sos = nullptr;
  int sos_len = 0;
  while (sos == nullptr) {
    if (p + 2 > n || d[p] != 0xFF) return kJpBadMarker;
    while (p + 1 < n && d[p + 1] == 0xFF) ++p;
    if (p + 2 > n) return kJpTruncated;
    const int m = d[p + 1];
    p += 2;
    if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01 || m == 0x00) return kJpMarkerBeforeScan;
    if (p + 2 > n) return kJpTruncated;
    const int L = (d[p] << 8) | d[p + 1];
    if (L < 2 || p + L > n) return kJpTruncated;
    const uint8_t* s = d + p + 2;
    const int ls = L - 2;
    if (m == 0xC0 || m == 0xC1) {
      if (have_frame || ls < 6) return kJpFrameHeader;
      H = (s[1] << 8) | s[2];
      W = (s[3] << 8) | s[4];
      nf = s[5];
      if (s[0] != 8 || (nf != 1 && nf != 3) || ls != 6 + 3 * nf || H < 1 || W < 1 || H > kJpMaxSide ||
          W > kJpMaxSide)
        return kJpFrameParams;
      for (int i = 0; i < nf; ++i) {
        cid[i] = s[6 + 3 * i];
        ch[i] = s[7 + 3 * i] >> 4;
        cv[i] = s[7 + 3 * i] & 15;
        cq[i] = s[8 + 3 * i];
      }
      have_frame = true;
    } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      return kJpSof;
    } else if (m == 0xC4) {
      int q = 0;
      while (q < ls) {
        if (q + 17 > ls) return kJpDht;
        const int tc = s[q] >> 4, th = s[q] & 15;
        int cnt = 0;
        for (int i = 0; i < 16; ++i) cnt += s[q + 1 + i];
        if (tc > 1 || th > 3 || cnt > 256 || q + 17 + cnt > ls) return kJpDht;
        h_at[tc][th] = int32_t(s + q + 1 - d);
        q += 17 + cnt;
      }
    } else if (m == 0xDB) {
      int q = 0;
      while (q < ls) {
        const int pq = s[q] >> 4, tq = s[q] & 15;
        const int len = 64 * (pq + 1);
        if (pq > 1 || tq > 3 || q + 1 + len > ls) return kJpDqt;
        q_at[tq] = int32_t(s + q + 1 - d);
        q_prec[tq] = pq;
        q += 1 + len;
      }
    } else if (m == 0xDD) {
      if (ls != 2) return kJpDri;
      restart = (s[0] << 8) | s[1];
    } else if (m == 0xE0) {
      if (ls >= 5 && jp_same(s, "JFIF\0", 5)) {
        if (ls < 14) return kJpShortJfif;
        jfif = true;
      }
    } else if (m == 0xEE) {
      if (ls >= 5 && jp_same(s, "Adobe", 5)) {
        if (ls < 12) return kJpShortAdobe;
        adobe = s[11];
      }
    } else if (m == 0xDA) {
      sos = s;
      sos_len = ls;
    } else if (!((m >= 0xE0 && m <= 0xEF) || m == 0xFE)) {
      return kJpMarker;
    }
    p += L;
  }
  if (!have_frame) return kJpNoFrame;
  if (sos_len != 4 + 2 * nf || sos[0] != nf) return kJpScanHeader;
  int td[3], ta[3];
  for (int i = 0; i < nf; ++i) {
    if (sos[1 + 2 * i] != cid[i]) return kJpScanOrder;
    td[i] = sos[2 + 2 * i] >> 4;
    ta[i] = sos[2 + 2 * i] & 15;
    if (cq[i] > 3 || q_at[cq[i]] < 0 || td[i] > 3 || ta[i] > 3 || h_at[0][td[i]] < 0 || h_at[1][ta[i]] < 0)
      return kJpUndefTable;
  }
  if (sos[1 + 2 * nf] != 0 || sos[2 + 2 * nf] != 63 || sos[3 + 2 * nf] != 0) return kJpSpectral;
  int hmax = 1, vmax = 1;
  if (nf == 1) {
    // one component, non-interleaved: the MCU is one block whatever the declared factors
    if (ch[0] < 1 || ch[0] > 4 || cv[0] < 1 || cv[0] > 4) return kJpSampling;
  } else {
    const bool y_ok = (ch[0] == 1 && cv[0] == 1) || (ch[0] == 2 && cv[0] == 1) || (ch[0] == 2 && cv[0] == 2);
    if (!y_ok || ch[1] != 1 || cv[1] != 1 || ch[2] != 1 || cv[2] != 1) return kJpSampling;
    if (!jfif) {
      if (adobe >= 0 && adobe != 1) return kJpAdobeTransform;
      if (adobe < 0 && !(cid[0] == 1 && cid[1] == 2 && cid[2] == 3)) return kJpComponentIds;
    }
    hmax = ch[0];
    vmax = cv[0];
  }
  // descriptor tables
  memset(o->blk_comp, 0, sizeof(*o) - offsetof(bdbnn_jpeg_desc, blk_comp));
  g->H = H;
  g->W = W;
  g->ncomp = nf;
  g->hmax = hmax;
  g->vmax = vmax;
  g->mcux = (W + 8 * hmax - 1) / (8 * hmax);
  g->mcuy = (H + 8 * vmax - 1) / (8 * vmax);
  g->restart = restart;
  g->scan = p;
  int bpm = 0;
  for (int i = 0; i < hmax * vmax; ++i) o->blk_comp[bpm++] = 0;
  for (int c = 1; c < nf; ++c) o->blk_comp[bpm++] = uint8_t(c);
  g->bpm = bpm;
  int dslot[4] = {-1, -1, -1, -1}, aslot[4] = {-1, -1, -1, -1}, nd = 0, na = 0;
  for (int i = 0; i < nf; ++i) {
    const uint8_t* qv = d + q_at[cq[i]];
    for (int k = 0; k < 64; ++k) {
#ifdef __CUDA_ARCH__
      const int z = c_zigzag[k];
#else
      const int z = kZigzag[k];
#endif
      o->qt[i][z] = q_prec[cq[i]] ? uint16_t((qv[2 * k] << 8) | qv[2 * k + 1]) : qv[k];
    }
    if (dslot[td[i]] < 0) {
      if (nd == 2) return kJpDcTables;
      dslot[td[i]] = nd;
      const uint8_t* b = d + h_at[0][td[i]];
      if (int why = jp_build_huff(b, b + 16, true, &o->dc[nd])) return why;
      ++nd;
    }
    if (aslot[ta[i]] < 0) {
      if (na == 2) return kJpAcTables;
      aslot[ta[i]] = na;
      const uint8_t* b = d + h_at[1][ta[i]];
      if (int why = jp_build_huff(b, b + 16, false, &o->ac[na])) return why;
      ++na;
    }
    o->comp_dc[i] = uint8_t(dslot[td[i]]);
    o->comp_ac[i] = uint8_t(aslot[ta[i]]);
  }
  return kJpOk;
}

// ---- host parse ----------------------------------------------------------------------------------------------------
#define JP_REJECT(...)                \
  do {                                \
    ::bdbnn::set_error(__VA_ARGS__);  \
    return BDBNN_ERR_UNSUPPORTED;     \
  } while (0)

static int jp_parse(const uint8_t* d, int64_t n, bdbnn_jpeg_desc* o, uint8_t* out, int64_t out_cap,
                    uint32_t* seg_off, int32_t seg_cap) {
  memset(o, 0, sizeof(*o));
  JpHead g;
  if (int why = jp_parse_head(d, n, &g, o)) JP_REJECT("jpeg_parse: %s", kJpWhy[why]);
  o->H = g.H;
  o->W = g.W;
  o->ncomp = g.ncomp;
  o->hmax = g.hmax;
  o->vmax = g.vmax;
  o->mcux = g.mcux;
  o->mcuy = g.mcuy;
  o->bpm = g.bpm;
  o->restart = g.restart;
  const int restart = g.restart;
  int64_t p = g.scan;
  // entropy-coded data: unstuff, split at RSTn, end at EOI
  const int64_t total = int64_t(o->mcux) * o->mcuy;
  int64_t w = 0;
  int nseg = 0, expect = 0;
  if (seg_cap < 1) JP_REJECT("jpeg_parse: segment table full");
  seg_off[nseg++] = 0;
  for (;;) {
    if (p >= n) JP_REJECT("jpeg_parse: no EOI");
    const uint8_t c = d[p];
    if (c != 0xFF) {
      if (w >= out_cap) JP_REJECT("jpeg_parse: data buffer full");
      out[w++] = c;
      ++p;
      continue;
    }
    if (p + 1 >= n) JP_REJECT("jpeg_parse: no EOI");
    const uint8_t c2 = d[p + 1];
    p += 2;
    if (c2 == 0x00) {
      if (w >= out_cap) JP_REJECT("jpeg_parse: data buffer full");
      out[w++] = 0xFF;
    } else if (c2 >= 0xD0 && c2 <= 0xD7) {
      if (restart == 0 || c2 - 0xD0 != expect) JP_REJECT("jpeg_parse: restart marker out of sequence");
      expect = (expect + 1) & 7;
      if (nseg >= seg_cap) JP_REJECT("jpeg_parse: segment table full");
      seg_off[nseg++] = uint32_t(w);
    } else if (c2 == 0xD9) {
      break;
    } else {
      JP_REJECT("jpeg_parse: marker 0x%02x in the scan", c2);
    }
  }
  const int64_t R = restart ? restart : total;
  if (nseg != (total + R - 1) / R) JP_REJECT("jpeg_parse: %d segments for %lld MCUs", nseg, (long long)total);
  if (w >= (int64_t(1) << 27)) JP_REJECT("jpeg_parse: scan too large");
  o->nseg = nseg;
  o->data_bytes = int32_t(w);
  return BDBNN_OK;
}

// ---- Huffman, on the device and in the host index builder (bdbnn_jpeg_index_file) ----------------------------------
struct JpBits {
  const uint8_t* p;
  int32_t nbytes;
  uint64_t buf;                                   // left-aligned
  int32_t have, next, pos;

  __host__ __device__ void init(const uint8_t* data, int32_t nb, int32_t bitpos) {
    p = data;
    nbytes = nb;
    next = bitpos >> 3;
    buf = 0;
    have = 0;
    pos = bitpos & ~7;
    fill();
    skip(bitpos & 7);
  }
  __host__ __device__ __forceinline__ void fill() {
    while (have <= 56) {
#ifdef __CUDA_ARCH__
      const uint32_t b = next < nbytes ? uint32_t(__ldg(p + next)) : 0u;   // zeros past the end
#else
      const uint32_t b = next < nbytes ? uint32_t(p[next]) : 0u;
#endif
      buf |= uint64_t(b) << (56 - have);
      ++next;
      have += 8;
    }
  }
  __host__ __device__ __forceinline__ void skip(int n) {
    buf <<= n;
    have -= n;
    pos += n;
  }
};

__host__ __device__ __forceinline__ uint64_t jp_pack(int32_t pos, int b, int k) {
  return (uint64_t(uint32_t(pos)) << 16) | (uint64_t(b) << 8) | uint64_t(k);
}

// Decode codewords from (pos, b, k) until pos >= stop_pos or stop_blocks blocks are complete.  WRITE stores each
// value at coef[block * 64 + natural index] (DC differences at index 0).  Returns the status bits of the first fault
// (decoding stops there); `done` counts the completed blocks.  The host (index builder) runs only jp_run<false>.
template <bool WRITE>
__host__ __device__ int jp_run(const bdbnn_jpeg_desc* __restrict__ d, const uint8_t* seg, int32_t nbits, int32_t& pos,
                      int& b, int& k, int32_t stop_pos, int32_t stop_blocks, int32_t& done, int16_t* coef) {
  done = 0;
  if (pos >= stop_pos || stop_blocks <= 0) return 0;
  JpBits br;
  br.init(seg, nbits >> 3, pos);
  int ci = d->blk_comp[b];
  while (br.pos < stop_pos && done < stop_blocks) {
    br.fill();
    const bdbnn_jpeg_huff* t = k == 0 ? &d->dc[d->comp_dc[ci] & 1] : &d->ac[d->comp_ac[ci] & 1];
    const uint32_t e = t->lut[uint32_t(br.buf >> 55)];
    int L, sym;
    if (e) {
      L = int(e >> 8);
      sym = int(e & 255u);
    } else {
      const int32_t c16 = int32_t(br.buf >> 48);
      L = 10;
      while (L <= 16 && (c16 >> (16 - L)) > t->maxcode[L]) ++L;
      if (L > 16) {
        pos = br.pos;
        return BDBNN_JPEG_BAD_CODE;
      }
      sym = t->vals[((c16 >> (16 - L)) + t->valoff[L]) & 255];
    }
    int r, s;
    if (k == 0) {
      r = 0;
      s = sym & 15;
    } else {
      r = sym >> 4;
      s = sym & 15;
    }
    if (br.pos + L + s > nbits) {
      pos = br.pos;
      return BDBNN_JPEG_PAST_END;
    }
    br.skip(L);
    int v = 0;
    if (s) {
      v = int(uint32_t(br.buf >> (64 - s)));
      if (v < (1 << (s - 1))) v -= (1 << s) - 1;
      br.skip(s);
    }
    if (k == 0) {
      if (WRITE) coef[int64_t(done) * 64] = int16_t(v);
      k = 1;
    } else if (s) {
      k += r;
      if (k > 63) {
        pos = br.pos;
        return BDBNN_JPEG_K_OVERFLOW;
      }
      if constexpr (WRITE) {
#ifdef __CUDA_ARCH__
        coef[int64_t(done) * 64 + c_zigzag[k]] = int16_t(v);
#else
        coef[int64_t(done) * 64 + kZigzag[k]] = int16_t(v);
#endif
      }
      ++k;
    } else if (r == 15) {
      k += 16;
      if (k > 64) {
        pos = br.pos;
        return BDBNN_JPEG_K_OVERFLOW;
      }
    } else {
      k = 64;
    }
    if (k == 64) {
      k = 0;
      b = b + 1 == d->bpm ? 0 : b + 1;
      ci = d->blk_comp[b];
      ++done;
    }
  }
  pos = br.pos;
  return 0;
}

__device__ __forceinline__ int jp_find_seg(const bdbnn_jpeg_seg* segs, int nseg, int64_t i) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (segs[mid].sub0 <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

struct JpSub {
  const bdbnn_jpeg_desc* d;
  const uint8_t* data;
  int32_t nbits, end, first_in_seg;
};

__device__ __forceinline__ JpSub jp_sub(const bdbnn_jpeg_desc* descs, const bdbnn_jpeg_seg* segs, int nseg,
                                        const uint8_t* data, int64_t i, int S, int* seg_out) {
  const int s = jp_find_seg(segs, nseg, i);
  const bdbnn_jpeg_seg g = segs[s];
  const int32_t j = int32_t(i - g.sub0);
  JpSub r;
  r.d = descs + g.img;
  r.data = data + g.off;
  r.nbits = g.nbytes * 8;
  r.end = j + 1 == g.nsub ? INT_MAX : min((j + 1) * S, r.nbits);
  r.first_in_seg = j == 0;
  *seg_out = s;
  return r;
}

// Barrier rounds inside the CTA: every thread adopts its predecessor's exit (sh_exit) and decodes again until no
// start changes.  `again` starts the loop with a change already made.  Returns the rounds taken.
__device__ __forceinline__ int jp_local_fixpoint(const JpSub& q, bool active, uint64_t& st, uint64_t& ex, int32_t& nb,
                                 uint64_t* sh_exit, int again) {
  const int t = threadIdx.x;
  int rounds = 0;
  for (;;) {
    if (!__syncthreads_or(again)) break;
    ++rounds;
    const uint64_t pred = (active && t > 0 && !q.first_in_seg) ? sh_exit[t - 1] : st;
    __syncthreads();
    again = 0;
    if (active && pred != st) {
      st = pred;
      again = 1;
      int32_t pos = int32_t(st >> 16);
      int b = int((st >> 8) & 255), k = int(st & 255);
      jp_run<false>(q.d, q.data, q.nbits, pos, b, k, q.end, INT_MAX, nb, nullptr);
      ex = jp_pack(pos, b, k);
      sh_exit[t] = ex;
    }
  }
  return rounds;
}

// Phases 1 and 2 in one launch.  Each CTA takes the next tile of kJpThreads subsequences from an atomic counter, so
// a CTA only ever waits for tiles taken before it (already running).  Phase 1: decode from the guessed starts, then
// barrier rounds to the CTA's own fixed point.  Phase 2: unless its first subsequence starts a segment, the CTA waits
// for the previous tile's ready flag, adopts that tile's last exit (exact by induction) and runs barrier rounds
// again; then it publishes its exits and sets its own flag.  rounds_max: the most barrier rounds of a CTA.  (The
// minimum of one block per SM lifts ptxas's default 32-register budget here, which spilled.)
__global__ void __launch_bounds__(kJpThreads, 1)
jpeg_sync_kernel(const bdbnn_jpeg_desc* __restrict__ descs, const bdbnn_jpeg_seg* __restrict__ segs, int nseg,
                 const uint8_t* __restrict__ data, int64_t n_sub, int S, uint64_t* start, uint64_t* exit_state,
                 int32_t* __restrict__ cnt, int32_t* tile_counter, int32_t* ready, int32_t* rounds_max) {
  __shared__ uint64_t sh_exit[kJpThreads];
  __shared__ uint64_t sh_pred;
  __shared__ int sh_tile;
  const int t = threadIdx.x;
  if (t == 0) sh_tile = atomicAdd(tile_counter, 1);
  __syncthreads();
  const int tile = sh_tile;
  const int64_t i = int64_t(tile) * kJpThreads + t;
  const bool active = i < n_sub;
  JpSub q{};
  uint64_t st = 0, ex = 0;
  int32_t nb = 0;
  if (active) {
    int s;
    q = jp_sub(descs, segs, nseg, data, i, S, &s);
    st = q.first_in_seg ? 0 : jp_pack(int32_t((i - segs[s].sub0) * S), 0, 0);
    int32_t pos = int32_t(st >> 16);
    int b = 0, k = 0;
    jp_run<false>(q.d, q.data, q.nbits, pos, b, k, q.end, INT_MAX, nb, nullptr);
    ex = jp_pack(pos, b, k);
  }
  sh_exit[t] = ex;
  int rounds = jp_local_fixpoint(q, active, st, ex, nb, sh_exit, 1);
  if (t == 0) {
    sh_pred = st;
    if (active && !q.first_in_seg) {
      const volatile int32_t* flag = ready + tile - 1;
      while (*flag == 0) __nanosleep(64);
      __threadfence();
      sh_pred = *(reinterpret_cast<const volatile uint64_t*>(exit_state) + (i - 1));
    }
  }
  __syncthreads();
  int again = 0;
  if (t == 0 && active && sh_pred != st) {
    st = sh_pred;
    again = 1;
    int32_t pos = int32_t(st >> 16);
    int b = int((st >> 8) & 255), k = int(st & 255);
    jp_run<false>(q.d, q.data, q.nbits, pos, b, k, q.end, INT_MAX, nb, nullptr);
    ex = jp_pack(pos, b, k);
    sh_exit[0] = ex;
  }
  rounds += jp_local_fixpoint(q, active, st, ex, nb, sh_exit, again);
  if (active) {
    start[i] = st;
    exit_state[i] = ex;
    cnt[i] = nb;
  }
  __threadfence();
  __syncthreads();
  if (t == 0) {
    atomicExch(ready + tile, 1);
    atomicMax(rounds_max, rounds);
  }
}

// Index entry of subsequence j >= 1 of a segment (bdbnn_jpeg_index_file): its start state, the exit of subsequence
// j - 1, as bits 0-4 the overshoot pos - j S past its first bit, bits 5-7 the block in the MCU, bits 8-13 the
// zig-zag index.  Bits 14-15 are zero.
constexpr int kJpEntryOvershoot = 31;

__host__ __device__ __forceinline__ bool jp_entry_pack(int32_t pos, int b, int k, int32_t j, int S, uint16_t* e) {
  const int64_t ov = int64_t(pos) - int64_t(j) * S;
  if (ov < 0 || ov >= kJpEntryOvershoot || b < 0 || b > 7 || k < 0 || k > 63) return false;
  *e = uint16_t(ov | (b << 5) | (k << 8));
  return true;
}

__host__ __device__ __forceinline__ uint64_t jp_entry_state(uint16_t e, int32_t j, int S) {
  return jp_pack(j * S + (e & 31), (e >> 5) & 7, (e >> 8) & 63);
}

// Replaces phases 1-2 when the starts come from an index: thread i takes its start from the entries (the segment's
// first subsequence starts at (0, 0, 0); segment s's entries begin at sub0 - s), decodes to its exit as phase 1 does
// and writes start[i] and cnt[i] for phases 3-4.  If the exit is not the segment's next stored start, or a stored
// start is malformed, the image gets BDBNN_JPEG_INDEX.  No waits: when every exit equals the next stored start, the
// stored starts are the sequential decode's states by induction from the segment's first, so phases 3-4 see what
// they see after phase 2.  A malformed start is replaced by the guess (j S, 0, 0) so that the later kernels stay in
// bounds.  (Four blocks per SM lift ptxas's default register budget, which spilled.)
__global__ void __launch_bounds__(kJpThreads, 4)
jpeg_index_check_kernel(const bdbnn_jpeg_desc* __restrict__ descs, const bdbnn_jpeg_seg* __restrict__ segs, int nseg,
                        const uint8_t* __restrict__ data, int64_t n_sub, int S, const uint16_t* __restrict__ entries,
                        uint64_t* __restrict__ start, int32_t* __restrict__ cnt, int32_t* __restrict__ status) {
  const int64_t i = int64_t(blockIdx.x) * kJpThreads + threadIdx.x;
  if (i >= n_sub) return;
  int s;
  const JpSub q = jp_sub(descs, segs, nseg, data, i, S, &s);
  const bdbnn_jpeg_seg g = segs[s];
  const int32_t j = int32_t(i - g.sub0);
  bool bad = false;
  uint64_t st = 0;
  if (j > 0) {
    const uint16_t e = entries[i - s - 1];
    st = jp_entry_state(e, j, S);
    if ((e >> 14) != 0 || ((e >> 5) & 7) >= q.d->bpm) {
      bad = true;
      st = jp_pack(j * S, 0, 0);
    }
  }
  int32_t pos = int32_t(st >> 16), nb = 0;
  int b = int((st >> 8) & 255), k = int(st & 255);
  jp_run<false>(q.d, q.data, q.nbits, pos, b, k, q.end, INT_MAX, nb, nullptr);
  start[i] = st;
  cnt[i] = nb;
  if (j + 1 < g.nsub && jp_pack(pos, b, k) != jp_entry_state(entries[i - s], j + 1, S)) bad = true;
  if (bad) atomicOr(status + g.img, BDBNN_JPEG_INDEX);
}

// ---- device: parse and unstuff of the original files (bdbnn_jpeg_decode_batch_files) -------------------------------
// One thread per image: the header half of the host parse, building the descriptor's tables in place.  The
// geometry the host took from the image's record stays as it is and is compared with the file's; any difference, or
// anything the host parse refuses, flags the image with BDBNN_JPEG_RECORD and sets its scan offset to -1.
__global__ void __launch_bounds__(128)
jpeg_parse_kernel(const uint8_t* __restrict__ files, bdbnn_jpeg_file* __restrict__ ftab,
                  bdbnn_jpeg_desc* __restrict__ descs, int n_img, int32_t* __restrict__ status) {
  const int i = int(blockIdx.x) * 128 + int(threadIdx.x);
  if (i >= n_img) return;
  const bdbnn_jpeg_file f = ftab[i];
  bdbnn_jpeg_desc* o = descs + i;
  JpHead g;
  const int why = jp_parse_head(files + f.off, f.size, &g, o);
  const bool bad = why != kJpOk || g.H != o->H || g.W != o->W || g.ncomp != o->ncomp || g.hmax != o->hmax ||
                   g.vmax != o->vmax || g.mcux != o->mcux || g.mcuy != o->mcuy || g.bpm != o->bpm ||
                   g.restart != o->restart;
  ftab[i].scan = bad ? -1 : int32_t(g.scan);
  if (bad) atomicOr(status + i, BDBNN_JPEG_RECORD);
}

constexpr int kJpUnBytes = 16;                    // scan bytes per thread per tile of jpeg_unstuff_kernel

__device__ __forceinline__ int jp_first_seg(const bdbnn_jpeg_seg* segs, int nseg, int img) {
  int lo = 0, hi = nseg;                          // first segment of an image >= img
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (segs[mid].img < img) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Block-wide exclusive sum of v (every thread of a kJpThreads block calls it); *total receives the sum.
__device__ __forceinline__ uint64_t jp_block_scan(uint64_t v, uint64_t* sh_warp, uint64_t* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint64_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) sh_warp[wid] = incl;
  __syncthreads();
  uint64_t before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kJpThreads / 32; ++w) {
    const uint64_t x = sh_warp[w];
    before += w < wid ? x : 0;
    all += x;
  }
  __syncthreads();
  *total = all;
  return before + incl - v;
}

// One CUDA block per image: the host parse's unstuff and RST split, in parallel over tiles of kJpThreads x
// kJpUnBytes scan bytes.  Within the scan an FF pairs with the next byte (00: a data FF, D0-D7: a segment end, D9:
// the end of the scan, anything else refused), so a byte's fate follows from its predecessor: each thread counts the
// data bytes and RST markers of its bytes before the scan's end, a block scan gives their positions, and a second
// walk writes the bytes to data at the image's data_off.  The RST sequence, each segment's start (the record's, in
// segs) and the total against data_bytes are checked; any difference sets BDBNN_JPEG_RECORD.  No byte is written at
// or past data_off + data_bytes, and no byte past the file is read.
__global__ void __launch_bounds__(kJpThreads)
jpeg_unstuff_kernel(const uint8_t* __restrict__ files, const bdbnn_jpeg_file* __restrict__ ftab,
                    const bdbnn_jpeg_desc* __restrict__ descs, const bdbnn_jpeg_seg* __restrict__ segs, int nseg,
                    uint8_t* __restrict__ data, int32_t* __restrict__ status) {
  __shared__ uint64_t sh_warp[kJpThreads / 32];
  __shared__ unsigned long long sh_end;
  const int img = blockIdx.x, t = threadIdx.x;
  const bdbnn_jpeg_file f = ftab[img];
  if (f.scan < 0) return;                         // the parse flagged the image
  const bdbnn_jpeg_desc* d = descs + img;
  const uint8_t* src = files + f.off;
  const int s0 = jp_first_seg(segs, nseg, img), s1 = jp_first_seg(segs, nseg, img + 1);
  const int64_t size = f.size, scan = f.scan, nbytes = d->data_bytes;
  uint8_t* out = data + d->data_off;
  int64_t out0 = 0, rst0 = 0;
  bool bad = false, ended = false;
  for (int64_t base = scan; base < size; base += int64_t(kJpThreads) * kJpUnBytes) {
    const int64_t p0 = base + int64_t(t) * kJpUnBytes;
    uint8_t b[kJpUnBytes + 1];
#pragma unroll
    for (int j = 0; j <= kJpUnBytes; ++j) b[j] = p0 + j < size ? __ldg(src + p0 + j) : 0;
    const bool prev_ff = p0 > scan && p0 - 1 < size && __ldg(src + p0 - 1) == 0xFF;
    // pair starts: an FF whose predecessor is not an FF; the end is the first pair start followed by D9
    if (t == 0) sh_end = ULLONG_MAX;
    __syncthreads();
    int64_t end = INT64_MAX;
#pragma unroll
    for (int j = 0; j < kJpUnBytes; ++j) {
      const bool tail = j == 0 ? prev_ff : b[j - 1] == 0xFF;
      if (end == INT64_MAX && p0 + j + 1 < size && b[j] == 0xFF && !tail && b[j + 1] == 0xD9) end = p0 + j;
    }
    if (end != INT64_MAX) atomicMin(&sh_end, (unsigned long long)end);
    __syncthreads();
    const int64_t e = sh_end == ULLONG_MAX ? INT64_MAX : int64_t(sh_end);
    uint32_t n_data = 0, n_rst = 0;
#pragma unroll
    for (int j = 0; j < kJpUnBytes; ++j) {
      const int64_t p = p0 + j;
      const bool tail = j == 0 ? prev_ff : b[j - 1] == 0xFF;
      if (p >= e || p >= size || tail) continue;
      if (b[j] != 0xFF) {
        ++n_data;
      } else if (p + 1 < size) {
        const uint8_t c2 = b[j + 1];
        if (c2 == 0x00) ++n_data;
        else if (c2 >= 0xD0 && c2 <= 0xD7) ++n_rst;
        else bad = true;                          // FF FF, or a foreign marker, before the end
      }
    }
    uint64_t tile;
    const uint64_t before = jp_block_scan((uint64_t(n_rst) << 32) | n_data, sh_warp, &tile);
    int64_t w = out0 + int64_t(before & 0xFFFFFFFFu), k = rst0 + int64_t(before >> 32);
#pragma unroll
    for (int j = 0; j < kJpUnBytes; ++j) {
      const int64_t p = p0 + j;
      const bool tail = j == 0 ? prev_ff : b[j - 1] == 0xFF;
      if (p >= e || p >= size || tail) continue;
      if (b[j] != 0xFF || (p + 1 < size && b[j + 1] == 0x00)) {
        if (w < nbytes) out[w] = b[j];
        ++w;
      } else if (p + 1 < size && b[j + 1] >= 0xD0 && b[j + 1] <= 0xD7) {
        // RST k ends segment k: it must be D0 + k mod 8, and segment k + 1 must start where the record says
        if (d->restart == 0 || b[j + 1] - 0xD0 != int(k & 7) || s0 + k + 1 >= s1 ||
            segs[s0 + k + 1].off - d->data_off != w)
          bad = true;
        ++k;
      }
    }
    out0 += int64_t(tile & 0xFFFFFFFFu);
    rst0 += int64_t(tile >> 32);
    if (e != INT64_MAX) {
      ended = true;
      break;
    }
  }
  bad = __syncthreads_or(bad);
  if (t == 0 && (bad || !ended || out0 != nbytes || rst0 + 1 != s1 - s0)) atomicOr(status + img, BDBNN_JPEG_RECORD);
}

// Phase 3: first[i] = blocks completed by the segment's earlier subsequences (one warp per segment).
__global__ void jpeg_scan_kernel(const bdbnn_jpeg_seg* __restrict__ segs, int nseg, const int32_t* __restrict__ cnt,
                                 int32_t* __restrict__ first) {
  const int s = int((int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (s >= nseg) return;
  const bdbnn_jpeg_seg g = segs[s];
  int64_t base = 0;
  for (int j0 = 0; j0 < g.nsub; j0 += 32) {
    const int j = j0 + lane;
    const int64_t v = j < g.nsub ? cnt[g.sub0 + j] : 0;
    int64_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (j < g.nsub) first[g.sub0 + j] = int32_t(min(base + incl - v, int64_t(INT_MAX)));
    base += __shfl_sync(0xffffffffu, incl, 31);
  }
}

// Phase 4: decode from the synchronised starts and write the coefficients.
__global__ void __launch_bounds__(kJpThreads)
jpeg_write_kernel(const bdbnn_jpeg_desc* __restrict__ descs, const bdbnn_jpeg_seg* __restrict__ segs, int nseg,
                  const uint8_t* __restrict__ data, int64_t n_sub, int S, const uint64_t* __restrict__ start,
                  const int32_t* __restrict__ first, int16_t* __restrict__ coef, int32_t* __restrict__ status) {
  const int64_t i = int64_t(blockIdx.x) * kJpThreads + threadIdx.x;
  if (i >= n_sub) return;
  int s;
  const JpSub q = jp_sub(descs, segs, nseg, data, i, S, &s);
  const bdbnn_jpeg_seg g = segs[s];
  const int32_t total = g.nmcu * q.d->bpm;
  const int32_t b0 = first[i];
  if (b0 >= total) return;
  const uint64_t st = start[i];
  int32_t pos = int32_t(st >> 16), done = 0;
  int b = int((st >> 8) & 255), k = int(st & 255);
  int16_t* out = coef + (q.d->coef_off + int64_t(g.mcu0) * q.d->bpm + b0) * 64;
  int f = jp_run<true>(q.d, q.data, q.nbits, pos, b, k, q.end, total - b0, done, out);
  if (b0 + done == total && q.nbits - pos > 7) f |= BDBNN_JPEG_PADDING;
  if (f) atomicOr(status + g.img, f);
}

// DC prediction: per-component running sums of the DC differences within each segment, in decode order.
__global__ void __launch_bounds__(128)
jpeg_dc_kernel(const bdbnn_jpeg_desc* __restrict__ descs, const bdbnn_jpeg_seg* __restrict__ segs,
               int16_t* __restrict__ coef, int32_t* __restrict__ status) {
  __shared__ long long sums[3][128];
  const bdbnn_jpeg_seg g = segs[blockIdx.x];
  const bdbnn_jpeg_desc* d = descs + g.img;
  const int bpm = d->bpm, t = threadIdx.x;
  int16_t* base = coef + (d->coef_off + int64_t(g.mcu0) * bpm) * 64;
  const int per = (g.nmcu + 127) / 128;
  const int m0 = min(t * per, g.nmcu), m1 = min(m0 + per, g.nmcu);
  long long a0 = 0, a1 = 0, a2 = 0;                // per component, in registers
  for (int m = m0; m < m1; ++m)
    for (int j = 0; j < bpm; ++j) {
      const int c = d->blk_comp[j];
      const long long v = base[(int64_t(m) * bpm + j) * 64];
      a0 += c == 0 ? v : 0;
      a1 += c == 1 ? v : 0;
      a2 += c == 2 ? v : 0;
    }
  sums[0][t] = a0;
  sums[1][t] = a1;
  sums[2][t] = a2;
  __syncthreads();
  if (t < 3) {
    long long run = 0;
    for (int u = 0; u < 128; ++u) {
      const long long v = sums[t][u];
      sums[t][u] = run;
      run += v;
    }
  }
  __syncthreads();
  a0 = sums[0][t];
  a1 = sums[1][t];
  a2 = sums[2][t];
  bool bad = false;
  for (int m = m0; m < m1; ++m)
    for (int j = 0; j < bpm; ++j) {
      int16_t* p = base + (int64_t(m) * bpm + j) * 64;
      const int c = d->blk_comp[j];
      long long a = (c == 0 ? a0 : (c == 1 ? a1 : a2)) + *p;
      if (c == 0) a0 = a;
      else if (c == 1) a1 = a;
      else a2 = a;
      bad |= a < -32768 || a > 32767;
      *p = int16_t(a);
    }
  if (bad) atomicOr(status + g.img, BDBNN_JPEG_DC_RANGE);
}

// ---- device: pixels ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int jp_find_img(const bdbnn_jpeg_desc* descs, int n, int64_t v, bool by_rgb) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const int64_t o = by_rgb ? descs[mid].rgb_off / 3 : descs[mid].coef_off;
    if (o <= v) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

constexpr int kCB = 13, kP1 = 2;
// jidctint.c's 1-D pass on in[0..7] (64-bit, as JLONG), outputs DESCALEd by `shift`.
__device__ __forceinline__ void jp_idct_1d(const long long* in, long long* out, int shift) {
  long long z2 = in[2], z3 = in[6];
  long long z1 = (z2 + z3) * 4433;
  const long long tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
  const long long tmp0 = (in[0] + in[4]) * (1LL << kCB), tmp1 = (in[0] - in[4]) * (1LL << kCB);
  const long long t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  long long o0 = in[7], o1 = in[5], o2 = in[3], o3 = in[1];
  z1 = o0 + o3;
  z2 = o1 + o2;
  z3 = o0 + o2;
  long long z4 = o1 + o3;
  const long long z5 = (z3 + z4) * 9633;
  o0 *= 2446;
  o1 *= 16819;
  o2 *= 25172;
  o3 *= 12299;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  o0 += z1 + z3;
  o1 += z2 + z4;
  o2 += z2 + z3;
  o3 += z1 + z4;
  const long long r = 1LL << (shift - 1);
  out[0] = (t10 + o3 + r) >> shift;
  out[7] = (t10 - o3 + r) >> shift;
  out[1] = (t11 + o2 + r) >> shift;
  out[6] = (t11 - o2 + r) >> shift;
  out[2] = (t12 + o1 + r) >> shift;
  out[5] = (t12 - o1 + r) >> shift;
  out[3] = (t13 + o0 + r) >> shift;
  out[4] = (t13 - o0 + r) >> shift;
}

// jpeg_idct_islow, 8 threads per block: thread c runs column c (pass 1) then row c (pass 2) and stores 8 samples
// into the component's plane.  The all-zero-AC shortcuts of jidctint.c give the same values as the general path.
__global__ void __launch_bounds__(kJpThreads)
jpeg_idct_kernel(const bdbnn_jpeg_desc* __restrict__ descs, int n_img, int64_t n_blocks,
                 const int16_t* __restrict__ coef, uint8_t* __restrict__ planes, int32_t* __restrict__ status) {
  __shared__ int32_t ws[kJpThreads / 8][64];
  const int64_t g = (int64_t(blockIdx.x) * kJpThreads + threadIdx.x) >> 3;
  const int c = threadIdx.x & 7, lb = threadIdx.x >> 3;
  const bool active = g < n_blocks;
  int img = 0;
  bool risky = false;
  if (active) {
    img = jp_find_img(descs, n_img, g, false);
    const bdbnn_jpeg_desc* d = descs + img;
    const int64_t local = g - d->coef_off;
    const int bi = int(local % d->bpm);
    const int ci = d->blk_comp[bi] % 3;
    const int16_t* cf = coef + g * 64;
    long long in[8], out[8];
    for (int r = 0; r < 8; ++r) {
      in[r] = (long long)cf[r * 8 + c] * d->qt[ci][r * 8 + c];
      risky |= in[r] > 32767 || in[r] < -32768;
    }
    jp_idct_1d(in, out, kCB - kP1);
    for (int r = 0; r < 8; ++r) {
      const int32_t w = int32_t(out[r]);
      risky |= w > 32767 || w < -32768;
      ws[lb][r * 8 + c] = w;
    }
  }
  __syncwarp();
  if (active) {
    const bdbnn_jpeg_desc* d = descs + img;
    const int64_t local = g - d->coef_off;
    const int64_t mcu = local / d->bpm;
    const int bi = int(local % d->bpm);
    const int ci = d->blk_comp[bi] % 3;
    const int my = int(mcu / d->mcux), mx = int(mcu % d->mcux);
    const int h = ci == 0 ? d->hmax : 1, v = ci == 0 ? d->vmax : 1;
    const int by = my * v + (ci == 0 ? bi / h : 0), bx = mx * h + (ci == 0 ? bi % h : 0);
    const int64_t luma = int64_t(d->mcux) * d->mcuy * d->hmax * d->vmax * 64;
    const int64_t chroma = int64_t(d->mcux) * d->mcuy * 64;
    uint8_t* plane = planes + d->coef_off * 64 + (ci == 0 ? 0 : luma + (ci - 1) * chroma);
    const int pw = d->mcux * h * 8;
    long long in[8], out[8];
    for (int x = 0; x < 8; ++x) in[x] = ws[lb][c * 8 + x];
    jp_idct_1d(in, out, kCB + kP1 + 3);
    uint8_t* o = plane + int64_t(by * 8 + c) * pw + bx * 8;
    for (int x = 0; x < 8; ++x) {
      const long long val = out[x];
      risky |= val > 511 || val < -512;
      const int w = int(val & 1023);                  // range_limit[x & RANGE_MASK]
      o[x] = uint8_t(w < 128 ? w + 128 : (w < 512 ? 255 : (w < 896 ? 0 : w - 896)));
    }
  }
  if (active && risky) atomicOr(status + img, BDBNN_JPEG_IDCT_RANGE);
}

__device__ __forceinline__ int jp_clamp8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// Chroma sample at output (y, x) of a plane with row pitch pw: libjpeg-turbo's upsampler for (hmax, vmax), fancy when
// the downsampled width exceeds 2, else replication; the first and last real rows serve as the context rows.
__device__ __forceinline__ int jp_chroma(const uint8_t* c, int pw, int y, int x, int hmax, int vmax, int dw, int dh) {
  if (hmax == 1) return c[int64_t(y) * pw + x];
  const int cx = x >> 1, cy = vmax == 2 ? y >> 1 : y;
  if (dw <= 2) return c[int64_t(cy) * pw + cx];
  const uint8_t* row = c + int64_t(cy) * pw;
  if (vmax == 1) {
    if ((x & 1) == 0) return cx == 0 ? row[0] : (3 * row[cx] + row[cx - 1] + 1) >> 2;
    return cx == dw - 1 ? row[cx] : (3 * row[cx] + row[cx + 1] + 2) >> 2;
  }
  const int fy = (y & 1) == 0 ? max(cy - 1, 0) : min(cy + 1, dh - 1);
  const uint8_t* far = c + int64_t(fy) * pw;
  const int cs = 3 * row[cx] + far[cx];
  if ((x & 1) == 0) return cx == 0 ? (4 * cs + 8) >> 4 : (3 * cs + 3 * row[cx - 1] + far[cx - 1] + 8) >> 4;
  return cx == dw - 1 ? (4 * cs + 7) >> 4 : (3 * cs + 3 * row[cx + 1] + far[cx + 1] + 7) >> 4;
}

// One thread per output pixel: upsampling and ycc_rgb_convert (build_ycc_rgb_table's fixed point), or gray.
__global__ void __launch_bounds__(kJpThreads)
jpeg_color_kernel(const bdbnn_jpeg_desc* __restrict__ descs, int n_img, int64_t n_pix,
                  const uint8_t* __restrict__ planes, uint8_t* __restrict__ rgb) {
  const int64_t g = int64_t(blockIdx.x) * kJpThreads + threadIdx.x;
  if (g >= n_pix) return;
  const bdbnn_jpeg_desc* d = descs + jp_find_img(descs, n_img, g, true);
  const int64_t p = g - d->rgb_off / 3;
  const int y = int(p / d->W), x = int(p % d->W);
  const uint8_t* py = planes + d->coef_off * 64;
  const int pwy = d->mcux * d->hmax * 8;
  const int Y = py[int64_t(y) * pwy + x];
  uint8_t* o = rgb + d->rgb_off + p * 3;
  if (d->ncomp == 1) {
    o[0] = o[1] = o[2] = uint8_t(Y);
    return;
  }
  const int64_t luma = int64_t(d->mcux) * d->mcuy * d->hmax * d->vmax * 64;
  const int64_t chroma = int64_t(d->mcux) * d->mcuy * 64;
  const int pwc = d->mcux * 8;
  const int dw = (d->W + d->hmax - 1) / d->hmax, dh = (d->H + d->vmax - 1) / d->vmax;
  const int cb = jp_chroma(py + luma, pwc, y, x, d->hmax, d->vmax, dw, dh) - 128;
  const int cr = jp_chroma(py + luma + chroma, pwc, y, x, d->hmax, d->vmax, dw, dh) - 128;
  o[0] = uint8_t(jp_clamp8(Y + ((91881 * cr + 32768) >> 16)));
  o[1] = uint8_t(jp_clamp8(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)));
  o[2] = uint8_t(jp_clamp8(Y + ((116130 * cb + 32768) >> 16)));
}

struct JpWork {
  int16_t* coef;
  uint8_t* planes;
  uint64_t *start, *exit;
  int32_t *cnt, *first, *ready, *counters;     // counters: tile counter, rounds
};

static size_t jp_align(size_t v) { return (v + 255) & ~size_t(255); }

static size_t jp_layout(int64_t n_blocks, int64_t n_sub, uint8_t* base, JpWork* w) {
  size_t o = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? base + o : nullptr;
    o += jp_align(bytes);
    return p;
  };
  JpWork t;
  t.coef = reinterpret_cast<int16_t*>(take(size_t(n_blocks) * 128));
  t.planes = take(size_t(n_blocks) * 64);
  t.start = reinterpret_cast<uint64_t*>(take(size_t(n_sub) * 8));
  t.exit = reinterpret_cast<uint64_t*>(take(size_t(n_sub) * 8));
  t.cnt = reinterpret_cast<int32_t*>(take(size_t(n_sub) * 4));
  t.first = reinterpret_cast<int32_t*>(take(size_t(n_sub) * 4));
  t.ready = reinterpret_cast<int32_t*>(take(size_t((n_sub + kJpThreads - 1) / kJpThreads) * 4));
  t.counters = reinterpret_cast<int32_t*>(take(8));
  if (w) *w = t;
  return o;
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_jpeg_parse(const uint8_t* file_host, int64_t file_bytes, bdbnn_jpeg_desc* desc_host,
                                uint8_t* data_host, int64_t data_cap, uint32_t* seg_off_host, int32_t seg_cap) {
  BDBNN_REQUIRE(file_host && desc_host && data_host && seg_off_host, "jpeg_parse: NULL pointer");
  BDBNN_REQUIRE(file_bytes >= 0 && data_cap >= 0 && seg_cap >= 0, "jpeg_parse: negative size");
  return jp_parse(file_host, file_bytes, desc_host, data_host, data_cap, seg_off_host, seg_cap);
}

// Scratch of bdbnn_jpeg_index_file: the descriptor, the segment offsets, the unstuffed data.
static size_t jp_index_scratch(int64_t file_bytes, size_t* seg_at, size_t* data_at) {
  *seg_at = jp_align(sizeof(bdbnn_jpeg_desc));
  *data_at = *seg_at + jp_align(size_t(file_bytes / 3 + 2) * 4);
  return *data_at + size_t(file_bytes);
}

extern "C" int bdbnn_debug_jpeg_index_entry(int32_t pos, int32_t b, int32_t k, int32_t j, int32_t S, uint16_t* entry,
                                            int32_t* state) {
  BDBNN_REQUIRE(entry && state, "debug_jpeg_index_entry: NULL pointer");
  BDBNN_REQUIRE(j >= 1 && S >= 8 && S <= (1 << 20) && int64_t(j) * S + 31 < INT_MAX,
                "debug_jpeg_index_entry: j = %d, S = %d outside range", j, S);
  if (!jp_entry_pack(pos, b, k, j, S, entry)) return BDBNN_ERR_UNSUPPORTED;
  const uint64_t st = jp_entry_state(*entry, j, S);
  state[0] = int32_t(st >> 16);
  state[1] = int32_t((st >> 8) & 255);
  state[2] = int32_t(st & 255);
  return BDBNN_OK;
}

extern "C" size_t bdbnn_jpeg_index_scratch_bytes(int64_t file_bytes) {
  if (file_bytes < 0 || file_bytes >= (int64_t(1) << 31)) return 0;
  size_t seg_at, data_at;
  return jp_index_scratch(file_bytes, &seg_at, &data_at);
}

// The sequential decode of each segment, cut at the same subsequence ends with the same unlimited block count as
// phase 1, so each recorded exit is the start phase 2 converges to.  The last subsequence is decoded to the segment's
// last block, as phase 4 decodes it, so that a stream the device would flag (cut short, corrupt, padded by more than
// 7 bits) is refused here and goes to the host decoder without a trip through the device.
extern "C" int bdbnn_jpeg_index_file(const uint8_t* file_host, int64_t file_bytes, int32_t S, void* scratch,
                                     size_t scratch_cap, uint16_t* entries, int64_t entry_cap, int64_t* n_entries,
                                     int32_t* n_seg) {
  BDBNN_REQUIRE(file_host && scratch && entries && n_entries && n_seg, "jpeg_index_file: NULL pointer");
  BDBNN_REQUIRE(file_bytes >= 0 && file_bytes < (int64_t(1) << 31) && entry_cap >= 0,
                "jpeg_index_file: file of %lld bytes or entry_cap %lld outside range", (long long)file_bytes,
                (long long)entry_cap);
  BDBNN_REQUIRE(S >= 8 && S <= (1 << 20), "jpeg_index_file: S = %d outside [8, 2^20]", S);
  BDBNN_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "jpeg_index_file: scratch not 8-byte aligned");
  size_t seg_at, data_at;
  BDBNN_REQUIRE(scratch_cap >= jp_index_scratch(file_bytes, &seg_at, &data_at),
                "jpeg_index_file: scratch of %zu bytes, need %zu", scratch_cap,
                jp_index_scratch(file_bytes, &seg_at, &data_at));
  uint8_t* base = static_cast<uint8_t*>(scratch);
  bdbnn_jpeg_desc* d = reinterpret_cast<bdbnn_jpeg_desc*>(base);
  uint32_t* seg_off = reinterpret_cast<uint32_t*>(base + seg_at);
  uint8_t* data = base + data_at;
  if (int rc = jp_parse(file_host, file_bytes, d, data, file_bytes, seg_off, int32_t(file_bytes / 3 + 2))) return rc;
  const int64_t total = int64_t(d->mcux) * d->mcuy, R = d->restart ? d->restart : total;
  int64_t n = 0;
  for (int sg = 0; sg < d->nseg; ++sg) {
    const uint32_t off = seg_off[sg];
    const int32_t nbytes = int32_t((sg + 1 < d->nseg ? seg_off[sg + 1] : uint32_t(d->data_bytes)) - off);
    const int32_t nbits = nbytes * 8;
    const int32_t nsub = std::max(1, int32_t((int64_t(nbits) + S - 1) / S));
    const int64_t nblk = std::min(R, total - sg * R) * d->bpm;
    int32_t pos = 0, done = 0;
    int b = 0, k = 0;
    int64_t blocks = 0;
    for (int32_t j = 1; j < nsub; ++j) {
      if (int f = jp_run<false>(d, data + off, nbits, pos, b, k, j * S, INT_MAX, done, nullptr))
        JP_REJECT("jpeg_index_file: segment %d: status %d before bit %lld", sg, f, (long long)j * S);
      blocks += done;
      BDBNN_REQUIRE(n < entry_cap, "jpeg_index_file: more than entry_cap = %lld entries", (long long)entry_cap);
      if (!jp_entry_pack(pos, b, k, j, S, entries + n))
        JP_REJECT("jpeg_index_file: segment %d: state (%d, %d, %d) at subsequence %d has no entry", sg, pos, b, k, j);
      ++n;
    }
    if (blocks > nblk) JP_REJECT("jpeg_index_file: segment %d: data past its last block", sg);
    const int f = jp_run<false>(d, data + off, nbits, pos, b, k, INT_MAX, int32_t(nblk - blocks), done, nullptr);
    if (f || blocks + done != nblk || nbits - pos > 7)
      JP_REJECT("jpeg_index_file: segment %d: status %d, %lld of %lld blocks, %d bits left", sg, f,
                (long long)(blocks + done), (long long)nblk, nbits - pos);
  }
  *n_entries = n;
  *n_seg = d->nseg;
  return BDBNN_OK;
}

extern "C" int bdbnn_jpeg_subseq_bits(void) { return jp_sub_bits(); }

extern "C" int bdbnn_debug_jpeg_subseq_bits(int32_t bits) {
  BDBNN_REQUIRE(bits == 0 || (bits >= 8 && bits <= (1 << 20)), "debug_jpeg_subseq_bits: %d outside {0} U [8, 2^20]",
                bits);
  g_jp_sub_bits.store(bits);
  return BDBNN_OK;
}

extern "C" size_t bdbnn_jpeg_workspace_bytes(int64_t n_blocks, int64_t n_sub) {
  if (n_blocks < 0 || n_sub < 0) return 0;
  return jp_layout(n_blocks, n_sub, nullptr, nullptr);
}

// Host validation of a batch's tables against the buffer sizes (bdbnn_jpeg_check_batch); on success the batch's
// blocks, pixels and subsequences.
static int jp_check(const bdbnn_jpeg_desc* desc_host, int32_t n_img, const bdbnn_jpeg_seg* seg_host, int32_t n_seg,
                    int64_t data_bytes, int64_t rgb_bytes, size_t work_bytes, int64_t* blocks_out, int64_t* pix_out,
                    int64_t* n_sub_out) {
  BDBNN_REQUIRE(desc_host && seg_host, "jpeg_check_batch: NULL pointer");
  BDBNN_REQUIRE(n_img >= 1 && n_seg >= n_img, "jpeg_check_batch: need n_img >= 1 and n_seg >= n_img, got %d, %d",
                n_img, n_seg);
  BDBNN_REQUIRE(data_bytes >= 0 && rgb_bytes >= 0, "jpeg_check_batch: negative size");
  const int S = jp_sub_bits();
  int64_t blocks = 0, pix = 0;
  for (int i = 0; i < n_img; ++i) {
    const bdbnn_jpeg_desc& d = desc_host[i];
    BDBNN_REQUIRE(d.H >= 1 && d.W >= 1 && d.H <= kJpMaxSide && d.W <= kJpMaxSide,
                  "jpeg_check_batch: image %d: %d x %d outside [1, %d]", i, d.H, d.W, kJpMaxSide);
    const bool samp = d.ncomp == 1 ? (d.hmax == 1 && d.vmax == 1 && d.bpm == 1)
                                   : (d.ncomp == 3 && d.bpm == d.hmax * d.vmax + 2 &&
                                      ((d.hmax == 1 && d.vmax == 1) || (d.hmax == 2 && (d.vmax == 1 || d.vmax == 2))));
    BDBNN_REQUIRE(samp, "jpeg_check_batch: image %d: unsupported sampling", i);
    BDBNN_REQUIRE(d.mcux == (d.W + 8 * d.hmax - 1) / (8 * d.hmax) && d.mcuy == (d.H + 8 * d.vmax - 1) / (8 * d.vmax),
                  "jpeg_check_batch: image %d: MCU grid inconsistent with the size", i);
    for (int j = 0; j < d.bpm; ++j)
      BDBNN_REQUIRE(d.blk_comp[j] == (j < d.hmax * d.vmax ? 0 : j - d.hmax * d.vmax + 1),
                    "jpeg_check_batch: image %d: block %d of the MCU has the wrong component", i, j);
    BDBNN_REQUIRE(d.coef_off == blocks, "jpeg_check_batch: image %d: coef_off %lld, expected %lld", i,
                  (long long)d.coef_off, (long long)blocks);
    BDBNN_REQUIRE(d.rgb_off == pix * 3, "jpeg_check_batch: image %d: rgb_off %lld, expected %lld", i,
                  (long long)d.rgb_off, (long long)(pix * 3));
    BDBNN_REQUIRE(d.data_off >= 0 && d.data_bytes >= 0 && d.data_off + d.data_bytes <= data_bytes,
                  "jpeg_check_batch: image %d: data outside the arena", i);
    blocks += int64_t(d.mcux) * d.mcuy * d.bpm;
    pix += int64_t(d.H) * d.W;
  }
  BDBNN_REQUIRE(pix * 3 <= rgb_bytes, "jpeg_check_batch: rgb holds %lld bytes, need %lld", (long long)rgb_bytes,
                (long long)(pix * 3));
  auto mcus = [&](int i) { return int64_t(desc_host[i].mcux) * desc_host[i].mcuy; };
  int64_t n_sub = 0, next_mcu = 0;
  int img = -1;
  for (int s = 0; s < n_seg; ++s) {
    const bdbnn_jpeg_seg& g = seg_host[s];
    if (g.img != img) {
      BDBNN_REQUIRE(g.img == img + 1 && g.img < n_img, "jpeg_check_batch: segment %d: image %d out of order", s,
                    g.img);
      BDBNN_REQUIRE(img < 0 || next_mcu == mcus(img), "jpeg_check_batch: image %d: segments do not cover its MCUs",
                    img);
      img = g.img;
      next_mcu = 0;
    }
    const bdbnn_jpeg_desc& d = desc_host[g.img];
    BDBNN_REQUIRE(g.nbytes >= 0 && g.off >= d.data_off && g.off + g.nbytes <= d.data_off + d.data_bytes,
                  "jpeg_check_batch: segment %d: bytes outside its image's data", s);
    BDBNN_REQUIRE(g.mcu0 == next_mcu && g.nmcu >= 1, "jpeg_check_batch: segment %d: MCUs [%d, +%d), expected %lld",
                  s, g.mcu0, g.nmcu, (long long)next_mcu);
    next_mcu += g.nmcu;
    const int64_t want = std::max<int64_t>(1, (int64_t(g.nbytes) * 8 + S - 1) / S);
    BDBNN_REQUIRE(g.sub0 == n_sub && g.nsub == want,
                  "jpeg_check_batch: segment %d: subsequences (%d, %d), expected (%lld, %lld) at %d bits", s,
                  g.sub0, g.nsub, (long long)n_sub, (long long)want, S);
    n_sub += want;
    BDBNN_REQUIRE(n_sub < (int64_t(1) << 31), "jpeg_check_batch: too many subsequences");
  }
  BDBNN_REQUIRE(img == n_img - 1 && next_mcu == mcus(img), "jpeg_check_batch: segments do not cover every image's MCUs");
  const size_t need = jp_layout(blocks, n_sub, nullptr, nullptr);
  BDBNN_REQUIRE(work_bytes >= need, "jpeg_check_batch: workspace of %zu bytes, need %zu", work_bytes, need);
  *blocks_out = blocks;
  *pix_out = pix;
  *n_sub_out = n_sub;
  return BDBNN_OK;
}

extern "C" int bdbnn_jpeg_check_batch(const bdbnn_jpeg_desc* desc_host, int32_t n_img, const bdbnn_jpeg_seg* seg_host,
                                      int32_t n_seg, int64_t data_bytes, int64_t rgb_bytes, size_t work_bytes) {
  int64_t blocks, pix, n_sub;
  return jp_check(desc_host, n_img, seg_host, n_seg, data_bytes, rgb_bytes, work_bytes, &blocks, &pix, &n_sub);
}

// The original files of bdbnn_jpeg_decode_batch_files, parsed and unstuffed on the device.
struct JpFiles {
  const uint8_t* host;
  uint8_t* dev;
  int64_t bytes;
  const bdbnn_jpeg_file* tab_host;
  bdbnn_jpeg_file* tab_dev;
};

// bdbnn_jpeg_decode_batch, or with entries_dev set bdbnn_jpeg_decode_batch_indexed: jpeg_index_check_kernel
// in place of jpeg_sync_kernel, the rest as it is.  With files set (bdbnn_jpeg_decode_batch_files, entries_dev set
// too), jpeg_parse_kernel and jpeg_unstuff_kernel build the tables and data_dev from the files first, and data_host
// is NULL.
static int jp_decode(const bdbnn_jpeg_desc* desc_host, bdbnn_jpeg_desc* desc_dev, int32_t n_img,
                     const bdbnn_jpeg_seg* seg_host, bdbnn_jpeg_seg* seg_dev, int32_t n_seg, const uint8_t* data_host,
                     uint8_t* data_dev, int64_t data_bytes, const uint16_t* entries_host, uint16_t* entries_dev,
                     int64_t n_entries, void* work, size_t work_bytes, uint8_t* rgb, int64_t rgb_bytes,
                     int32_t* status_dev, int32_t* status_host, int32_t* rounds_host, void* stream,
                     const JpFiles* files = nullptr) {
  int64_t blocks, pix, n_sub;
  if (int rc = jp_check(desc_host, n_img, seg_host, n_seg, data_bytes, rgb_bytes, work_bytes, &blocks, &pix, &n_sub))
    return rc;
  if (files) {
    BDBNN_REQUIRE(files->bytes >= 0, "jpeg_decode_batch_files: negative files_bytes");
    for (int i = 0; i < n_img; ++i) {
      const bdbnn_jpeg_file& f = files->tab_host[i];
      BDBNN_REQUIRE(f.off >= 0 && f.size >= 0 && f.off <= files->bytes - f.size,
                    "jpeg_decode_batch_files: image %d: file [%lld, +%d) outside the %lld bytes of files", i,
                    (long long)f.off, f.size, (long long)files->bytes);
    }
  }
  const int S = jp_sub_bits();
  BDBNN_REQUIRE(!entries_dev || n_entries == n_sub - n_seg,
                "jpeg_decode_batch_indexed: %lld entries, the segments' nsub - 1 sum to %lld", (long long)n_entries,
                (long long)(n_sub - n_seg));
  BDBNN_REQUIRE((reinterpret_cast<uintptr_t>(work) & 255) == 0, "jpeg_decode_batch: workspace not 256-byte aligned");

  const cudaStream_t st = cudaStream_t(stream);
  JpWork w;
  jp_layout(blocks, n_sub, static_cast<uint8_t*>(work), &w);
  BDBNN_CUDA(cudaMemcpyAsync(desc_dev, desc_host, size_t(n_img) * sizeof(bdbnn_jpeg_desc), cudaMemcpyHostToDevice, st));
  BDBNN_CUDA(cudaMemcpyAsync(seg_dev, seg_host, size_t(n_seg) * sizeof(bdbnn_jpeg_seg), cudaMemcpyHostToDevice, st));
  if (!files)
    BDBNN_CUDA(cudaMemcpyAsync(data_dev, data_host, size_t(data_bytes), cudaMemcpyHostToDevice, st));
  BDBNN_CUDA(cudaMemsetAsync(w.coef, 0, size_t(blocks) * 128, st));
  BDBNN_CUDA(cudaMemsetAsync(status_dev, 0, size_t(n_img) * 4, st));
  if (files) {
    BDBNN_CUDA(cudaMemcpyAsync(files->dev, files->host, size_t(files->bytes), cudaMemcpyHostToDevice, st));
    BDBNN_CUDA(cudaMemcpyAsync(files->tab_dev, files->tab_host, size_t(n_img) * sizeof(bdbnn_jpeg_file),
                               cudaMemcpyHostToDevice, st));
    jpeg_parse_kernel<<<unsigned((n_img + 127) / 128), 128, 0, st>>>(files->dev, files->tab_dev, desc_dev, n_img,
                                                                     status_dev);
    if (int rc = check_launch("jpeg_parse_kernel")) return rc;
    jpeg_unstuff_kernel<<<unsigned(n_img), kJpThreads, 0, st>>>(files->dev, files->tab_dev, desc_dev, seg_dev, n_seg,
                                                                data_dev, status_dev);
    if (int rc = check_launch("jpeg_unstuff_kernel")) return rc;
  }

  const unsigned sub_grid = unsigned((n_sub + kJpThreads - 1) / kJpThreads);
  if (entries_dev) {
    BDBNN_CUDA(cudaMemsetAsync(w.counters, 0, 8, st));         // rounds_host receives 0
    if (n_entries > 0)
      BDBNN_CUDA(cudaMemcpyAsync(entries_dev, entries_host, size_t(n_entries) * 2, cudaMemcpyHostToDevice, st));
    jpeg_index_check_kernel<<<sub_grid, kJpThreads, 0, st>>>(desc_dev, seg_dev, n_seg, data_dev, n_sub, S,
                                                              entries_dev, w.start, w.cnt, status_dev);
    if (int rc = check_launch("jpeg_index_check_kernel")) return rc;
  } else {
    BDBNN_CUDA(cudaMemsetAsync(w.ready, 0, size_t(sub_grid) * 4, st));
    BDBNN_CUDA(cudaMemsetAsync(w.counters, 0, 8, st));
    jpeg_sync_kernel<<<sub_grid, kJpThreads, 0, st>>>(desc_dev, seg_dev, n_seg, data_dev, n_sub, S, w.start, w.exit,
                                                       w.cnt, w.counters, w.ready, w.counters + 1);
    if (int rc = check_launch("jpeg_sync_kernel")) return rc;
  }
  jpeg_scan_kernel<<<unsigned((int64_t(n_seg) * 32 + 255) / 256), 256, 0, st>>>(seg_dev, n_seg, w.cnt, w.first);
  if (int rc = check_launch("jpeg_scan_kernel")) return rc;
  jpeg_write_kernel<<<sub_grid, kJpThreads, 0, st>>>(desc_dev, seg_dev, n_seg, data_dev, n_sub, S, w.start, w.first,
                                                      w.coef, status_dev);
  if (int rc = check_launch("jpeg_write_kernel")) return rc;
  jpeg_dc_kernel<<<unsigned(n_seg), 128, 0, st>>>(desc_dev, seg_dev, w.coef, status_dev);
  if (int rc = check_launch("jpeg_dc_kernel")) return rc;
  jpeg_idct_kernel<<<unsigned((blocks * 8 + kJpThreads - 1) / kJpThreads), kJpThreads, 0, st>>>(
      desc_dev, n_img, blocks, w.coef, w.planes, status_dev);
  if (int rc = check_launch("jpeg_idct_kernel")) return rc;
  jpeg_color_kernel<<<unsigned((pix + kJpThreads - 1) / kJpThreads), kJpThreads, 0, st>>>(desc_dev, n_img, pix,
                                                                                          w.planes, rgb);
  if (int rc = check_launch("jpeg_color_kernel")) return rc;
  BDBNN_CUDA(cudaMemcpyAsync(status_host, status_dev, size_t(n_img) * 4, cudaMemcpyDeviceToHost, st));
  if (rounds_host) BDBNN_CUDA(cudaMemcpyAsync(rounds_host, w.counters + 1, 4, cudaMemcpyDeviceToHost, st));
  return BDBNN_OK;
}

extern "C" int bdbnn_jpeg_decode_batch(const bdbnn_jpeg_desc* desc_host, bdbnn_jpeg_desc* desc_dev, int32_t n_img,
                                       const bdbnn_jpeg_seg* seg_host, bdbnn_jpeg_seg* seg_dev, int32_t n_seg,
                                       const uint8_t* data_host, uint8_t* data_dev, int64_t data_bytes, void* work,
                                       size_t work_bytes, uint8_t* rgb, int64_t rgb_bytes, int32_t* status_dev,
                                       int32_t* status_host, int32_t* rounds_host, void* stream) {
  BDBNN_REQUIRE(desc_host && desc_dev && seg_host && seg_dev && data_host && data_dev && work && rgb && status_dev &&
                    status_host,
                "jpeg_decode_batch: NULL pointer");
  return jp_decode(desc_host, desc_dev, n_img, seg_host, seg_dev, n_seg, data_host, data_dev, data_bytes, nullptr,
                   nullptr, 0, work, work_bytes, rgb, rgb_bytes, status_dev, status_host, rounds_host, stream);
}

extern "C" int bdbnn_jpeg_decode_batch_indexed(const bdbnn_jpeg_desc* desc_host, bdbnn_jpeg_desc* desc_dev,
                                               int32_t n_img, const bdbnn_jpeg_seg* seg_host, bdbnn_jpeg_seg* seg_dev,
                                               int32_t n_seg, const uint8_t* data_host, uint8_t* data_dev,
                                               int64_t data_bytes, const uint16_t* entries_host,
                                               uint16_t* entries_dev, int64_t n_entries, void* work,
                                               size_t work_bytes, uint8_t* rgb, int64_t rgb_bytes,
                                               int32_t* status_dev, int32_t* status_host, int32_t* rounds_host,
                                               void* stream) {
  BDBNN_REQUIRE(desc_host && desc_dev && seg_host && seg_dev && data_host && data_dev && entries_host &&
                    entries_dev && work && rgb && status_dev && status_host,
                "jpeg_decode_batch_indexed: NULL pointer");
  return jp_decode(desc_host, desc_dev, n_img, seg_host, seg_dev, n_seg, data_host, data_dev, data_bytes,
                   entries_host, entries_dev, n_entries, work, work_bytes, rgb, rgb_bytes, status_dev, status_host,
                   rounds_host, stream);
}

extern "C" int bdbnn_jpeg_decode_batch_files(const uint8_t* files_host, uint8_t* files_dev, int64_t files_bytes,
                                             const bdbnn_jpeg_file* file_host, bdbnn_jpeg_file* file_dev,
                                             const bdbnn_jpeg_desc* desc_host, bdbnn_jpeg_desc* desc_dev,
                                             int32_t n_img, const bdbnn_jpeg_seg* seg_host, bdbnn_jpeg_seg* seg_dev,
                                             int32_t n_seg, uint8_t* data_dev, int64_t data_bytes,
                                             const uint16_t* entries_host, uint16_t* entries_dev, int64_t n_entries,
                                             void* work, size_t work_bytes, uint8_t* rgb, int64_t rgb_bytes,
                                             int32_t* status_dev, int32_t* status_host, void* stream) {
  BDBNN_REQUIRE(files_host && files_dev && file_host && file_dev && desc_host && desc_dev && seg_host && seg_dev &&
                    data_dev && entries_host && entries_dev && work && rgb && status_dev && status_host,
                "jpeg_decode_batch_files: NULL pointer");
  const JpFiles files{files_host, files_dev, files_bytes, file_host, file_dev};
  return jp_decode(desc_host, desc_dev, n_img, seg_host, seg_dev, n_seg, nullptr, data_dev, data_bytes, entries_host,
                   entries_dev, n_entries, work, work_bytes, rgb, rgb_bytes, status_dev, status_host, nullptr, stream,
                   &files);
}
