// Baseline JPEG decoding for sm_90a, bit-identical to the C code paths of libjpeg-turbo that PIL.Image.open runs
// (jdhuff.c, jidctint.c's jpeg_idct_islow, jdsample.c's fancy upsampling, jdcolor.c's ycc_rgb_convert).  Four launches
// after the workspace memsets:
//
//   unstuff   the entropy-coded bytes of every image, 4 KB per CTA in ticket order: drop the 0x00 after each 0xFF,
//             drop each RSTn and mark the compacted byte its interval starts at, compact with the decoupled look-back
//             of common.cuh.  Any other marker sets status 8.
//   huffman   the self-synchronising parallel decode of Weissenberger & Schmidt: each thread owns kSub bits of the
//             compacted stream and decodes from a guessed state (bit position, block within the MCU, zig-zag index);
//             inside the CTA every thread re-decodes from its predecessor's exit state until all entry states agree
//             (at most one round per thread; a dozen at q95, DESIGN §6).  CTAs form a chain in ticket order: a CTA
//             first takes its predecessor's speculative exit (posted as soon as that CTA settled), scans its block
//             counts, then waits for the exact exit and posts its own at once when the two agree, re-running the fixed
//             point and the scan only when they differ.  The exact exit carries the block count and the DC
//             predictors, so the CTA knows where every block goes; a second decode of its bits writes the quantised
//             coefficients with undifferenced DC.  Exactness never depends on how fast the states synchronise: the
//             fixed point runs until nothing changes, and the worst case is a serial decode.  A restart interval
//             ends where the decoder completes an MCU within the < 8 one-bits before a marked byte (no code is all
//             ones, T.81 Annex C); the exact pass checks the MCU count and the marker number there.
//   idct      jpeg_idct_islow per 8 x 8 block of the MCU rows the requested rows (and their upsampling context) need,
//             64-bit intermediates like its JLONG, the int workspace, range_limit's 10-bit wrap; uint8 planes.
//   colour    fancy upsampling (h2v1 / h2v2, plain replication below three chroma columns as jdsample.c chooses),
//             context rows replicated from the component's last real row, then ycc_rgb_convert; uint8 HWC rows.
#include "common.cuh"

namespace p3d {
namespace jpeg {

constexpr int kUnstuffThreads = 256, kUnstuffBytes = 16, kTile = kUnstuffThreads * kUnstuffBytes;
constexpr int kHuffThreads = 128;
constexpr int kSub = 512;                           // bits per subsequence (one thread)
constexpr int kCtaBits = kHuffThreads * kSub;
constexpr int kFastBits = 10;
constexpr int kIdctThreads = 128, kColourThreads = 256;

enum : int { kBadCode = 1, kBadRestart = 2, kTruncated = 4, kBadMarker = 8, kBadDesc = 16 };

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct Geo {
  int mrows, mcols, bpm, total_mcus;
  long long total_blocks;
};

__device__ __forceinline__ Geo geometry(const p3d_jpeg_desc &d) {
  Geo g;
  g.mrows = (d.height + 8 * d.vs - 1) / (8 * d.vs);
  g.mcols = (d.width + 8 * d.hs - 1) / (8 * d.hs);
  g.bpm = d.hs * d.vs + 2;
  g.total_mcus = g.mrows * g.mcols;
  g.total_blocks = static_cast<long long>(g.total_mcus) * g.bpm;
  return g;
}

// A descriptor the call can decode: its size, a supported sampling, a segment inside data and within max_bytes.
__device__ __forceinline__ bool desc_ok(const p3d_jpeg_desc &d, int H, int W, long long data_bytes, long long max_bytes) {
  const bool samp = (d.hs == 1 && d.vs == 1) || (d.hs == 2 && d.vs == 1) || (d.hs == 2 && d.vs == 2);
  return samp && d.height == H && d.width == W && d.length >= 0 && d.length <= max_bytes && d.offset >= 0 &&
         d.offset + d.length <= data_bytes;
}

struct Work {  // the workspace, carved the same way on the host (sizing) and the device
  unsigned int *tickets;        // [2][N]
  int *lengths;                 // [N] compacted bytes
  unsigned long long *lb;       // [N][tiles] look-back descriptors of the unstuff pass
  unsigned long long *spec;     // [N][ctas] speculative exit states (bit 63 = posted)
  int *exact;                   // [N][ctas][8]: state lo, hi, blocks lo, hi, dc0..2, flag
  uint8_t *stream;              // [N][stream_stride] compacted bytes
  uint8_t *marks;               // [N][stream_stride] 0x80 | n: RSTn precedes this compacted byte
  int16_t *coef;                // [N][max_blocks][64]
  uint8_t *planes;              // [N][3][plane_bytes]
  size_t control_bytes, marks_bytes, coef_bytes;
  long long stream_stride, max_blocks, plane_pitch, plane_rows;
  int tiles, ctas;
};

inline long long max_blocks(int H, int W) {
  const long long b444 = 3ll * ((H + 7) / 8) * ((W + 7) / 8);
  const long long b422 = 4ll * ((H + 7) / 8) * ((W + 15) / 16);
  const long long b420 = 6ll * ((H + 15) / 16) * ((W + 15) / 16);
  return b444 > b422 ? (b444 > b420 ? b444 : b420) : (b422 > b420 ? b422 : b420);
}

inline Work carve(void *base, int N, int H, int W, long long max_bytes) {
  Work w;
  w.tiles = static_cast<int>((max_bytes + kTile - 1) / kTile);
  if (w.tiles < 1) w.tiles = 1;
  w.ctas = static_cast<int>((max_bytes * 8 + kCtaBits - 1) / kCtaBits);
  if (w.ctas < 1) w.ctas = 1;
  w.stream_stride = static_cast<long long>(align_up(static_cast<size_t>(max_bytes) + 16, 16));
  w.max_blocks = max_blocks(H, W);
  w.plane_pitch = (W + 15) / 16 * 16;
  w.plane_rows = (H + 15) / 16 * 16;
  Carver c(base);
  w.tickets = c.take<unsigned int>(2 * N);
  w.lengths = c.take<int>(N);
  w.lb = c.take<unsigned long long>(static_cast<size_t>(N) * w.tiles);
  w.spec = c.take<unsigned long long>(static_cast<size_t>(N) * w.ctas);
  w.exact = c.take<int>(static_cast<size_t>(N) * w.ctas * 8);
  w.control_bytes = c.off;
  w.marks = c.take<uint8_t>(static_cast<size_t>(N) * w.stream_stride);
  w.marks_bytes = c.off - w.control_bytes;
  const size_t coef0 = c.off;
  w.coef = c.take<int16_t>(static_cast<size_t>(N) * w.max_blocks * 64);
  w.coef_bytes = c.off - coef0;
  w.stream = c.take<uint8_t>(static_cast<size_t>(N) * w.stream_stride);
  w.planes = c.take<uint8_t>(static_cast<size_t>(N) * 3 * w.plane_pitch * w.plane_rows);
  return w;
}

struct Args {
  const uint8_t *data;
  long long data_bytes, max_bytes;
  const p3d_jpeg_desc *desc;
  int N, H, W, y0, y1;
  uint8_t *out;
  int *status;  // [N]
  Work w;
};

// ------------------------------------------------------------------------------------------------ unstuff

__global__ void __launch_bounds__(kUnstuffThreads) unstuff_kernel(const Args a) {
  const int n = blockIdx.y, tid = threadIdx.x;
  __shared__ unsigned int s_tile;
  __shared__ int s_warp[kUnstuffThreads / 32];
  __shared__ int s_prefix;
  __shared__ bool s_ok;
  if (tid == 0) {
    s_tile = atomicAdd(a.w.tickets + n, 1u);
    s_ok = desc_ok(a.desc[n], a.H, a.W, a.data_bytes, a.max_bytes);
  }
  __syncthreads();
  const unsigned int t = s_tile;
  if (!s_ok) return;
  const long long len = a.desc[n].length;
  const long long i0 = static_cast<long long>(t) * kTile;
  if (i0 >= len) return;
  const uint8_t *src = a.data + a.desc[n].offset;
  // classify this thread's bytes: keep (data), drop (stuffing / marker), mark (an RSTn starts here)
  const long long b0 = i0 + static_cast<long long>(tid) * kUnstuffBytes;
  uint8_t v[kUnstuffBytes + 2];  // v[0] = byte before, v[1..16] = own, v[17] = byte after
#pragma unroll
  for (int j = 0; j < kUnstuffBytes + 2; ++j) {
    const long long i = b0 + j - 1;
    v[j] = (i >= 0 && i < len) ? __ldg(src + i) : 0;
  }
  unsigned int keep = 0;
  int bad = 0;
#pragma unroll
  for (int j = 1; j <= kUnstuffBytes; ++j) {
    const long long i = b0 + j - 1;
    if (i >= len) break;
    if (i > 0 && v[j - 1] == 0xFF) continue;  // second byte of a stuffed pair or a marker
    if (v[j] != 0xFF) {
      keep |= 1u << j;
      continue;
    }
    const uint8_t nx = v[j + 1];
    if (i + 1 < len && nx == 0x00) keep |= 1u << j;
    else if (!(i + 1 < len && nx >= 0xD0 && nx <= 0xD7)) bad = 1;
  }
  if (bad) atomicOr(a.status + n, kBadMarker);
  const int cnt = __popc(keep);
  // CTA-wide exclusive scan of the counts, then the look-back across the image's tiles
  const int lane = tid & 31, warp = tid >> 5;
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  int warp_off = 0, total = 0;
  for (int k = 0; k < kUnstuffThreads / 32; ++k) {
    if (k < warp) warp_off += s_warp[k];
    total += s_warp[k];
  }
  if (warp == 0) {
    const int pre = lookback_exclusive_prefix(a.w.lb + static_cast<size_t>(n) * a.w.tiles, t, total);
    if (lane == 0) s_prefix = pre;
  }
  __syncthreads();
  int pos = s_prefix + warp_off + incl - cnt;
  uint8_t *dst = a.w.stream + static_cast<size_t>(n) * a.w.stream_stride;
  uint8_t *marks = a.w.marks + static_cast<size_t>(n) * a.w.stream_stride;
#pragma unroll
  for (int j = 1; j <= kUnstuffBytes; ++j) {
    const long long i = b0 + j - 1;
    if (i >= len) break;
    if (keep & (1u << j)) {
      dst[pos++] = v[j];
    } else if (v[j] == 0xFF && !(i > 0 && v[j - 1] == 0xFF) && i + 1 < len && v[j + 1] >= 0xD0 && v[j + 1] <= 0xD7) {
      marks[pos] = static_cast<uint8_t>(0x80 | (v[j + 1] - 0xD0));
    }
  }
  if (i0 + kTile >= len && tid == kUnstuffThreads - 1) a.w.lengths[n] = pos;  // the last tile: the stream's length
}

// ------------------------------------------------------------------------------------------------ Huffman decode

struct Tables {
  uint16_t fast[6][1 << kFastBits];  // (length << 8) | symbol for codes of <= kFastBits bits, 0 otherwise
  int maxcode[6][17];                // largest code of each length, -1 if none
  int valoff[6][17];                 // index into vals of code 0 of each length
  uint8_t vals[6][256];
};

// State of the decoder at a symbol boundary: bit position p, block b within the MCU, zig-zag index k.
__device__ __forceinline__ unsigned long long pack(uint32_t p, int b, int k) {
  return (static_cast<unsigned long long>(p) << 12) | (static_cast<unsigned long long>(b) << 7) | static_cast<unsigned>(k);
}
__device__ __forceinline__ uint32_t st_p(unsigned long long s) { return static_cast<uint32_t>(s >> 12); }
__device__ __forceinline__ int st_b(unsigned long long s) { return static_cast<int>((s >> 7) & 31); }
__device__ __forceinline__ int st_k(unsigned long long s) { return static_cast<int>(s & 127); }

struct Dc {  // DC differences summed since the last reset, per component; mask = components reset
  int sum[3];
  int reset;
};
__device__ __forceinline__ Dc dc_zero() { return Dc{{0, 0, 0}, 0}; }
__device__ __forceinline__ Dc dc_then(const Dc &x, const Dc &y) {  // x, then y
  Dc r;
#pragma unroll
  for (int c = 0; c < 3; ++c) r.sum[c] = (y.reset >> c) & 1 ? y.sum[c] : x.sum[c] + y.sum[c];
  r.reset = x.reset | y.reset;
  return r;
}

struct Stream {
  const uint32_t *words;  // compacted bytes, big-endian within each 32-bit load
  const uint8_t *marks;
  uint32_t nbits, nbytes;
};

// Word w of the stream (bits [32 w, 32 w + 32), most significant first); bits at or past the end read as 0.
__device__ __forceinline__ uint32_t load_word(const Stream &s, uint32_t w) {
  const uint32_t bit0 = w * 32u;
  if (bit0 >= s.nbits) return 0u;
  uint32_t v = __byte_perm(__ldg(s.words + w), 0, 0x0123);
  const uint32_t valid = s.nbits - bit0;
  if (valid < 32u) v &= ~(0xffffffffu >> valid);
  return v;
}

// A 64-bit window on the stream at bit p: at least 32 valid bits after every refill.
struct Reader {
  uint64_t buf;
  int cnt;
  uint32_t next;
};
__device__ __forceinline__ void reader_at(Reader &r, const Stream &s, uint32_t p) {
  const uint32_t w = p >> 5;
  r.buf = ((static_cast<uint64_t>(load_word(s, w)) << 32) | load_word(s, w + 1)) << (p & 31);
  r.cnt = 64 - static_cast<int>(p & 31);
  r.next = w + 2;
}
__device__ __forceinline__ void reader_refill(Reader &r, const Stream &s) {
  if (r.cnt <= 32) {
    r.buf |= static_cast<uint64_t>(load_word(s, r.next++)) << (32 - r.cnt);
    r.cnt += 32;
  }
}
__device__ __forceinline__ void reader_skip(Reader &r, const Stream &s, int n) {
  r.buf <<= n;
  r.cnt -= n;
  reader_refill(r, s);
}

struct Exact {  // what the writing pass needs
  int16_t *coef;
  long long block;        // absolute index of the block being decoded
  long long total_blocks;
  int pred0, pred1, pred2;
  int ri, bpm, total_mcus;
  int *status;
};

// Decode from state (p, b, k) while the next symbol starts before `limit`.  Counts completed blocks and sums DC
// differences (speculative passes); with WRITE, writes coefficients and checks the restart structure.
template <bool WRITE>
__device__ __forceinline__ void decode(const Stream &s, const Tables &T, int hv, int bpm, uint32_t limit, uint32_t &p,
                                       int &b, int &k, int &blocks, Dc &dc, Exact &ex) {
  int err = 0;
  Reader r;
  reader_at(r, s, p);
  while (p < limit) {
    const uint32_t v = static_cast<uint32_t>(r.buf >> 32);
    const int comp = b < hv ? 0 : b - hv + 1;
    const int tab = (k == 0 ? 0 : 3) + comp;
    int len, sym;
    const uint32_t e = T.fast[tab][v >> (32 - kFastBits)];
    if (e) {
      len = e >> 8;
      sym = e & 255;
    } else {
      len = 0;
      sym = 0;
#pragma unroll
      for (int l = kFastBits + 1; l <= 16; ++l) {
        const int code = static_cast<int>(v >> (32 - l));
        if (len == 0 && code <= T.maxcode[tab][l]) {
          len = l;
          sym = T.vals[tab][(T.valoff[tab][l] + code) & 255];
        }
      }
      if (len == 0) {  // undefined code: skip one bit (a speculative decoder resynchronises; the exact one flags it)
        if (WRITE && ex.block < ex.total_blocks) err |= kBadCode;
        p += 1;
        reader_skip(r, s, 1);
        continue;
      }
    }
    const int sz = k == 0 ? min(sym, 15) : (sym & 15);  // a DC category past 11 only in corrupt tables
    const int run = k == 0 ? 0 : (sym >> 4);
    int val = sz ? static_cast<int>((v << len) >> (32 - sz)) : 0;
    if (sz && val < (1 << (sz - 1))) val -= (1 << sz) - 1;
    p += len + sz;
    reader_skip(r, s, len + sz);
    if (k == 0) {
      dc.sum[0] += comp == 0 ? val : 0;
      dc.sum[1] += comp == 1 ? val : 0;
      dc.sum[2] += comp == 2 ? val : 0;
      if (WRITE) {
        ex.pred0 += comp == 0 ? val : 0;
        ex.pred1 += comp == 1 ? val : 0;
        ex.pred2 += comp == 2 ? val : 0;
        const int pred = comp == 0 ? ex.pred0 : (comp == 1 ? ex.pred1 : ex.pred2);
        if (ex.block < ex.total_blocks) ex.coef[ex.block * 64] = static_cast<int16_t>(pred);
      }
      k = 1;
    } else if (sz) {
      k += run;
      if (k > 63) {
        if (WRITE && ex.block < ex.total_blocks) err |= kBadCode;
        k = 64;
      } else {
        if (WRITE && ex.block < ex.total_blocks) ex.coef[ex.block * 64 + kZigzag[k]] = static_cast<int16_t>(val);
        ++k;
      }
    } else if (run == 15) {
      k += 16;
    } else {
      k = 64;  // EOB
    }
    if (k < 64) continue;
    // the block is complete
    k = 0;
    ++blocks;
    if (WRITE) ++ex.block;
    if (++b < bpm) continue;
    b = 0;
    // an MCU is complete: does a restart interval end here?
    const uint32_t q = (p + 7) >> 3;
    bool jump = false;
    int mark = 0;
    if (q < s.nbytes) {
      mark = s.marks[q];
      if (mark) {
        const int pad = static_cast<int>(q * 8 - p);
        jump = pad == 0 || static_cast<uint32_t>(r.buf >> (64 - pad)) == (1u << pad) - 1u;
      }
    }
    if (jump) {
      p = q * 8;
      reader_at(r, s, p);
      dc.sum[0] = dc.sum[1] = dc.sum[2] = 0;
      dc.reset = 7;
    }
    if (WRITE) {
      const long long mcu = ex.block / ex.bpm;
      if (mcu < ex.total_mcus) {
        const bool boundary = ex.ri > 0 && mcu % ex.ri == 0;
        if (jump != boundary || (jump && (mark & 7) != static_cast<int>(((mcu / ex.ri) - 1) & 7))) err |= kBadRestart;
      }
      if (jump) ex.pred0 = ex.pred1 = ex.pred2 = 0;
    }
  }
  if (WRITE && err) atomicOr(ex.status, err);
}

__device__ void build_tables(Tables &T, const p3d_jpeg_desc &d, int tid) {
  if (tid < 6) {
    const int c = tid % 3;
    const uint8_t *bits = tid < 3 ? d.dc_bits[c] : d.ac_bits[c];
    const uint8_t *vals = tid < 3 ? d.dc_vals[c] : d.ac_vals[c];
    const int nv = tid < 3 ? 16 : 256;
    for (int i = 0; i < nv; ++i) T.vals[tid][i] = vals[i];
    int code = 0, j = 0;
    T.maxcode[tid][0] = -1;
    T.valoff[tid][0] = 0;
    for (int l = 1; l <= 16; ++l) {
      const int cnt = bits[l - 1];
      T.valoff[tid][l] = j - code;
      T.maxcode[tid][l] = cnt ? code + cnt - 1 : -1;
      code += cnt;
      j += cnt;
      code <<= 1;
    }
  }
  __syncthreads();
  for (int i = tid; i < 6 * (1 << kFastBits); i += blockDim.x) {
    const int tab = i >> kFastBits, e = i & ((1 << kFastBits) - 1);
    uint16_t r = 0;
    for (int l = 1; l <= kFastBits; ++l) {
      const int code = e >> (kFastBits - l);
      if (code <= T.maxcode[tab][l]) {
        const int vi = T.valoff[tab][l] + code;
        r = static_cast<uint16_t>((l << 8) | T.vals[tab][vi & 255]);
        break;
      }
    }
    T.fast[tab][e] = r;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kHuffThreads) huffman_kernel(const Args a) {
  __shared__ Tables T;
  __shared__ unsigned long long s_exit[kHuffThreads];
  __shared__ unsigned long long s_entry0;
  __shared__ unsigned int s_t;
  __shared__ bool s_ok;
  __shared__ int s_scan_blocks[kHuffThreads];
  __shared__ Dc s_scan_dc[kHuffThreads];
  __shared__ long long s_pred_blocks;
  __shared__ Dc s_pred_dc;
  __shared__ bool s_redo;
  const int n = blockIdx.y, tid = threadIdx.x;
  if (tid == 0) {
    s_t = atomicAdd(a.w.tickets + a.N + n, 1u);
    s_ok = desc_ok(a.desc[n], a.H, a.W, a.data_bytes, a.max_bytes);
  }
  __syncthreads();
  const unsigned int t = s_t;
  if (!s_ok) {
    if (t == 0 && tid == 0) atomicOr(a.status + n, kBadDesc);
    return;
  }
  const p3d_jpeg_desc &d = a.desc[n];
  const Geo g = geometry(d);
  Stream s;
  s.nbytes = static_cast<uint32_t>(a.w.lengths[n]);
  s.nbits = s.nbytes * 8u;
  s.words = reinterpret_cast<const uint32_t *>(a.w.stream + static_cast<size_t>(n) * a.w.stream_stride);
  s.marks = a.w.marks + static_cast<size_t>(n) * a.w.stream_stride;
  const unsigned long long cta0 = static_cast<unsigned long long>(t) * kCtaBits;
  if (cta0 >= s.nbits) {
    if (t == 0 && tid == 0) atomicOr(a.status + n, kTruncated);  // no entropy-coded data at all
    return;
  }
  build_tables(T, d, tid);
  const int hv = d.hs * d.vs;
  const uint32_t start = static_cast<uint32_t>(cta0) + tid * kSub;
  const uint32_t limit = min(start + kSub, s.nbits);

  // speculative pass from a guessed state: a symbol boundary at the subsequence's first bit, first block, DC
  unsigned long long entry = pack(start, 0, 0);
  uint32_t p = start;
  int b = 0, k = 0, blocks = 0;
  Dc dc = dc_zero();
  Exact ex{};  // the writing pass's; unused by the speculative ones
  decode<false>(s, T, hv, g.bpm, limit, p, b, k, blocks, dc, ex);
  s_exit[tid] = pack(p, b, k);
  if (tid == 0) s_entry0 = entry;

  // fixed point: every entry state equals the predecessor's exit state (thread 0's: s_entry0)
  auto settle = [&]() {
    while (true) {
      __syncthreads();
      const unsigned long long e = tid ? s_exit[tid - 1] : s_entry0;
      const bool changed = e != entry;
      __syncthreads();
      if (changed) {
        entry = e;
        p = st_p(e);
        b = st_b(e);
        k = st_k(e);
        blocks = 0;
        dc = dc_zero();
        decode<false>(s, T, hv, g.bpm, limit, p, b, k, blocks, dc, ex);
        s_exit[tid] = pack(p, b, k);
      }
      if (!__syncthreads_or(changed)) break;
    }
  };
  // inclusive scan of block counts and DC summaries over the CTA's threads
  auto scan = [&]() {
    s_scan_blocks[tid] = blocks;
    s_scan_dc[tid] = dc;
    __syncthreads();
    for (int o = 1; o < kHuffThreads; o <<= 1) {
      int bb = 0;
      Dc dd = dc_zero();
      const bool has = tid >= o;
      if (has) {
        bb = s_scan_blocks[tid - o];
        dd = s_scan_dc[tid - o];
      }
      __syncthreads();
      if (has) {
        s_scan_blocks[tid] += bb;
        s_scan_dc[tid] = dc_then(dd, s_scan_dc[tid]);
      }
      __syncthreads();
    }
  };
  settle();
  volatile unsigned long long *spec = a.w.spec + static_cast<size_t>(n) * a.w.ctas;
  volatile int *exact = a.w.exact + static_cast<size_t>(n) * a.w.ctas * 8;
  if (tid == kHuffThreads - 1) spec[t] = (1ull << 63) | s_exit[tid];  // a hint for the successor
  if (t > 0) {
    // the predecessor's speculative exit: almost always its exact one already
    if (tid == 0) {
      unsigned long long v;
      while (!((v = spec[t - 1]) >> 63)) __nanosleep(32);
      s_entry0 = v & ~(1ull << 63);
    }
    settle();
  }
  scan();
  // the chain: the predecessor's exact exit state, block count and DC predictors.  When its exit state is the entry
  // state settled on (the common case) the CTA posts its own at once; otherwise it settles and scans again first.
  auto post = [&]() {
    const long long cum = s_pred_blocks + s_scan_blocks[kHuffThreads - 1];
    const Dc cdc = dc_then(s_pred_dc, s_scan_dc[kHuffThreads - 1]);
    volatile int *r = exact + t * 8;
    const unsigned long long st = s_exit[kHuffThreads - 1];
    r[0] = static_cast<int>(static_cast<uint32_t>(st));
    r[1] = static_cast<int>(static_cast<uint32_t>(st >> 32));
    r[2] = static_cast<int>(static_cast<uint32_t>(cum));
    r[3] = static_cast<int>(cum >> 32);
    r[4] = cdc.sum[0];
    r[5] = cdc.sum[1];
    r[6] = cdc.sum[2];
    __threadfence();
    r[7] = 1;
    if (cta0 + kCtaBits >= s.nbits && cum < g.total_blocks) atomicOr(a.status + n, kTruncated);  // the last CTA
  };
  if (tid == 0) {
    bool redo = false;
    if (t > 0) {
      volatile int *r = exact + (t - 1) * 8;
      while (r[7] == 0) __nanosleep(32);
      __threadfence();
      const unsigned long long st = static_cast<unsigned long long>(static_cast<uint32_t>(r[0])) |
                                    (static_cast<unsigned long long>(static_cast<uint32_t>(r[1])) << 32);
      s_pred_blocks = static_cast<long long>(static_cast<uint32_t>(r[2])) | (static_cast<long long>(r[3]) << 32);
      s_pred_dc = Dc{{r[4], r[5], r[6]}, 7};
      redo = st != s_entry0;
      s_entry0 = st;
    } else {
      s_pred_blocks = 0;
      s_pred_dc = Dc{{0, 0, 0}, 7};
    }
    s_redo = redo;
    if (!redo) post();
  }
  __syncthreads();
  if (s_redo) {
    settle();
    scan();
    if (tid == 0) post();
  }
  const long long excl_blocks = s_pred_blocks + s_scan_blocks[tid] - blocks;
  // the exclusive DC predictors of this thread: predecessor CTAs, then the CTA's threads before it
  Dc pre = s_pred_dc;
  if (tid > 0) pre = dc_then(pre, s_scan_dc[tid - 1]);
  // writing pass from the exact entry state
  ex.coef = a.w.coef + static_cast<size_t>(n) * a.w.max_blocks * 64;
  ex.block = excl_blocks;
  ex.total_blocks = g.total_blocks;
  ex.pred0 = pre.sum[0];
  ex.pred1 = pre.sum[1];
  ex.pred2 = pre.sum[2];
  ex.ri = d.restart_interval;
  ex.bpm = g.bpm;
  ex.total_mcus = g.total_mcus;
  ex.status = a.status + n;
  p = st_p(entry);
  b = st_b(entry);
  k = st_k(entry);
  blocks = 0;
  dc = dc_zero();
  decode<true>(s, T, hv, g.bpm, limit, p, b, k, blocks, dc, ex);
}

// ------------------------------------------------------------------------------------------------ IDCT

constexpr long long FIX_0_298631336 = 2446, FIX_0_390180644 = 3196, FIX_0_541196100 = 4433, FIX_0_765366865 = 6270,
                    FIX_0_899976223 = 7373, FIX_1_175875602 = 9633, FIX_1_501321110 = 12299, FIX_1_847759065 = 15137,
                    FIX_1_961570560 = 16069, FIX_2_053119869 = 16819, FIX_2_562915447 = 20995, FIX_3_072711026 = 25172;
constexpr int CONST_BITS = 13, PASS1_BITS = 2;

// One pass of jpeg_idct_islow on (i0..i7), before its descale, in JLONG (64-bit) arithmetic.
__device__ __forceinline__ void idct_1d(long long i0, long long i1, long long i2, long long i3, long long i4, long long i5,
                                        long long i6, long long i7, long long o[8]) {
  long long z1 = (i2 + i6) * FIX_0_541196100;
  const long long tmp2 = z1 + i6 * -FIX_1_847759065;
  const long long tmp3 = z1 + i2 * FIX_0_765366865;
  const long long tmp0 = (i0 + i4) * (1ll << CONST_BITS);
  const long long tmp1 = (i0 - i4) * (1ll << CONST_BITS);
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  long long t0 = i7, t1 = i5, t2 = i3, t3 = i1;
  z1 = t0 + t3;
  long long z2 = t1 + t2, z3 = t0 + t2, z4 = t1 + t3;
  const long long z5 = (z3 + z4) * FIX_1_175875602;
  t0 *= FIX_0_298631336;
  t1 *= FIX_2_053119869;
  t2 *= FIX_3_072711026;
  t3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223;
  z2 *= -FIX_2_562915447;
  z3 = z3 * -FIX_1_961570560 + z5;
  z4 = z4 * -FIX_0_390180644 + z5;
  t0 += z1 + z3;
  t1 += z2 + z4;
  t2 += z2 + z3;
  t3 += z1 + z4;
  o[0] = tmp10 + t3;
  o[7] = tmp10 - t3;
  o[1] = tmp11 + t2;
  o[6] = tmp11 - t2;
  o[2] = tmp12 + t1;
  o[5] = tmp12 - t1;
  o[3] = tmp13 + t0;
  o[4] = tmp13 - t0;
}

__device__ __forceinline__ long long descale(long long x, int n) { return (x + (1ll << (n - 1))) >> n; }

// IDCT_range_limit[x & RANGE_MASK]: a 10-bit wrap, then the clamp of the sample shifted by 128.
__device__ __forceinline__ uint32_t range_limit(long long x) {
  const int s = static_cast<int>((x + 512) & 1023) - 512 + 128;
  return static_cast<uint32_t>(s < 0 ? 0 : (s > 255 ? 255 : s));
}

// MCU rows [mr0, mr1) that rows [y0, y1) and their upsampling context need.
__device__ __forceinline__ void mcu_rows(const p3d_jpeg_desc &d, int y0, int y1, const Geo &g, int &mr0, int &mr1) {
  if (d.vs == 2) {
    const int dh = (d.height + 1) / 2;
    const int c0 = max(0, y0 / 2 - 1), c1 = min(dh - 1, (y1 - 1) / 2 + 1);
    mr0 = c0 / 8;
    mr1 = c1 / 8 + 1;
  } else {
    mr0 = y0 / 8;
    mr1 = (y1 - 1) / 8 + 1;
  }
  mr1 = min(mr1, g.mrows);
}

__global__ void __launch_bounds__(kIdctThreads) idct_kernel(const Args a) {
  __shared__ int q_s[3][64];
  const int n = blockIdx.y;
  const p3d_jpeg_desc &d = a.desc[n];
  if (!desc_ok(d, a.H, a.W, a.data_bytes, a.max_bytes)) return;
  for (int i = threadIdx.x; i < 3 * 64; i += blockDim.x) q_s[i / 64][i % 64] = static_cast<int16_t>(d.quant[i / 64][i % 64]);  // ISLOW_MULT_TYPE: short
  __syncthreads();
  const Geo g = geometry(d);
  int mr0, mr1;
  mcu_rows(d, a.y0, a.y1, g, mr0, mr1);
  const long long first = static_cast<long long>(mr0) * g.mcols * g.bpm;
  const long long blk = first + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (blk >= static_cast<long long>(mr1) * g.mcols * g.bpm) return;
  const int hv = d.hs * d.vs;
  const long long mcu = blk / g.bpm;
  const int bi = static_cast<int>(blk % g.bpm);
  const int my = static_cast<int>(mcu / g.mcols), mx = static_cast<int>(mcu % g.mcols);
  int comp, by, bx;
  if (bi < hv) {
    comp = 0;
    by = my * d.vs + bi / d.hs;
    bx = mx * d.hs + bi % d.hs;
  } else {
    comp = bi - hv + 1;
    by = my;
    bx = mx;
  }
  const int4 *src = reinterpret_cast<const int4 *>(a.w.coef + (static_cast<size_t>(n) * a.w.max_blocks + blk) * 64);
  int c[64];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int4 v = src[i];
    const int w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      c[8 * i + 2 * j] = static_cast<int16_t>(w[j] & 0xffff) * q_s[comp][8 * i + 2 * j];
      c[8 * i + 2 * j + 1] = static_cast<int16_t>(w[j] >> 16) * q_s[comp][8 * i + 2 * j + 1];
    }
  }
  int ws[64];
#pragma unroll
  for (int col = 0; col < 8; ++col) {  // pass 1: columns
    long long o[8];
    idct_1d(c[col], c[8 + col], c[16 + col], c[24 + col], c[32 + col], c[40 + col], c[48 + col], c[56 + col], o);
#pragma unroll
    for (int r = 0; r < 8; ++r) ws[8 * r + col] = static_cast<int>(descale(o[r], CONST_BITS - PASS1_BITS));
  }
  uint8_t *plane = a.w.planes + (static_cast<size_t>(n) * 3 + comp) * a.w.plane_pitch * a.w.plane_rows;
#pragma unroll
  for (int r = 0; r < 8; ++r) {  // pass 2: rows
    long long o[8];
    idct_1d(ws[8 * r], ws[8 * r + 1], ws[8 * r + 2], ws[8 * r + 3], ws[8 * r + 4], ws[8 * r + 5], ws[8 * r + 6],
            ws[8 * r + 7], o);
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      lo |= range_limit(descale(o[j], CONST_BITS + PASS1_BITS + 3)) << (8 * j);
      hi |= range_limit(descale(o[j + 4], CONST_BITS + PASS1_BITS + 3)) << (8 * j);
    }
    *reinterpret_cast<uint2 *>(plane + static_cast<size_t>(by * 8 + r) * a.w.plane_pitch + bx * 8) = make_uint2(lo, hi);
  }
}

// ------------------------------------------------------------------------------------------------ upsample + colour

// One pixel: its chroma sample c of plane P after jdsample.c's upsampling (dw, dh: the plane's real size).
__device__ __forceinline__ int chroma(const uint8_t *P, long long pitch, int x, int y, int hs, int vs, int dw, int dh) {
  if (hs == 1) return P[y * pitch + x];
  if (dw <= 2) return P[(y / vs) * pitch + x / 2];  // plain replication
  const int i = x >> 1;
  const int nb = (x & 1) ? min(i + 1, dw - 1) : max(i - 1, 0);
  if (vs == 1) {
    const uint8_t *row = P + y * pitch;
    return (3 * row[i] + row[nb] + 1 + (x & 1)) >> 2;  // h2v1: biases 1, 2
  }
  const int near = y >> 1;
  const int far = min(max((y & 1) ? near + 1 : near - 1, 0), dh - 1);  // context rows: the last real row
  const uint8_t *r0 = P + near * pitch, *r1 = P + far * pitch;
  const int cs = 3 * r0[i] + r1[i], cn = 3 * r0[nb] + r1[nb];
  return (3 * cs + cn + 8 - (x & 1)) >> 4;  // h2v2: biases 8, 7
}

// Four pixels per thread: upsampled chroma, ycc_rgb_convert, 12 bytes stored as three words when aligned.
__global__ void __launch_bounds__(kColourThreads) colour_kernel(const Args a) {
  const int n = blockIdx.z;
  const p3d_jpeg_desc &d = a.desc[n];
  const int x0 = 4 * (blockIdx.x * blockDim.x + threadIdx.x);
  const int y = a.y0 + blockIdx.y;
  if (x0 >= a.W || !desc_ok(d, a.H, a.W, a.data_bytes, a.max_bytes)) return;
  const long long pitch = a.w.plane_pitch, psize = pitch * a.w.plane_rows;
  const uint8_t *Y = a.w.planes + static_cast<size_t>(n) * 3 * psize;
  const int dw = (a.W + d.hs - 1) / d.hs, dh = (a.H + d.vs - 1) / d.vs;
  uint32_t px[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int x = min(x0 + j, a.W - 1);
    const int yv = Y[y * pitch + x];
    const int cb = chroma(Y + psize, pitch, x, y, d.hs, d.vs, dw, dh) - 128;
    const int cr = chroma(Y + 2 * psize, pitch, x, y, d.hs, d.vs, dw, dh) - 128;
    const int r = yv + ((91881 * cr + 32768) >> 16);                   // Cr_r_tab
    const int g = yv + ((-22554 * cb + 32768 + -46802 * cr) >> 16);    // Cb_g_tab + Cr_g_tab, shifted once
    const int bl = yv + ((116130 * cb + 32768) >> 16);                 // Cb_b_tab
    px[j] = static_cast<uint32_t>(min(max(r, 0), 255)) | (static_cast<uint32_t>(min(max(g, 0), 255)) << 8) |
            (static_cast<uint32_t>(min(max(bl, 0), 255)) << 16);
  }
  uint8_t *o = a.out + ((static_cast<size_t>(n) * (a.y1 - a.y0) + blockIdx.y) * a.W + x0) * 3;
  if (x0 + 4 <= a.W && (reinterpret_cast<uintptr_t>(o) & 3) == 0) {
    uint32_t *o32 = reinterpret_cast<uint32_t *>(o);
    o32[0] = px[0] | (px[1] << 24);
    o32[1] = (px[1] >> 8) | (px[2] << 16);
    o32[2] = (px[2] >> 16) | (px[3] << 8);
  } else {
    for (int j = 0; j < 4 && x0 + j < a.W; ++j) {
      o[3 * j] = static_cast<uint8_t>(px[j]);
      o[3 * j + 1] = static_cast<uint8_t>(px[j] >> 8);
      o[3 * j + 2] = static_cast<uint8_t>(px[j] >> 16);
    }
  }
}

inline bool limits_ok(int N, int H, int W, long long max_bytes) {
  return N <= P3D_JPEG_MAX_IMAGES && H <= P3D_JPEG_MAX_SIDE && W <= P3D_JPEG_MAX_SIDE && max_bytes <= (1ll << 28);
}

}  // namespace jpeg
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_jpeg_decode_workspace_bytes(int N, int H, int W, int64_t max_bytes) {
  if (N < 1 || H < 1 || W < 1 || max_bytes < 1 || !jpeg::limits_ok(N, H, W, max_bytes)) return 0;
  jpeg::Work w = jpeg::carve(nullptr, N, H, W, max_bytes);
  return reinterpret_cast<size_t>(w.planes) +
         static_cast<size_t>(N) * 3 * static_cast<size_t>(w.plane_pitch) * static_cast<size_t>(w.plane_rows);
}

extern "C" int p3d_jpeg_decode_u8(const uint8_t *data, int64_t data_bytes, const p3d_jpeg_desc *desc, int N, int H, int W,
                                  int y0, int y1, int64_t max_bytes, uint8_t *out, int32_t *status_dev, void *workspace,
                                  size_t workspace_bytes, p3d_stream_t stream) {
  if (!data || !desc || !out || !status_dev || !workspace) return P3D_ERR_INVALID_ARG;
  if (N < 1 || H < 1 || W < 1 || data_bytes < 1 || max_bytes < 1 || y0 < 0 || y1 <= y0 || y1 > H) return P3D_ERR_INVALID_ARG;
  if (!jpeg::limits_ok(N, H, W, max_bytes)) return P3D_ERR_UNSUPPORTED;
  if (workspace_bytes < p3d_jpeg_decode_workspace_bytes(N, H, W, max_bytes)) return P3D_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  jpeg::Args a;
  a.data = data;
  a.data_bytes = data_bytes;
  a.max_bytes = max_bytes;
  a.desc = desc;
  a.N = N;
  a.H = H;
  a.W = W;
  a.y0 = y0;
  a.y1 = y1;
  a.out = out;
  a.status = status_dev;
  a.w = jpeg::carve(workspace, N, H, W, max_bytes);
  P3D_CUDA_CHECK(cudaMemsetAsync(workspace, 0, a.w.control_bytes + a.w.marks_bytes + a.w.coef_bytes, st));
  jpeg::unstuff_kernel<<<dim3(a.w.tiles, N), jpeg::kUnstuffThreads, 0, st>>>(a);
  P3D_LAUNCH_CHECK();
  jpeg::huffman_kernel<<<dim3(a.w.ctas, N), jpeg::kHuffThreads, 0, st>>>(a);
  P3D_LAUNCH_CHECK();
  // blocks of the MCU rows the band needs, for the sampling that needs the most of them
  long long most = 0;
  const int modes[3][2] = {{1, 1}, {2, 1}, {2, 2}};
  for (const auto &m : modes) {
    const int hs = m[0], vs = m[1], mh = 8 * vs;
    const int mcols = (W + 8 * hs - 1) / (8 * hs), mrows = (H + mh - 1) / mh;
    int mr0, mr1;
    if (vs == 2) {
      const int dh = (H + 1) / 2, c0 = y0 / 2 - 1 > 0 ? y0 / 2 - 1 : 0, c1 = (y1 - 1) / 2 + 1 < dh - 1 ? (y1 - 1) / 2 + 1 : dh - 1;
      mr0 = c0 / 8;
      mr1 = c1 / 8 + 1;
    } else {
      mr0 = y0 / 8;
      mr1 = (y1 - 1) / 8 + 1;
    }
    if (mr1 > mrows) mr1 = mrows;
    const long long blocks = static_cast<long long>(mr1 - mr0) * mcols * (hs * vs + 2);
    if (blocks > most) most = blocks;
  }
  jpeg::idct_kernel<<<dim3(div_up(most, jpeg::kIdctThreads), N), jpeg::kIdctThreads, 0, st>>>(a);
  P3D_LAUNCH_CHECK();
  jpeg::colour_kernel<<<dim3(div_up(W, 4 * jpeg::kColourThreads), y1 - y0, N), jpeg::kColourThreads, 0, st>>>(a);
  P3D_LAUNCH_CHECK();
  return P3D_OK;
}
