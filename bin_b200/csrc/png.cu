// PNG encoder of the evaluation loop's outputs (test.py / demo.py write every output with cv2.imwrite): n same-size
// uint8 (h, w, 3) BGR images -> n complete PNG files whose inflated IDAT payload is the one cv2.imwrite writes (every
// row filter type 1, Sub; zlib at level 1 with Z_RLE: literals and matches at distance 1 only).
//
// The filtered payload of an image (h * (3w + 1) bytes) is cut into kSeg-byte segments; the cut depends only on (h, w).
// Each segment becomes one deflate block:
//   png_segment_kernel  one CTA per segment: generates the Sub bytes straight from the image into shared memory,
//                       parses runs as Z_RLE does (each thread a 128-byte chunk; block scans give every chunk the run
//                       that crosses its edges), takes the histograms, builds length-limited canonical Huffman codes
//                       (15 bits; 7 for the code-length code), prices the dynamic and fixed block and keeps the
//                       Adler-32 partial of the segment.
//   png_plan_kernel     one thread per image walks its segments in order: picks the cheapest of dynamic, fixed and
//                       stored at the block's actual bit offset (a stored block pads to a byte), sets each block's bit
//                       offset, combines the Adler-32 and sizes the zlib stream and the file.
//   png_emit_kernel     one CTA per segment re-derives its tokens and writes its block at its offset.  Words owned by
//                       one thread are stored, words shared with a neighbouring range are merged with atomicOr into the
//                       zeroed buffer: OR commutes, so the bytes do not depend on the order.
//   png_frame_kernel    one warp per 8192-byte IDAT chunk: signature, IHDR, the zlib header 78 01, the data, the
//                       Adler-32 and IEND, each chunk's CRC-32 from per-lane partials combined in GF(2).
// Every grid depends only on (h, w) and n (one grid row per image), every sum is an integer, so the bytes depend only
// on the pixels and (h, w): not on the stream, the SM count, n or the image's position in the batch.
#include <stdint.h>

#include "internal.h"

namespace binb {

constexpr int kSeg = 32768;                     // payload bytes per deflate block
constexpr int kPngThreads = 256;
constexpr int kChunk = kSeg / kPngThreads;      // payload bytes per thread
constexpr int kIdat = 8192;                     // data bytes per IDAT chunk (libpng's default, as cv2 writes)
constexpr int kFrameWarps = 8;
constexpr int kMaxBits = 15, kClMaxBits = 7;
constexpr int kStored = 0, kFixed = 1, kDynamic = 2;   // BTYPE
constexpr uint32_t kAdlerMod = 65521;

__constant__ uint16_t kLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                      31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// What the segment pass hands to the plan and emit passes.
struct SegPlan {
  uint32_t len;                          // payload bytes of the segment
  uint32_t adler_a, adler_b;             // sum p_i, sum (len - i) p_i, both mod 65521
  uint32_t dyn_bits, fixed_bits;         // whole block, 3-bit header and end-of-block code included
  uint32_t hdr_bits;                     // 3-bit header + dynamic code description
  uint16_t hlit, hdist, hclen, nrle;     // code counts of the dynamic header; run-length-coded code lengths
  uint8_t lit_len[288], dist_len[32], cl_len[20];
  uint8_t rle_sym[320], rle_extra[320];
};

struct PngBlock {
  unsigned long long bit;                // offset of the block in the deflate stream
  int type, pad;
};

struct PngInfo {
  unsigned long long zlen;               // zlib stream bytes: 2 + deflate + 4
  uint32_t adler;
  int nidat;
};

struct PngSmem {
  uint8_t buf[kSeg + 8];                 // buf[0] = payload byte before the segment, buf[1 + i] = byte i
  uint32_t lit_freq[288], dist_freq[32], cl_freq[20];
  uint16_t lit_code[288], dist_code[32], cl_code[20];
  uint8_t lit_len[288], dist_len[32], cl_len[20];
  uint8_t len_sym[260];                  // match length -> length code - 257
  int w[288], sorted[288], A[288];
  unsigned scan[kPngThreads];
  unsigned long long adler_a, adler_b;
  unsigned extra_bits;
  int nused;
  uint8_t all_len[320];
};

// ------------------------------------------------------------------------------------------------------ helpers
__host__ __device__ inline long long png_payload_bytes(int h, int w) { return (long long)h * (3ll * w + 1); }
static inline int png_nseg(long long L) { return (int)((L + kSeg - 1) / kSeg); }
static inline long long png_deflate_cap(long long L) { return 5ll * png_nseg(L) + L; }   // all blocks stored
static inline size_t png_zbuf_bytes(long long L) { return (size_t)((png_deflate_cap(L) + 8 + 255) / 256 * 256); }
static inline size_t png_align(size_t x) { return (x + 255) / 256 * 256; }

static inline bool png_shape_ok(int h, int w) {
  return h >= 1 && w >= 1 && h <= 65535 && w <= 65535 && png_payload_bytes(h, w) < (1ll << 31);
}
static inline size_t png_file_bytes(long long zlen) {      // signature, IHDR, the IDAT chunks, IEND
  return (size_t)(8 + 25 + 12 * ((zlen + kIdat - 1) / kIdat) + zlen + 12);
}

// Stage the segment's Sub-filtered payload bytes [g0, g0 + len) and the byte before it.
__device__ void stage_payload(const uint8_t* __restrict__ img, int w3, long long g0, int len, uint8_t* buf) {
  const int rowlen = w3 + 1;
  for (int i = threadIdx.x; i <= len; i += kPngThreads) {
    const int q = (int)(g0 + i - 1);
    uint8_t v = 0;
    if (q >= 0) {
      const int row = q / rowlen, k = q - row * rowlen;
      if (k == 0) {
        v = w3 == 3 ? 0 : 1;                           // filter type: Sub (None for one-pixel rows, as libpng)
      } else {
        const uint8_t* r = img + (size_t)row * w3;
        const int x = k - 1, src = x + 2 - 2 * (x % 3);   // the file stores RGB: byte x of the row is BGR byte src
        v = (uint8_t)(r[src] - (x >= 3 ? r[src - 3] : 0));
      }
    }
    buf[i] = v;
  }
}

// Inclusive Hillis-Steele scan over the CTA (reverse: from the last thread down); returns the exclusive value.
template <typename Op>
__device__ unsigned block_excl_scan(unsigned v, unsigned identity, bool reverse, unsigned* sh, Op op) {
  const int t = reverse ? kPngThreads - 1 - (int)threadIdx.x : (int)threadIdx.x;
  __syncthreads();
  sh[t] = v;
  __syncthreads();
  for (int d = 1; d < kPngThreads; d <<= 1) {
    unsigned x = sh[t];
    if (t >= d) x = op(sh[t - d], x);
    __syncthreads();
    sh[t] = x;
    __syncthreads();
  }
  const unsigned r = t > 0 ? sh[t - 1] : identity;
  __syncthreads();
  return r;
}

// Run context of this thread's chunk: e(i) = byte i repeats the byte before it (a distance-1 match may cover it).
// prev_zero = last i < c0 with e(i) = 0 (-1 if none), next_zero = first i >= c1 with e(i) = 0 (len if none).
struct ChunkRuns {
  int c0, c1, prev_zero, next_zero;
};

__device__ __forceinline__ bool repeats(const uint8_t* buf, bool stream_start, int i) {
  return !(stream_start && i == 0) && buf[1 + i] == buf[i];
}

__device__ ChunkRuns chunk_runs(const uint8_t* buf, bool stream_start, int len, unsigned* sh) {
  ChunkRuns c;
  c.c0 = min((int)threadIdx.x * kChunk, len);
  c.c1 = min(c.c0 + kChunk, len);
  int lz = -1, fz = len;
  for (int i = c.c0; i < c.c1; ++i)
    if (!repeats(buf, stream_start, i)) {
      lz = i;
      if (fz == len) fz = i;
    }
  c.prev_zero = (int)block_excl_scan((unsigned)(lz + 1), 0u, false, sh, [](unsigned a, unsigned b) { return max(a, b); }) - 1;
  c.next_zero = (int)block_excl_scan((unsigned)fz, (unsigned)len, true, sh, [](unsigned a, unsigned b) { return min(a, b); });
  return c;
}

// The tokens that start in [c0, c1), in order, as zlib's deflate_rle parses them: at each position the run r of bytes
// equal to the previous byte; r >= 3 gives a match of min(r, 258), otherwise a literal.  Runs are cut at the segment's
// start (its first byte may still repeat the previous segment's last byte).  lit(byte), match(length).
template <typename Lit, typename Match>
__device__ void walk_tokens(const uint8_t* buf, bool stream_start, const ChunkRuns& c, Lit lit, Match match) {
  int i = c.c0;
  while (i < c.c1) {
    if (!repeats(buf, stream_start, i)) {
      lit(buf[1 + i]);
      ++i;
      continue;
    }
    const int s = i == c.c0 ? c.prev_zero + 1 : i;        // i > c0: the byte before started no run
    int t = i + 1;
    while (t < c.c1 && repeats(buf, stream_start, t)) ++t;
    if (t == c.c1) t = c.next_zero;
    const int m = t - s, full = m - m % 258, rem = m % 258, end = min(t, c.c1);
    int o = i - s;
    while (s + o < end) {
      if (o < full) {
        if (o % 258 == 0) match(258);
        o = (o / 258 + 1) * 258;
      } else if (rem >= 3) {
        if (o == full) match(rem);
        break;
      } else {
        lit(buf[1 + s + o]);
        ++o;
      }
    }
    i = end;
  }
}

__device__ void init_len_sym(PngSmem& S) {
  for (int L = threadIdx.x; L < 260; L += kPngThreads) {
    int k = 27;                                        // 258 has its own code; 227..257 share code 284
    while (k > 0 && (int)kLenBase[k] > L) --k;
    S.len_sym[L] = (uint8_t)(L == 258 ? 28 : k);
  }
}

// Moffat and Katajainen's in-place minimum-redundancy code lengths over ascending weights A[0..n), n >= 2.
__device__ void min_redundancy_lengths(int* A, int n) {
  A[0] += A[1];
  int root = 0, leaf = 2;
  for (int next = 1; next < n - 1; ++next) {
    if (leaf >= n || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = next; }
    else A[next] = A[leaf++];
    if (leaf >= n || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = next; }
    else A[next] += A[leaf++];
  }
  A[n - 2] = 0;
  for (int next = n - 3; next >= 0; --next) A[next] = A[A[next]] + 1;
  int avbl = 1, used = 0, dpth = 0, root2 = n - 2, next = n - 1;
  while (avbl > 0) {
    while (root2 >= 0 && A[root2] == dpth) { ++used; --root2; }
    while (avbl > used) { A[next--] = dpth; --avbl; }
    avbl = 2 * used;
    ++dpth;
    used = 0;
  }
}

// Length-limited Huffman code lengths of freq[0..n) (all threads call).  At least two symbols get a code, as zlib
// forces, so a single distance code is sent with one bit.
__device__ void build_lengths(const uint32_t* freq, int n, int maxbits, uint8_t* len, PngSmem& S) {
  __syncthreads();
  if (threadIdx.x == 0) {
    int used = 0;
    for (int i = 0; i < n; ++i) {
      S.w[i] = (int)freq[i];
      used += freq[i] > 0;
    }
    for (int i = 0; i < n && used < 2; ++i)
      if (S.w[i] == 0) { S.w[i] = 1; ++used; }
    S.nused = used;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += kPngThreads) {
    len[i] = 0;
    const int wi = S.w[i];
    if (wi > 0) {
      int rank = 0;
      for (int j = 0; j < n; ++j) {
        const int wj = S.w[j];
        rank += wj > 0 && (wj < wi || (wj == wi && j < i));
      }
      S.sorted[rank] = i;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int m = S.nused;
    for (int k = 0; k < m; ++k) S.A[k] = S.w[S.sorted[k]];
    min_redundancy_lengths(S.A, m);
    int num[kMaxBits + 1] = {};
    for (int k = 0; k < m; ++k) num[min(S.A[k], maxbits)]++;
    // Clamping shortened codes, so the Kraft sum may exceed 1: give up one longest code and split a shorter one
    // until it is exactly 1 (each step lowers the sum by 2^-maxbits and keeps the number of codes).
    unsigned total = 0;
    for (int l = 1; l <= maxbits; ++l) total += (unsigned)num[l] << (maxbits - l);
    while (total != (1u << maxbits)) {
      num[maxbits]--;
      for (int l = maxbits - 1; l > 0; --l)
        if (num[l]) { num[l]--; num[l + 1] += 2; break; }
      total--;
    }
    int j = 0;                                        // least frequent first: the longest codes
    for (int l = maxbits; l > 0; --l)
      for (int c = num[l]; c > 0; --c) len[S.sorted[j++]] = (uint8_t)l;
  }
  __syncthreads();
}

// Canonical codes of len[0..n), bit-reversed for deflate's LSB-first packing (one thread).
__device__ void canonical_codes(const uint8_t* len, int n, uint16_t* code) {
  int count[kMaxBits + 1] = {}, next[kMaxBits + 1];
  for (int i = 0; i < n; ++i) count[len[i]]++;
  count[0] = 0;
  int c = 0;
  for (int b = 1; b <= kMaxBits; ++b) {
    c = (c + count[b - 1]) << 1;
    next[b] = c;
  }
  for (int i = 0; i < n; ++i)
    if (len[i]) code[i] = (uint16_t)(__brev((unsigned)next[len[i]]++) >> (32 - len[i]));
}

__device__ __forceinline__ int fixed_lit_len(int s) { return s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8; }
__device__ __forceinline__ int cl_extra_bits(int s) { return s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0; }

struct PngImages {
  const uint8_t* img[BIN_PNG_MAX_BATCH];
};

// ------------------------------------------------------------------------------------------------ segment pass
__global__ void __launch_bounds__(kPngThreads) png_segment_kernel(PngImages imgs, int h, int w, int nseg,
                                                                  SegPlan* __restrict__ plans) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  PngSmem& S = *reinterpret_cast<PngSmem*>(smem_raw);
  const int tid = threadIdx.x, seg = blockIdx.x, im = blockIdx.y;
  const long long L = png_payload_bytes(h, w), g0 = (long long)seg * kSeg;
  const int len = (int)min((long long)kSeg, L - g0);
  const bool stream_start = seg == 0;
  SegPlan& P = plans[(size_t)im * nseg + seg];

  stage_payload(imgs.img[im], 3 * w, g0, len, S.buf);
  init_len_sym(S);
  for (int i = tid; i < 288; i += kPngThreads) S.lit_freq[i] = 0;
  if (tid < 32) S.dist_freq[tid] = 0;
  if (tid < 20) S.cl_freq[tid] = 0;
  if (tid == 0) { S.adler_a = 0; S.adler_b = 0; S.extra_bits = 0; }
  __syncthreads();
  if (tid == 0) S.lit_freq[256] = 1;                 // end of block

  const ChunkRuns c = chunk_runs(S.buf, stream_start, len, S.scan);
  unsigned extra = 0;
  walk_tokens(
      S.buf, stream_start, c, [&](int b) { atomicAdd(&S.lit_freq[b], 1u); },
      [&](int m) {
        const int k = S.len_sym[m];
        atomicAdd(&S.lit_freq[257 + k], 1u);
        atomicAdd(&S.dist_freq[0], 1u);
        extra += kLenExtra[k];
      });
  unsigned long long a = 0, b = 0;
  for (int i = c.c0; i < c.c1; ++i) {
    const unsigned v = S.buf[1 + i];
    a += v;
    b += (unsigned long long)(len - i) * v;
  }
  atomicAdd(&S.adler_a, a);
  atomicAdd(&S.adler_b, b);
  atomicAdd(&S.extra_bits, extra);
  __syncthreads();

  build_lengths(S.lit_freq, 286, kMaxBits, S.lit_len, S);
  build_lengths(S.dist_freq, 30, kMaxBits, S.dist_len, S);
  if (tid == 0) {
    int hlit = 286, hdist = 30;
    while (hlit > 257 && S.lit_len[hlit - 1] == 0) --hlit;
    while (hdist > 1 && S.dist_len[hdist - 1] == 0) --hdist;
    for (int i = 0; i < hlit; ++i) S.all_len[i] = S.lit_len[i];
    for (int i = 0; i < hdist; ++i) S.all_len[hlit + i] = S.dist_len[i];
    // run-length code the lengths (16: repeat the previous 3-6 times, 17: 3-10 zeros, 18: 11-138 zeros)
    const int N = hlit + hdist;
    int nrle = 0;
    auto put = [&](int sym, int x) { P.rle_sym[nrle] = (uint8_t)sym; P.rle_extra[nrle] = (uint8_t)x; ++nrle; S.cl_freq[sym]++; };
    for (int k = 0; k < N;) {
      const int v = S.all_len[k];
      int r = 1;
      while (k + r < N && S.all_len[k + r] == v) ++r;
      int rr = r;
      if (v == 0) {
        while (rr >= 11) { const int q = min(rr, 138); put(18, q - 11); rr -= q; }
        if (rr >= 3) { put(17, rr - 3); rr = 0; }
        for (; rr > 0; --rr) put(0, 0);
      } else {
        put(v, 0);
        --rr;
        while (rr >= 3) { const int q = min(rr, 6); put(16, q - 3); rr -= q; }
        for (; rr > 0; --rr) put(v, 0);
      }
      k += r;
    }
    P.hlit = (uint16_t)hlit;
    P.hdist = (uint16_t)hdist;
    P.nrle = (uint16_t)nrle;
  }
  build_lengths(S.cl_freq, 19, kClMaxBits, S.cl_len, S);
  if (tid == 0) {
    int hclen = 19;
    while (hclen > 4 && S.cl_len[kClOrder[hclen - 1]] == 0) --hclen;
    unsigned hdr = 3 + 14 + 3 * hclen;
    for (int s = 0; s < 19; ++s) hdr += S.cl_freq[s] * (S.cl_len[s] + cl_extra_bits(s));
    unsigned dyn = hdr + S.extra_bits, fix = 3 + S.extra_bits;
    for (int s = 0; s < 286; ++s) {
      dyn += S.lit_freq[s] * S.lit_len[s];
      fix += S.lit_freq[s] * fixed_lit_len(s);
    }
    dyn += S.dist_freq[0] * S.dist_len[0];
    fix += S.dist_freq[0] * 5;
    P.len = (uint32_t)len;
    P.adler_a = (uint32_t)(S.adler_a % kAdlerMod);
    P.adler_b = (uint32_t)(S.adler_b % kAdlerMod);
    P.dyn_bits = dyn;
    P.fixed_bits = fix;
    P.hdr_bits = hdr;
    P.hclen = (uint16_t)hclen;
  }
  for (int i = tid; i < 288; i += kPngThreads) P.lit_len[i] = i < 286 ? S.lit_len[i] : 0;
  if (tid < 32) P.dist_len[tid] = tid < 30 ? S.dist_len[tid] : 0;
  if (tid < 20) P.cl_len[tid] = tid < 19 ? S.cl_len[tid] : 0;
}

// ------------------------------------------------------------------------------------------------ plan pass
__global__ void png_plan_kernel(const SegPlan* __restrict__ plans, int nseg, PngBlock* __restrict__ blocks,
                                PngInfo* __restrict__ info, int64_t* __restrict__ sizes) {
  if (threadIdx.x != 0) return;
  const int im = blockIdx.x;
  const SegPlan* P = plans + (size_t)im * nseg;
  PngBlock* B = blocks + (size_t)im * nseg;
  unsigned long long bit = 0;
  uint32_t A = 1, Bsum = 0;
  for (int s = 0; s < nseg; ++s) {
    const SegPlan& p = P[s];
    const int pad = (int)((8 - ((bit + 3) & 7)) & 7);
    const unsigned long long stored = 3ull + pad + 32 + 8ull * p.len;
    unsigned long long cost = p.dyn_bits;
    int type = kDynamic;
    if (p.fixed_bits < cost) { cost = p.fixed_bits; type = kFixed; }
    if (stored < cost) { cost = stored; type = kStored; }
    B[s].bit = bit;
    B[s].type = type;
    B[s].pad = pad;
    bit += cost;
    Bsum = (uint32_t)((Bsum + (unsigned long long)p.len % kAdlerMod * A + p.adler_b) % kAdlerMod);
    A = (A + p.adler_a) % kAdlerMod;
  }
  const unsigned long long zlen = 2 + (bit + 7) / 8 + 4;
  info[im].zlen = zlen;
  info[im].adler = (Bsum << 16) | A;
  info[im].nidat = (int)((zlen + kIdat - 1) / kIdat);
  sizes[im] = (int64_t)(8 + 25 + 12 * ((zlen + kIdat - 1) / kIdat) + zlen + 12);
}

// ------------------------------------------------------------------------------------------------ emit pass
// Writes bits [lo, hi) of the stream: whole words inside the range are stored, the others ORed in.
struct BitWriter {
  uint32_t* buf;
  unsigned long long lo, hi, word, acc;
  int fill;
  __device__ BitWriter(uint32_t* b, unsigned long long start, unsigned long long end)
      : buf(b), lo(start), hi(end), word(start >> 5), acc(0), fill((int)(start & 31)) {}
  __device__ __forceinline__ void flush_word() {
    const uint32_t v = (uint32_t)acc;
    const unsigned long long w0 = word << 5;
    if (w0 >= lo && w0 + 32 <= hi) buf[word] = v;
    else if (v) atomicOr(buf + word, v);
    acc >>= 32;
    fill -= 32;
    ++word;
  }
  __device__ __forceinline__ void put(uint32_t bits, int n) {   // n <= 16
    acc |= (unsigned long long)bits << fill;
    fill += n;
    if (fill >= 32) flush_word();
  }
  __device__ void finish() {
    if (fill > 0) {
      const uint32_t v = (uint32_t)acc;
      if (v) atomicOr(buf + word, v);
    }
  }
};

__global__ void __launch_bounds__(kPngThreads) png_emit_kernel(PngImages imgs, int h, int w, int nseg,
                                                               const SegPlan* __restrict__ plans,
                                                               const PngBlock* __restrict__ blocks, uint32_t* zbuf,
                                                               size_t zbuf_words) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  PngSmem& S = *reinterpret_cast<PngSmem*>(smem_raw);
  const int tid = threadIdx.x, seg = blockIdx.x, im = blockIdx.y;
  const long long L = png_payload_bytes(h, w), g0 = (long long)seg * kSeg;
  const int len = (int)min((long long)kSeg, L - g0);
  const bool stream_start = seg == 0, last = seg == nseg - 1;
  const SegPlan& P = plans[(size_t)im * nseg + seg];
  const PngBlock blk = blocks[(size_t)im * nseg + seg];
  uint32_t* out = zbuf + (size_t)im * zbuf_words;

  stage_payload(imgs.img[im], 3 * w, g0, len, S.buf);
  init_len_sym(S);
  if (blk.type != kStored) {
    for (int i = tid; i < 288; i += kPngThreads) S.lit_len[i] = blk.type == kDynamic ? P.lit_len[i] : fixed_lit_len(i);
    if (tid < 32) S.dist_len[tid] = blk.type == kDynamic ? P.dist_len[tid] : (tid < 30 ? 5 : 0);
    if (tid < 20) S.cl_len[tid] = P.cl_len[tid];
  }
  __syncthreads();
  if (blk.type != kStored && tid == 0) {
    canonical_codes(S.lit_len, 288, S.lit_code);
    canonical_codes(S.dist_len, 32, S.dist_code);
    if (blk.type == kDynamic) canonical_codes(S.cl_len, 19, S.cl_code);
  }
  const ChunkRuns c = chunk_runs(S.buf, stream_start, len, S.scan);   // its scans synchronise the CTA

  unsigned bits = 0;
  if (blk.type == kStored) {
    bits = 8u * (c.c1 - c.c0);
  } else {
    walk_tokens(
        S.buf, stream_start, c, [&](int b) { bits += S.lit_len[b]; },
        [&](int m) {
          const int k = S.len_sym[m];
          bits += S.lit_len[257 + k] + kLenExtra[k] + S.dist_len[0];
        });
    if (tid == kPngThreads - 1) bits += S.lit_len[256];
  }
  const unsigned off = block_excl_scan(bits, 0u, false, S.scan, [](unsigned a, unsigned b) { return a + b; });
  const unsigned hdr_bits = blk.type == kStored ? 3 + blk.pad + 32 : blk.type == kFixed ? 3 : P.hdr_bits;
  if (tid == 0) {
    BitWriter bw(out, blk.bit, blk.bit + hdr_bits);
    bw.put((last ? 1u : 0u) | ((unsigned)blk.type << 1), 3);
    if (blk.type == kStored) {
      bw.put(0, blk.pad);
      bw.put((uint32_t)len, 16);
      bw.put((uint32_t)(~len) & 0xffffu, 16);
    } else if (blk.type == kDynamic) {
      bw.put(P.hlit - 257, 5);
      bw.put(P.hdist - 1, 5);
      bw.put(P.hclen - 4, 4);
      for (int k = 0; k < P.hclen; ++k) bw.put(S.cl_len[kClOrder[k]], 3);
      for (int r = 0; r < P.nrle; ++r) {
        const int s = P.rle_sym[r];
        bw.put(S.cl_code[s], S.cl_len[s]);
        if (s >= 16) bw.put(P.rle_extra[r], cl_extra_bits(s));
      }
    }
    bw.finish();
  }
  if (bits > 0) {
    const unsigned long long start = blk.bit + hdr_bits + off;
    BitWriter bw(out, start, start + bits);
    if (blk.type == kStored) {
      for (int i = c.c0; i < c.c1; ++i) bw.put(S.buf[1 + i], 8);
    } else {
      walk_tokens(
          S.buf, stream_start, c, [&](int b) { bw.put(S.lit_code[b], S.lit_len[b]); },
          [&](int m) {
            const int k = S.len_sym[m];
            bw.put(S.lit_code[257 + k], S.lit_len[257 + k]);
            if (kLenExtra[k]) bw.put((uint32_t)(m - kLenBase[k]), kLenExtra[k]);
            bw.put(S.dist_code[0], S.dist_len[0]);
          });
      if (tid == kPngThreads - 1) bw.put(S.lit_code[256], S.lit_len[256]);
    }
    bw.finish();
  }
}

// ------------------------------------------------------------------------------------------------ framing pass
// CRC-32 (reflected, polynomial 0xedb88320) without the final inversion is linear in (state, data), so
// crc(S, A || B) = crc(S, A) * x^(8|B|) mod P  xor  crc(0, B).
__device__ uint32_t gf2_mulmod(uint32_t a, uint32_t b) {      // a * b mod P, bit 31 = x^0
  uint32_t p = 0;
  for (int k = 0; k < 32; ++k) {
    if (a & (0x80000000u >> k)) p ^= b;
    b = (b & 1) ? (b >> 1) ^ 0xedb88320u : b >> 1;
  }
  return p;
}
__device__ uint32_t x_pow_8n(unsigned n) {                    // x^(8n) mod P
  uint32_t r = 0x80000000u, base = 0x80000000u >> 8;
  for (; n; n >>= 1) {
    if (n & 1) r = gf2_mulmod(base, r);
    base = gf2_mulmod(base, base);
  }
  return r;
}

__device__ __forceinline__ uint8_t zbyte(const uint8_t* z, unsigned long long zlen, uint32_t adler, unsigned long long j) {
  if (j < 2) return j == 0 ? 0x78 : 0x01;                    // deflate, 32K window, no dictionary (what cv2 writes)
  if (j >= zlen - 4) return (uint8_t)(adler >> (8 * (3 - (int)(j - (zlen - 4)))));
  return z[j - 2];
}

__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
  p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}

__global__ void __launch_bounds__(kFrameWarps * 32) png_frame_kernel(int h, int w, const PngInfo* __restrict__ info,
                                                                     const uint32_t* __restrict__ zbuf, size_t zbuf_words,
                                                                     uint8_t* __restrict__ out, size_t out_stride) {
  __shared__ uint32_t table[256];
  {
    uint32_t c = threadIdx.x;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xedb88320u : c >> 1;
    table[threadIdx.x] = c;
  }
  __syncthreads();
  const int im = blockIdx.y, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * kFrameWarps + (threadIdx.x >> 5);
  const PngInfo inf = info[im];
  if (chunk >= inf.nidat) return;
  uint8_t* file = out + (size_t)im * out_stride;
  const uint8_t* z = reinterpret_cast<const uint8_t*>(zbuf + (size_t)im * zbuf_words);
  auto crc_bytes = [&](uint32_t s, const uint8_t* p, int n) {
    for (int i = 0; i < n; ++i) s = table[(s ^ p[i]) & 0xff] ^ (s >> 8);
    return s;
  };

  if (chunk == 0 && lane == 0) {
    const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
    for (int i = 0; i < 8; ++i) file[i] = sig[i];
    uint8_t* c = file + 8;
    put_be32(c, 13);
    c[4] = 'I'; c[5] = 'H'; c[6] = 'D'; c[7] = 'R';
    put_be32(c + 8, (uint32_t)w);
    put_be32(c + 12, (uint32_t)h);
    c[16] = 8; c[17] = 2; c[18] = 0; c[19] = 0; c[20] = 0;   // 8-bit truecolour, deflate, filter 0, no interlace
    put_be32(c + 21, ~crc_bytes(0xffffffffu, c + 4, 17));
  }

  const unsigned long long d0 = (unsigned long long)chunk * kIdat;
  const int dlen = (int)min((unsigned long long)kIdat, inf.zlen - d0);
  uint8_t* c = file + 33 + (size_t)chunk * (kIdat + 12);
  const int per = kIdat / 32, b0 = min(lane * per, dlen), b1 = min(b0 + per, dlen);
  uint32_t s = 0;
  if (lane == 0) {
    put_be32(c, (uint32_t)dlen);
    c[4] = 'I'; c[5] = 'D'; c[6] = 'A'; c[7] = 'T';
    s = crc_bytes(0xffffffffu, c + 4, 4);
  }
  for (int i = b0; i < b1; ++i) {
    const uint8_t v = zbyte(z, inf.zlen, inf.adler, d0 + i);
    c[8 + i] = v;
    s = table[(s ^ v) & 0xff] ^ (s >> 8);
  }
  uint32_t crc = s;
  for (int l = 1; l < 32; ++l) {
    const uint32_t sl = __shfl_sync(0xffffffffu, s, l);
    const int nl = __shfl_sync(0xffffffffu, b1 - b0, l);
    if (lane == 0 && nl > 0) crc = gf2_mulmod(x_pow_8n((unsigned)nl), crc) ^ sl;
  }
  if (lane == 0) {
    put_be32(c + 8 + dlen, ~crc);
    if (chunk == inf.nidat - 1) {
      uint8_t* e = c + 12 + dlen;
      const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xae, 0x42, 0x60, 0x82};
      for (int i = 0; i < 12; ++i) e[i] = iend[i];
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
size_t png_max_bytes(int h, int w) {
  if (!png_shape_ok(h, w)) return 0;
  return png_file_bytes(2 + png_deflate_cap(png_payload_bytes(h, w)) + 4);
}

struct PngLayout {
  size_t plans, blocks, info, zbuf, total, zbuf_bytes;
};
static PngLayout png_layout(int n, int h, int w) {
  const long long L = png_payload_bytes(h, w);
  const size_t nseg = (size_t)png_nseg(L);
  PngLayout o;
  o.plans = 0;
  o.blocks = o.plans + png_align((size_t)n * nseg * sizeof(SegPlan));
  o.info = o.blocks + png_align((size_t)n * nseg * sizeof(PngBlock));
  o.zbuf = o.info + png_align((size_t)n * sizeof(PngInfo));
  o.zbuf_bytes = png_zbuf_bytes(L);
  o.total = o.zbuf + (size_t)n * o.zbuf_bytes;
  return o;
}

size_t png_workspace_bytes(int n, int h, int w) {
  if (n < 1 || n > BIN_PNG_MAX_BATCH || !png_shape_ok(h, w)) return 0;
  return png_layout(n, h, w).total;
}

int launch_png_encode_u8(const uint8_t* const* imgs_host, int n, int h, int w, uint8_t* out, size_t out_stride,
                         int64_t* sizes, void* workspace, size_t workspace_bytes, cudaStream_t s) {
  // every check precedes the first CUDA call
  if (!imgs_host || !out || !sizes || !workspace) return fail(BIN_ERR_ARG, "png_encode: null argument");
  if (n < 1 || n > BIN_PNG_MAX_BATCH) return fail(BIN_ERR_ARG, "png_encode: n must be in 1..BIN_PNG_MAX_BATCH");
  if (!png_shape_ok(h, w))
    return fail(BIN_ERR_ARG, "png_encode: h and w must be in 1..65535 with h*(3w+1) < 2^31");
  PngImages imgs{};
  for (int i = 0; i < n; ++i) {
    if (!imgs_host[i]) return fail(BIN_ERR_ARG, "png_encode: null image pointer");
    imgs.img[i] = imgs_host[i];
  }
  if (out_stride < png_max_bytes(h, w))
    return fail(BIN_ERR_ARG, "png_encode: out_stride below bin_png_max_bytes(h, w)");
  if (out_stride > SIZE_MAX / (size_t)n) return fail(BIN_ERR_ARG, "png_encode: n * out_stride overflows");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(BIN_ERR_ARG, "png_encode: workspace must be 256-byte aligned");
  if (reinterpret_cast<uintptr_t>(sizes) & 7) return fail(BIN_ERR_ARG, "png_encode: sizes must be 8-byte aligned");
  const PngLayout lay = png_layout(n, h, w);
  if (workspace_bytes < lay.total)
    return fail(BIN_ERR_WORKSPACE, "png_encode: workspace too small (see bin_png_workspace_bytes)");

  static std::atomic<unsigned long long> seg_mask{0}, emit_mask{0};
  BIN_TRY(ensure_dynamic_smem(png_segment_kernel, (int)sizeof(PngSmem), seg_mask));
  BIN_TRY(ensure_dynamic_smem(png_emit_kernel, (int)sizeof(PngSmem), emit_mask));
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  SegPlan* plans = reinterpret_cast<SegPlan*>(ws + lay.plans);
  PngBlock* blocks = reinterpret_cast<PngBlock*>(ws + lay.blocks);
  PngInfo* info = reinterpret_cast<PngInfo*>(ws + lay.info);
  uint32_t* zbuf = reinterpret_cast<uint32_t*>(ws + lay.zbuf);
  const size_t zwords = lay.zbuf_bytes / 4;
  const int nseg = png_nseg(png_payload_bytes(h, w));

  BIN_CUDA_OK(cudaMemsetAsync(zbuf, 0, (size_t)n * lay.zbuf_bytes, s));
  png_segment_kernel<<<dim3(nseg, n), kPngThreads, sizeof(PngSmem), s>>>(imgs, h, w, nseg, plans);
  BIN_CUDA_OK(cudaGetLastError());
  png_plan_kernel<<<n, 32, 0, s>>>(plans, nseg, blocks, info, sizes);
  BIN_CUDA_OK(cudaGetLastError());
  png_emit_kernel<<<dim3(nseg, n), kPngThreads, sizeof(PngSmem), s>>>(imgs, h, w, nseg, plans, blocks, zbuf, zwords);
  BIN_CUDA_OK(cudaGetLastError());
  const long long zmax = 2 + png_deflate_cap(png_payload_bytes(h, w)) + 4;
  const int max_idat = (int)((zmax + kIdat - 1) / kIdat);
  png_frame_kernel<<<dim3((max_idat + kFrameWarps - 1) / kFrameWarps, n), kFrameWarps * 32, 0, s>>>(
      h, w, info, zbuf, zwords, out, out_stride);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}

}  // namespace binb
