// FAST-9 corner detector (16-pixel ring, >= 9 contiguous brighter-or-darker pixels).
// Reference: vpp/algorithms/fast_detector/fast.hpp:253-508 (SIMD pruning tree == the 9-arc
// predicate on the ring *as implemented*, whose slots 4 and 12 are sampled on row r-3),
// :36-77 (score, true ring), :663-673 / :889-928 / :745-799 (plain, local-maxima, blockwise),
// mask semantics :310-317 (mask byte bit 4 gates the brighter arc, bit 0 the darker arc).
//
// GPU structure: pass 1 puts one warp on 32 consecutive pixels of a row; the two "necessary"
// ring pixels (top/bottom) are tested first and __any_sync lets the whole warp skip the other
// 14 loads when no lane can be a corner; the corner flags of the 32 lanes are collected with
// __ballot_sync into one word of a bitmask (1 bit / pixel).  Maxima modes refine that bitmask.
// Pass 2 scans per-row counts and emits keypoints in raster order (deterministic, unlike the
// reference's per-thread buffers flushed under `omp critical`).
// HBM-bound: 1 byte read per pixel (+1 with a mask) + 8 bytes per keypoint.
#include "common.cuh"

#include <atomic>
#include "tma.cuh"

namespace vppb {

// ring slot -> (dr, dc).  Row 0: as implemented by fast9() (fast.hpp:327-461); row 1: true ring.
__constant__ signed char c_ring[2][16][2] = {
    {{-3, 0}, {-3, 1}, {-2, 2}, {-1, 3}, {-3, 3}, {1, 3}, {2, 2}, {3, 1}, {3, 0}, {3, -1}, {2, -2}, {1, -3}, {-3, -3}, {-1, -3}, {-2, -2}, {-3, -1}},
    {{-3, 0}, {-3, 1}, {-2, 2}, {-1, 3}, {0, 3}, {1, 3}, {2, 2}, {3, 1}, {3, 0}, {3, -1}, {2, -2}, {1, -3}, {0, -3}, {-1, -3}, {-2, -2}, {-3, -1}}};

__device__ __forceinline__ bool arc9(uint32_t m16) {
  uint32_t x = m16 | (m16 << 16);
  x &= x >> 1;
  x &= x >> 2;
  x &= x >> 4;  // 8 contiguous
  x &= x >> 1;  // 9 contiguous
  return x != 0;
}

// fast.hpp:36-77: sum of |v - a| over ring pixels beyond the threshold, max of the two polarities
__device__ __forceinline__ int fast9_score_at(const Img& im, int r, int c, int th) {
  const unsigned char* p = im.base + (long long)r * im.pitch + c;
  const int v = *p;
  int sum_inf = 0, sum_sup = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) {
    const int a = p[(long long)c_ring[1][i][0] * im.pitch + c_ring[1][i][1]];
    const int diff = v - a;
    if (diff < -th) sum_inf -= diff;
    else if (diff > th) sum_sup += diff;
  }
  return max(sum_sup, sum_inf);
}

// pass 1: detection -> bitmask words (row-major, wpr words per row) and per-row counts
__global__ void __launch_bounds__(256) k_fast9_detect(Img im, Img mask, int has_mask, int th, int ring, uint32_t* bits, int wpr, int* rowcount) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long total = (long long)im.nrows * wpr;
  const int thb = th & 255;  // S::repeat(th) replicates the low byte
  for (long long w = warp0; w < total; w += nwarps) {
    const int r = (int)(w / wpr);
    const int c = (int)(w - (long long)r * wpr) * 32 + lane;
    const bool inside = c < im.ncols;
    const unsigned char* p = im.base + (long long)r * im.pitch + c;
    int m = 0xFF;
    if (has_mask) m = inside ? (int)__ldg(mask.base + (long long)r * mask.pitch + c) : 0;
    int v = 0, hi = 0, lo = 0;
    bool cand_b = false, cand_d = false;
    if (inside && m != 0) {
      v = __ldg(p);
      hi = min(v + thb, 255);  // u_adds
      lo = max(v - thb, 0);    // u_subs
      const int a0 = __ldg(p + (long long)c_ring[ring][0][0] * im.pitch + c_ring[ring][0][1]);
      const int a8 = __ldg(p + (long long)c_ring[ring][8][0] * im.pitch + c_ring[ring][8][1]);
      // every 9-arc of the 16-ring contains slot 0 or slot 8 (fast.hpp:326-337)
      cand_b = (m & 0x10) && (a0 > hi || a8 > hi);
      cand_d = (m & 0x01) && (a0 < lo || a8 < lo);
    }
    bool corner = false;
    if (__any_sync(0xffffffffu, cand_b || cand_d)) {
      if (cand_b || cand_d) {
        uint32_t mb = 0, md = 0;
#pragma unroll
        for (int i = 0; i < 16; i++) {
          const int a = __ldg(p + (long long)c_ring[ring][i][0] * im.pitch + c_ring[ring][i][1]);
          mb |= (uint32_t)(a > hi) << i;
          md |= (uint32_t)(a < lo) << i;
        }
        corner = (cand_b && arc9(mb)) || (cand_d && arc9(md));
      }
    }
    const uint32_t word = __ballot_sync(0xffffffffu, corner);
    if (lane == 0) {
      bits[w] = word;
      if (word) atomicAdd(&rowcount[r], __popc(word));
    }
  }
}

// ------------------------------------------------------------------ band kernel (TMA-staged detection)
// One CTA per band of FB_ROWS image rows; the band is walked in boxes of 2016 pixels.  Thread 0 keeps two TMA boxes in
// flight (2048 bytes = 16 halo + 2016 + 16 halo, by FB_ROWS + 6 rows), the CTA works on one while the other lands.
//   phase 1 (prefilter, 4 pixels per thread per step, packed bytes): every 9-arc of the ring contains slot 0 (r-3, c) or
//     slot 8 (r+3, c) (fast.hpp:326-337), and both sit in the same column as the centre, so |v - a0| > th or |v - a8| > th
//     is evaluated on whole aligned words: VABSDIFF4 + a 3-instruction packed "greater than th".  Survivors (a few percent
//     of a natural frame, the pixels within 3 rows of a strong horizontal contrast) are appended to a candidate list in
//     shared memory.
//   phase 2 (exact test, one candidate per thread, no idle lanes): the 16 ring bytes come from the staged box; bright /
//     dark flags are shifted into two 16-bit masks (one subtraction + one funnel shift per slot and polarity), the 9-arc
//     test is the bit trick of arc9(); corners set their bit in the band's bitmask (shared memory).
// After the last box the band's bitmask rows and their per-row / per-band counts go to global memory; k_fast9_emit_bands
// turns them into raster-ordered keypoints.  No atomics on global memory, nothing to zero beforehand.
constexpr int FB_ROWS = 4;   // rows per tile: small tiles = many CTAs per SM and fine-grained balance (a 4K frame is 1080 tiles over 792 resident CTAs on 132 SMs)
constexpr int FE_ROWS = 8;   // rows per CTA of the emit kernel (one warp each)
constexpr int FB_BOXW = 2048;
constexpr int FB_INNER = FB_BOXW - 32;
constexpr int FB_INH = FB_ROWS + 6;
constexpr int FB_STAGE = FB_INH * FB_BOXW;
constexpr int FB_THREADS = 256;
constexpr int FB_WARPS = FB_THREADS / 32;
constexpr int FB_WCOLS = FB_INNER / FB_WARPS;  // 252 pixels = 63 words of a box row per warp
constexpr int FB_MAXW = 65535;

constexpr int FB_BOXWORDS = FB_INNER / 32;  // 63 bitmask words per box row
constexpr int FB_SMEM = FB_STAGE + FB_ROWS * FB_INNER * 2 + FB_ROWS * FB_BOXWORDS * 4 + 8 + (FB_WARPS + FB_ROWS) * 4 + 32;

template <int RING, bool has_mask>
__global__ void __launch_bounds__(FB_THREADS, 5) k_fast9_band(const __grid_constant__ CUtensorMap tmap, Img im, Img mask, int th, int nboxes,
                                                              int wpr, uint32_t* bits, int* rowcount, int* bandtotal) {
  extern __shared__ __align__(128) unsigned char smem[];
  unsigned char* st = smem;
  unsigned short* lists = reinterpret_cast<unsigned short*>(smem + FB_STAGE);
  uint32_t* bm = reinterpret_cast<uint32_t*>(smem + FB_STAGE + FB_ROWS * FB_INNER * 2);   // [FB_ROWS][FB_BOXWORDS]: this box's columns only
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + FB_STAGE + FB_ROWS * FB_INNER * 2 + FB_ROWS * FB_BOXWORDS * 4);
  int* ncand = reinterpret_cast<int*>(bar + 1);    // [FB_WARPS], one counter per warp
  int* rowcnt = ncand + FB_WARPS;                  // [FB_ROWS]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  grid_launch_dependents();  // the emit kernel may be scheduled as SMs free up; it waits for this grid before it reads anything
  const int band = blockIdx.x / nboxes, k = blockIdx.x - band * nboxes, r0 = band * FB_ROWS;
  const int rows_here = min(FB_ROWS, im.nrows - r0);
  const int thb = th & 255;  // S::repeat(th) replicates the low byte (fast.hpp:120-126)
  const int xbase = k * FB_INNER;                        // image column of box byte 16
  const int cols_here = min(FB_INNER, im.ncols - xbase);

  if (tid == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
    // tensor origin = 16 bytes left of column 0 and 3 rows above row 0; 8-byte elements, 252 elements per inner box
    mbar_arrive_expect_tx(bar, FB_STAGE);
    tma_load_2d(st, &tmap, k * (FB_INNER / 8), r0, bar);
  }
  if (tid < FB_WARPS) ncand[tid] = 0;
  for (int i = tid; i < FB_ROWS * FB_BOXWORDS; i += FB_THREADS) bm[i] = 0;
  __syncthreads();

  // packed "byte > thb":  u = thb + 1;  x >= u  <=>  bit 7 of ((x | H) - (U & ~H)) combined with bit 7 of x
  const uint32_t H = 0x80808080u;
  const uint32_t K = (((uint32_t)(thb + 1) & 0x7Fu) * 0x01010101u);
  const bool u_high = (thb + 1) >= 128;
  // every warp owns a column strip of the box (FB_WCOLS pixels = 2 words per lane) and works on it alone: its own
  // candidate list, __syncwarp between its two phases; the CTA only meets at the very end
  unsigned short* list = lists + warp * (FB_ROWS * FB_WCOLS);

  if (thb < 255) {
    mbar_wait(bar, 0);
    // ---- phase 1: lane = word column; the 14 rows of the column are loaded once, every row serves as slot 0 of the row 3
    //      below it, as centre, and as slot 8 of the row 3 above it
#pragma unroll
    for (int half = 0; half < 2; half++) {
      const int wi = warp * (FB_WCOLS / 4) + half * 32 + lane;   // word of the box-inner row
      const int x = 4 * wi;
      if (half * 32 + lane < FB_WCOLS / 4 && x < cols_here) {
        const unsigned char* colp = st + 16 + x;
        uint32_t w[FB_INH];
#pragma unroll
        for (int j = 0; j < FB_INH; j++) w[j] = *reinterpret_cast<const uint32_t*>(colp + j * FB_BOXW);
        uint32_t edge = 0xFFFFFFFFu;
        if (x + 4 > cols_here) edge = (1u << (8 * (cols_here - x))) - 1u;  // bytes right of the image
#pragma unroll
        for (int j = 0; j < FB_ROWS; j++) {
          const uint32_t v = w[j + 3];
          const uint32_t d0 = __vabsdiffu4(v, w[j]), d8 = __vabsdiffu4(v, w[j + 6]);
          const uint32_t t0 = (d0 | H) - K, t8 = (d8 | H) - K;
          uint32_t g = u_high ? ((t0 & d0) | (t8 & d8)) : (t0 | d0 | t8 | d8);
          g &= H & edge;
          if (g && j < rows_here) {
            if (has_mask) {
              const unsigned char* mp = mask.base + (long long)(r0 + j) * mask.pitch + xbase + x;
#pragma unroll
              for (int q = 0; q < 4; q++)
                if (((g >> (8 * q + 7)) & 1u) && __ldg(mp + q) == 0) g &= ~(0x80u << (8 * q));
            }
            while (g) {
              const int q = (__ffs(g) - 1) >> 3;
              g &= g - 1;
              const int idx = atomicAdd(&ncand[warp], 1);
              list[idx] = (unsigned short)((j << 11) | (16 + x + q));
            }
          }
        }
      }
    }
    __syncthreads();
    // ---- phase 2: exact test, one candidate per thread; the candidates of all strips are shared out evenly over the CTA
    //      (strips that cross a strong edge hold most of them)
    int start[FB_WARPS + 1];
    start[0] = 0;
#pragma unroll
    for (int w = 0; w < FB_WARPS; w++) start[w + 1] = start[w] + ncand[w];
    for (int e = tid; e < start[FB_WARPS]; e += FB_THREADS) {
      int w = 0;
#pragma unroll
      for (int q = 1; q < FB_WARPS; q++) w += (e >= start[q]) ? 1 : 0;
      const int code = lists[w * (FB_ROWS * FB_WCOLS) + (e - start[w])];
      const int j = code >> 11, xl = code & 2047;
      const unsigned char* p = st + (j + 3) * FB_BOXW + xl;
      const int v = p[0];
      const int cb = v + thb, cd = v - thb;  // brighter: a > cb (== a > min(v+th,255)); darker: a < cd
      uint32_t mb = 0, md = 0;
#define VPPB_FAST_SLOT(DR, DC)                                                  \
      {                                                                         \
        const int a = p[(DR) * FB_BOXW + (DC)];                                 \
        mb = __funnelshift_l((uint32_t)(cb - a), mb, 1);                        \
        md = __funnelshift_l((uint32_t)(a - cd), md, 1);                        \
      }
      VPPB_FAST_SLOT(-3, 0) VPPB_FAST_SLOT(-3, 1) VPPB_FAST_SLOT(-2, 2) VPPB_FAST_SLOT(-1, 3)
      if (RING == 0) VPPB_FAST_SLOT(-3, 3) else VPPB_FAST_SLOT(0, 3)
      VPPB_FAST_SLOT(1, 3) VPPB_FAST_SLOT(2, 2) VPPB_FAST_SLOT(3, 1) VPPB_FAST_SLOT(3, 0) VPPB_FAST_SLOT(3, -1)
      VPPB_FAST_SLOT(2, -2) VPPB_FAST_SLOT(1, -3)
      if (RING == 0) VPPB_FAST_SLOT(-3, -3) else VPPB_FAST_SLOT(0, -3)
      VPPB_FAST_SLOT(-1, -3) VPPB_FAST_SLOT(-2, -2) VPPB_FAST_SLOT(-3, -1)
#undef VPPB_FAST_SLOT
      const int c = xbase + xl - 16;
      int m = 0xFF;
      if (has_mask) m = __ldg(mask.base + (long long)(r0 + j) * mask.pitch + c);
      const bool corner = ((m & 0x10) && arc9(mb & 0xFFFFu)) || ((m & 0x01) && arc9(md & 0xFFFFu));
      if (corner) atomicOr(&bm[j * FB_BOXWORDS + ((xl - 16) >> 5)], 1u << ((xl - 16) & 31));
    }
  }
  __syncthreads();
  // ---- this box's bitmask columns and per-row counts to global memory (2016 = 63 words: boxes start on word boundaries)
  if (warp < FB_ROWS) {
    int cnt = 0;
    if (warp < rows_here) {
      const int w0 = xbase >> 5, nw = (cols_here + 31) >> 5;
      for (int w = lane; w < nw; w += 32) {
        const uint32_t word = bm[warp * FB_BOXWORDS + w];
        bits[(long long)(r0 + warp) * wpr + w0 + w] = word;
        cnt += __popc(word);
      }
    }
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) {
      rowcnt[warp] = cnt;
      if (warp < rows_here) rowcount[(long long)(r0 + warp) * nboxes + k] = cnt;
    }
  }
  __syncthreads();
  if (tid == 0) {
    int t = 0;
    for (int j = 0; j < FB_ROWS; j++) t += rowcnt[j];
    bandtotal[band * nboxes + k] = t;
  }
}

// out of line: the emit loop is unrolled over the words a lane holds, the 16 ring loads of a score must not be copied 16 times
__device__ __noinline__ int fast9_score_out(const Img& im, int r, int c, int th, int score_div) {
  const int sc = fast9_score_at(im, r, c, th);
  return score_div ? ((sc / 16) & 255) : sc;
}

// Raster-ordered emission from the band kernel's output: CTA = band; its first keypoint index is the sum of the totals of
// the (band, box) tiles above (summed by the CTA itself - no scan launch), one warp per row walks the bitmask, whose
// words it has all loaded up front (independent loads: one memory latency per row, not one per 32 words).
// The last band also stores the total count.
constexpr int FE_MAXW = 16;  // bitmask words per lane staged per pass: rows up to 16 * 32 * 32 = 16384 pixels in one pass
__global__ void __launch_bounds__(FB_THREADS) k_fast9_emit_bands(Img im, int th, const uint32_t* bits, int wpr, const int* rowcount, const int* bandtotal,
                                                                int nbands, int nboxes, vppb_int2* kps, int* scores, int score_div, int capacity, int* count_dev) {
  __shared__ int part[FB_THREADS / 32];
  __shared__ int base_s;
  __shared__ uint32_t rowbits[FB_THREADS / 32][FE_MAXW * 32];  // a row's words, loaded up front (independent loads), consumed by a rolled loop
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r0 = blockIdx.x * FE_ROWS, band = r0 / FB_ROWS;   // FE_ROWS is a multiple of FB_ROWS: the CTA starts on a band boundary
  const int r = r0 + warp;
  const bool row_ok = warp < FE_ROWS && r < im.nrows;
  grid_dependency_wait();  // launched programmatically behind the tile kernel: its bitmask and counts are complete from here on
#pragma unroll
  for (int q = 0; q < FE_MAXW; q++) {
    const int wi = q * 32 + lane;
    rowbits[warp][wi] = (row_ok && wi < wpr) ? __ldg(&bits[(long long)r * wpr + wi]) : 0u;
  }
  int rc = 0;  // lane j < FE_ROWS: keypoints of row r0 + j (all boxes)
  if (lane < FE_ROWS && r0 + lane < im.nrows)
    for (int k = 0; k < nboxes; k++) rc += __ldg(&rowcount[(long long)(r0 + lane) * nboxes + k]);
  int acc = 0;
  const int before = band * nboxes;
  for (int i = tid; i < before; i += FB_THREADS) acc += __ldg(&bandtotal[i]);
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) part[warp] = acc;
  __syncthreads();
  if (tid == 0) {
    int b = 0;
    for (int i = 0; i < FB_THREADS / 32; i++) b += part[i];
    base_s = b;
    if (blockIdx.x == gridDim.x - 1 && count_dev) {
      int t = b;
      for (int i = before; i < nbands * nboxes; i++) t += bandtotal[i];
      *count_dev = t;
    }
  }
  __syncthreads();
  if (!row_ok) return;
  int off = base_s, mine = 0;
  for (int j = 0; j < FE_ROWS; j++) {
    const int cj = __shfl_sync(0xffffffffu, rc, j);
    if (j < warp) off += cj;
    if (j == warp) mine = cj;
  }
  if (mine == 0) return;
#pragma unroll 1
  for (int w0 = 0; w0 < wpr; w0 += 32) {
    const int wi = w0 + lane;
    uint32_t word = w0 < FE_MAXW * 32 ? rowbits[warp][wi] : (wi < wpr ? bits[(long long)r * wpr + wi] : 0u);  // rows wider than 16384 pixels: the rest loads as it goes
    const int cnt = __popc(word);
    int incl = cnt;
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    int pos = off + incl - cnt;
    while (word) {
      const int b = __ffs(word) - 1;
      word &= word - 1;
      if (pos < capacity) {
        const int c = wi * 32 + b;
        kps[pos] = vppb_int2{r, c};
        if (scores) scores[pos] = fast9_score_out(im, r, c, th, score_div);
      }
      pos++;
    }
    off += __shfl_sync(0xffffffffu, incl, 31);
  }
}

__device__ __forceinline__ bool bit_at(const uint32_t* bits, int wpr, int nrows, int ncols, int r, int c) {
  if (r < 0 || r >= nrows || c < 0 || c >= ncols) return false;
  return (bits[(long long)r * wpr + (c >> 5)] >> (c & 31)) & 1u;
}

// local maxima (fast.hpp:889-928): keep a detected corner iff its u8 score (score/16) is strictly
// greater than the 8 neighbours' entries of the score image (0 where no corner was detected).
__global__ void __launch_bounds__(256) k_fast9_local_max(Img im, int th, const uint32_t* bits, uint32_t* bits_out, int wpr, int* rowcount) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long total = (long long)im.nrows * wpr;
  for (long long w = warp0; w < total; w += nwarps) {
    const uint32_t word = bits[w];
    bool keep = false;
    if (word) {  // warp-uniform
      const int r = (int)(w / wpr);
      const int c = (int)(w - (long long)r * wpr) * 32 + lane;
      if ((word >> lane) & 1u) {
        const int a = (fast9_score_at(im, r, c, th) / 16) & 255;
        keep = true;
#pragma unroll
        for (int dr = -1; dr <= 1; dr++)
#pragma unroll
          for (int dc = -1; dc <= 1; dc++) {
            if (dr == 0 && dc == 0) continue;
            int n = 0;
            if (bit_at(bits, wpr, im.nrows, im.ncols, r + dr, c + dc)) n = (fast9_score_at(im, r + dr, c + dc, th) / 16) & 255;
            keep = keep && (a > n);
          }
      }
    }
    const uint32_t out = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) {
      bits_out[w] = out;
      if (out) atomicAdd(&rowcount[(int)(w / wpr)], __popc(out));
    }
  }
}

// blockwise maxima (fast.hpp:745-799): per block_size x block_size cell anchored at (0,0), raster
// scan, strict '>' (first maximum wins), kept iff max > 0.  One thread per cell; bits_out zeroed by caller.
__global__ void __launch_bounds__(128) k_fast9_block_max(Img im, int th, int bs, const uint32_t* bits, unsigned* cellkp, int wpr,
                                                        int* rowcount, int cells_r, int cells_c) {
  const long long total = (long long)cells_r * cells_c;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r0 = (int)(i / cells_c) * bs, c0 = (int)(i % cells_c) * bs;
    unsigned vmax = 0;
    int pr = -1, pc = -1;
    for (int r = r0; r < min(r0 + bs, im.nrows); r++) {
      int c = c0;
      const int cend = min(c0 + bs, im.ncols);
      while (c < cend) {
        const int wi = c >> 5;
        uint32_t word = bits[(long long)r * wpr + wi] >> (c & 31);
        const int span = min(32 - (c & 31), cend - c);
        if (span < 32) word &= (1u << span) - 1u;
        while (word) {
          const int b = __ffs(word) - 1;
          word &= word - 1;
          const unsigned v = (unsigned)((fast9_score_at(im, r, c + b, th) / 16) & 255);
          if (v > vmax) { vmax = v; pr = r; pc = c + b; }
        }
        c += span;
      }
    }
    // one keypoint at most per cell; emitted in CELL raster order.  Unsigned: rows up to 65535 survive the packing, 0xFFFFFFFF = none
    cellkp[i] = vmax > 0 ? (((unsigned)pr << 16) | (unsigned)pc) : 0xFFFFFFFFu;
    if (vmax > 0) atomicAdd(&rowcount[(int)(i / cells_c)], 1);
  }
}

// exclusive scan of the per-row counts; single CTA. rowoff[nrows] = total.
__global__ void __launch_bounds__(1024) k_fast9_scan(const int* rowcount, int* rowoff, int nrows) {
  __shared__ int warp_sums[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nrows; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < nrows ? rowcount[i] : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, x, o);
      if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      int s = warp_sums[threadIdx.x];
      for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, s, o);
        if (threadIdx.x >= o) s += y;
      }
      warp_sums[threadIdx.x] = s;
    }
    __syncthreads();
    const int warp_prefix = (threadIdx.x >> 5) ? warp_sums[(threadIdx.x >> 5) - 1] : 0;
    const int incl = x + warp_prefix + carry;
    if (i < nrows) rowoff[i] = incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry = incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) rowoff[nrows] = carry;
}

// pass 2: one warp per row walks the bitmask and writes keypoints (and scores) in raster order
__global__ void __launch_bounds__(256) k_fast9_emit(Img im, int th, const uint32_t* bits, int wpr, const int* rowoff, vppb_int2* kps,
                                                   int* scores, int score_div, int capacity) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int nwarps = (int)(((long long)gridDim.x * blockDim.x) >> 5);
  for (int r = warp0; r < im.nrows; r += nwarps) {
    int off = rowoff[r];
    if (rowoff[r + 1] == off) continue;
    for (int w0 = 0; w0 < wpr; w0 += 32) {
      const int wi = w0 + lane;
      uint32_t word = wi < wpr ? bits[(long long)r * wpr + wi] : 0u;
      const int cnt = __popc(word);
      int incl = cnt;
      for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      int pos = off + incl - cnt;
      while (word) {
        const int b = __ffs(word) - 1;
        word &= word - 1;
        if (pos < capacity) {
          const int c = wi * 32 + b;
          kps[pos].r = r;
          kps[pos].c = c;
          if (scores) {
            const int s = fast9_score_at(im, r, c, th);
            scores[pos] = score_div ? ((s / 16) & 255) : s;
          }
        }
        pos++;
      }
      off += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
}

// blockwise emit: one warp per row of cells, keypoints leave in cell raster order (the serial order of fast.hpp:763-790)
__global__ void __launch_bounds__(256) k_fast9_emit_cells(Img im, int th, const unsigned* cellkp, int cells_r, int cells_c, const int* rowoff, vppb_int2* kps,
                                                         int* scores, int capacity) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int nwarps = (int)(((long long)gridDim.x * blockDim.x) >> 5);
  for (int cr = warp0; cr < cells_r; cr += nwarps) {
    int off = rowoff[cr];
    if (rowoff[cr + 1] == off) continue;
    for (int c0 = 0; c0 < cells_c; c0 += 32) {
      const int cc = c0 + lane;
      const unsigned v = cc < cells_c ? cellkp[(long long)cr * cells_c + cc] : 0xFFFFFFFFu;
      const unsigned m = __ballot_sync(0xffffffffu, v != 0xFFFFFFFFu);
      if (v != 0xFFFFFFFFu) {
        const int pos = off + __popc(m & ((1u << lane) - 1u));
        if (pos < capacity) {
          const int r = (int)(v >> 16), c = (int)(v & 0xFFFFu);
          kps[pos].r = r; kps[pos].c = c;
          if (scores) scores[pos] = (fast9_score_at(im, r, c, th) / 16) & 255;
        }
      }
      off += __popc(m);
    }
  }
}

// fast_detector9_blockwise_rank (fast.hpp:801-886) on the raw score image of fast_detector9_maxima2 (fast.hpp:710-740): per block the strict
// 3x3 maxima of the raw scores (0 where nothing was detected) enter a table of maxp slots by the reference's rule - a candidate REPLACES
// the first slot whose score is smaller -, the table is sorted by decreasing score (stable), slot k of a block is rank k.  One thread
// per block; the tables go to cellpts / cellsc (maxp entries per block, (row << 16 | col) and raw score), cellcnt = used slots.
constexpr int FR_MAXP = 16;
__global__ void __launch_bounds__(128) k_fast9_block_rank(Img im, int th, int bs, int maxp, const uint32_t* bits, int wpr, unsigned* cellpts, int* cellsc,
                                                         int* cellcnt, int* rowcount, int cells_r, int cells_c) {
  const long long total = (long long)cells_r * cells_c;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r0 = (int)(i / cells_c) * bs, c0 = (int)(i % cells_c) * bs;
    int pv[FR_MAXP];
    unsigned pp[FR_MAXP];
    for (int k = 0; k < maxp; k++) { pv[k] = 0; pp[k] = 0; }
    for (int r = r0; r < min(r0 + bs, im.nrows); r++) {
      int c = c0;
      const int cend = min(c0 + bs, im.ncols);
      while (c < cend) {
        uint32_t word = bits[(long long)r * wpr + (c >> 5)] >> (c & 31);
        const int span = min(32 - (c & 31), cend - c);
        if (span < 32) word &= (1u << span) - 1u;
        while (word) {
          const int b = __ffs(word) - 1;
          word &= word - 1;
          const int cc = c + b;
          const int v = fast9_score_at(im, r, cc, th);
          if (v <= 0) continue;  // detected on the reference's ring, scored on the true one: the score can be 0 (fast.hpp:839)
          bool is_max = true;
          for (int dr = -1; dr <= 1 && is_max; dr++)
            for (int dc = -1; dc <= 1; dc++) {
              if (dr == 0 && dc == 0) continue;
              const int nv = bit_at(bits, wpr, im.nrows, im.ncols, r + dr, cc + dc) ? fast9_score_at(im, r + dr, cc + dc, th) : 0;
              if (!(v > nv)) { is_max = false; break; }
            }
          if (is_max)
            for (int k = 0; k < maxp; k++)
              if (pv[k] < v) { pv[k] = v; pp[k] = ((unsigned)r << 16) | (unsigned)cc; break; }
        }
        c += span;
      }
    }
    for (int a = 1; a < maxp; a++) {  // std::sort on <= 16 elements == insertion sort: stable
      const int v = pv[a];
      const unsigned q = pp[a];
      int j = a - 1;
      while (j >= 0 && pv[j] < v) { pv[j + 1] = pv[j]; pp[j + 1] = pp[j]; j--; }
      pv[j + 1] = v; pp[j + 1] = q;
    }
    int cnt = 0;
    for (int k = 0; k < maxp; k++) {
      cellpts[i * maxp + k] = pp[k];
      cellsc[i * maxp + k] = pv[k];
      cnt += pv[k] > 0 ? 1 : 0;
    }
    cellcnt[i] = cnt;
    if (cnt) atomicAdd(&rowcount[(int)(i / cells_c)], cnt);
  }
}

// one warp per row of blocks: records (row, col, rank) leave in block raster order, ranks ascending
__global__ void __launch_bounds__(256) k_fast9_emit_rank(const unsigned* cellpts, const int* cellsc, const int* cellcnt, int cells_r, int cells_c, int maxp,
                                                        const int* rowoff, int* kps3, int* scores, int capacity) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int nwarps = (int)(((long long)gridDim.x * blockDim.x) >> 5);
  for (int cr = warp0; cr < cells_r; cr += nwarps) {
    int off = rowoff[cr];
    if (rowoff[cr + 1] == off) continue;
    for (int c0 = 0; c0 < cells_c; c0 += 32) {
      const int cc = c0 + lane;
      const long long cell = (long long)cr * cells_c + cc;
      const int cnt = cc < cells_c ? cellcnt[cell] : 0;
      int incl = cnt;
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      int pos = off + incl - cnt;
      for (int k = 0; k < cnt; k++, pos++)
        if (pos < capacity) {
          const unsigned v = cellpts[cell * maxp + k];
          kps3[3 * pos] = (int)(v >> 16); kps3[3 * pos + 1] = (int)(v & 0xFFFFu); kps3[3 * pos + 2] = k;
          if (scores) scores[pos] = cellsc[cell * maxp + k];
        }
      off += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
}

__global__ void k_fast9_scores(Img im, int th, const vppb_int2* kps, int n, int* scores) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const bool inside = kps[i].r >= 0 && kps[i].r < im.nrows && kps[i].c >= 0 && kps[i].c < im.ncols;  // the ring of an in-frame point stays inside the 3-px border
    scores[i] = inside ? fast9_score_at(im, kps[i].r, kps[i].c, th) : 0;
  }
}

struct FastWs {
  uint32_t* bits_a;
  uint32_t* bits_b;
  int* rowcount;
  int* rowoff;
  int* bandtotal;
  int* count;   // device copy of the keypoint count of the last call
  unsigned* cellkp;
  long long bytes;
};

static FastWs fast_ws_layout(void* base, int nrows, int ncols, int block_size) {
  FastWs w;
  const long long wpr = (ncols + 31) / 32;
  const long long bits_bytes = ((long long)nrows * wpr * 4 + 255) / 256 * 256;
  const long long nboxes = (ncols + FB_INNER - 1) / FB_INNER;
  const long long rows_bytes = (((long long)nrows + 8) * nboxes * 4 + 255) / 256 * 256;  // per (row, box) counts of the band kernel; the other paths use the first nrows + 1
  unsigned char* p = static_cast<unsigned char*>(base);
  w.bits_a = reinterpret_cast<uint32_t*>(p);
  w.bits_b = reinterpret_cast<uint32_t*>(p + bits_bytes);
  w.rowcount = reinterpret_cast<int*>(p + 2 * bits_bytes);
  w.rowoff = reinterpret_cast<int*>(p + 2 * bits_bytes + rows_bytes);
  w.bandtotal = reinterpret_cast<int*>(p + 2 * bits_bytes + 2 * rows_bytes);   // <= nrows / FB_ROWS + 1 entries fit in rows_bytes
  w.count = reinterpret_cast<int*>(p + 2 * bits_bytes + 3 * rows_bytes);
  w.cellkp = reinterpret_cast<unsigned*>(p + 2 * bits_bytes + 3 * rows_bytes + 256);
  // the cell array only exists for the blockwise mode; block_size <= 0 sizes it for the smallest block the library
  // accepts there (1 pixel), so that a workspace sized without knowing the mode is always large enough
  const int bs = block_size > 0 ? block_size : 1;
  const long long cells = (long long)((nrows + bs - 1) / bs) * ((ncols + bs - 1) / bs);
  w.bytes = 2 * bits_bytes + 3 * rows_bytes + 256 + ((cells * 4 + 255) / 256) * 256;
  return w;
}

}  // namespace vppb

using namespace vppb;

// TMA needs the library layout (>= 16 addressable bytes left of column 0, 16-byte aligned rows); FB_MAXW bounds the band bitmask
static bool fast_band_eligible(const vppb_img* img) {
  if (img->align < 16 || ((uintptr_t)img->base % 16) || (img->pitch % 16)) return false;
  long long bs = (long long)img->border * img->elem_bytes;
  if (bs % img->align) bs += img->align - (bs % img->align);
  long long pch = (long long)img->ncols * img->elem_bytes + 2 * bs;
  if (pch % img->align) pch += img->align - (pch % img->align);
  if (pch != img->pitch || bs < 16) return false;
  return img->ncols <= FB_MAXW;
}

struct FastRank { int maxp; int* kps3; };  // fast_detector9_blockwise_rank: a blockwise run that reports up to maxp ranked points per block
static long long fast_rank_bytes(int nrows, int ncols, int block_size, int maxp) {
  const long long cells = (long long)((nrows + block_size - 1) / block_size) * ((ncols + block_size - 1) / block_size);
  return ((cells * (2LL * maxp + 1) * 4 + 255) / 256) * 256;
}

static int fast9_core(const vppb_img* img, int32_t th, const vppb_img* mask, int32_t mode, int32_t block_size, int32_t ring, void* workspace,
                      int64_t workspace_bytes, vppb_int2* kps_out, int32_t* scores_out, int32_t capacity, int32_t* count_dev, int** count_src, void* stream,
                      const char* name, const FastRank* rank = nullptr) {
  VPPB_REQUIRE(img && img->base && workspace, VPPB_E_ARG, "%s: NULL argument", name);
  VPPB_REQUIRE(img->elem_bytes == 1, VPPB_E_ARG, "%s: image must be u8", name);
  // fast.hpp:937-938
  VPPB_REQUIRE(img->border >= 3, VPPB_E_BORDER, "Image need a border of 3px at least for the FAST detector");
  VPPB_REQUIRE(mode >= 0 && mode <= 2 && (ring == 0 || ring == 1), VPPB_E_ARG, "%s: bad mode/ring", name);
  VPPB_REQUIRE(mode != VPPB_FAST_BLOCKWISE || block_size > 0, VPPB_E_ARG, "%s: block_size must be > 0", name);
  VPPB_REQUIRE(capacity == 0 || kps_out || (rank && rank->kps3), VPPB_E_ARG, "%s: NULL keypoint buffer", name);
  const bool has_mask = mask && mask->base;
  if (has_mask)
    VPPB_REQUIRE(mask->elem_bytes == 1 && mask->nrows >= img->nrows && mask->ncols >= img->ncols, VPPB_E_ARG, "%s: mask must be u8 and cover the image", name);
  VPPB_REQUIRE(img->nrows < 65536 && img->ncols < 65536, VPPB_E_ARG, "%s: image larger than 65535 in one dimension", name);
  // the reference ignores block_size outside the blockwise mode: so does the workspace rule
  FastWs ws = fast_ws_layout(workspace, img->nrows, img->ncols, mode == VPPB_FAST_BLOCKWISE && !rank ? block_size : (1 << 30));
  const long long need = ws.bytes + (rank ? fast_rank_bytes(img->nrows, img->ncols, block_size, rank->maxp) : 0);
  VPPB_REQUIRE((uintptr_t)workspace % 256 == 0, VPPB_E_ARG, "%s: workspace not 256-byte aligned", name);
  VPPB_REQUIRE(workspace_bytes >= need, VPPB_E_ARG, "%s: workspace %lld < %lld bytes", name, (long long)workspace_bytes, need);
  cudaStream_t st = as_stream(stream);
  const int wpr = (img->ncols + 31) / 32;
  const long long words = (long long)img->nrows * wpr;
  Img im = view(img);
  Img mk = has_mask ? view(mask) : im;
  const int sms = sm_count();
  int* cnt = count_dev ? count_dev : ws.count;
  *count_src = cnt;
  const int nbands = (img->nrows + FB_ROWS - 1) / FB_ROWS;

  static int force_old = -1;
  if (force_old < 0) {
    const char* e = getenv("VPPB_FAST_IMPL");
    force_old = (e && !strcmp(e, "warp")) ? 1 : 0;
  }
  const bool band_path = fast_band_eligible(img) && !force_old;
  if (band_path) {
    CUtensorMap tmap;
    unsigned char* origin = static_cast<unsigned char*>(img->base) - 3LL * img->pitch - 16;
    const uint64_t width_el = ((uint64_t)img->ncols + 32 + 7) / 8;
    int rc = encode_tensor_map_2d(&tmap, origin, CU_TENSOR_MAP_DATA_TYPE_UINT64, 8, width_el, (uint64_t)img->nrows + 6, (uint64_t)img->pitch, FB_BOXW / 8, FB_INH);
    if (rc) return rc;
    static std::atomic<int> attr_done{0};
    if (!attr_done.load(std::memory_order_acquire)) {
      VPPB_CUDA(cudaFuncSetAttribute(k_fast9_band<0, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, FB_SMEM));
      VPPB_CUDA(cudaFuncSetAttribute(k_fast9_band<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, FB_SMEM));
      VPPB_CUDA(cudaFuncSetAttribute(k_fast9_band<0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, FB_SMEM));
      VPPB_CUDA(cudaFuncSetAttribute(k_fast9_band<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, FB_SMEM));
      attr_done.store(1, std::memory_order_release);
    }
    const int nboxes = (img->ncols + FB_INNER - 1) / FB_INNER;
    const int grid = nbands * nboxes;
    if (ring == 0 && !has_mask) k_fast9_band<0, false><<<grid, FB_THREADS, FB_SMEM, st>>>(tmap, im, mk, th, nboxes, wpr, ws.bits_a, ws.rowcount, ws.bandtotal);
    else if (ring == 0) k_fast9_band<0, true><<<grid, FB_THREADS, FB_SMEM, st>>>(tmap, im, mk, th, nboxes, wpr, ws.bits_a, ws.rowcount, ws.bandtotal);
    else if (!has_mask) k_fast9_band<1, false><<<grid, FB_THREADS, FB_SMEM, st>>>(tmap, im, mk, th, nboxes, wpr, ws.bits_a, ws.rowcount, ws.bandtotal);
    else k_fast9_band<1, true><<<grid, FB_THREADS, FB_SMEM, st>>>(tmap, im, mk, th, nboxes, wpr, ws.bits_a, ws.rowcount, ws.bandtotal);
    if (mode == VPPB_FAST_ALL) {
      VPPB_CUDA(launch_dependent(k_fast9_emit_bands, (img->nrows + FE_ROWS - 1) / FE_ROWS, FB_THREADS, 0, st, im, th, (const uint32_t*)ws.bits_a, wpr, (const int*)ws.rowcount,
                                 (const int*)ws.bandtotal, nbands, nboxes, kps_out, (int*)scores_out, 0, (int)capacity, cnt));
      VPPB_LAUNCH_CHECK(name);
      return VPPB_OK;
    }
  } else {
    VPPB_CUDA(cudaMemsetAsync(ws.rowcount, 0, ((size_t)img->nrows + 1) * sizeof(int), st));
    long long blocks = (words + 7) / 8;  // 8 warps per CTA
    int grid = (int)(blocks < (long long)sms * 8 ? blocks : (long long)sms * 8);
    k_fast9_detect<<<grid, 256, 0, st>>>(im, mk, has_mask ? 1 : 0, th, ring, ws.bits_a, wpr, ws.rowcount);
  }
  const uint32_t* final_bits = ws.bits_a;
  if (mode != VPPB_FAST_ALL) {
    VPPB_CUDA(cudaMemsetAsync(ws.rowcount, 0, ((size_t)img->nrows + 1) * sizeof(int), st));
    if (mode == VPPB_FAST_LOCAL_MAXIMA) {
      long long blocks = (words + 7) / 8;
      int grid = (int)(blocks < (long long)sms * 8 ? blocks : (long long)sms * 8);
      k_fast9_local_max<<<grid, 256, 0, st>>>(im, th, ws.bits_a, ws.bits_b, wpr, ws.rowcount);
    } else {
      const int cells_r = (img->nrows + block_size - 1) / block_size, cells_c = (img->ncols + block_size - 1) / block_size;
      long long cells = (long long)cells_r * cells_c;
      long long blocks = (cells + 127) / 128;
      int grid = (int)(blocks < (long long)sms * 16 ? blocks : (long long)sms * 16);
      if (rank) {
        unsigned* cellpts = reinterpret_cast<unsigned*>(static_cast<unsigned char*>(workspace) + ws.bytes);
        int* cellsc = reinterpret_cast<int*>(cellpts + cells * rank->maxp);
        int* cellcnt = cellsc + cells * rank->maxp;
        k_fast9_block_rank<<<grid, 128, 0, st>>>(im, th, block_size, rank->maxp, ws.bits_a, wpr, cellpts, cellsc, cellcnt, ws.rowcount, cells_r, cells_c);
        k_fast9_scan<<<1, 1024, 0, st>>>(ws.rowcount, ws.rowoff, cells_r);
        long long eb = ((long long)cells_r + 7) / 8;
        k_fast9_emit_rank<<<(int)(eb < (long long)sms * 8 ? eb : (long long)sms * 8), 256, 0, st>>>(cellpts, cellsc, cellcnt, cells_r, cells_c, rank->maxp, ws.rowoff,
                                                                                                  rank->kps3, scores_out, capacity);
        VPPB_LAUNCH_CHECK(name);
        *count_src = ws.rowoff + cells_r;
        if (count_dev) VPPB_CUDA(cudaMemcpyAsync(count_dev, ws.rowoff + cells_r, sizeof(int), cudaMemcpyDeviceToDevice, st));
        return VPPB_OK;
      }
      k_fast9_block_max<<<grid, 128, 0, st>>>(im, th, block_size, ws.bits_a, ws.cellkp, wpr, ws.rowcount, cells_r, cells_c);
      k_fast9_scan<<<1, 1024, 0, st>>>(ws.rowcount, ws.rowoff, cells_r);
      long long eb = ((long long)cells_r + 7) / 8;
      k_fast9_emit_cells<<<(int)(eb < (long long)sms * 8 ? eb : (long long)sms * 8), 256, 0, st>>>(im, th, ws.cellkp, cells_r, cells_c, ws.rowoff, kps_out, scores_out,
                                                                                                 capacity);
      VPPB_LAUNCH_CHECK(name);
      *count_src = ws.rowoff + cells_r;
      if (count_dev) VPPB_CUDA(cudaMemcpyAsync(count_dev, ws.rowoff + cells_r, sizeof(int), cudaMemcpyDeviceToDevice, st));
      return VPPB_OK;
    }
    final_bits = ws.bits_b;
  }
  k_fast9_scan<<<1, 1024, 0, st>>>(ws.rowcount, ws.rowoff, img->nrows);
  {
    long long blocks = ((long long)img->nrows + 7) / 8;
    int grid = (int)(blocks < (long long)sms * 8 ? blocks : (long long)sms * 8);
    k_fast9_emit<<<grid, 256, 0, st>>>(im, th, final_bits, wpr, ws.rowoff, kps_out, scores_out, mode != VPPB_FAST_ALL ? 1 : 0, capacity);
  }
  VPPB_LAUNCH_CHECK(name);
  *count_src = ws.rowoff + img->nrows;
  if (count_dev) VPPB_CUDA(cudaMemcpyAsync(count_dev, ws.rowoff + img->nrows, sizeof(int), cudaMemcpyDeviceToDevice, st));
  return VPPB_OK;
}

extern "C" {

int64_t vppb_fast9_workspace_bytes(int32_t nrows, int32_t ncols, int32_t block_size) {
  if (nrows <= 0 || ncols <= 0) return 0;
  return fast_ws_layout(nullptr, nrows, ncols, block_size).bytes;
}

int vppb_fast9_u8(const vppb_img* img, int32_t th, const vppb_img* mask, int32_t mode, int32_t block_size, int32_t ring,
                  void* workspace, int64_t workspace_bytes, vppb_int2* kps_out, int32_t* scores_out, int32_t capacity,
                  int32_t* count_out, void* stream) {
  VPPB_REQUIRE(count_out, VPPB_E_ARG, "vppb_fast9_u8: NULL argument");
  int* src = nullptr;
  int rc = fast9_core(img, th, mask, mode, block_size, ring, workspace, workspace_bytes, kps_out, scores_out, capacity, nullptr, &src, stream, "vppb_fast9_u8");
  if (rc) return rc;
  int total = 0;
  VPPB_CUDA(cudaMemcpyAsync(&total, src, sizeof(int), cudaMemcpyDeviceToHost, as_stream(stream)));
  VPPB_CUDA(cudaStreamSynchronize(as_stream(stream)));
  *count_out = total;
  VPPB_REQUIRE(total <= capacity, VPPB_E_CAPACITY, "vppb_fast9_u8: %d keypoints exceed the capacity %d", total, capacity);
  return VPPB_OK;
}

int vppb_fast9_u8_async(const vppb_img* img, int32_t th, const vppb_img* mask, int32_t mode, int32_t block_size, int32_t ring,
                        void* workspace, int64_t workspace_bytes, vppb_int2* kps_out, int32_t* scores_out, int32_t capacity,
                        int32_t* count_dev, void* stream) {
  VPPB_REQUIRE(count_dev, VPPB_E_ARG, "vppb_fast9_u8_async: NULL argument");
  int* src = nullptr;
  return fast9_core(img, th, mask, mode, block_size, ring, workspace, workspace_bytes, kps_out, scores_out, capacity, count_dev, &src, stream, "vppb_fast9_u8_async");
}

int64_t vppb_fast9_rank_workspace_bytes(int32_t nrows, int32_t ncols, int32_t block_size, int32_t max_points) {
  if (nrows <= 0 || ncols <= 0 || block_size <= 0 || max_points < 1 || max_points > FR_MAXP) return 0;
  return fast_ws_layout(nullptr, nrows, ncols, 1 << 30).bytes + fast_rank_bytes(nrows, ncols, block_size, max_points);
}

int vppb_fast9_blockwise_rank_u8(const vppb_img* img, int32_t th, const vppb_img* mask, int32_t block_size, int32_t max_points, int32_t ring,
                                 void* workspace, int64_t workspace_bytes, int32_t* kps3_out, int32_t* scores_out, int32_t capacity, int32_t* count_out,
                                 void* stream) {
  VPPB_REQUIRE(count_out, VPPB_E_ARG, "vppb_fast9_blockwise_rank_u8: NULL argument");
  VPPB_REQUIRE(max_points >= 1 && max_points <= FR_MAXP && block_size > 0, VPPB_E_ARG, "vppb_fast9_blockwise_rank_u8: 1 <= max_points <= %d, block_size > 0", FR_MAXP);
  FastRank rk{max_points, kps3_out};
  int* src = nullptr;
  int rc = fast9_core(img, th, mask, VPPB_FAST_BLOCKWISE, block_size, ring, workspace, workspace_bytes, nullptr, scores_out, capacity, nullptr, &src, stream,
                      "vppb_fast9_blockwise_rank_u8", &rk);
  if (rc) return rc;
  int total = 0;
  VPPB_CUDA(cudaMemcpyAsync(&total, src, sizeof(int), cudaMemcpyDeviceToHost, as_stream(stream)));
  VPPB_CUDA(cudaStreamSynchronize(as_stream(stream)));
  *count_out = total;
  VPPB_REQUIRE(total <= capacity, VPPB_E_CAPACITY, "vppb_fast9_blockwise_rank_u8: %d records exceed the capacity %d", total, capacity);
  return VPPB_OK;
}

int vppb_fast9_scores(const vppb_img* img, int32_t th, const vppb_int2* kps, int32_t n, int32_t* scores_out, void* stream) {
  VPPB_REQUIRE(img && img->base && (n == 0 || (kps && scores_out)), VPPB_E_ARG, "vppb_fast9_scores: NULL argument");
  VPPB_REQUIRE(img->elem_bytes == 1, VPPB_E_ARG, "vppb_fast9_scores: image must be u8");
  VPPB_REQUIRE(img->border >= 3, VPPB_E_BORDER, "vppb_fast9_scores: border %d < 3", img->border);
  if (n == 0) return VPPB_OK;
  int grid = (n + 255) / 256;
  k_fast9_scores<<<grid, 256, 0, as_stream(stream)>>>(view(img), th, kps, n, scores_out);
  VPPB_LAUNCH_CHECK("vppb_fast9_scores");
  return VPPB_OK;
}

}  // extern "C"
