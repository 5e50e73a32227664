// 5x5 box stencil:  out = (sum of the 25 neighbours) / 25, per channel, integer division.
// Reference: the relative_access / box_nbh2d user kernels of benchmarks/box_5x5_filter2.cc:71-81
// (image2d<int>) and examples/box_filter.cc:23-32 (image2d<vuchar3>, vint3 accumulator).
//
// Byte images (u8, vuchar3) run as byte streams: a vuchar3 row is 3*ncols bytes and the
// horizontal taps sit CS = 3 bytes apart.  Tiles are staged in shared memory by TMA
// (cp.async.bulk.tensor.2d + mbarrier); see k_box5_bytes_tma below for the two-phase scheme.
#include "common.cuh"

#include <algorithm>
#include <atomic>
#include "tma.cuh"

namespace vppb {

// ------------------------------------------------------------------ tensor map encoding
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode_tensor_map_2d(CUtensorMap* map, void* origin, CUtensorMapDataType elem, int elem_bytes, uint64_t width,
                         uint64_t height, uint64_t pitch, uint32_t box_w, uint32_t box_h) {
  static std::atomic<PFN_tmapEncodeTiled> cached{nullptr};
  PFN_tmapEncodeTiled fn = cached.load(std::memory_order_acquire);
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
      set_error("cuTensorMapEncodeTiled entry point unavailable (%d)", (int)e);
      return VPPB_E_CUDA;
    }
    fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
    cached.store(fn, std::memory_order_release);
  }
  (void)elem_bytes;
  cuuint64_t gdim[2] = {width, height};
  cuuint64_t gstr[1] = {pitch};
  cuuint32_t box[2] = {box_w, box_h};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, elem, 2, origin, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): origin %p w %llu h %llu pitch %llu box %ux%u", (int)r, origin,
              (unsigned long long)width, (unsigned long long)height, (unsigned long long)pitch, box_w, box_h);
    return VPPB_E_CUDA;
  }
  return VPPB_OK;
}

// ------------------------------------------------------------------ direct kernels (any layout)
// One thread per output element; used for images the TMA path cannot describe (unaligned
// external buffers) and as the int32 path.  T = element, CS = tap stride in elements.
template <typename T, typename ACC, int CS>
__global__ void k_box5_direct(Img in, Img out, int row_elems) {
  long long total = (long long)out.nrows * row_elems;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int r = (int)(i / row_elems);
    int x = (int)(i - (long long)r * row_elems);
    ACC s = 0;
#pragma unroll
    for (int dy = -2; dy <= 2; dy++) {
      const T* p = row_ptr<T>(in, r + dy) + x;
#pragma unroll
      for (int dx = -2; dx <= 2; dx++) s += (ACC)p[dx * CS];
    }
    row_ptr<T>(out, r)[x] = (T)(s / 25);
  }
}

// ------------------------------------------------------------------ TMA tile kernel (bytes)
// One CTA per tile of 992 x 16 output bytes.  Thread 0 issues ONE TMA load of the 1024-byte x
// 20-row input box (16 bytes of halo-and-alignment left and right, 2 rows above/below) and the
// whole CTA waits on its mbarrier.
//   phase 1 (vertical): thread = (16-byte column group, 8 output rows).  Bytes are split into
//     packed 16-bit lanes E = (b0,b2), O = (b1,b3) of each word and the 5-row column sums are kept
//     as a running window in registers (ring of 5 rows), written to shared memory as u16 pairs.
//   phase 2 (horizontal + divide): thread = (row, 16-byte output group).  The 5 taps CS bytes
//     apart are whole or word-straddling lane pairs of the column sums (one PRMT each), summed
//     with IADD3, divided by 25 with an exact multiply-shift and packed back to bytes.
// 4 CTAs (16 warps) are resident per SM; every input byte is fetched once per tile (+25 % halo
// rows, served by L2).  HBM-bound: 2 bytes of traffic per output byte.
constexpr int BX_BOXW = 1024;           // bytes per box row (64 column groups of 16 bytes)
constexpr int BX_OUTW = 992;            // output bytes per tile row (62 groups)
constexpr int BX_THREADS = 128;
constexpr int BX_CS_ROW_WORDS = BX_BOXW / 4;              // 256 words per plane per row
// TH = output rows per tile (16: 4 CTAs/SM, +25 % halo rows; 8: 8 CTAs/SM, +50 % halo rows)
template <int TH> struct BoxCfg {
  static constexpr int INH = TH + 4;                          // input rows per tile
  static constexpr int RAW_BYTES = INH * BX_BOXW;
  static constexpr int CS_BYTES = TH * 2 * BX_CS_ROW_WORDS * 4;  // E and O planes
  static constexpr int SMEM = RAW_BYTES + CS_BYTES + 16;
};
constexpr unsigned BX_DIV25 = 671089u;  // floor(s/25) == (s * 671089) >> 24 for 0 <= s <= 6375 (checked exhaustively)

// a + b (and a - b) on the FMA pipe: with a runtime multiplier ptxas must keep the IMAD, which moves the
// packed-lane additions off the half-rate ALU pipe (PRMT/LOP3/IADD3/SHF) that bounds this kernel.
__device__ __forceinline__ uint32_t fadd_u32(uint32_t a, uint32_t mul, uint32_t b) { return a * mul + b; }  // mul = +1 / -1 at run time

// floor(lane / 25) of both 16-bit lanes of se (lanes x, x+2) and so (lanes x+1, x+3), packed to 4 bytes.
// lo lanes: (v * 671089) >> 24.  hi lanes: mulhi(se, 671089) = (hi*M + ((lo*M) >> 16)) >> 16, whose byte 1 is
// floor(hi/25): the carry-in (< 2^16) is far below the slack of the magic number (exhaustively checked in
// tests/test_abi.py::test_box_division_magic).
__device__ __forceinline__ uint32_t box_div_pack(uint32_t se, uint32_t so) {
  const uint32_t pel = (se & 0xFFFFu) * BX_DIV25, pol = (so & 0xFFFFu) * BX_DIV25;
  const uint32_t peh = __umulhi(se, BX_DIV25), poh = __umulhi(so, BX_DIV25);
  const uint32_t lo = __byte_perm(pel, pol, 0x0073);  // (q(x), q(x+1)): byte 3 of the products
  const uint32_t hi = __byte_perm(peh, poh, 0x0051);  // (q(x+2), q(x+3)): byte 1 of the high products
  return __byte_perm(lo, hi, 0x5410);
}

// ---------------- phase 1 of a tile: 5-row column sums of the raw box -> E / O planes in shared memory
template <int BX_TH>
__device__ __forceinline__ void box_phase1(const unsigned char* raw, uint32_t* csE, uint32_t* csO, int tid, uint32_t minus_one) {
  constexpr int RG_ROWS = BX_TH / 2;  // output rows per phase-1 row group
  const int cg = tid & 63, rg = tid >> 6;
  const unsigned char* col = raw + (rg * RG_ROWS) * BX_BOXW + cg * 16;
  uint32_t ringE[5][4], ringO[5][4], VE[4], VO[4];
#pragma unroll
  for (int q = 0; q < 4; q++) { VE[q] = 0; VO[q] = 0; }
#pragma unroll
  for (int j = 0; j < RG_ROWS + 4; j++) {
    const uint4 v = *reinterpret_cast<const uint4*>(col + j * BX_BOXW);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    const int slot = j % 5;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const uint32_t e = w[q] & 0x00FF00FFu, o = __byte_perm(w[q], 0u, 0x4341);
      if (j >= 5) {
        VE[q] = fadd_u32(ringE[slot][q], minus_one, VE[q] + e);   // V += e - old  (one IADD3 + one IMAD)
        VO[q] = fadd_u32(ringO[slot][q], minus_one, VO[q] + o);
      } else { VE[q] += e; VO[q] += o; }
      ringE[slot][q] = e;
      ringO[slot][q] = o;
    }
    if (j >= 4) {
      const int orow = rg * RG_ROWS + j - 4;
      *reinterpret_cast<uint4*>(csE + orow * BX_CS_ROW_WORDS + cg * 4) = make_uint4(VE[0], VE[1], VE[2], VE[3]);
      *reinterpret_cast<uint4*>(csO + orow * BX_CS_ROW_WORDS + cg * 4) = make_uint4(VO[0], VO[1], VO[2], VO[3]);
    }
  }
}

// ---------------- phase 2 of a tile: horizontal taps, divide, store (out_base / out_pitch: the image the tile belongs to)
template <int CS, int BX_TH>
__device__ __forceinline__ void box_phase2(const uint32_t* csE, const uint32_t* csO, unsigned char* out_base, long long out_pitch, int out_nrows,
                                           int rowbytes, int x0, int y0, int vec_store, int tid, uint32_t one) {
  const int rows_here = min(BX_TH, out_nrows - y0);
  for (int u = tid; u < BX_TH * 62; u += BX_THREADS) {
    const int row = u / 62, og = u - row * 62;
    const int x = x0 + og * 16;
    if (row >= rows_here || x >= rowbytes) continue;
    // own words are box words 4og+4 .. 4og+7 (the box starts 16 bytes left of x0); window = words k-2 .. k+5
    const uint32_t* pe = csE + row * BX_CS_ROW_WORDS + og * 4 + 2;
    const uint32_t* po = csO + row * BX_CS_ROW_WORDS + og * 4 + 2;
    const uint2 e0 = *reinterpret_cast<const uint2*>(pe), e2 = *reinterpret_cast<const uint2*>(pe + 6);
    const uint4 e1 = *reinterpret_cast<const uint4*>(pe + 2);
    const uint2 o0 = *reinterpret_cast<const uint2*>(po), o2 = *reinterpret_cast<const uint2*>(po + 6);
    const uint4 o1 = *reinterpret_cast<const uint4*>(po + 2);
    const uint32_t E[8] = {e0.x, e0.y, e1.x, e1.y, e1.z, e1.w, e2.x, e2.y};
    const uint32_t O[8] = {o0.x, o0.y, o1.x, o1.y, o1.z, o1.w, o2.x, o2.y};
    uint32_t SE[7], SO[7];
#pragma unroll
    for (int i = 0; i < 7; i++) {
      SE[i] = __byte_perm(E[i], E[i + 1], 0x5432);  // lanes (byte2 of word i, byte0 of word i+1)
      SO[i] = __byte_perm(O[i], O[i + 1], 0x5432);  // lanes (byte3 of word i, byte1 of word i+1)
    }
    uint32_t ow[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int i = j + 2;
      uint32_t he, ho;
      if (CS == 3) {
        // lanes (x, x+2): taps x-6, x-3, x, x+3, x+6 ; lanes (x+1, x+3) likewise.  3 terms on the ALU (IADD3), 2 on the FMA pipe.
        he = fadd_u32(SE[i + 1], one, fadd_u32(SO[i], one, SE[i - 2] + O[i - 1] + E[i]));
        ho = fadd_u32(SO[i + 1], one, fadd_u32(E[i + 1], one, SO[i - 2] + SE[i - 1] + O[i]));
      } else {
        he = fadd_u32(SE[i], one, fadd_u32(O[i], one, SE[i - 1] + SO[i - 1] + E[i]));  // CS == 1: taps x-2 .. x+2
        ho = fadd_u32(SO[i], one, fadd_u32(SE[i], one, SO[i - 1] + E[i] + O[i]));
      }
      ow[j] = box_div_pack(he, ho);
    }
    unsigned char* dst = out_base + (long long)(y0 + row) * out_pitch + x;
    if (vec_store && x + 16 <= rowbytes) {
      *reinterpret_cast<uint4*>(dst) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
    } else {
      for (int k = 0; k < 16; k++)
        if (x + k < rowbytes) dst[k] = (unsigned char)(ow[k >> 2] >> ((k & 3) * 8));
    }
  }
}

// Persistent: each CTA walks tiles blockIdx.x, blockIdx.x + gridDim.x, ...; the TMA load of the NEXT tile is
// issued right after phase 1 (the raw box is dead once the column sums are in shared memory), so its
// latency hides behind phase 2.
template <int CS, int BX_TH>
__global__ void __launch_bounds__(BX_THREADS, BX_TH == 16 ? 4 : 6) k_box5_bytes_tma(const __grid_constant__ CUtensorMap tmap, Img out, int rowbytes, int strips,
                                                                 int ntiles, int vec_store, uint32_t one) {
  constexpr int BX_RAW_BYTES = BoxCfg<BX_TH>::RAW_BYTES, BX_CS_BYTES = BoxCfg<BX_TH>::CS_BYTES;
  extern __shared__ __align__(128) unsigned char smem[];
  unsigned char* raw = smem;
  uint32_t* csE = reinterpret_cast<uint32_t*>(smem + BX_RAW_BYTES);
  uint32_t* csO = csE + BX_TH * BX_CS_ROW_WORDS;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + BX_RAW_BYTES + BX_CS_BYTES);
  const int tid = threadIdx.x;
  const uint32_t minus_one = 0u - one;
  grid_launch_dependents();
  if (tid == 0) mbar_init(bar, 1);
  grid_dependency_wait();  // launched programmatically behind the previous kernel of the stream

  if (tid == 0) {
    fence_barrier_init();
    mbar_arrive_expect_tx(bar, BX_RAW_BYTES);
    // tensor origin = 16 bytes left of x = 0, 2 rows above y = 0; elements are 8 bytes; the box starts at
    // x0 - 16.  (The innermost box coordinate times the element size is kept a multiple of 16 bytes: a conservative
    // rule the emulator enforces (tests/emu/tma.cuh), not a documented TMA limit, and not probed on an H100.)
    tma_load_2d(raw, &tmap, (blockIdx.x % strips) * (BX_OUTW / 8), (blockIdx.x / strips) * BX_TH, bar);
  }
  __syncthreads();  // barrier init visible to the waiters
  uint32_t parity = 0;

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int x0 = (tile % strips) * BX_OUTW, y0 = (tile / strips) * BX_TH;
    mbar_wait(bar, parity);
    parity ^= 1;
    box_phase1<BX_TH>(raw, csE, csO, tid, minus_one);
    __syncthreads();
    // the raw box is dead: prefetch the next tile of this CTA behind phase 2
    if (tid == 0 && tile + (int)gridDim.x < ntiles) {
      const int nt = tile + gridDim.x;
      mbar_arrive_expect_tx(bar, BX_RAW_BYTES);
      tma_load_2d(raw, &tmap, (nt % strips) * (BX_OUTW / 8), (nt / strips) * BX_TH, bar);
    }
    box_phase2<CS, BX_TH>(csE, csO, out.base, out.pitch, out.nrows, rowbytes, x0, y0, vec_store, tid, one);
    __syncthreads();  // column sums consumed before the next tile's phase 1 overwrites them
  }
}

// ------------------------------------------------------------------ streaming kernel (bytes)
// A task is a band of R output rows of one image across S adjacent strips of its rows (a whole 1080p vuchar3 row; a 4K row is two
// bands wide, an 8K row four), so a CTA streams nearly contiguous memory: the library pads a 1080p row of 5760 bytes to a 6016-byte
// pitch.  A strip is G <= 126 16-byte output groups, one per lane of a group of BS_CWARPS consumer warps; a row is cut into strips as
// equal as whole groups allow (1080p, 4K and 8K vuchar3 rows are 3, 6 and 12 strips of 120 groups), and into bands of as equal
// strip counts, at most BS_MAX_S.  The CTA is S groups of consumer warps and one producer warp.  Lane 0 of the producer walks the
// CTA's tasks and keeps a ring of stages in flight; a stage is S TMA boxes (one per strip: 16 bytes left + 16 G + 16 right by
// BS_K = 5 rows) on one "full" mbarrier, and an "empty" mbarrier takes one arrival per consumer warp done reading it.  Nothing in
// the loop waits on a CTA-wide barrier, and the pipeline runs on from one task of the CTA into the next.  Per input row a consumer
// lane
//   loads its window from its strip's box (LDS.64 + LDS.128 + LDS.64: bytes x-8 .. x+23),
//   splits the words into packed 16-bit lanes E = (b0,b2), O = (b1,b3) and forms the 5 horizontal taps CS bytes apart
//     (whole or word-straddling lane pairs, one PRMT each)  ->  H = horizontal 5-sum of the raw row, 8 registers,
//   slides the vertical window in registers: S += H - H(5 rows ago)  (ring of 5 rows, statically indexed because a
//     stage is exactly 5 rows),
//   and for every completed window divides by 25 (exact multiply-shift) and stores its 16 bytes as one 16-byte store.
// Horizontal-first means the only data exchanged between lanes is the raw halo, which TMA already put in shared memory.
constexpr int BS_K = 5;            // rows per stage == rows of the vertical window
constexpr int BS_MAX_BATCH = 128;  // images per launch (their tensor maps travel in the 32 KB kernel parameter space)
constexpr int BS_CWARPS = 4;       // consumer warps per strip; one more warp per CTA produces
constexpr int BS_MAX_S = 3;        // strips per band: 3 x 4 consumer warps + the producer = 416 threads
constexpr int BS_MAX_THREADS = 32 * (BS_CWARPS * BS_MAX_S + 1);
constexpr int BS_MAX_G = 126;      // 16-byte groups per strip: a box row of 16 G + 32 bytes stays within TMA's 256 8-byte elements
constexpr int BS_BOX_BYTES = BS_K * 2048;  // one strip's box of a stage; a multiple of 128 (TMA destination alignment)
// per band width S = 1, 2, 3: CTAs resident per SM (registers: <= 96 per thread, -Xptxas -v) and stages in each CTA's ring, so that
// the rings fill about the same 180 - 200 KB of the H100's 228 KB of shared memory per SM
constexpr int BS_CTAS_PER_SM[BS_MAX_S + 1] = {0, 3, 2, 1};
constexpr int BS_STAGES[BS_MAX_S + 1] = {0, 6, 5, 6};
inline int bs_smem(int S) { return BS_STAGES[S] * S * BS_BOX_BYTES + 2 * BS_STAGES[S] * 8; }

template <int NB>
struct BoxStream {
  CUtensorMap maps[NB];
  unsigned char* out_base[NB];
  // row tiles (multi-GPU): pixel (0,0) of the tile itself and of the tiles above / below it (NULL: none, the tile's own
  // border rows are the halo).  The neighbours' memory may be a peer GPU's, mapped into this process.
  const unsigned char* in_base[NB];
  const unsigned char* up_base[NB];
  const unsigned char* dn_base[NB];
  int nimg, out_pitch, nrows, rowbytes, strips, G, boxw, chunks, R, groups, vec_store, total;
  int S, bands, stages;     // strips per band, bands per row, stages in the ring
  int in_pitch, row_room;   // row_room: addressable bytes of a row from pixel (0,0) to the end of its pitch
};

// A stage that straddles a row-tile seam: row by row for each strip of the band, each row from the tile that owns it - the halo
// rows come straight from the neighbour's (peer GPU's) memory as 1-D bulk copies, so the transfer is part of the kernel's own load
// pipeline.
template <int NB>
__device__ __noinline__ void box_stage_from_tiles(const BoxStream<NB>& p, unsigned char* stage, uint64_t* bar, int img, int strip0, int nstrips, int ty) {
  const unsigned char* up = p.up_base[img];
  const unsigned char* dn = p.dn_base[img];
  int rows = 0, bytes = 0;
  for (int i = 0; i < BS_K; i++) rows += (ty + i - 2 <= p.nrows + 1) ? 1 : 0;
  for (int s = 0; s < nstrips; s++) bytes += rows * min(p.boxw, p.row_room - ((strip0 + s) * 16 * p.G - 16));
  mbar_arrive_expect_tx(bar, bytes);
  for (int s = 0; s < nstrips; s++) {
    const int xoff = (strip0 + s) * 16 * p.G - 16;
    const int len = min(p.boxw, p.row_room - xoff);
    for (int i = 0; i < BS_K; i++) {
      const int v = ty + i - 2;  // image row of the tile
      if (v > p.nrows + 1) continue;
      const unsigned char* src = (v < 0 && up) ? up + (long long)(p.nrows + v) * p.in_pitch
                               : (v >= p.nrows && dn) ? dn + (long long)(v - p.nrows) * p.in_pitch
                                                      : p.in_base[img] + (long long)v * p.in_pitch;
      tma_load_1d(stage + s * BS_BOX_BYTES + i * p.boxw, src + xoff, len, bar);
    }
  }
}

// Ablations for tools/box_bench.py and tools/box_ceiling.py (VPPB_BOX_ABLATE; their outputs are NOT the box filter):
//   BOX_COPY:    the same tasks, TMA boxes and stores, the arithmetic replaced by storing each staged row's own bytes;
//   BOX_COMPUTE: the first ring of stages is fetched once and then re-read for every later stage (no new TMA), and the
//                results are folded into one word per lane and task instead of being stored row by row.
enum { BOX_FILTER = 0, BOX_COPY = 1, BOX_COMPUTE = 2 };

template <int CS, int NB, int MODE = BOX_FILTER>
__global__ void __launch_bounds__(BS_MAX_THREADS, 1) k_box5_stream(const __grid_constant__ BoxStream<NB> p) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int stage_bytes = p.S * BS_BOX_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.stages * stage_bytes);
  uint64_t* empty = full + p.stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per_img = p.bands * p.chunks;

  grid_launch_dependents();  // the next kernel of the stream may be scheduled while this one drains (it waits before it reads)
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; s++) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], BS_CWARPS * p.S);
    }
    fence_barrier_init();
  }
  __syncthreads();           // barrier init visible to every warp
  grid_dependency_wait();    // launched programmatically: everything above overlapped the previous kernel's tail; its writes are visible now

  if (warp == BS_CWARPS * p.S) {
    // producer: a task is decoded once (two divisions), a stage costs a handful of instructions per strip; only stages that
    // straddle a row-tile seam take the (out-of-line) row-by-row path
    if (lane != 0) return;
    int slot = 0;
    uint32_t round = 0;  // completed passes over the ring
    for (int task = blockIdx.x; task < p.total; task += gridDim.x) {
      const int img = task / per_img, rem = task - img * per_img;
      const int chunk = rem / p.bands, band = rem - chunk * p.bands;
      const int strip0 = band * p.S, nstrips = min(p.S, p.strips - strip0);
      int y = chunk * p.R;  // the stage is rows [y, y + 5) of the tensor map = image rows y - 2 .. y + 2
      const bool seam = (p.up_base[img] && y < 2) || (p.dn_base[img] && y + p.groups * BS_K > p.nrows + 2);
      for (int g = 0; g < p.groups; g++, y += BS_K) {
        if (round > 0) mbar_wait(&empty[slot], (round - 1) & 1);  // every consumer warp is done with the slot's previous stage
        unsigned char* stage = smem + slot * stage_bytes;
        if (MODE == BOX_COMPUTE && round > 0)
          mbar_arrive(&full[slot]);
        else if (seam && ((p.up_base[img] && y < 2) || (p.dn_base[img] && y + BS_K > p.nrows + 2)))
          box_stage_from_tiles<NB>(p, stage, &full[slot], img, strip0, nstrips, y);
        else {
          mbar_arrive_expect_tx(&full[slot], nstrips * BS_K * p.boxw);
          // tensor origin = 16 bytes left of x = 0 and 2 rows above y = 0; 8-byte elements (x coordinate * 8 is a multiple of 16)
          for (int s = 0; s < nstrips; s++) tma_load_2d(stage + s * BS_BOX_BYTES, &p.maps[img], (strip0 + s) * 2 * p.G, y, &full[slot]);
        }
        if (++slot == p.stages) { slot = 0; round++; }
      }
    }
    return;
  }

  const int sg = warp / BS_CWARPS;                        // this warp's strip of the band
  const int cl = (warp - sg * BS_CWARPS) * 32 + lane;     // this lane's 16-byte group of the strip
  const int cr = min(cl, p.G - 1);   // lanes right of the strip read the last group's window and store nothing
  int slot = 0;
  uint32_t parity = 0;
  for (int task = blockIdx.x; task < p.total; task += gridDim.x) {
    const int img = task / per_img, rem = task - img * per_img;
    const int chunk = rem / p.bands, band = rem - chunk * p.bands;
    const int strip = band * p.S + sg;  // >= p.strips: a strip group of a narrower last band (reads a stale box, stores nothing)
    const int x = strip * 16 * p.G + 16 * cl;
    const int y0 = chunk * p.R, yend = min(y0 + p.R, p.nrows);
    const int nbytes = cl < p.G ? min(16, p.rowbytes - x) : 0;  // <= 0: nothing of this lane's group is in the image
    const bool vec = nbytes == 16 && p.vec_store;
    unsigned char* const dst = p.out_base[img] + (long long)y0 * p.out_pitch + x;

    uint32_t rE[BS_K][4], rO[BS_K][4], SE[4], SO[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
      SE[q] = 0; SO[q] = 0;
#pragma unroll
      for (int j = 0; j < BS_K; j++) { rE[j][q] = 0; rO[j][q] = 0; }
    }
    uint32_t acc = 0;

    unsigned char* drow = dst - 5LL * p.out_pitch;  // advanced once per input row: the row its window completes
    for (int g = 0; g < p.groups; g++) {
      mbar_wait(&full[slot], parity);
      const unsigned char* st = smem + slot * stage_bytes + sg * BS_BOX_BYTES + 16 * cr;
#pragma unroll
      for (int j = 0; j < BS_K; j++) {
        const unsigned char* rp = st + j * p.boxw;
        const uint2 wl = *reinterpret_cast<const uint2*>(rp + 8);
        const uint4 wm = *reinterpret_cast<const uint4*>(rp + 16);
        const uint2 wr = *reinterpret_cast<const uint2*>(rp + 32);
        const uint32_t w[8] = {wl.x, wl.y, wm.x, wm.y, wm.z, wm.w, wr.x, wr.y};  // 2 words left, 4 own, 2 right
        uint32_t E[8], O[8], XE[7], XO[7];
#pragma unroll
        for (int i = 0; i < 8; i++) { E[i] = w[i] & 0x00FF00FFu; O[i] = __byte_perm(w[i], 0u, 0x4341); }
#pragma unroll
        for (int i = 0; i < 7; i++) { XE[i] = __byte_perm(E[i], E[i + 1], 0x5432); XO[i] = __byte_perm(O[i], O[i + 1], 0x5432); }
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int i = q + 2;
          uint32_t he, ho;
          if (CS == 3) {  // lanes (x, x+2): taps x-6, x-3, x, x+3, x+6; lanes (x+1, x+3) likewise
            he = XE[i + 1] + XO[i] + XE[i - 2] + O[i - 1] + E[i];
            ho = XO[i + 1] + E[i + 1] + XO[i - 2] + XE[i - 1] + O[i];
          } else {        // CS == 1: taps x-2 .. x+2
            he = XE[i] + O[i] + XE[i - 1] + XO[i - 1] + E[i];
            ho = XO[i] + XE[i] + XO[i - 1] + E[i] + O[i];
          }
          SE[q] = SE[q] + he - rE[j][q];  // one IADD3 with a negated operand
          SO[q] = SO[q] + ho - rO[j][q];
          rE[j][q] = he;
          rO[j][q] = ho;
        }
        drow += p.out_pitch;
        if (g > 0 || j == BS_K - 1) {  // input rows 0 .. 3 of a task only fill the window
          const int y = y0 + g * BS_K + j - 4;
          if (y < yend && nbytes > 0) {
            uint32_t ow[4];
#pragma unroll
            for (int q = 0; q < 4; q++) ow[q] = MODE == BOX_COPY ? w[2 + q] : box_div_pack(SE[q], SO[q]);
            if (MODE == BOX_COMPUTE) {
              acc ^= ow[0] ^ ow[1] ^ ow[2] ^ ow[3];
            } else if (vec) {  // one 16-byte store (a plain uint4 store of this loop is split into 4-byte stores by NVVM)
              st_stream(reinterpret_cast<int4*>(drow), make_int4((int)ow[0], (int)ow[1], (int)ow[2], (int)ow[3]));
            } else {  // the right edge of the image, or an output without 16-byte alignment: byte stores, statically indexed
#pragma unroll
              for (int k = 0; k < 16; k++)
                if (k < nbytes) drow[k] = (unsigned char)(ow[k >> 2] >> ((k & 3) * 8));
            }
          }
        }
      }
      __syncwarp();  // every lane of the warp is done reading the stage
      if (lane == 0) mbar_arrive(&empty[slot]);
      if (++slot == p.stages) { slot = 0; parity ^= 1; }
    }
    if (MODE == BOX_COMPUTE && vec) *reinterpret_cast<uint32_t*>(dst) = acc;
  }
}

static int layout_pitch(const vppb_img* i) {
  if (i->align <= 0) return -1;
  long long bs = (long long)i->border * i->elem_bytes;
  if (bs % i->align) bs += i->align - (bs % i->align);
  long long p = (long long)i->ncols * i->elem_bytes + 2 * bs;
  if (p % i->align) p += i->align - (p % i->align);
  return (int)p;
}

// TMA needs: library layout (so the bytes left/right of the domain belong to the row),
// 16-byte aligned pixel (0,0) and pitch, border >= 2 with at least 16 bytes of row before column 0.
static bool tma_eligible(const vppb_img* in) {
  if (in->align < 16 || in->border < 2) return false;
  if (((uintptr_t)in->base % 16) || (in->pitch % 16)) return false;
  if (layout_pitch(in) != in->pitch) return false;
  return true;
}

// rows per tile: 16 amortises the 4 halo rows better, 8 gives twice the CTAs (small frames cannot
// fill 132 SMs x 4 CTAs with 16-row tiles).  VPPB_BOX_TH=8|16 overrides for experiments.
static int box_tile_rows(int nrows, int rowbytes) {
  static int forced = -1;
  if (forced < 0) {
    const char* e = getenv("VPPB_BOX_TH");
    forced = e ? atoi(e) : 0;
  }
  if (forced == 8 || forced == 16) return forced;
  const long long tiles16 = (long long)((rowbytes + BX_OUTW - 1) / BX_OUTW) * ((nrows + 15) / 16);
  return tiles16 >= 4LL * sm_count() ? 16 : 8;
}

// Rows per task: R = 5 m - 4 (a task then reads exactly m stages).  Small R = more tasks (parallelism for few frames) but 4 extra
// input rows per task; pick the R with the smallest makespan estimate over the resident CTAs, up to one band height per image
// (1080p x 128: one task per image on the H100's 132 resident CTAs).
static int box_stream_rows(long long bands_x_imgs, int nrows, long long ctas, int* chunks_out) {
  static int forced = -1;
  if (forced < 0) {
    const char* e = getenv("VPPB_BOX_R");
    forced = e ? atoi(e) : 0;
  }
  const int m_max = std::max(4, (nrows + 4 + BS_K - 1) / BS_K);
  int best_r = 16;
  double best = 1e300;
  for (int m = 4; m <= m_max; m++) {
    const int r = 5 * m - 4;
    if (forced > 0 && r != forced) continue;
    const long long chunks = (nrows + r - 1) / r, tasks = chunks * bands_x_imgs;
    const long long waves = (tasks + ctas - 1) / ctas;
    // per task: m stages of 5 rows + ~2 stages of pipeline fill; a wave costs its slowest CTA
    const double cost = (double)waves * (5.0 * m + 2.0);
    if (cost < best) { best = cost; best_r = r; }
  }
  *chunks_out = (nrows + best_r - 1) / best_r;
  return best_r;
}

// n equally shaped, TMA-eligible images (n <= NB) in one launch of the streaming kernel
template <int CS, int NB, int MODE>
static int box5_stream_launch_nb(const vppb_img* ins, const vppb_img* ups, const vppb_img* dns, const vppb_img* outs, int n, cudaStream_t st, const char* name) {
  const int rowbytes = ins[0].ncols * CS, nrows = ins[0].nrows;
  static std::atomic<unsigned long long> attr_done{0};
  int dev = 0;
  VPPB_CUDA(cudaGetDevice(&dev));
  const unsigned long long bit = 1ULL << (dev & 63);
  if (!(attr_done.load(std::memory_order_acquire) & bit)) {
    int most = 0;
    for (int s = 1; s <= BS_MAX_S; s++) most = std::max(most, bs_smem(s));
    VPPB_CUDA(cudaFuncSetAttribute(k_box5_stream<CS, NB, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
    attr_done.fetch_or(bit, std::memory_order_release);
  }
  BoxStream<NB> p;
  memset(&p, 0, sizeof(p));
  p.nimg = n;
  p.out_pitch = outs[0].pitch;
  p.nrows = nrows;
  p.rowbytes = rowbytes;
  const int row_groups = (rowbytes + 15) / 16;
  p.strips = (row_groups + BS_MAX_G - 1) / BS_MAX_G;
  p.G = (row_groups + p.strips - 1) / p.strips;
  p.boxw = 16 * p.G + 32;
  p.bands = (p.strips + BS_MAX_S - 1) / BS_MAX_S;
  p.S = (p.strips + p.bands - 1) / p.bands;
  p.stages = BS_STAGES[p.S];
  const long long resident = (long long)sm_count() * BS_CTAS_PER_SM[p.S];
  p.R = box_stream_rows((long long)p.bands * n, nrows, resident, &p.chunks);
  p.groups = (p.R + 4 + BS_K - 1) / BS_K;
  p.vec_store = (((uintptr_t)outs[0].base % 16) == 0 && (outs[0].pitch % 16) == 0) ? 1 : 0;
  p.total = n * p.bands * p.chunks;
  const uint64_t width_el = ((uint64_t)rowbytes + 32 + 7) / 8;
  for (int k = 0; k < n; k++) {
    const vppb_img* in = &ins[k];
    unsigned char* origin = static_cast<unsigned char*>(in->base) - 2LL * in->pitch - 16;
    int rc = encode_tensor_map_2d(&p.maps[k], origin, CU_TENSOR_MAP_DATA_TYPE_UINT64, 8, width_el, (uint64_t)nrows + 4, (uint64_t)in->pitch,
                                  p.boxw / 8, BS_K);
    if (rc) return rc;
    p.out_base[k] = static_cast<unsigned char*>(outs[k].base);
    p.in_base[k] = static_cast<const unsigned char*>(in->base);
    p.up_base[k] = (ups && ups[k].base) ? static_cast<const unsigned char*>(ups[k].base) : nullptr;
    p.dn_base[k] = (dns && dns[k].base) ? static_cast<const unsigned char*>(dns[k].base) : nullptr;
  }
  {
    long long bs = (long long)ins[0].border * ins[0].elem_bytes;
    if (bs % ins[0].align) bs += ins[0].align - (bs % ins[0].align);
    p.in_pitch = ins[0].pitch;
    p.row_room = ins[0].pitch - (int)bs;
  }
  const int grid = (int)std::min<long long>(p.total, resident);
  VPPB_CUDA(launch_dependent(k_box5_stream<CS, NB, MODE>, grid, 32 * (BS_CWARPS * p.S + 1), bs_smem(p.S), st, p));
  VPPB_LAUNCH_CHECK(name);
  return VPPB_OK;
}

// the kernel parameters carry one tensor map per image: a single image travels with a 1-entry block (launching a kernel
// with kilobytes of parameters costs microseconds), batches with up to 128
template <int CS>
static int box5_stream_launch(const vppb_img* ins, const vppb_img* ups, const vppb_img* dns, const vppb_img* outs, int n, cudaStream_t st, const char* name) {
  static int ablate = -1;
  if (ablate < 0) {
    const char* e = getenv("VPPB_BOX_ABLATE");
    ablate = !e ? BOX_FILTER : !strcmp(e, "copy") ? BOX_COPY : !strcmp(e, "compute") ? BOX_COMPUTE : BOX_FILTER;
  }
  if (ablate == BOX_COPY) return box5_stream_launch_nb<CS, BS_MAX_BATCH, BOX_COPY>(ins, ups, dns, outs, n, st, name);
  if (ablate == BOX_COMPUTE) return box5_stream_launch_nb<CS, BS_MAX_BATCH, BOX_COMPUTE>(ins, ups, dns, outs, n, st, name);
  if (n == 1) return box5_stream_launch_nb<CS, 1, BOX_FILTER>(ins, ups, dns, outs, n, st, name);
  if (n <= 4) return box5_stream_launch_nb<CS, 4, BOX_FILTER>(ins, ups, dns, outs, n, st, name);
  if (n <= 32) return box5_stream_launch_nb<CS, 32, BOX_FILTER>(ins, ups, dns, outs, n, st, name);
  return box5_stream_launch_nb<CS, BS_MAX_BATCH, BOX_FILTER>(ins, ups, dns, outs, n, st, name);
}

template <int CS>
static int box5_bytes(const vppb_img* in, const vppb_img* out, void* stream, const char* name) {
  VPPB_REQUIRE(in && out && in->base && out->base, VPPB_E_ARG, "%s: NULL image", name);
  VPPB_REQUIRE(in->elem_bytes == CS && out->elem_bytes == CS, VPPB_E_ARG, "%s: element size must be %d", name, CS);
  VPPB_REQUIRE(same_domain(in, out), VPPB_E_ARG, "%s: domains differ", name);
  VPPB_REQUIRE(in->border >= 2, VPPB_E_BORDER, "%s: input border %d < 2", name, in->border);
  cudaStream_t st = as_stream(stream);
  const int rowbytes = in->ncols * CS;
  // one frame per launch: the launch is dominated by fixed costs, where the CTA tile kernel (one TMA box per CTA) is cheaper than
  // the streaming kernel (tools/box_bench.py, single_* with and without VPPB_BOX_SINGLE=stream; figures in DESIGN §3.1), so single
  // frames below 96 MiB take the tile kernel
  static int single_policy = -1;
  if (single_policy < 0) {
    const char* e = getenv("VPPB_BOX_SINGLE");
    single_policy = (e && !strcmp(e, "stream")) ? 1 : 0;
  }
  const bool small = (long long)rowbytes * in->nrows < 96LL * 1024 * 1024;
  if (tma_eligible(in) && (single_policy == 1 || !small)) return box5_stream_launch<CS>(in, nullptr, nullptr, out, 1, st, name);
  if (tma_eligible(in)) {
    CUtensorMap tmap;
    unsigned char* origin = static_cast<unsigned char*>(in->base) - 2LL * in->pitch - 16;
    const uint64_t width_el = ((uint64_t)rowbytes + 32 + 7) / 8;
    const int th = box_tile_rows(in->nrows, rowbytes);
    int rc = encode_tensor_map_2d(&tmap, origin, CU_TENSOR_MAP_DATA_TYPE_UINT64, 8, width_el, (uint64_t)in->nrows + 4,
                                  (uint64_t)in->pitch, BX_BOXW / 8, th + 4);
    if (rc) return rc;
    const int strips = (rowbytes + BX_OUTW - 1) / BX_OUTW;
    const int row_tiles = (in->nrows + th - 1) / th;
    const int vec_store = (((uintptr_t)out->base % 16) == 0 && (out->pitch % 16) == 0) ? 1 : 0;
    // the opt-in shared-memory size is a per-device function attribute: set it once per device (bit = device ordinal)
    static std::atomic<unsigned long long> attr_done{0};
    int dev = 0;
    VPPB_CUDA(cudaGetDevice(&dev));
    const unsigned long long bit = 1ULL << (dev & 63);
    if (!(attr_done.load(std::memory_order_acquire) & bit)) {
      VPPB_CUDA(cudaFuncSetAttribute(k_box5_bytes_tma<CS, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, BoxCfg<16>::SMEM));
      VPPB_CUDA(cudaFuncSetAttribute(k_box5_bytes_tma<CS, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, BoxCfg<8>::SMEM));
      attr_done.fetch_or(bit, std::memory_order_release);
    }
    const int ntiles = strips * row_tiles;
    const int resident = sm_count() * (th == 16 ? 4 : 6);
    const int grid = ntiles < resident ? ntiles : resident;
    if (th == 16)
      VPPB_CUDA(launch_dependent(k_box5_bytes_tma<CS, 16>, grid, BX_THREADS, BoxCfg<16>::SMEM, st, tmap, view(out), rowbytes, strips, ntiles, vec_store, 1u));
    else
      VPPB_CUDA(launch_dependent(k_box5_bytes_tma<CS, 8>, grid, BX_THREADS, BoxCfg<8>::SMEM, st, tmap, view(out), rowbytes, strips, ntiles, vec_store, 1u));
  } else {
    long long total = (long long)in->nrows * rowbytes;
    long long blocks = (total + 255) / 256;
    long long cap = (long long)sm_count() * 16;
    k_box5_direct<unsigned char, int, CS><<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(view(in), view(out), rowbytes);
  }
  VPPB_LAUNCH_CHECK(name);
  return VPPB_OK;
}

// A batch of equally shaped images in one launch of the streaming kernel per <= 128 images.  Anything the batched
// kernel cannot take (mixed shapes, a view or an unaligned buffer among them) falls back to one launch per image -
// same results either way.
template <int CS>
static int box5_bytes_batch(const vppb_img* ins, const vppb_img* outs, int n, void* stream, const char* name) {
  VPPB_REQUIRE(ins && outs && n >= 0, VPPB_E_ARG, "%s: NULL batch", name);
  if (n == 0) return VPPB_OK;
  bool uniform = true;
  for (int i = 0; i < n; i++) {
    const vppb_img *in = &ins[i], *out = &outs[i];
    VPPB_REQUIRE(in->base && out->base, VPPB_E_ARG, "%s: NULL image %d", name, i);
    VPPB_REQUIRE(in->elem_bytes == CS && out->elem_bytes == CS, VPPB_E_ARG, "%s: element size must be %d (image %d)", name, CS, i);
    VPPB_REQUIRE(same_domain(in, out), VPPB_E_ARG, "%s: domains differ (image %d)", name, i);
    VPPB_REQUIRE(in->border >= 2, VPPB_E_BORDER, "%s: input border %d < 2 (image %d)", name, in->border, i);
    uniform = uniform && tma_eligible(in) && same_domain(in, &ins[0]) && out->pitch == outs[0].pitch &&
              (((uintptr_t)out->base % 16) == 0) == (((uintptr_t)outs[0].base % 16) == 0);
  }
  if (!uniform || n == 1) {
    for (int i = 0; i < n; i++) {
      int rc = box5_bytes<CS>(&ins[i], &outs[i], stream, name);
      if (rc) return rc;
    }
    return VPPB_OK;
  }
  cudaStream_t st = as_stream(stream);
  for (int i0 = 0; i0 < n; i0 += BS_MAX_BATCH) {
    int rc = box5_stream_launch<CS>(ins + i0, nullptr, nullptr, outs + i0, std::min(BS_MAX_BATCH, n - i0), st, name);
    if (rc) return rc;
  }
  return VPPB_OK;
}

// Row tiles: equally shaped TMA-eligible tiles; neighbours given per tile (base == NULL: none)
template <int CS>
static int box5_bytes_tiles(const vppb_img* ins, const vppb_img* ups, const vppb_img* dns, const vppb_img* outs, int n, void* stream, const char* name) {
  VPPB_REQUIRE(ins && outs && n >= 0, VPPB_E_ARG, "%s: NULL batch", name);
  for (int i = 0; i < n; i++) {
    const vppb_img *in = &ins[i], *out = &outs[i];
    VPPB_REQUIRE(in->base && out->base, VPPB_E_ARG, "%s: NULL image %d", name, i);
    VPPB_REQUIRE(in->elem_bytes == CS && out->elem_bytes == CS, VPPB_E_ARG, "%s: element size must be %d (image %d)", name, CS, i);
    VPPB_REQUIRE(same_domain(in, out) && same_domain(in, &ins[0]), VPPB_E_ARG, "%s: domains differ (image %d)", name, i);
    VPPB_REQUIRE(in->border >= 2 && in->nrows >= 2, VPPB_E_BORDER, "%s: tile %d needs border >= 2 and at least 2 rows", name, i);
    VPPB_REQUIRE(tma_eligible(in) && in->pitch == ins[0].pitch && in->border == ins[0].border && in->align == ins[0].align, VPPB_E_ARG,
                 "%s: tiles must share the library layout (image %d)", name, i);
    VPPB_REQUIRE(out->pitch == outs[0].pitch && (((uintptr_t)out->base % 16) == 0) == (((uintptr_t)outs[0].base % 16) == 0), VPPB_E_ARG,
                 "%s: outputs must share pitch and alignment (image %d)", name, i);
    for (const vppb_img* nb : {ups ? &ups[i] : nullptr, dns ? &dns[i] : nullptr})
      if (nb && nb->base)
        VPPB_REQUIRE(nb->pitch == in->pitch && nb->ncols == in->ncols && nb->nrows >= 2 && nb->elem_bytes == CS && nb->border == in->border &&
                         nb->align == in->align && ((uintptr_t)nb->base % 16) == 0,
                     VPPB_E_ARG, "%s: neighbour of tile %d must have the tile's layout", name, i);
    // the tile above contributes its LAST rows: they are addressed from its pixel (0,0) with ITS row count
    VPPB_REQUIRE(!(ups && ups[i].base) || ups[i].nrows == in->nrows, VPPB_E_ARG, "%s: the tile above tile %d must have as many rows (pass a sub-image of its last rows otherwise)", name, i);
  }
  cudaStream_t st = as_stream(stream);
  for (int i0 = 0; i0 < n; i0 += BS_MAX_BATCH) {
    int rc = box5_stream_launch<CS>(ins + i0, ups ? ups + i0 : nullptr, dns ? dns + i0 : nullptr, outs + i0, std::min(BS_MAX_BATCH, n - i0), st, name);
    if (rc) return rc;
  }
  return VPPB_OK;
}

}  // namespace vppb

using namespace vppb;

extern "C" {

int vppb_box5x5_u8c3_batch(const vppb_img* ins, const vppb_img* outs, int32_t n, void* stream) {
  return box5_bytes_batch<3>(ins, outs, n, stream, "vppb_box5x5_u8c3_batch");
}
int vppb_box5x5_u8_batch(const vppb_img* ins, const vppb_img* outs, int32_t n, void* stream) {
  return box5_bytes_batch<1>(ins, outs, n, stream, "vppb_box5x5_u8_batch");
}

int vppb_box5x5_u8c3_tiles(const vppb_img* ins, const vppb_img* ups, const vppb_img* downs, const vppb_img* outs, int32_t n, void* stream) {
  return box5_bytes_tiles<3>(ins, ups, downs, outs, n, stream, "vppb_box5x5_u8c3_tiles");
}
int vppb_box5x5_u8_tiles(const vppb_img* ins, const vppb_img* ups, const vppb_img* downs, const vppb_img* outs, int32_t n, void* stream) {
  return box5_bytes_tiles<1>(ins, ups, downs, outs, n, stream, "vppb_box5x5_u8_tiles");
}

int vppb_box5x5_u8c3(const vppb_img* in, const vppb_img* out, void* stream) {
  return box5_bytes<3>(in, out, stream, "vppb_box5x5_u8c3");
}

int vppb_box5x5_u8(const vppb_img* in, const vppb_img* out, void* stream) {
  return box5_bytes<1>(in, out, stream, "vppb_box5x5_u8");
}

int vppb_box5x5_i32(const vppb_img* in, const vppb_img* out, void* stream) {
  VPPB_REQUIRE(in && out && in->base && out->base, VPPB_E_ARG, "vppb_box5x5_i32: NULL image");
  VPPB_REQUIRE(in->elem_bytes == 4 && out->elem_bytes == 4, VPPB_E_ARG, "vppb_box5x5_i32: element size must be 4");
  VPPB_REQUIRE(same_domain(in, out), VPPB_E_ARG, "vppb_box5x5_i32: domains differ");
  VPPB_REQUIRE(in->border >= 2, VPPB_E_BORDER, "vppb_box5x5_i32: input border %d < 2", in->border);
  long long total = (long long)in->nrows * in->ncols;
  long long blocks = (total + 255) / 256;
  long long cap = (long long)sm_count() * 16;
  // int accumulation wraps like the reference's `int sum` on two's-complement hardware
  k_box5_direct<int, int, 1><<<(int)(blocks < cap ? blocks : cap), 256, 0, as_stream(stream)>>>(view(in), view(out), in->ncols);
  VPPB_LAUNCH_CHECK("vppb_box5x5_i32");
  return VPPB_OK;
}

}  // extern "C"
