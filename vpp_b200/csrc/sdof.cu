// Semi-dense optical flow of video_extruder: coarse-to-fine SAD block matching on a grid of
// patchsize x patchsize cells, greedy 8-neighbour descent, neighbour propagation sweeps.
// Reference: vpp/algorithms/optical_flow/semi_dense_optical_flow.hpp:17-214,
// vpp/algorithms/optical_flow/gradient_descent.hh:10-89.
//
// The reference is sequentially defined (and racy under OpenMP): the FIRST keypoint that reaches a
// cell claims it, and the propagation sweeps are Gauss-Seidel in raster order.  The GPU keeps the
// serial semantics exactly:
//   - claim: atomicMin of the keypoint index per cell, then only the owner matches (the match of a
//     cell depends on nothing the other keypoints do);
//   - propagation: iteration (kr, kc) of a sweep only depends on iterations (kr, kc-1) and
//     (kr-1, kc-1..kc+1), so all iterations with kc + 2 kr = t are independent: one launch per
//     wavefront t, one warp per cell, in the sweep's own direction.
// One warp evaluates a SAD (winsize^2 <= 225 byte pairs over 32 lanes, integer shuffle reduction);
// the row-wise early exit of the reference only skips sums that already exceed the threshold, so the
// full SAD gives the same comparisons.  Gather / latency bound, not HBM bound.
#include "common.cuh"

#include <limits.h>
#include <string.h>

#include <vector>

namespace vppb {

constexpr unsigned FULLM = 0xffffffffu;

struct SdofLevel {
  Img i1, i2;
  // one 64-bit record per cell: flow.x (16 bits, signed) | flow.y (16) | distance (24, 0xFFFFFF = INT_MAX) | sweep (8: the last
  // sweep, 1-based, of this scale that has finished with the cell).  A single word so that the dataflow sweeps get a
  // neighbour's flow together with its "done" stamp in ONE acquire load, and publish both with one release store.
  unsigned long long* rec;  // cells: (cr + 2) x (cc + 2) entries, row stride = cstride
  unsigned char* mark;
  int* owner;
  int cr, cc, cstride;   // cell-map domain (pf_domain pyramid level) and row stride
  // relaxation schedule (k_sdof_fused): second record buffer (a sweep reads `old`, writes `cur`), a stamp per cell that dedups the
  // work lists, the list of marked cells and two alternating work lists
  unsigned long long* rec2;
  int* stamp;
  int* mlist;
  int* wl[2];
};

__device__ __forceinline__ unsigned long long rec_pack(int fx, int fy, int dist, int sweep) {
  const unsigned d = dist == INT_MAX ? 0xFFFFFFu : (unsigned)dist;
  return (unsigned long long)((unsigned)fx & 0xFFFFu) | ((unsigned long long)((unsigned)fy & 0xFFFFu) << 16) | ((unsigned long long)(d & 0xFFFFFFu) << 32) |
         ((unsigned long long)((unsigned)sweep & 0xFFu) << 56);
}
__device__ __forceinline__ int rec_fx(unsigned long long r) { return (int)(short)(r & 0xFFFFu); }
__device__ __forceinline__ int rec_fy(unsigned long long r) { return (int)(short)((r >> 16) & 0xFFFFu); }
__device__ __forceinline__ int rec_dist(unsigned long long r) { const unsigned d = (unsigned)((r >> 32) & 0xFFFFFFu); return d == 0xFFFFFFu ? INT_MAX : (int)d; }
__device__ __forceinline__ int rec_sweep(unsigned long long r) { return (int)(r >> 56); }

__constant__ int c_c8_it[9][2] = {{6, 3}, {0, 3}, {0, 5}, {2, 5}, {2, 7}, {4, 7}, {4, 1}, {6, 1}, {0, 0}};
__constant__ int c_c8[8][2] = {{-1, 1}, {0, 1}, {1, 1}, {-1, 0}, {1, 0}, {-1, -1}, {0, -1}, {1, -1}};
// c_c8 for a lane-dependent index without a constant-bank replay: (offset + 1) in 2-bit fields
__device__ __forceinline__ int c8_dr(int i) { return (int)((0x9224u >> (2 * i)) & 3u) - 1; }
__device__ __forceinline__ int c8_dc(int i) { return (int)((0x016Au >> (2 * i)) & 3u) - 1; }

// ---- batched SADs -----------------------------------------------------------------------------------------------------------
// A propagation iteration needs the SADs of up to 8 candidate flows, a descent step those of the 8 neighbours of the current
// position: independent sums that the reference evaluates one after the other.  Here a group of 4 lanes owns one candidate
// (8 candidates per warp at once); a lane sums whole window rows (rows sub, sub + 4, ...) with aligned 32-bit loads, a funnel
// shift to the window's byte offset and VABSDIFF4-with-sum, all loads of a lane in flight together: one memory round trip per
// batch instead of one per candidate.  Integer sums: the grouping changes nothing in the result.
__device__ __forceinline__ unsigned sad_rows(const unsigned char* pa, long long apitch, const unsigned char* pb, long long bpitch, int ws, int sub, int nl) {
  unsigned s = 0;
  const bool words = ((apitch | bpitch) & 3) == 0;  // aligned words never leave a row allocation whose pitch is a multiple of 4
  if (!words) {  // rows whose pitch is not a multiple of 4 (wrapped user memory): byte loads
    for (int row = sub; row < ws; row += nl)
      for (int x = 0; x < ws; x++) s += (unsigned)abs((int)pa[row * apitch + x] - (int)pb[row * bpitch + x]);
    return s;
  }
#pragma unroll
  for (int j = 0; j < 5; j++) {  // nl = 4: rows sub, sub + 4, ... (j = 4 never below ws <= 15 ... 16); nl = 3: up to 5 rows per lane
    const int row = sub + j * nl;
    if (row < ws) {
      const unsigned char* ra = pa + row * apitch;
      const unsigned char* rb = pb + row * bpitch;
      const unsigned oa = (unsigned)(unsigned long long)ra & 3u, ob = (unsigned)(unsigned long long)rb & 3u;
      const unsigned* wa = reinterpret_cast<const unsigned*>(ra - oa);
      const unsigned* wb = reinterpret_cast<const unsigned*>(rb - ob);
      const int la = (int)(oa + ws - 1) >> 2, lb = (int)(ob + ws - 1) >> 2;  // last aligned word the row touches
      unsigned a[5], b[5];
#pragma unroll
      for (int q = 0; q < 5; q++) {
        a[q] = q <= la ? wa[q] : 0u;
        b[q] = q <= lb ? wb[q] : 0u;
      }
#pragma unroll
      for (int q = 0; q < 4; q++) {
        if (q * 4 < ws) {
          unsigned va = __funnelshift_r(a[q], a[q + 1], oa * 8), vb = __funnelshift_r(b[q], b[q + 1], ob * 8);
          const int rem = ws - q * 4;
          if (rem < 4) { const unsigned m = (1u << (8 * rem)) - 1u; va &= m; vb &= m; }
          s += __vsadu4(va, vb);
        }
      }
    }
  }
  return s;
}

__device__ __forceinline__ bool sad_inside(const Img& a, const Img& b, int ar, int ac, int br, int bc) {
  return !(ar < 0 || ar >= a.nrows || ac < 0 || ac >= a.ncols || br < 0 || br >= b.nrows || bc < 0 || bc >= b.ncols);  // :102-108
}

// one SAD by the whole warp (a lane per window row)
__device__ __forceinline__ int sad_warp(const Img& a, const Img& b, int ar, int ac, int br, int bc, int ws) {
  if (!sad_inside(a, b, ar, ac, br, bc)) return INT_MAX;
  const int lane = threadIdx.x & 31, h = ws / 2;
  unsigned s = sad_rows(a.base + (long long)(ar - h) * a.pitch + (ac - h), a.pitch, b.base + (long long)(br - h) * b.pitch + (bc - h), b.pitch, ws, lane, 32);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(FULLM, s, o);
  return (int)s;
}

// the SAD of the candidate of this lane's group of 4 (all four lanes pass the same arguments); every lane of the warp calls it
__device__ __forceinline__ int sad_group4(const Img& a, const Img& b, int ar, int ac, int br, int bc, int ws, bool active) {
  const bool inside = sad_inside(a, b, ar, ac, br, bc);
  const int h = ws / 2;
  unsigned s = 0;
  if (active && inside)
    s = sad_rows(a.base + (long long)(ar - h) * a.pitch + (ac - h), a.pitch, b.base + (long long)(br - h) * b.pitch + (bc - h), b.pitch, ws, threadIdx.x & 3, 4);
  s += __shfl_xor_sync(FULLM, s, 1);
  s += __shfl_xor_sync(FULLM, s, 2);
  return inside ? (int)s : INT_MAX;
}

// the same with groups of 3 lanes: ten candidates per warp (lanes 30, 31 idle) - the eight neighbours of a position AND the position
// itself in one batch; for winsize 9 a lane sums exactly 3 rows, as the busiest lane of a group of 4 does
__device__ __forceinline__ int sad_group3(const Img& a, const Img& b, int ar, int ac, int br, int bc, int ws, bool active) {
  const int lane = threadIdx.x & 31;
  const bool inside = sad_inside(a, b, ar, ac, br, bc);
  const int h = ws / 2, g3 = lane / 3;
  unsigned s = 0;
  if (active && inside && lane < 30)
    s = sad_rows(a.base + (long long)(ar - h) * a.pitch + (ac - h), a.pitch, b.base + (long long)(br - h) * b.pitch + (bc - h), b.pitch, ws, lane - 3 * g3, 3);
  const int base = min(3 * g3, 29);
  const unsigned t = __shfl_sync(FULLM, s, base) + __shfl_sync(FULLM, s, base + 1) + __shfl_sync(FULLM, s, base + 2);
  return inside ? (int)t : INT_MAX;
}

// gradient_descent.hh:10-89 for a match that starts at its prediction: the SAD at the prediction (the reference evaluates it first,
// :52) rides in the batch of the first step's eight neighbours (group 8), so a match that stays where it was predicted - the usual
// case below the coarsest scale - costs ONE memory round trip.  Later steps as descent_warp.
__device__ __forceinline__ void descent_from_prediction(const Img& a, const Img& b, int pr, int pc, int predr, int predc, int ws, int max_it, int& flr,
                                                        int& flc, int& dist) {
  const int lane = threadIdx.x & 31;
  const int g3 = min(lane / 3, 8);  // groups 0..7: the neighbours c_c8[g], group 8 (lanes 24..26): the position itself; lanes 27..31 idle
  const int gdr = g3 < 8 ? c8_dr(g3) : 0, gdc = g3 < 8 ? c8_dc(g3) : 0;
  int mr = predr, mc = predc, md = INT_MAX;
  int mi = 8;
  for (int search = 0; search < max_it; search++) {
    const int dg = sad_group3(a, b, pr, pc, predr + gdr, predc + gdc, ws, lane < (search == 0 ? 27 : 24));
    if (search == 0) md = __shfl_sync(FULLM, dg, 24);
    int i = c_c8_it[mi][0];
    const int end = c_c8_it[mi][1];
    bool first = true;
    while (first || i != end) {
      first = false;
      const int d = __shfl_sync(FULLM, dg, i * 3);
      if (d < md) { mr = predr + c_c8[i][0]; mc = predc + c_c8[i][1]; mi = i; md = d; }
      i = (i + 1) & 7;
    }
    if (predr == mr && predc == mc) break;
    predr = mr; predc = mc;
  }
  flr = mr - pr; flc = mc - pc; dist = md;
}

// gradient_descent.hh:10-89 (whole warp, uniform control flow).  `md` = the SAD at the prediction (the caller has it).  A step
// evaluates the 8 neighbours of the current position at once (group i <-> c_c8[i]) and then replays the reference's visiting
// order and strict comparisons on the eight values, so the walk is the reference's.
__device__ __forceinline__ void descent_warp(const Img& a, const Img& b, int pr, int pc, int predr, int predc, int ws, int max_it, int md, int& flr,
                                             int& flc, int& dist) {
  const int g = (threadIdx.x & 31) >> 2;
  const int gdr = c8_dr(g), gdc = c8_dc(g);
  int mr = predr, mc = predc;
  int mi = 8;
  for (int search = 0; search < max_it; search++) {
    const int dg = sad_group4(a, b, pr, pc, predr + gdr, predc + gdc, ws, true);
    int i = c_c8_it[mi][0];
    const int end = c_c8_it[mi][1];
    bool first = true;
    while (first || i != end) {
      first = false;
      const int d = __shfl_sync(FULLM, dg, i * 4);
      if (d < md) { mr = predr + c_c8[i][0]; mc = predc + c_c8[i][1]; mi = i; md = d; }
      i = (i + 1) & 7;
    }
    if (predr == mr && predc == mc) break;
    predr = mr; predc = mc;
  }
  flr = mr - pr; flc = mc - pc; dist = md;
}

__global__ void k_sdof_clear(SdofLevel L) {
  const int total = (L.cr + 2) * L.cstride;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) { L.mark[i] = 0; L.owner[i] = INT_MAX; L.rec[i] = 0ull; }
}

// a keypoint outside the frame (level 0) claims nothing and is reported invalid, also where a coarser level, rounded up, would hold it
__device__ __forceinline__ bool kp_in_frame(vppb_int2 k, int nrows0, int ncols0) { return k.r >= 0 && k.c >= 0 && k.r < nrows0 && k.c < ncols0; }

__global__ void k_sdof_claim(SdofLevel L, const vppb_int2* kps, int n, int scale_div, int patch, int nrows0, int ncols0) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!kp_in_frame(kps[i], nrows0, ncols0)) continue;
    const int fr = (kps[i].r / scale_div) / patch, fc = (kps[i].c / scale_div) / patch;
    if (fr >= L.cr || fc >= L.cc || kps[i].r / scale_div >= L.i1.nrows || kps[i].c / scale_div >= L.i1.ncols) continue;
    atomicMin(&L.owner[fr * L.cstride + fc], i);
  }
}

// :114-143, one warp per keypoint; only the owner (lowest index == first in serial order) of a cell matches
__global__ void __launch_bounds__(128) k_sdof_match(SdofLevel L, SdofLevel coarser, int has_coarser, const vppb_int2* kps, int n, int scale_div,
                                                    int patch, int ws) {
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nwarps) {
    if (kps[i].r < 0 || kps[i].c < 0) continue;  // warp-uniform
    const int pr = kps[i].r / scale_div, pc = kps[i].c / scale_div;
    if (pr >= L.i1.nrows || pc >= L.i1.ncols || pr / patch >= L.cr || pc / patch >= L.cc) continue;
    const int cell = (pr / patch) * L.cstride + (pc / patch);
    if (L.owner[cell] != i) continue;  // warp-uniform
    int predr = pr, predc = pc;
    if (has_coarser) {
      const int m = (pr / (2 * patch)) * coarser.cstride + (pc / (2 * patch));
      if (coarser.mark[m]) { const unsigned long long cr_ = coarser.rec[m]; predr = pr + rec_fx(cr_) * 2; predc = pc + rec_fy(cr_) * 2; }
    }
    int flr, flc, d;
    descent_from_prediction(L.i1, L.i2, pr, pc, predr, predc, ws, 5, flr, flc, d);
    if (lane == 0) { L.rec[cell] = rec_pack(flr, flc, d, 0); L.mark[cell] = 2; }
  }
}

// :149-189, iteration (kr, kc) of a propagation sweep, executed by one warp; forward sweeps start at pixel 0 and step
// +patch, backward sweeps start at the last pixel and step -patch (so p is not the cell corner there)
// `epoch` > 0 (dataflow sweeps): the lanes that hold a PREDECESSOR of the sweep order wait until its record carries this sweep's number;
// the cell's own record is published with it.  epoch == 0 (launch-ordered schedules): plain loads, the stamp stays 0.
// the arithmetic of one iteration: lanes 0..8 hold the mark and the record of the 3 x 3 cells around the iteration's cell (lane 4 = the
// cell itself); returns the cell's new flow and distance on every lane
__device__ __forceinline__ void sdof_prop_eval(const SdofLevel& L, int r, int c, int ws, int nmark, unsigned long long nrec, int2& cur, int& d1) {
  const int lane = threadIdx.x & 31;
  const unsigned long long own = __shfl_sync(FULLM, nrec, 4);
  cur = make_int2(rec_fx(own), rec_fy(own));
  const int2 prev = cur;
  d1 = rec_dist(own);
  // the SADs of all marked neighbours' flows at once: group g of 4 lanes <-> neighbour k = g (+1 past the centre)
  const int g = lane >> 2, kg = g + (g >= 4);
  const int mg = __shfl_sync(FULLM, nmark, kg);
  const unsigned long long rg = __shfl_sync(FULLM, nrec, kg);
  // a neighbour whose flow is within 2 pixels of the cell's pre-sweep flow is skipped whatever happens (the `prev` half of the test
  // below): its SAD is never looked at.  In a smooth flow field that is every neighbour - no window is read at all.
  const int q0 = prev.x - rec_fx(rg), q1 = prev.y - rec_fy(rg);
  const bool need = mg != 0 && q0 * q0 + q1 * q1 >= 9;
  if (!__any_sync(FULLM, need)) return;
  const int dg = sad_group4(L.i1, L.i2, r, c, r + rec_fx(rg), c + rec_fy(rg), ws, need);
#pragma unroll 1
  for (int k = 0; k < 9; k++) {
    if (k == 4) continue;
    if (!__shfl_sync(FULLM, nmark, k)) continue;  // outside the cell map or unmarked
    const unsigned long long nr_ = __shfl_sync(FULLM, nrec, k);
    const int2 nf = make_int2(rec_fx(nr_), rec_fy(nr_));
    const int a0 = cur.x - nf.x, a1 = cur.y - nf.y, b0 = prev.x - nf.x, b1 = prev.y - nf.y;
    if (a0 * a0 + a1 * a1 < 9 || b0 * b0 + b1 * b1 < 9) continue;  // integer norm() > 2
    const int d2 = __shfl_sync(FULLM, dg, (k - (k > 4)) * 4);
    if (d2 < d1) {
      int flr, flc, d;
      descent_warp(L.i1, L.i2, r, c, r + nf.x, c + nf.y, ws, 5, d2, flr, flc, d);
      if (d < d1) { cur = make_int2(flr, flc); d1 = d; }
    }
  }
}

__device__ __forceinline__ void sdof_prop_cell(const SdofLevel& L, int kr, int kc, int forward, int patch, int ws, int lane, int epoch = 0, int nkc = 0) {
  const int inr = L.i1.nrows, inc = L.i1.ncols;
  const int r = forward ? kr * patch : inr - 1 - kr * patch, c = forward ? kc * patch : inc - 1 - kc * patch;
  const int fr = r / patch, fc = c / patch;
  const int cell = fr * L.cstride + fc;
  if (!L.mark[cell]) return;  // warp-uniform
  // the cell's own record and its 8 neighbours' are fetched at once, one per lane (lane k = (dr + 1) * 3 + (dc + 1); lane 4 = the
  // cell itself)
  int nmark = 0;
  bool pred = false;
  unsigned long long nrec = 0;
  const unsigned long long* nptr = L.rec;
  if (lane < 9) {
    const int dr = lane / 3 - 1, dc = lane % 3 - 1;
    const int nr = fr + dr, nc = fc + dc;
    if (nr >= 0 && nr < L.cr && nc >= 0 && nc < L.cc) {
      const int ncell = nr * L.cstride + nc;
      nmark = L.mark[ncell];
      if (nmark) {
        nptr = &L.rec[ncell];
        if (epoch > 0) {
          // predecessors in sweep coordinates: (kr, kc-1), (kr-1, kc-1), (kr-1, kc), (kr-1, kc+1); a step of +1 in sweep coordinates is a
          // step of sgn in cell coordinates
          const int sgn = forward ? 1 : -1;
          const int skr = dr * sgn, skc = dc * sgn;  // the neighbour's offset in sweep coordinates
          pred = (skr == -1 || (skr == 0 && skc == -1)) && kr + skr >= 0 && kc + skc >= 0 && kc + skc < nkc;
          nrec = ld_acquire64(nptr);
        } else {
          nrec = __ldcg(nptr);
        }
      }
    }
  }
  const int d0 = rec_dist(__shfl_sync(FULLM, nrec, 4));
  const int2 prev = make_int2(rec_fx(__shfl_sync(FULLM, nrec, 4)), rec_fy(__shfl_sync(FULLM, nrec, 4)));
  int2 cur;
  int d1;
  // Dataflow sweeps SPECULATE: the iteration is evaluated on the records as they are now, without waiting for the predecessors; only
  // then do the lanes that hold a predecessor wait for its stamp of this sweep.  A record whose flow did not change (the usual case: a
  // sweep moves few cells) validates the speculation - the result is a function of the nine flows and the cell's own distance - and the
  // warp publishes at once: the chain of dependent iterations then costs one flag hop per cell instead of hop + SADs.  Otherwise
  // the iteration is redone on the final records (successors cannot have changed: they wait for this cell's stamp).
  sdof_prop_eval(L, r, c, ws, nmark, nrec, cur, d1);
  if (epoch > 0) {
    unsigned long long fin = nrec;
    if (pred)
      while (rec_sweep(fin) < epoch) { spin_pause(); fin = ld_acquire64(nptr); }
    const bool moved = nmark && (unsigned)fin != (unsigned)nrec;  // flow.x | flow.y are the low 32 bits
    if (__any_sync(FULLM, moved)) sdof_prop_eval(L, r, c, ws, nmark, fin, cur, d1);
  }
  const bool changed = cur.x != prev.x || cur.y != prev.y || d1 != d0;
  if (lane == 0) {
    if (changed) L.mark[cell] = 1;
    if (epoch > 0) st_release64(&L.rec[cell], rec_pack(cur.x, cur.y, d1, epoch));  // flow, distance and the "done" stamp in one store
    else if (changed) L.rec[cell] = rec_pack(cur.x, cur.y, d1, 0);
  }
}

// the iterations (kr, kc) of one sweep with kc + 2 kr == t: iteration (kr, kc) only reads what (kr, kc-1) and
// (kr-1, kc-1..kc+1) wrote, so a whole anti-diagonal is independent
__global__ void __launch_bounds__(128) k_sdof_prop_wave(SdofLevel L, int t, int forward, int nkr, int nkc, int patch, int ws) {
  const int lane = threadIdx.x & 31;
  const int kr_lo = max(0, (t - (nkc - 1) + 1) / 2), kr_hi = min(nkr - 1, t / 2);
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int kr = kr_lo + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5); kr <= kr_hi; kr += nwarps) {
    const int kc = t - 2 * kr;
    if (kc < 0 || kc >= nkc) continue;
    sdof_prop_cell(L, kr, kc, forward, patch, ws, lane);
  }
}

// ---- dataflow schedule of a sweep (propagation > 30, or VPPB_SDOF_SCHEDULE=dataflow): ONE persistent launch per sweep ---
// Only marked cells do anything in a sweep and a marked cell only reads its marked 8-neighbours, so the Gauss-Seidel order
// is a partial order on the marked cells: (kr, kc) must come after its marked predecessors (kr, kc-1), (kr-1, kc-1..kc+1)
// and before its marked successors.  Warps draw iterations from a ticket counter in WAVEFRONT order (anti-diagonal
// t = kc + 2 kr, then kr): consecutive tickets are independent iterations, so as many warps as a diagonal has marked cells
// work at once.  Before its iteration a warp waits until the `done` flag of every marked predecessor carries this sweep's
// number (acquire loads at GPU scope), afterwards it publishes its own flag (release store).  Every predecessor sits on an
// earlier diagonal, i.e. holds a smaller ticket, which a running warp already owns: no deadlock.  The critical path is
// the longest chain of adjacent marked cells times one flag hop, instead of (columns + 2 rows) kernel launches.
__global__ void __launch_bounds__(128) k_sdof_sweep(SdofLevel L, int forward, int nkr, int nkc, int patch, int ws, int epoch, int* ticket) {
  const int lane = threadIdx.x & 31;
  const int inr = L.i1.nrows, inc = L.i1.ncols;
  const int total = nkr * nkc;
  // wavefront order: diagonal t holds the iterations kr in [lo(t), hi(t)], lo = max(0, ceil((t - nkc + 1) / 2)), hi = min(nkr - 1, t / 2).
  // first(t) = number of iterations on the diagonals before t, in closed form for the three regimes of the band
  // (growing, full width, shrinking) would need case analysis: a warp instead walks the diagonals incrementally - its
  // tickets only grow.
  int t = 0, first = 0;  // current diagonal and the ticket of its first iteration
  auto diag_len = [&](int tt) {
    const int lo = max(0, (tt - (nkc - 1) + 1) / 2), hi = min(nkr - 1, tt / 2);
    return hi >= lo ? hi - lo + 1 : 0;
  };
  for (;;) {
    int i = 0;
    if (lane == 0) i = atomicAdd(ticket, 1);
    i = __shfl_sync(FULLM, i, 0);
    if (i >= total) break;
    int len = diag_len(t);
    while (i >= first + len) { first += len; t++; len = diag_len(t); }  // warp-uniform
    const int kr = max(0, (t - (nkc - 1) + 1) / 2) + (i - first), kc = t - 2 * kr;
    const int r = forward ? kr * patch : inr - 1 - kr * patch, c = forward ? kc * patch : inc - 1 - kc * patch;
    const int fr = r / patch, fc = c / patch;
    const int cell = fr * L.cstride + fc;
    if (!L.mark[cell]) continue;  // marks only go from 2 to 1 during the sweeps: "marked" never changes
    sdof_prop_cell(L, kr, kc, forward, patch, ws, lane, epoch, nkc);
  }
}

// ---- dependency-level schedule of a sweep (opt-in, VPPB_SDOF_SCHEDULE=levels) ---------------------------------
// Only marked cells do anything in a sweep, and a marked cell only interacts with its marked 8-neighbours.  Give every
// marked cell the level 1 + max(level of the marked neighbours that PRECEDE it in the sweep) (0 if none): two
// adjacent marked cells always get different levels, ordered as the serial sweep orders them, so running the levels
// one after another - all cells of a level at once - reproduces the Gauss-Seidel sweep exactly, in (longest chain of
// adjacent marked cells) launches instead of (cols + 2 rows) anti-diagonals.  With video_extruder's keypoints (one per
// 10 x 10 block, cells of 5 px) the finest scale needs a handful of levels instead of ~800 wavefronts.
// k_sdof_levels: ONE CTA walks the anti-diagonals (integer work only, a __syncthreads per diagonal), then buckets the
// marked cells by level.  sched[0] = number of levels, sched[1] = number of marked cells, start = sched + 2 (cap + 1
// entries: bucket starts, then the total), hist = start + cap + 1 (scratch: histogram, then bucket cursors).
// cells: kr * nkc + kc of the marked cells, grouped by level (order inside a level is irrelevant: its cells are independent).
__global__ void __launch_bounds__(1024) k_sdof_levels(SdofLevel L, int forward, int nkr, int nkc, int patch, int* level, int* sched, int cap, unsigned* cells) {
  const int inr = L.i1.nrows, inc = L.i1.ncols;
  const int waves = nkc + 2 * (nkr - 1);
  int* start = sched + 2;
  int* hist = start + cap + 1;
  __shared__ int s_max, s_cnt;
  if (threadIdx.x == 0) { s_max = -1; s_cnt = 0; }
  for (int i = threadIdx.x; i < cap; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  const int sgn = forward ? 1 : -1;  // a step of +1 in sweep coordinates is a step of sgn in cell coordinates
  for (int t = 0; t < waves; t++) {
    const int kr_lo = max(0, (t - (nkc - 1) + 1) / 2), kr_hi = min(nkr - 1, t / 2);
    for (int kr = kr_lo + (int)threadIdx.x; kr <= kr_hi; kr += blockDim.x) {
      const int kc = t - 2 * kr;
      if (kc < 0 || kc >= nkc) continue;
      const int r = forward ? kr * patch : inr - 1 - kr * patch, c = forward ? kc * patch : inc - 1 - kc * patch;
      const int fr = r / patch, fc = c / patch;
      const int cell = fr * L.cstride + fc;
      if (!L.mark[cell]) continue;
      int lv = 0;
      // predecessors in sweep order: (kr, kc-1), (kr-1, kc-1), (kr-1, kc), (kr-1, kc+1) - counted only where sdof_prop_cell reads them
      const int pr[4] = {fr, fr - sgn, fr - sgn, fr - sgn}, pc[4] = {fc - sgn, fc - sgn, fc, fc + sgn};
      for (int k = 0; k < 4; k++) {
        if (pr[k] < 0 || pr[k] >= L.cr || pc[k] < 0 || pc[k] >= L.cc) continue;
        const int pcell = pr[k] * L.cstride + pc[k];
        if (L.mark[pcell]) lv = max(lv, level[pcell] + 1);
      }
      level[cell] = lv;
      atomicMax(&s_max, lv);
      atomicAdd(&s_cnt, 1);
      atomicAdd(&hist[lv], 1);
    }
    __syncthreads();
  }
  const int nlevels = s_max + 1;
  if (threadIdx.x == 0) {
    sched[0] = nlevels;
    sched[1] = s_cnt;
    int run = 0;
    for (int l = 0; l < nlevels; l++) { start[l] = run; run += hist[l]; hist[l] = start[l]; }  // hist becomes the fill cursor
    start[nlevels] = run;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nkr * nkc; i += blockDim.x) {
    const int kr = i / nkc, kc = i - kr * nkc;
    const int r = forward ? kr * patch : inr - 1 - kr * patch, c = forward ? kc * patch : inc - 1 - kc * patch;
    const int cell = (r / patch) * L.cstride + (c / patch);
    if (!L.mark[cell]) continue;
    cells[atomicAdd(&hist[level[cell]], 1)] = (unsigned)i;  // i = kr * nkc + kc: frames may be wider than 65535 cells
  }
}

// one level of the schedule: n independent iterations, one warp each
__global__ void __launch_bounds__(128) k_sdof_prop_list(SdofLevel L, const unsigned* cells, int n, int forward, int nkc, int patch, int ws) {
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nwarps) {
    const int v = (int)cells[i];
    sdof_prop_cell(L, v / nkc, v % nkc, forward, patch, ws, lane);
  }
}

// ---- relaxation schedule (default): the WHOLE flow (all scales: clear, claim, match, sweeps, emit) in ONE cooperative launch ----
// A Gauss-Seidel sweep is the unique solution X of  X(c) = f(old(c), X(predecessors of c), old(successors of c))  over the marked
// cells, where the predecessors of an iteration are the 4 neighbours the sweep visits before it.  That system is triangular, so it
// can also be solved by relaxation:  round 0 evaluates every marked cell on the pre-sweep records (all cells at once); round k >= 1
// re-evaluates exactly the cells one of whose predecessors changed its FLOW in round k-1 (a work list, deduplicated by a stamp per
// cell), reading predecessors from `cur` and successors / the cell itself from `old`.  A cell read while its predecessor is being
// rewritten is re-queued by that predecessor, so when a round queues nothing every cell has been evaluated on the final records of
// its predecessors: the fixed point is the serial sweep, bit for bit, whatever the order inside a round.  A sweep moves few cells,
// so the number of rounds is the length of the longest chain of *moving* cells (a handful), not the number of anti-diagonals; each
// round is one grid-wide barrier.  Worst case (a flow that propagates along a whole row): as many rounds as the dataflow schedule
// has hops.
struct SdofFused {
  SdofLevel L[8];
  int nscales, min_scale, patch, ws, propagation, n;
  const vppb_int2* kps;
  vppb_int2* out_pos;
  int* out_dist;
  unsigned char* out_valid;
  int* ctr;  // zeroed before the launch: [0] grid barrier, [1], [2] statistics, [8 + 128 * scale] marked cells of the scale, [.. + 4 + 4 * sweep + 0..2] work-list lengths
};

// one evaluation of cell `cell` in a relaxation round (one warp).  first: round 0 of the sweep (everything read from `old`, `cur`
// written unconditionally); later rounds compare with the cell's previous `cur`.  A cell whose flow moved queues its successors.
__device__ __forceinline__ void sdof_relax_cell(const SdofLevel& L, const unsigned long long* old, unsigned long long* cur, int cell, int forward, int nkr,
                                                int nkc, int patch, int ws, bool first, int stampval, int* wl_next, int* cnt_next) {
  const int lane = threadIdx.x & 31;
  const int inr = L.i1.nrows, inc = L.i1.ncols;
  const int fr = cell / L.cstride, fc = cell - fr * L.cstride;
  const int kr = forward ? fr : (inr - 1) / patch - fr, kc = forward ? fc : (inc - 1) / patch - fc;
  if (kr < 0 || kr >= nkr || kc < 0 || kc >= nkc) {  // a marked cell no iteration of the sweep visits keeps its record (warp-uniform)
    if (first && lane == 0) __stcg(cur + cell, __ldcg(old + cell));
    return;
  }
  const int r = forward ? kr * patch : inr - 1 - kr * patch, c = forward ? kc * patch : inc - 1 - kc * patch;
  const int sgn = forward ? 1 : -1;  // a step of +1 in sweep coordinates is a step of sgn in cell coordinates
  int nmark = 0;
  unsigned long long nrec = 0;
  if (lane < 9) {
    const int dr = lane / 3 - 1, dc = lane % 3 - 1;
    const int nr = fr + dr, nc = fc + dc;
    if (nr >= 0 && nr < L.cr && nc >= 0 && nc < L.cc) {
      const int ncell = nr * L.cstride + nc;
      nmark = __ldcg(L.mark + ncell);
      if (nmark) {
        const int skr = dr * sgn, skc = dc * sgn;
        const bool pred = !first && (skr == -1 || (skr == 0 && skc == -1)) && kr + skr >= 0 && kc + skc >= 0 && kc + skc < nkc;
        nrec = __ldcg(pred ? cur + ncell : old + ncell);
      }
    }
  }
  unsigned long long mine = 0;
  if (lane == 9 && !first) mine = __ldcg(cur + cell);
  const unsigned long long ref = first ? __shfl_sync(FULLM, nrec, 4) : __shfl_sync(FULLM, mine, 9);
  int2 res;
  int d1;
  sdof_prop_eval(L, r, c, ws, nmark, nrec, res, d1);
  const unsigned long long out = rec_pack(res.x, res.y, d1, 0);
  if ((first || out != ref) && lane == 0) __stcg(cur + cell, out);
  if ((unsigned)out != (unsigned)ref && lane < 4) {  // flow.x | flow.y are the low 32 bits
    // successors in sweep coordinates: (0, +1), (+1, -1), (+1, 0), (+1, +1)
    const int skr = lane == 0 ? 0 : 1, skc = lane == 0 ? 1 : lane - 2;
    const int kr2 = kr + skr, kc2 = kc + skc;
    const int nr = fr + skr * sgn, nc = fc + skc * sgn;
    if (kr2 < nkr && kc2 >= 0 && kc2 < nkc && nr >= 0 && nr < L.cr && nc >= 0 && nc < L.cc) {
      const int ncell = nr * L.cstride + nc;
      if (__ldcg(L.mark + ncell) && atomicMax(L.stamp + ncell, stampval) < stampval) wl_next[atomicAdd(cnt_next, 1)] = ncell;
    }
  }
}

template <int MINB>
__global__ void __launch_bounds__(256, MINB) k_sdof_fused(const SdofFused P) {
  const int lane = threadIdx.x & 31;
  const int gthreads = gridDim.x * blockDim.x, gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nwarps = gthreads >> 5, gwarp = gtid >> 5;
  int gen = 0;
  int* const bar = P.ctr;
  // clear + claim of every scale (a claim depends on nothing but the keypoints)
  for (int scale = P.nscales - 1; scale >= P.min_scale; scale--) {
    const SdofLevel& L = P.L[scale];
    const int total = (L.cr + 2) * L.cstride;
    for (int i = gtid; i < total; i += gthreads) { L.mark[i] = 0; L.owner[i] = INT_MAX; L.stamp[i] = 0; }
  }
  grid_barrier(bar, gen);
  for (int scale = P.nscales - 1; scale >= P.min_scale; scale--) {
    const SdofLevel& L = P.L[scale];
    const int scale_div = 1 << scale;
    for (int i = gtid; i < P.n; i += gthreads) {
      const int kr_ = P.kps[i].r, kc_ = P.kps[i].c;
      if (!kp_in_frame(P.kps[i], P.L[0].i1.nrows, P.L[0].i1.ncols)) continue;
      const int fr = (kr_ / scale_div) / P.patch, fc = (kc_ / scale_div) / P.patch;
      if (fr >= L.cr || fc >= L.cc || kr_ / scale_div >= L.i1.nrows || kc_ / scale_div >= L.i1.ncols) continue;
      atomicMin(&L.owner[fr * L.cstride + fc], i);
    }
  }
  grid_barrier(bar, gen);
  const unsigned long long* coarser_rec = nullptr;  // final records of the scale above
  for (int scale = P.nscales - 1; scale >= P.min_scale; scale--) {
    const SdofLevel& L = P.L[scale];
    const int scale_div = 1 << scale;
    int* const sctr = P.ctr + 8 + 128 * scale;
    // match (:114-143): the owner of a cell (lowest keypoint index == first in serial order), one warp per keypoint
    for (int i = gwarp; i < P.n; i += nwarps) {
      const int kr_ = P.kps[i].r, kc_ = P.kps[i].c;
      if (kr_ < 0 || kc_ < 0) continue;  // warp-uniform
      const int pr = kr_ / scale_div, pc = kc_ / scale_div;
      if (pr >= L.i1.nrows || pc >= L.i1.ncols || pr / P.patch >= L.cr || pc / P.patch >= L.cc) continue;
      const int cell = (pr / P.patch) * L.cstride + (pc / P.patch);
      if (__ldcg(L.owner + cell) != i) continue;  // warp-uniform
      int predr = pr, predc = pc;
      if (coarser_rec) {
        const SdofLevel& C = P.L[scale + 1];
        const int m = (pr / (2 * P.patch)) * C.cstride + (pc / (2 * P.patch));
        if (__ldcg(C.mark + m)) { const unsigned long long cr_ = __ldcg(coarser_rec + m); predr = pr + rec_fx(cr_) * 2; predc = pc + rec_fy(cr_) * 2; }
      }
      int flr, flc, d;
      descent_from_prediction(L.i1, L.i2, pr, pc, predr, predc, P.ws, 5, flr, flc, d);
      if (lane == 0) { __stcg(L.rec + cell, rec_pack(flr, flc, d, 0)); L.mark[cell] = 2; L.mlist[atomicAdd(sctr, 1)] = cell; }
    }
    grid_barrier(bar, gen);
    const int nm = __ldcg(sctr);
    const int nkr = (L.i1.nrows + P.patch - 1) / P.patch, nkc = (L.i1.ncols + P.patch - 1) / P.patch;
    unsigned long long* old = L.rec;
    unsigned long long* cur = L.rec2;
    for (int Ki = 0; Ki < P.propagation; Ki++) {
      const int forward = Ki % 2;  // :191-200: odd iterations forward, even (incl. the first) backward
      int* const cnt = sctr + 4 + 4 * Ki;
      const int stamp0 = Ki << 20;
      for (int i = gwarp; i < nm; i += nwarps)
        sdof_relax_cell(L, old, cur, __ldcg(L.mlist + i), forward, nkr, nkc, P.patch, P.ws, true, stamp0 + 1, L.wl[0], cnt);
      grid_barrier(bar, gen);
      for (int k = 1;; k++) {
        const int nq = __ldcg(cnt + (k - 1) % 3);
        if (nq == 0) break;  // grid-uniform: the counter is stable until every CTA has passed the next barrier
        if (gtid == 0) { cnt[(k + 1) % 3] = 0; P.ctr[1] += 1; P.ctr[2] += nq; }  // statistics: rounds and re-evaluations of the call
        for (int i = gwarp; i < nq; i += nwarps)
          sdof_relax_cell(L, old, cur, __ldcg(L.wl[(k - 1) & 1] + i), forward, nkr, nkc, P.patch, P.ws, false, stamp0 + k + 1, L.wl[k & 1], cnt + k % 3);
        grid_barrier(bar, gen);
      }
      unsigned long long* t = old; old = cur; cur = t;
    }
    coarser_rec = old;  // the last sweep's result (or the matches if there is no sweep)
  }
  // results (:205-212)
  const SdofLevel& L = P.L[P.min_scale];
  const int div = P.patch * (1 << P.min_scale), mul = 1 << P.min_scale;
  for (int i = gtid; i < P.n; i += gthreads) {
    const int kr_ = P.kps[i].r, kc_ = P.kps[i].c;
    const int fr = kr_ / div, fc = kc_ / div;
    int v = 0, pr = 0, pc = 0, d = 0;
    if (kp_in_frame(P.kps[i], P.L[0].i1.nrows, P.L[0].i1.ncols) && fr < L.cr && fc < L.cc && __ldcg(L.mark + fr * L.cstride + fc)) {
      const unsigned long long rc_ = __ldcg(coarser_rec + fr * L.cstride + fc);
      v = 1; pr = kr_ + rec_fx(rc_) * mul; pc = kc_ + rec_fy(rc_) * mul; d = rec_dist(rc_);
    }
    P.out_valid[i] = (unsigned char)v; P.out_pos[i].r = pr; P.out_pos[i].c = pc; P.out_dist[i] = d;
  }
}


__global__ void k_sdof_emit(SdofLevel L, const vppb_int2* kps, int n, int div, int mul, int nrows0, int ncols0, vppb_int2* pos, int* dist,
                            unsigned char* valid) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int fr = kps[i].r / div, fc = kps[i].c / div;
    int v = 0, pr = 0, pc = 0, d = 0;
    if (kp_in_frame(kps[i], nrows0, ncols0) && fr < L.cr && fc < L.cc && L.mark[fr * L.cstride + fc]) {
      const int cell = fr * L.cstride + fc;
      const unsigned long long rc_ = L.rec[cell];
      v = 1; pr = kps[i].r + rec_fx(rc_) * mul; pc = kps[i].c + rec_fy(rc_) * mul; d = rec_dist(rc_);
    }
    valid[i] = (unsigned char)v; pos[i].r = pr; pos[i].c = pc; dist[i] = d;
  }
}

static void cell_dims(int nrows, int ncols, int patch, int level, int& cr, int& cc) {
  cr = nrows / patch; cc = ncols / patch;
  for (int s = 0; s < level; s++) { cr = (int)(1 + cr / 2.f); cc = (int)(1 + cc / 2.f); }  // pyramid.hh:140 on pf_domain
}
// buffers of the dependency-level schedule (sized for the finest scale): level per cell, the cell list, sched[]
static void sched_dims(int nrows, int ncols, int patch, long long& cells, int& cap) {
  const int nkr = (nrows + patch - 1) / patch, nkc = (ncols + patch - 1) / patch;
  cells = (long long)(nkr + 3) * (nkc + 3);
  cap = nkc + 2 * nkr + 2;  // more than the number of anti-diagonals = upper bound of the number of levels
}
constexpr long long kCtrBytes = 8192;  // 2048 ints: dataflow tickets (256) or the relaxation schedule's barrier + 128 per scale
static long long sched_bytes(int nrows, int ncols, int patch) {
  long long cells; int cap;
  sched_dims(nrows, ncols, patch, cells, cap);
  return ((cells * 8 + (2LL + 2LL * (cap + 1)) * 4 + 255) / 256) * 256 + 256 + kCtrBytes;  // + the counters of the dataflow / relaxation sweeps
}
static long long level_bytes(int cr, int cc) {
  const long long cells = (long long)(cr + 2) * (cc + 2);
  return ((cells * (8 + 8 + 4 + 4 + 3 * 4 + 1) + 255) / 256) * 256 + 1024;  // rec, rec2, owner, stamp, mlist + 2 work lists, mark
}

}  // namespace vppb

using namespace vppb;

extern "C" {

int64_t vppb_sdof_workspace_bytes(int32_t nrows, int32_t ncols, const vppb_sdof_params* p) {
  if (!p || p->patchsize <= 0 || p->nscales <= 0 || p->nscales > 8) return 0;
  long long total = 0;
  for (int s = 0; s < p->nscales; s++) { int cr, cc; cell_dims(nrows, ncols, p->patchsize, s, cr, cc); total += level_bytes(cr, cc); }
  return total + sched_bytes(nrows, ncols, p->patchsize);
}

int vppb_sdof_u8(const vppb_img* pyr1, const vppb_img* pyr2, const vppb_sdof_params* p, const vppb_int2* kps, int32_t n, void* workspace,
                 int64_t workspace_bytes, vppb_int2* out_pos, int32_t* out_dist, unsigned char* out_valid, void* stream) {
  VPPB_REQUIRE(pyr1 && pyr2 && p && workspace, VPPB_E_ARG, "vppb_sdof_u8: NULL argument");
  VPPB_REQUIRE(n == 0 || (kps && out_pos && out_dist && out_valid), VPPB_E_ARG, "vppb_sdof_u8: NULL keypoint/output array");
  VPPB_REQUIRE(p->nscales >= 1 && p->nscales <= 8 && p->min_scale >= 0 && p->min_scale < p->nscales && p->patchsize >= 1 && p->winsize >= 1 &&
                   p->winsize <= 15 && p->propagation >= 0, VPPB_E_ARG, "vppb_sdof_u8: parameters out of range");
  VPPB_REQUIRE((uintptr_t)workspace % 256 == 0, VPPB_E_ARG, "vppb_sdof_u8: workspace not 256-byte aligned");
  VPPB_REQUIRE(workspace_bytes >= vppb_sdof_workspace_bytes(pyr1[0].nrows, pyr1[0].ncols, p), VPPB_E_ARG, "vppb_sdof_u8: workspace too small");
  cudaStream_t st = as_stream(stream);
  SdofLevel L[8];
  unsigned char* w = static_cast<unsigned char*>(workspace);
  for (int s = 0; s < p->nscales; s++) {
    VPPB_REQUIRE(pyr1[s].base && pyr2[s].base && pyr1[s].elem_bytes == 1 && pyr2[s].elem_bytes == 1 && same_domain(&pyr1[s], &pyr2[s]), VPPB_E_ARG,
                 "vppb_sdof_u8: level %d images invalid", s);
    // the SAD window is centred on in-domain pixels only, so winsize/2 border pixels suffice (the reference allocates 2*winsize)
    VPPB_REQUIRE(pyr1[s].border >= p->winsize / 2 && pyr2[s].border >= p->winsize / 2, VPPB_E_BORDER, "vppb_sdof_u8: level %d border < winsize/2", s);
    int cr, cc;
    cell_dims(pyr1[0].nrows, pyr1[0].ncols, p->patchsize, s, cr, cc);
    const long long cells = (long long)(cr + 2) * (cc + 2);
    L[s].i1 = view(&pyr1[s]); L[s].i2 = view(&pyr2[s]);
    L[s].cr = cr; L[s].cc = cc; L[s].cstride = cc + 2;
    L[s].rec = reinterpret_cast<unsigned long long*>(w);
    L[s].rec2 = reinterpret_cast<unsigned long long*>(w + cells * 8);
    L[s].owner = reinterpret_cast<int*>(w + cells * 16);
    L[s].stamp = reinterpret_cast<int*>(w + cells * 20);
    L[s].mlist = reinterpret_cast<int*>(w + cells * 24);
    L[s].wl[0] = reinterpret_cast<int*>(w + cells * 28);
    L[s].wl[1] = reinterpret_cast<int*>(w + cells * 32);
    L[s].mark = w + cells * 36;
    w += level_bytes(cr, cc);
  }
  // opt-in: VPPB_SDOF_SCHEDULE=levels runs every sweep as dependency levels of the marked cells when that is shorter than the
  // anti-diagonals (one blocking read-back of the schedule size per sweep), one launch per anti-diagonal otherwise
  const char* sched_env = getenv("VPPB_SDOF_SCHEDULE");
  const bool use_levels = sched_env && strcmp(sched_env, "levels") == 0;
  const bool use_waves = sched_env && strcmp(sched_env, "antidiagonals") == 0;
  const bool use_flags = sched_env && strcmp(sched_env, "dataflow") == 0;  // one persistent launch per sweep, flags between cells
  // default: the relaxation schedule, the whole call in ONE cooperative launch (needs the keypoints' outputs, at most 30 sweeps per scale)
  const bool use_relax = !use_levels && !use_waves && !use_flags && p->propagation <= 30;
  const bool use_dataflow = !use_levels && !use_waves && !use_relax;
  long long sched_cells; int sched_cap;
  sched_dims(pyr1[0].nrows, pyr1[0].ncols, p->patchsize, sched_cells, sched_cap);
  int* lvl = reinterpret_cast<int*>(w);
  unsigned* cell_list = reinterpret_cast<unsigned*>(w + sched_cells * 4);
  int* sched = reinterpret_cast<int*>(w + sched_cells * 8);
  int* tickets = reinterpret_cast<int*>(w + sched_bytes(pyr1[0].nrows, pyr1[0].ncols, p->patchsize) - kCtrBytes);  // 256 counters, one per (scale, sweep)
  // a dataflow sweep publishes its 1-based number in the record's 8-bit stamp: sweep 256 would read as 0 and its successors
  // would wait forever; the tickets hold one counter per (scale, sweep)
  VPPB_REQUIRE(!use_dataflow || (p->propagation <= 255 && p->nscales * p->propagation <= 256), VPPB_E_ARG,
               "vppb_sdof_u8: the dataflow schedule takes at most 255 sweeps per scale and 256 in all");
  if (use_dataflow) VPPB_CUDA(cudaMemsetAsync(tickets, 0, 1024, st));
  if (use_relax) {
    SdofFused F;
    memset(&F, 0, sizeof(F));
    for (int s = 0; s < p->nscales; s++) F.L[s] = L[s];
    F.nscales = p->nscales; F.min_scale = p->min_scale; F.patch = p->patchsize; F.ws = p->winsize; F.propagation = p->propagation; F.n = n;
    F.kps = kps; F.out_pos = out_pos; F.out_dist = out_dist; F.out_valid = out_valid; F.ctr = tickets;
    VPPB_CUDA(cudaMemsetAsync(tickets, 0, kCtrBytes, st));
    // work: a warp per keypoint / marked cell; the grid never exceeds what is resident at once (cooperative launch)
    int cr0, cc0;
    cell_dims(pyr1[0].nrows, pyr1[0].ncols, p->patchsize, p->min_scale, cr0, cc0);
    const long long want_warps = n > (long long)cr0 * cc0 ? n : (long long)cr0 * cc0;
    long long blocks = (want_warps + 7) / 8;
    const char* occ_env = getenv("VPPB_SDOF_OCC");  // experiment knob: CTAs of 256 threads per SM the kernel is compiled for (2, 3 or 4)
    const int occ = occ_env ? atoi(occ_env) : 2;
    void (*kern)(const SdofFused) = occ == 4 ? k_sdof_fused<4> : occ == 3 ? k_sdof_fused<3> : k_sdof_fused<2>;
    const int cap = cooperative_grid_limit(kern, 256);
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    VPPB_CUDA(launch_cooperative(kern, (int)blocks, 256, st, F));
    VPPB_LAUNCH_CHECK("vppb_sdof_u8 (fused)");
    if (getenv("VPPB_SDOF_STATS")) {  // debugging aid: blocks
      int h[3] = {0, 0, 0};
      VPPB_CUDA(cudaMemcpyAsync(h, tickets, sizeof(h), cudaMemcpyDeviceToHost, st));
      VPPB_CUDA(cudaStreamSynchronize(st));
      fprintf(stderr, "vppb_sdof_u8: grid %lld x 256, %d grid barriers, %d relaxation rounds after the first of each sweep, %d re-evaluations\n", blocks,
              h[0] / (int)blocks, h[1], h[2]);
    }
    return VPPB_OK;
  }
  std::vector<int> h_sched;
  const int sms = sm_count();
  for (int scale = p->nscales - 1; scale >= p->min_scale; scale--) {
    const int scale_div = 1 << scale;
    SdofLevel& Ls = L[scale];
    k_sdof_clear<<<sms * 2, 256, 0, st>>>(Ls);
    if (n > 0) {
      k_sdof_claim<<<(n + 255) / 256, 256, 0, st>>>(Ls, kps, n, scale_div, p->patchsize, pyr1[0].nrows, pyr1[0].ncols);
      const int blocks = (n + 3) / 4;
      k_sdof_match<<<blocks < sms * 16 ? blocks : sms * 16, 128, 0, st>>>(Ls, L[scale + 1 < p->nscales ? scale + 1 : scale], scale < p->nscales - 1 ? 1 : 0, kps,
                                                                        n, scale_div, p->patchsize, p->winsize);
    }
    const int nkr = (Ls.i1.nrows + p->patchsize - 1) / p->patchsize, nkc = (Ls.i1.ncols + p->patchsize - 1) / p->patchsize;
    for (int Ki = 0; Ki < p->propagation; Ki++) {
      const int forward = Ki % 2;  // :191-200: odd iterations forward, even (incl. the first) backward
      const int waves = nkc + 2 * (nkr - 1);
      if (use_dataflow) {
        const int blocks = (nkr * nkc + 3) / 4;
        k_sdof_sweep<<<blocks < sms * 8 ? blocks : sms * 8, 128, 0, st>>>(Ls, forward, nkr, nkc, p->patchsize, p->winsize, Ki + 1, tickets + scale * p->propagation + Ki);
        continue;
      }
      if (use_levels) {
        k_sdof_levels<<<1, 1024, 0, st>>>(Ls, forward, nkr, nkc, p->patchsize, lvl, sched, sched_cap, cell_list);
        VPPB_LAUNCH_CHECK("vppb_sdof_u8 (levels)");
        h_sched.assign((size_t)sched_cap + 3, 0);
        VPPB_CUDA(cudaMemcpyAsync(h_sched.data(), sched, ((size_t)sched_cap + 3) * sizeof(int), cudaMemcpyDeviceToHost, st));
        VPPB_CUDA(cudaStreamSynchronize(st));
        const int nlevels = h_sched[0];
        if (nlevels * 2 <= waves) {  // worth it: at most half as many launches as anti-diagonals
          for (int l = 0; l < nlevels; l++) {
            const int first = h_sched[2 + l], cnt = h_sched[2 + l + 1] - first;
            if (cnt <= 0) continue;
            const int blocks = (cnt + 3) / 4;
            k_sdof_prop_list<<<blocks < sms * 16 ? blocks : sms * 16, 128, 0, st>>>(Ls, cell_list + first, cnt, forward, nkc, p->patchsize, p->winsize);
          }
          continue;
        }
      }
      for (int t = 0; t < waves; t++) {
        const int width = (nkr < (nkc + 1) / 2 + 1 ? nkr : (nkc + 1) / 2 + 1);
        const int blocks = (width + 3) / 4;
        k_sdof_prop_wave<<<blocks, 128, 0, st>>>(Ls, t, forward, nkr, nkc, p->patchsize, p->winsize);
      }
    }
  }
  if (n > 0)
    k_sdof_emit<<<(n + 255) / 256, 256, 0, st>>>(L[p->min_scale], kps, n, p->patchsize * (1 << p->min_scale), 1 << p->min_scale, pyr1[0].nrows, pyr1[0].ncols,
                                                 out_pos, out_dist, out_valid);
  VPPB_LAUNCH_CHECK("vppb_sdof_u8");
  return VPPB_OK;
}

}  // extern "C"

// ==== sparse optical flow ========================================================================================================
// FAST keypoints of two frames matched by their patches, optionally refined by Lucas-Kanade.
// Reference: vpp/algorithms/optical_flow.hh:52-73 (the two declared overloads) and optical_flow/sparse_optical_flow.hh:36-112 (a body
// the reference keeps under `#if 0`; it never compiled, so the semantics below are this library's, see DESIGN §3.9).
//
// One call chains the existing entries on one stream: blockwise FAST on both frames (vppb_fast9_u8_async, one workspace reused),
// extract_patches on both keypoint sets, the grid-local SAD matcher, and in subpixel mode vppb_pyrlk_prepare + vppb_lk_match_u8.
// Two kernels of this section fill the gaps: k_sof_seed turns the matches into the integer flow (or LK's keypoints and predictions),
// k_sof_refine computes the SAD between frame 1's patch and frame 2's window at the refined position.  The only host
// synchronisation is the 8-byte read of the two keypoint counts after the detections: the patch, matcher and LK entries take
// their counts on the host.
// It sits in this file, next to the semi-dense flow, because the CPU emulator builds the library's sources from a fixed list.
namespace vppb {

constexpr int SOF_WARPS = 8;  // refine: keypoints (warps) per CTA

// One thread per K1 keypoint.  Integer mode: the outputs themselves.  Subpixel mode: position, LK's float keypoint and its prediction
// (K2[t] - K1[i], or (0, 0) without a match); k_sof_refine writes flow's fate, distance and valid afterwards.
__global__ void __launch_bounds__(256) k_sof_seed(const vppb_int2* k1, const vppb_int2* k2, const int32_t* idx, const int32_t* dist, int n, int nrows,
                                                  int ncols, int subpix, vppb_int2* pos, vppb_float2* flow, int32_t* dout, unsigned char* valid,
                                                  vppb_float2* kf, vppb_float2* pred) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const vppb_int2 p = k1[i];
  const int t = idx[i];
  vppb_float2 f;
  f.r = 0.f;
  f.c = 0.f;
  if (t >= 0) {  // 64-bit difference: a caller keypoint may lie anywhere
    const vppb_int2 q = k2[t];
    f.r = (float)((long long)q.r - p.r);
    f.c = (float)((long long)q.c - p.c);
  }
  pos[i] = p;
  if (subpix) {
    vppb_float2 k;
    k.r = (float)p.r;
    k.c = (float)p.c;
    kf[i] = k;
    pred[i] = f;
    return;
  }
  const bool ok = t >= 0 && p.r >= 0 && p.r < nrows && p.c >= 0 && p.c < ncols;
  vppb_float2 z;
  z.r = 0.f;
  z.c = 0.f;
  flow[i] = ok ? f : z;
  dout[i] = ok ? dist[i] : 0x7fffffff;
  valid[i] = ok ? 1 : 0;
}

// One warp per keypoint: SAD in int between row i of D1 and the winsize x winsize window of i2 centred on (int)(K1[i] + flow),
// truncated toward zero per component (the reference's extract_patch(vfloat2), patch.hh:66-79, in the row-major layout); a window
// that leaves i2's domain plus border, or a non-finite position, counts as all zeros (extract_patches' zero-row rule).  Lane l
// takes the 4-element groups l, l + 32, ... of the flattened window: D1's rows are 16-byte aligned, so its group is one word; the
// window's 4 bytes (consecutive columns of one row of i2, or the end of a row and the start of the next) are gathered, lanes
// reading consecutive bytes of a row; __vsadu4 sums the group.
__global__ void __launch_bounds__(32 * SOF_WARPS) k_sof_refine(Img i2, const vppb_int2* k1, Img d1, int n, int ws, vppb_float2* flow, int32_t* dout,
                                                              unsigned char* valid) {
  const int k = blockIdx.x * SOF_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= n) return;
  const vppb_int2 p = k1[k];
  if (!(p.r >= 0 && p.r < i2.nrows && p.c >= 0 && p.c < i2.ncols)) {  // a caller keypoint outside the frame is never valid
    if (lane == 0) {
      vppb_float2 z;
      z.r = 0.f;
      z.c = 0.f;
      flow[k] = z;
      dout[k] = 0x7fffffff;
      valid[k] = 0;
    }
    return;
  }
  const vppb_float2 f = flow[k];
  const float yr = __fadd_rn((float)p.r, f.r), yc = __fadd_rn((float)p.c, f.c);
  const int h = ws / 2;
  const long long b = i2.border;
  // |y| < 2^30: (int) is defined; any window beyond that lies outside every image the entry accepts
  bool inside = isfinite(yr) && isfinite(yc) && fabsf(yr) < 1073741824.f && fabsf(yc) < 1073741824.f;
  const int cr = inside ? (int)yr : 0, cc = inside ? (int)yc : 0;
  inside = inside && (long long)cr - h >= -b && (long long)cr - h + ws - 1 <= i2.nrows - 1 + b && (long long)cc - h >= -b &&
           (long long)cc - h + ws - 1 <= i2.ncols - 1 + b;
  const unsigned char* drow = d1.base + (long long)k * d1.pitch;
  const unsigned char* w0 = i2.base + (long long)(cr - h) * i2.pitch + (cc - h);
  const int n2 = ws * ws;
  unsigned s = 0;
  for (int g = lane; 4 * g < n2; g += 32) {
    const int e0 = 4 * g;
    unsigned dw, iw = 0;
    if (e0 + 3 < n2) {
      dw = *reinterpret_cast<const unsigned*>(drow + e0);
    } else {
      dw = 0;
      for (int j = 0; e0 + j < n2; j++) dw |= (unsigned)drow[e0 + j] << (8 * j);
    }
    if (inside) {
      int r = e0 / ws, c = e0 - r * ws;
      for (int j = 0; j < 4 && e0 + j < n2; j++) {
        iw |= (unsigned)w0[(long long)r * i2.pitch + c] << (8 * j);
        if (++c == ws) {
          c = 0;
          r++;
        }
      }
    }
    s = __vsadu4(dw, iw) + s;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    dout[k] = (int32_t)s;
    valid[k] = 1;
  }
}

// ---- workspace ----------------------------------------------------------------------------------------------------------------
static int64_t sof_al(int64_t n) { return (n + 255) & ~(int64_t)255; }

struct SofWs {
  int32_t* counts;  // [0] = |K1| (detection), [1] = |K2|
  vppb_int2 *k1, *k2;
  void* fast;
  int64_t fast_bytes;
  unsigned char *d1, *d2;
  int dpitch;
  void* match;
  int64_t match_bytes;
  int32_t *idx, *dist;
  vppb_float2 *kf, *pred;
  float* err;
  unsigned char* pyr;  // prev, next, grad pyramids: 3 * nscales levels, each sof_al(layout total)
  int64_t bytes;
};

static const int SOF_PYR_ALIGN = 128;

static void sof_level_dims(int nrows, int ncols, int l, int& nr, int& nc) {
  nr = nrows;
  nc = ncols;
  for (int k = 0; k < l; k++) {  // pyramid.hh:140,154: 1 + n / 2
    nr = 1 + nr / 2;
    nc = 1 + nc / 2;
  }
}

static int64_t sof_level_bytes(int nr, int nc, int elem, int border) {
  int32_t pitch;
  int64_t total, origin;
  if (vppb_layout(nr, nc, elem, border, SOF_PYR_ALIGN, &pitch, &total, &origin)) return -1;
  return sof_al(total);
}

// Carve the workspace (base may be NULL to size it).  n1 < 0: K1 comes from FAST on i1.
static SofWs sof_ws(unsigned char* base, int nrows, int ncols, const vppb_sof_params& P, int n1) {
  SofWs w;
  const int64_t cells = (int64_t)((nrows + P.block_size - 1) / P.block_size) * ((ncols + P.block_size - 1) / P.block_size);
  const int64_t c1 = n1 < 0 ? cells : n1, c2 = cells;
  const int64_t D = (int64_t)P.winsize * P.winsize;
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    unsigned char* p = base ? base + off : nullptr;
    off += sof_al(bytes);
    return p;
  };
  w.counts = reinterpret_cast<int32_t*>(take(8));
  w.k1 = reinterpret_cast<vppb_int2*>(take(n1 < 0 ? c1 * 8 : 0));
  w.k2 = reinterpret_cast<vppb_int2*>(take(c2 * 8));
  w.fast_bytes = vppb_fast9_workspace_bytes(nrows, ncols, P.block_size);
  w.fast = take(w.fast_bytes);
  w.dpitch = (int)((D + 15) & ~(int64_t)15);
  w.d1 = take(c1 * w.dpitch);
  w.d2 = take(c2 * w.dpitch);
  w.match_bytes = vppb_match_local_sad_workspace_bytes((int32_t)c1, (int32_t)c2, (int32_t)D, P.search_radius, P.cell_width);
  w.match = take(w.match_bytes);
  w.idx = reinterpret_cast<int32_t*>(take(c1 * 4));
  w.dist = reinterpret_cast<int32_t*>(take(c1 * 4));
  w.kf = w.pred = nullptr;
  w.err = nullptr;
  w.pyr = nullptr;
  if (P.subpixelic) {
    w.kf = reinterpret_cast<vppb_float2*>(take(c1 * 8));
    w.pred = reinterpret_cast<vppb_float2*>(take(c1 * 8));
    w.err = reinterpret_cast<float*>(take(c1 * 4));
    w.pyr = base ? base + off : nullptr;
    const int border = P.winsize / 2;
    for (int l = 0; l < P.nscales; l++) {
      int nr, nc;
      sof_level_dims(nrows, ncols, l, nr, nc);
      off += 2 * sof_level_bytes(nr, nc, 1, border) + sof_level_bytes(nr, nc, 8, border);
    }
  }
  w.bytes = off;
  return w;
}

// the argument checks a caller can satisfy: everything but the workspace, the outputs and the keypoint count
static int sof_check_params(const char* fn, int32_t nrows, int32_t ncols, const vppb_sof_params* P) {
  VPPB_REQUIRE(P, VPPB_E_ARG, "%s: NULL params", fn);
  VPPB_REQUIRE(nrows >= 1 && ncols >= 1 && nrows < 65536 && ncols < 65536, VPPB_E_ARG, "%s: image %dx%d outside 1 .. 65535", fn, nrows, ncols);
  VPPB_REQUIRE(P->block_size >= 1 && P->search_radius >= 0 && P->cell_width >= 1, VPPB_E_ARG,
               "%s: block_size %d and cell_width %d must be >= 1, search_radius %d >= 0", fn, P->block_size, P->cell_width, P->search_radius);
  VPPB_REQUIRE(P->winsize >= 1 && P->winsize <= 4096, VPPB_E_ARG, "%s: winsize %d out of [1, 4096]", fn, P->winsize);
  if (P->subpixelic) {
    VPPB_REQUIRE(P->winsize >= 5 && P->winsize <= 15 && (P->winsize & 1), VPPB_E_ARG, "%s: with subpixelic, winsize %d must be odd and in 5 .. 15",
                 fn, P->winsize);
    VPPB_REQUIRE(P->nscales >= 1 && P->nscales <= 8, VPPB_E_ARG, "%s: nscales %d outside 1 .. 8", fn, P->nscales);
    VPPB_REQUIRE(P->lk_iterations >= 0, VPPB_E_ARG, "%s: lk_iterations %d < 0", fn, P->lk_iterations);
  }
  return VPPB_OK;
}

}  // namespace vppb

using namespace vppb;

extern "C" {

int64_t vppb_sparse_flow_workspace_bytes(int32_t nrows, int32_t ncols, const vppb_sof_params* params, int32_t nkeypoints) {
  if (sof_check_params("vppb_sparse_flow_workspace_bytes", nrows, ncols, params)) return 0;
  return sof_ws(nullptr, nrows, ncols, *params, nkeypoints < 0 ? -1 : nkeypoints).bytes;
}

int vppb_sparse_flow_u8(const vppb_img* i1, const vppb_img* i2, const vppb_sof_params* params, const vppb_int2* keypoints, int32_t n,
                        void* workspace, int64_t workspace_bytes, vppb_int2* pos_out, vppb_float2* flow_out, int32_t* dist_out,
                        unsigned char* valid_out, int32_t capacity, int32_t* count_out, void* stream) {
  const char* fn = "vppb_sparse_flow_u8";
  VPPB_REQUIRE(i1 && i2 && i1->base && i2->base && count_out, VPPB_E_ARG, "%s: NULL argument", fn);
  VPPB_REQUIRE(i1->elem_bytes == 1 && i2->elem_bytes == 1, VPPB_E_ARG, "%s: unsigned char images expected", fn);
  VPPB_REQUIRE(same_domain(i1, i2), VPPB_E_ARG, "%s: domains %dx%d and %dx%d differ", fn, i1->nrows, i1->ncols, i2->nrows, i2->ncols);
  int rc = sof_check_params(fn, i1->nrows, i1->ncols, params);
  if (rc) return rc;
  const vppb_sof_params P = *params;
  const int need_border = P.winsize / 2 > 3 ? P.winsize / 2 : 3;
  VPPB_REQUIRE(i1->border >= need_border && i2->border >= need_border, VPPB_E_BORDER, "%s: borders %d and %d < max(3, winsize / 2) = %d", fn,
               i1->border, i2->border, need_border);
  const bool detect = keypoints == nullptr;
  VPPB_REQUIRE(detect || n >= 0, VPPB_E_ARG, "%s: negative keypoint count %d", fn, n);
  VPPB_REQUIRE(capacity >= 0 && (capacity == 0 || (pos_out && flow_out && dist_out && valid_out)), VPPB_E_ARG, "%s: NULL output or negative capacity",
               fn);
  if (P.subpixelic)  // what vppb_pyrlk_prepare checks of the pyramids built here: a mirror border no larger than any level
    for (int l = 0; l < P.nscales; l++) {
      int nr, nc;
      sof_level_dims(i1->nrows, i1->ncols, l, nr, nc);
      VPPB_REQUIRE(P.winsize / 2 <= nr && P.winsize / 2 <= nc, VPPB_E_BORDER, "%s: pyramid level %d (%dx%d) smaller than its border %d", fn, l, nr,
                   nc, P.winsize / 2);
    }
  const SofWs need = sof_ws(nullptr, i1->nrows, i1->ncols, P, detect ? -1 : n);
  VPPB_REQUIRE(workspace && workspace_bytes >= need.bytes && (uintptr_t)workspace % 256 == 0, VPPB_E_ARG,
               "%s: workspace %lld < %lld bytes (or not 256-byte aligned)", fn, (long long)workspace_bytes, (long long)need.bytes);
  if (!detect && n > capacity) {
    *count_out = n;
    VPPB_REQUIRE(false, VPPB_E_CAPACITY, "%s: %d keypoints exceed the capacity %d", fn, n, capacity);
  }
  if (!detect && n == 0) {
    *count_out = 0;
    return VPPB_OK;
  }
  const SofWs w = sof_ws(static_cast<unsigned char*>(workspace), i1->nrows, i1->ncols, P, detect ? -1 : n);
  cudaStream_t st = as_stream(stream);
  const int cells = (int)(((int64_t)(i1->nrows + P.block_size - 1) / P.block_size) * ((i1->ncols + P.block_size - 1) / P.block_size));

  // 1. blockwise FAST on both frames, one workspace; both counts come back in one 8-byte read
  const vppb_int2* k1 = detect ? w.k1 : keypoints;
  if (detect && (rc = vppb_fast9_u8_async(i1, P.detector_th, nullptr, VPPB_FAST_BLOCKWISE, P.block_size, VPPB_FAST_REFERENCE_RING, w.fast, w.fast_bytes,
                                          w.k1, nullptr, cells, w.counts, stream)))
    return rc;
  if ((rc = vppb_fast9_u8_async(i2, P.detector_th, nullptr, VPPB_FAST_BLOCKWISE, P.block_size, VPPB_FAST_REFERENCE_RING, w.fast, w.fast_bytes, w.k2,
                                nullptr, cells, w.counts + 1, stream)))
    return rc;
  int32_t counts[2] = {0, 0};
  VPPB_CUDA(cudaMemcpyAsync(counts, w.counts, sizeof(counts), cudaMemcpyDeviceToHost, st));
  VPPB_CUDA(cudaStreamSynchronize(st));
  const int n1 = detect ? counts[0] : n, n2 = counts[1];
  *count_out = n1;
  VPPB_REQUIRE(n1 <= capacity, VPPB_E_CAPACITY, "%s: %d keypoints exceed the capacity %d", fn, n1, capacity);
  if (n1 == 0) return VPPB_OK;

  // 2. patches of both sets: rows of winsize^2 bytes, 16-byte aligned
  const int D = P.winsize * P.winsize;
  vppb_img d1 = {w.d1, nullptr, n1, D, w.dpitch, 0, 1, 16};
  vppb_img d2 = {n2 ? w.d2 : nullptr, nullptr, n2, D, w.dpitch, 0, 1, 16};
  if ((rc = vppb_extract_patches(i1, k1, n1, P.winsize, &d1, stream))) return rc;
  if ((rc = vppb_extract_patches(i2, w.k2, n2, P.winsize, &d2, stream))) return rc;

  // 3. grid-local SAD match of frame 1's patches (queries) against frame 2's (trains)
  if ((rc = vppb_match_local_sad(&d1, &d2, k1, w.k2, P.search_radius, P.cell_width, w.match, w.match_bytes, w.idx, w.dist, stream))) return rc;
  k_sof_seed<<<(n1 + 255) / 256, 256, 0, st>>>(k1, w.k2, w.idx, w.dist, n1, i1->nrows, i1->ncols, P.subpixelic ? 1 : 0, pos_out, flow_out, dist_out,
                                               valid_out, w.kf, w.pred);
  VPPB_LAUNCH_CHECK(fn);
  if (!P.subpixelic) return VPPB_OK;

  // 4. lucas_kanade(i1, i2, _keypoints = K1, _prediction = integer flow, ...) (lucas_kanade.hpp:135-184), then the SAD at the result
  vppb_img prev[8], next[8], grad[8];
  unsigned char* p = w.pyr;
  const int border = P.winsize / 2;
  for (int l = 0; l < P.nscales; l++) {
    int nr, nc;
    sof_level_dims(i1->nrows, i1->ncols, l, nr, nc);
    const int64_t b1 = sof_level_bytes(nr, nc, 1, border), b8 = sof_level_bytes(nr, nc, 8, border);
    if ((rc = vppb_wrap(&prev[l], p, nr, nc, 1, border, SOF_PYR_ALIGN))) return rc;
    if ((rc = vppb_wrap(&next[l], p + b1, nr, nc, 1, border, SOF_PYR_ALIGN))) return rc;
    if ((rc = vppb_wrap(&grad[l], p + 2 * b1, nr, nc, 8, border, SOF_PYR_ALIGN))) return rc;
    p += 2 * b1 + b8;
  }
  if ((rc = vppb_pyrlk_prepare(i1, i2, prev, next, grad, P.nscales, 0, stream))) return rc;
  vppb_lk_params L;
  L.nlevels = P.nscales;
  L.min_scale = 0;
  L.winsize = P.winsize;
  L.max_iter = P.lk_iterations;
  L.grad_is_float = 0;
  L.err_mode = VPPB_LK_ERR_SAD;
  L.gate_on_max_err = 0;
  L.min_ev = 0.f;  // lucas_kanade.hpp:143-144 keeps min_ev = 0.0001 and delta = 0.1 in int
  L.delta = 0.f;
  L.max_err = 0.f;
  L.factor = 2.f;
  L.pred_div = (float)(1 << P.nscales);  // lucas_kanade.hpp:163
  if ((rc = vppb_lk_match_u8(prev, next, grad, &L, w.kf, w.pred, n1, flow_out, w.err, stream))) return rc;
  k_sof_refine<<<(n1 + SOF_WARPS - 1) / SOF_WARPS, 32 * SOF_WARPS, 0, st>>>(view(i2), k1, view(&d1), n1, P.winsize, flow_out, dist_out, valid_out);
  VPPB_LAUNCH_CHECK(fn);
  return VPPB_OK;
}

}  // extern "C"
