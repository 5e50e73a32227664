// Plain LSU copies of the box headline's bytes for tools/box_ceiling.py (not part of libvppb).  A launch covers n image pairs;
// a CTA owns one task = (image, band of rows, segment of seg_bytes bytes of the row) and walks down its rows, one 16-byte group per
// thread, U rows of loads in flight before their stores.  "strips" = 1920-byte segments over all rows (the streaming box kernel's
// column-strip traffic), "bands" = whole rows over a band of rows.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -Xcompiler -fPIC -shared -o box_ceiling.so box_ceiling.cu
#include <cuda_runtime.h>
#include <stdint.h>

enum { M_COPY = 0, M_READ = 1, M_WRITE = 2 };
constexpr int U = 8;

struct CopyArgs {
  const unsigned long long* in;   // device array of n input pixel (0,0) addresses
  const unsigned long long* out;  // device array of n output addresses
  int in_pitch, out_pitch, nrows, rowbytes;
  int seg_bytes, segs, band_rows, bands;
  unsigned* sink;                 // the read-only pass folds its loads into one word per thread; written only for one unlikely value
};

__device__ __forceinline__ uint4 ld16(const unsigned char* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st16(unsigned char* p, uint4 v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

template <int MODE>
__global__ void k_ceiling(CopyArgs a) {
  const int per_img = a.segs * a.bands;
  const int img = blockIdx.x / per_img, rem = blockIdx.x - img * per_img;
  const int band = rem / a.segs, seg = rem - band * a.segs;
  const int xo = 16 * threadIdx.x;
  const int x = seg * a.seg_bytes + xo;
  if (xo >= a.seg_bytes || x + 16 > a.rowbytes) return;
  const int y0 = band * a.band_rows, y1 = min(a.nrows, y0 + a.band_rows);
  const unsigned char* src = reinterpret_cast<const unsigned char*>(a.in[img]) + x;
  unsigned char* dst = reinterpret_cast<unsigned char*>(a.out[img]) + x;
  uint4 acc = make_uint4(0, 0, 0, 0);
  for (int y = y0; y < y1; y += U) {
    uint4 v[U];
    if (MODE != M_WRITE) {
#pragma unroll
      for (int u = 0; u < U; u++)
        if (y + u < y1) v[u] = ld16(src + (long long)(y + u) * a.in_pitch);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (y + u >= y1) break;
      if (MODE == M_COPY) st16(dst + (long long)(y + u) * a.out_pitch, v[u]);
      if (MODE == M_WRITE) st16(dst + (long long)(y + u) * a.out_pitch, make_uint4(y + u, x, img, 0));
      if (MODE == M_READ) { acc.x ^= v[u].x; acc.y ^= v[u].y; acc.z ^= v[u].z; acc.w ^= v[u].w; }
    }
  }
  if (MODE == M_READ && acc.x == 0x12345678u && acc.y == 0x9abcdef0u) a.sink[0] = acc.z;
}

extern "C" {

// mode: 0 copy, 1 read only, 2 write only; block = threads per CTA (>= seg_bytes / 16)
int ceiling_launch(int mode, const unsigned long long* in, const unsigned long long* out, int n, int in_pitch, int out_pitch, int nrows,
                   int rowbytes, int seg_bytes, int band_rows, int block, unsigned* sink, void* stream) {
  CopyArgs a;
  a.in = in; a.out = out; a.in_pitch = in_pitch; a.out_pitch = out_pitch; a.nrows = nrows; a.rowbytes = rowbytes;
  a.seg_bytes = seg_bytes; a.segs = (rowbytes + seg_bytes - 1) / seg_bytes;
  a.band_rows = band_rows; a.bands = (nrows + band_rows - 1) / band_rows; a.sink = sink;
  const int grid = n * a.segs * a.bands;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (mode == M_COPY) k_ceiling<M_COPY><<<grid, block, 0, st>>>(a);
  else if (mode == M_READ) k_ceiling<M_READ><<<grid, block, 0, st>>>(a);
  else k_ceiling<M_WRITE><<<grid, block, 0, st>>>(a);
  return (int)cudaGetLastError();
}

// cudaMemcpy2DAsync of every pair (host arrays of device addresses)
int ceiling_memcpy2d(const unsigned long long* in, const unsigned long long* out, int n, int in_pitch, int out_pitch, int nrows, int rowbytes,
                     void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int i = 0; i < n; i++) {
    cudaError_t e = cudaMemcpy2DAsync(reinterpret_cast<void*>(out[i]), out_pitch, reinterpret_cast<const void*>(in[i]), in_pitch, rowbytes, nrows,
                                      cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) return (int)e;
  }
  return 0;
}
}
