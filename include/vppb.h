/*
 * vppb.h — C-ABI of the H100-native dense-pixel path behind the Video++ (matt-42/vpp) API.
 *
 * Video++ is a header-only C++14 template library, so the reference has no FFI of its own for
 * this path: the boundary it exposes is the template API of vpp/core and vpp/algorithms.  This
 * header is the thin extern-"C" shim the new C++14 headers (vpp_b200/include/vpp) and the
 * Python/ctypes host (vpp_b200/capi.py) bind to; every entry point cites the reference
 * template (file:line, relative to the reference tree) whose work it performs on the GPU.
 *
 * Conventions
 *   - every function returns an int status: 0 = OK, <0 = VPPB_E_* ; vppb_last_error() gives text.
 *   - plain pointers and sizes only; `stream` is a cudaStream_t passed as void* (NULL = default).
 *   - coordinates are (row, col) as in the reference (vint2{r,c}).
 *   - images are described by vppb_img: `base` is the DEVICE address of pixel (0,0); rows are
 *     `pitch` bytes apart; `border` rows/cols of real, addressable memory surround the domain
 *     (imageNd.hpp:151-196).  No function allocates device memory unless it says so.
 *   - there is no CPU fallback: without a CUDA device every compute entry returns VPPB_E_CUDA.
 */
#ifndef VPPB_H_
#define VPPB_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VPPB_VERSION 100

enum {
  VPPB_OK = 0,
  VPPB_E_CUDA = -1,     /* CUDA runtime / driver error (text in vppb_last_error) */
  VPPB_E_ARG = -2,      /* invalid argument (NULL image, mismatched domains, bad element size) */
  VPPB_E_BORDER = -3,   /* image border too small for the stencil (fast.hpp:937-938 throws here) */
  VPPB_E_CAPACITY = -4, /* output capacity too small; count_out holds the required size */
  VPPB_E_NCCL = -5
};

/* imageNd<V,2> descriptor (imageNd.hh:16-40 imageNd_data). */
typedef struct vppb_img {
  void* base;         /* device pointer to pixel (0,0) == imageNd_data::begin_ */
  void* alloc;        /* start of the owned allocation (NULL for borrowed/_data views and subimages) */
  int32_t nrows;      /* domain rows */
  int32_t ncols;      /* domain cols */
  int32_t pitch;      /* bytes between successive rows */
  int32_t border;     /* addressable border pixels on each side */
  int32_t elem_bytes; /* sizeof(V): 1 (u8), 3 (vuchar3), 4 (int/float), 8 (vint2/vfloat2) ... */
  int32_t align;      /* row alignment in bytes the allocation was made with (0 = unknown) */
} vppb_img;

/* keypoint / flow records exchanged with the host (vint2 / vfloat2 are (row, col)). */
typedef struct vppb_int2 { int32_t r, c; } vppb_int2;
typedef struct vppb_float2 { float r, c; } vppb_float2;

/* ---- library ---------------------------------------------------------------------------- */
int vppb_version(void);
const char* vppb_last_error(void);
/* Select the CUDA device used by the calling thread and warm the context. */
int vppb_init(int device);
int vppb_device_count(int* n);
int vppb_sync(void* stream);

/* ---- image2d<V> storage (imageNd.hpp:151-196 allocate; :224-234 coords_to_offset) --------- */
/* Host-only layout arithmetic (no GPU needed): pitch, total buffer bytes and the byte offset of
 * pixel (0,0) from the aligned buffer start for an image of nrows x ncols elements of elem_bytes
 * with `border` and row alignment `align` (reference default 16/32, ours 128). */
int vppb_layout(int32_t nrows, int32_t ncols, int32_t elem_bytes, int32_t border, int32_t align,
                int32_t* pitch, int64_t* total_bytes, int64_t* origin_offset);
/* cudaMalloc an image with the reference layout; border content is uninitialised (as malloc). */
int vppb_alloc(vppb_img* out, int32_t nrows, int32_t ncols, int32_t elem_bytes, int32_t border, int32_t align);
/* Describe an image inside a caller-owned device buffer of at least total_bytes (vppb_layout)
 * — the `_data=`/`_pitch=` constructor (imageNd.hpp:99-141) for buffers laid out by vppb_layout. */
int vppb_wrap(vppb_img* out, void* device_buffer, int32_t nrows, int32_t ncols, int32_t elem_bytes,
              int32_t border, int32_t align);
int vppb_free(vppb_img* img);
/* img | box  (imageNd.hpp:324-341): view of rows [r0,r1] x cols [c0,c1], re-based to (0,0). */
int vppb_subimage(const vppb_img* img, int32_t r0, int32_t c0, int32_t r1, int32_t c1, vppb_img* out);
/* Host <-> device.  `host` addresses host pixel (0,0), rows host_pitch bytes apart; with_border
 * != 0 also transfers the border frame (host buffer must hold it at negative offsets). */
int vppb_upload(const vppb_img* dst, const void* host, int64_t host_pitch, int with_border, void* stream);
int vppb_download(const vppb_img* src, void* host, int64_t host_pitch, int with_border, void* stream);

/* ---- pixel_wise named kernels (pixel_wise.hpp:69-165) ------------------------------------- */
/* pixel_wise(A,B,C) | [](int& a,int& b,int& c){ a = b + c; }   benchmarks/image_add.cc:51-57 */
int vppb_pw_add_i32(const vppb_img* a, const vppb_img* b, const vppb_img* c, void* stream);
/* fill(img, v) fill.hh:12-15; `value` points to elem_bytes host bytes. with_border -> fill.hh:24-28 */
int vppb_fill(const vppb_img* img, const void* value, int with_border, void* stream);
/* copy(src,dst) copy.hh:10-19 (with_border=0) / copy_with_border copy.hh:22-27 (with_border=1) */
int vppb_copy2d(const vppb_img* src, const vppb_img* dst, int with_border, void* stream);
/* copy(src, dst) + fill_border_mirror(dst) in one launch (pyramid2d::update: copy then mirror, pyramid.hh:170,196).
 * Equal domains; dst->border <= dst size. */
int vppb_copy2d_mirror(const vppb_img* src, const vppb_img* dst, void* stream);
/* fill_border_with_value fill.hh:32-45 / fill_border_mirror :48-83 / fill_border_closest :86-121 */
int vppb_fill_border_value(const vppb_img* img, const void* value, void* stream);
int vppb_fill_border_mirror(const vppb_img* img, void* stream);
int vppb_fill_border_closest(const vppb_img* img, void* stream);
/* sum(img) sum.hh:12-19 for u8 / i8 / i32 images: promoted (int) accumulator, wraps like int. */
int vppb_sum_i32(const vppb_img* img, int is_signed, int64_t* out_host, void* stream);

/* ---- 5x5 box stencil (relative_access / box_nbh2d user kernel) ---------------------------- */
/* out = (sum of the 25 neighbours) / 25 per channel, integer division.
 * u8c3: image2d<vuchar3> (BASELINE config 2; vint3 accumulate, examples/box_filter.cc:23-32 form)
 * i32 : image2d<int>     (benchmarks/box_5x5_filter2.cc:71-81).  `in` needs border >= 2, filled. */
int vppb_box5x5_u8c3(const vppb_img* in, const vppb_img* out, void* stream);
int vppb_box5x5_i32(const vppb_img* in, const vppb_img* out, void* stream);
/* same on single-channel u8 (image2d<unsigned char>) */
int vppb_box5x5_u8(const vppb_img* in, const vppb_img* out, void* stream);
/* The same filter over a batch of n image pairs (the frames of a video step) with as few launches as possible: equally
 * shaped library-layout images go through ONE persistent launch per 32 images (the per-launch ramp-up and tail, which
 * rival the run time of a whole 1080p frame, are paid once per batch); any other mix is processed image by image.
 * ins / outs: arrays of n descriptors.  Results are identical to n calls of the single-image entry. */
int vppb_box5x5_u8c3_batch(const vppb_img* ins, const vppb_img* outs, int32_t n, void* stream);
int vppb_box5x5_u8_batch(const vppb_img* ins, const vppb_img* outs, int32_t n, void* stream);

/* ---- frame ingest: rgb_to_graylevel (colorspace_conversions.hh:10-47), SURVEY 8(f) N1 ------------------- */
/* out(p) = (in(p)[0] + in(p)[1] + in(p)[2]) / 3 (int, truncating) over out's domain_with_border, as
 * rgb_to_graylevel<unsigned char>(image2d<vuchar3 | vuchar4>) does; in: 3- or 4-byte pixels (4th channel ignored),
 * out: u8, same domain, in->border >= out->border (the reference builds `out` with the input's border). */
int vppb_rgb_to_graylevel_u8(const vppb_img* in, const vppb_img* out, void* stream);
/* The ingest every caller performs before the path - clone(frame, _border = b); fill_border_mirror;
 * rgb_to_graylevel (examples/video_extruder.cc:46-48) - in one launch: converts the domain and writes out's mirror
 * border from the mirrored domain pixels.  `in` needs no border (a decoder surface: tight rows are fine). */
int vppb_rgb_to_graylevel_u8_mirror(const vppb_img* in, const vppb_img* out, void* stream);

/* ---- Scharr + pyramid (scharr.hh:46-87, pyramid.hh:12-81,133-198) ------------------------- */
/* scharr(in u8, out vector<Vt,2>): out elem 8 bytes; as_float=0 -> vint2 (truncated), 1 -> vfloat2 */
int vppb_scharr_u8(const vppb_img* in, const vppb_img* out, int as_float, void* stream);
/* scharr + fill_border_mirror(out) in one launch (the gradient level 0 of lucas_kanade.hpp:156-157 /
 * video_extruder.hpp: scharr, then pyramid2d::propagate_level0 mirrors it first).  out->border <= out size. */
int vppb_scharr_u8_mirror(const vppb_img* in, const vppb_img* out, int as_float, void* stream);
/* One pyramid step: out(r,c) = lowpass5x5sep(in)(2r,2c)  (antialiasing_lowpass_filter + subsample2,
 * fused; the mirror-filled H temp of pyramid.hh:36 is reproduced by index mirroring).
 * kind: 0 = u8, 1 = vint2 (integer /16 per component), 2 = vfloat2.  `in` needs border >= 2, filled. */
int vppb_lowpass_sub2(const vppb_img* in, const vppb_img* out, int kind, void* stream);
/* The same step followed by fill_border_mirror(out) (what pyramid2d::propagate_level0 does for every level,
 * pyramid.hh:169-192), in ONE launch: the thread that produces out(r,c) also writes the <= 8 border pixels
 * that mirror it.  Needs out->border <= min(out->nrows, out->ncols) (VPPB_E_BORDER otherwise). */
int vppb_lowpass_sub2_mirror(const vppb_img* in, const vppb_img* out, int kind, void* stream);

/* Everything lucas_kanade() / a pyrlk_match caller builds before matching, in one call: pyramid2d<uchar>::update(i1) -> prev[],
 * ::update(i2) -> next[], scharr(prev[0], grad[0]) + propagate_level0 -> grad[] (lucas_kanade.hpp:150-157).  prev / next /
 * grad: nlevels descriptors each (allocated by the caller, borders >= 2 / >= 1; all distinct buffers); grad may be NULL: only the two
 * u8 pyramids are built (what semi_dense_optical_flow.hpp:70-100 needs).  Two forms: one launch per step with the three independent
 * chains on three streams forked from / joined into `stream` (default with a gradient pyramid), or ONE cooperative launch - the steps of
 * a level concatenated into a phase of work items, grid-wide barriers between the levels - for images in the library layout (16-byte
 * aligned rows, <= 8 levels; default without a gradient pyramid, which falls back to the streams form when the images or the level count
 * do not fit it).  VPPB_PREPARE=fused|streams overrides the choice; under `fused` a call that does not fit returns VPPB_E_ARG and says why
 * (the layout or more than 8 levels).  1 <= nlevels <= 16.  Every step is checked as its stand-alone entry point checks it
 * (vppb_copy2d_mirror, vppb_scharr_u8_mirror, vppb_lowpass_sub2_mirror) before anything is queued: a call rejected with VPPB_E_ARG or
 * VPPB_E_BORDER writes nothing. */
int vppb_pyrlk_prepare(const vppb_img* i1, const vppb_img* i2, const vppb_img* prev, const vppb_img* next, const vppb_img* grad,
                       int32_t nlevels, int32_t grad_is_float, void* stream);

/* ---- FAST9 (fast.hpp:253-508, 643-799, 889-955) ------------------------------------------- */
enum { VPPB_FAST_REFERENCE_RING = 0, VPPB_FAST_TRUE_RING = 1 };
enum { VPPB_FAST_ALL = 0, VPPB_FAST_LOCAL_MAXIMA = 1, VPPB_FAST_BLOCKWISE = 2 };
/* Workspace bytes needed by vppb_fast9_u8 for an nrows x ncols image (block_size: the blockwise cell side, or <= 0
 * for a workspace that is large enough for every mode and block size).  The workspace must be 256-byte aligned (any vppb_alloc or
 * cudaMalloc pointer is): vppb_fast9_u8, _async and vppb_fast9_blockwise_rank_u8 return VPPB_E_ARG for any other pointer. */
int64_t vppb_fast9_workspace_bytes(int32_t nrows, int32_t ncols, int32_t block_size);
/* fast9(A, th, [_local_maxima|_blockwise, _block_size=, _mask=, _scores=]).
 * mask may be NULL (== 0xFF everywhere).  kps_out (device, capacity records) receives the
 * keypoints in raster order; scores_out (device int32, may be NULL) the matching scores
 * (raw score for mode ALL, score/16 for the maxima modes, fast.hpp:670-671,698-704);
 * count_out (host) the number of keypoints found.  ring selects the reference's ring
 * (a4/a12 sampled on row r-3, fast.hpp:367-368) or the true Bresenham ring. */
int vppb_fast9_u8(const vppb_img* img, int32_t th, const vppb_img* mask, int32_t mode, int32_t block_size,
                  int32_t ring, void* workspace, int64_t workspace_bytes,
                  vppb_int2* kps_out, int32_t* scores_out, int32_t capacity, int32_t* count_out,
                  void* stream);
/* The same without any host synchronisation: the keypoint count is stored to count_dev (DEVICE int32), keypoints
 * beyond `capacity` are dropped (the count still tells how many there were).  What a pipeline that keeps its keypoints
 * on the device (video_extruder) calls; fast9() itself reads count_dev back once to size its std::vector. */
int vppb_fast9_u8_async(const vppb_img* img, int32_t th, const vppb_img* mask, int32_t mode, int32_t block_size,
                        int32_t ring, void* workspace, int64_t workspace_bytes,
                        vppb_int2* kps_out, int32_t* scores_out, int32_t capacity, int32_t* count_dev,
                        void* stream);
/* fast9_scores (fast.hpp:643-652): score of n given points (device arrays). */
int vppb_fast9_scores(const vppb_img* img, int32_t th, const vppb_int2* kps, int32_t n, int32_t* scores_out,
                      void* stream);

/* fast_detector9_blockwise_rank (fast.hpp:801-886, on fast_detector9_maxima2 fast.hpp:710-740): up to max_points (<= 16) ranked
 * keypoints per block_size x block_size block - the strict 3x3 maxima of the RAW score image (0 where nothing was detected), kept by
 * the reference's table rule and sorted by decreasing score.  kps3_out (device int32 triples): (row, col, rank), blocks in raster
 * order, ranks ascending; scores_out (device, may be NULL): raw scores; count_out (host).  Synchronises the stream.  Workspace:
 * 256-byte aligned (VPPB_E_ARG otherwise). */
int64_t vppb_fast9_rank_workspace_bytes(int32_t nrows, int32_t ncols, int32_t block_size, int32_t max_points);
int vppb_fast9_blockwise_rank_u8(const vppb_img* img, int32_t th, const vppb_img* mask, int32_t block_size, int32_t max_points,
                                 int32_t ring, void* workspace, int64_t workspace_bytes, int32_t* kps3_out, int32_t* scores_out,
                                 int32_t capacity, int32_t* count_out, void* stream);

/* ---- the remaining 3x3 stencils of the path (SURVEY 8(f) N4) ------------------------------- */
/* lbp_transform(A, B) (lbp_transform.hh:7-38), unsigned char -> unsigned char: bit k of B(r, c) = neighbour k of A(r, c) > A(r, c),
 * neighbours in raster order without the centre.  A needs a border >= 1, read as it is (the caller fills it). */
int vppb_lbp_u8(const vppb_img* in, const vppb_img* out, void* stream);
/* local_maxima_filter(A, nbh_size) (fast.hpp:555-575; nbh_size is ignored there too): IN PLACE, a pixel that is not strictly greater
 * than its 8 neighbours becomes 0 - with the reference's serial raster-order semantics (the neighbours above and to the left have
 * already been filtered).  unsigned char or int pixels, border >= 1 (read, never written).  One cooperative launch.  The workspace
 * (at least vppb_local_maxima_filter_workspace_bytes bytes) must be 256-byte aligned (VPPB_E_ARG otherwise). */
int64_t vppb_local_maxima_filter_workspace_bytes(int32_t nrows, int32_t ncols, int32_t elem_bytes);
int vppb_local_maxima_filter(const vppb_img* img, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- chamfer distance transforms (distance_transforms.hh:86-152) --------------------------------------------------------- */
/* d4_ / d8_ / d3_4_ / d5_7_11_distance_transform(A, S): the reference's generic_incremental_distance_transform with its four masks
 * (fill_with_border(S, B = nrows + ncols); S = 0 where A == 0; a forward and a backward raster pass), computed in parallel with the
 * identical result: every border pixel of `out`, at its whole width (a view's border is its parent's memory), becomes B, and every
 * domain pixel the mask distance to the nearest zero of `in`, capped at B.  `in`: unsigned char or int pixels compared with 0, its
 * border is not read; `out`: int, same domain, border >= 1 (>= 2 for d5-7-11: VPPB_E_BORDER), no memory shared with `in` (VPPB_E_ARG).
 * Pitch padding is never written.  A fixed number of launches per mask, no host synchronisation; `workspace` is device memory of at
 * least vppb_distance_transform_workspace_bytes bytes, 8-byte aligned (VPPB_E_ARG otherwise, unless that size is 0), used until the
 * work queued on `stream` completes. */
enum { VPPB_DT_D4 = 0, VPPB_DT_D8 = 1, VPPB_DT_D3_4 = 2, VPPB_DT_D5_7_11 = 3 };
int64_t vppb_distance_transform_workspace_bytes(int32_t nrows, int32_t ncols, int32_t kind);
int vppb_distance_transform(const vppb_img* in, const vppb_img* out, int32_t kind, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- SAD descriptor matching (descriptor_matcher/*.hh) and patch extraction (core/patch.hh:32-47) ------------------------- */
/* Descriptors are the rows of an image: `query` and `train` hold one descriptor per row, ncols = its length (>= 1, the same for
 * both), elem_bytes 1 (unsigned char) or 4 (int, rows 4-byte aligned), any pitch, views included.  The distance is the reference's
 * sad_distance (distances.hh:9-30), sum |q[k] - t[k]| in int, always summed in full (its early exit only drops candidates that
 * cannot win); for int descriptors the results are defined when every SAD fits in int32, as in the reference.  index_out and
 * dist_out are device arrays of query->nrows entries; a query without a candidate gets index -1 and distance INT32_MAX.  Nothing
 * synchronises the host; `workspace` is device memory of at least the *_workspace_bytes bytes, used until the work queued on
 * `stream` completes.  Every argument the host can see is checked before anything is queued: a rejected call writes nothing. */
/* bruteforce_matcher with sad_distance (bruteforce_matcher.hh:11-47): for every query i the train j of smallest SAD, ties to the
 * lowest j (the reference's strict < scan from j = 0) - index and distance equal the reference's.  Without trains every query
 * gets (-1, INT32_MAX), where the reference reads train 0 out of bounds.  Workspace: 8 bytes per query, 8-byte aligned. */
int64_t vppb_match_bruteforce_sad_workspace_bytes(int32_t nquery, int32_t ntrain, int32_t ncols);
int vppb_match_bruteforce_sad(const vppb_img* query, const vppb_img* train, void* workspace, int64_t workspace_bytes, int32_t* index_out,
                              int32_t* dist_out, void* stream);
/* local_index1d_sad_descriptor_matcher (local_index1d_sad_descriptor_matcher.hh:10-57, grid_index.hh:11-88, index1d.hh) at
 * _approximation = 1: a train's cell is (p.r / s, p.c / s), C division, s = cell_width >= 1; a query's window is the inclusive box
 * of cells ((q - R) / s, (q + R) / s), R = search_radius >= 0 (whole cells, not a disc of radius R).  The result is the smallest SAD
 * over the trains of the window's cells, ties to the smallest (cell row, cell col, train index).  The distance always equals the
 * reference's; the index equals it wherever the reference's choice is determined - inside one cell the reference orders ties by an
 * unstable std::sort (index1d.hh:41-45).  A train at a coordinate <= -s is never matched (the reference asserts).  Positions are
 * DEVICE arrays of (row, col).  Workspace (256-byte aligned) depends on ntrain only; the trains are binned by a stable device-side
 * radix sort on their cell. */
int64_t vppb_match_local_sad_workspace_bytes(int32_t nquery, int32_t ntrain, int32_t ncols, int32_t search_radius, int32_t cell_width);
int vppb_match_local_sad(const vppb_img* query, const vppb_img* train, const vppb_int2* query_positions, const vppb_int2* train_positions,
                         int32_t search_radius, int32_t cell_width, void* workspace, int64_t workspace_bytes, int32_t* index_out,
                         int32_t* dist_out, void* stream);
/* extract_patches(kps, img, winsize) (patch.hh:32-47): row k of `out` (n x winsize^2, img's element type) is the winsize x winsize
 * window centred on keypoints[k] (a DEVICE array), row-major from element 0: element (r + h) * winsize + (c + h) for r, c in
 * [-h, winsize - h), h = winsize / 2.  Deviation: the reference writes element r * winsize + c, before each row (out of bounds
 * for keypoint 0); this is the layout it plainly intends.  `img`: unsigned char or int, border >= h (VPPB_E_BORDER); a keypoint
 * whose window leaves the domain plus border gets a zero row (decided per keypoint on the device). */
int vppb_extract_patches(const vppb_img* img, const vppb_int2* keypoints, int32_t n, int32_t winsize, const vppb_img* out, void* stream);

/* ---- Lucas-Kanade (lucas_kanade.hpp:12-184, lk.hh:42-175, pyrlk_match.hh:15-55) ----------- */
enum { VPPB_LK_ERR_SAD = 0 /* lucas_kanade.hpp:116-128 */, VPPB_LK_ERR_SAD_OVER_MAD = 1 /* lk.hh:151-173 */ };
typedef struct vppb_lk_params {
  int32_t nlevels;      /* pyramid levels passed in prev/next/grad (level 0 = full resolution) */
  int32_t min_scale;    /* finest level processed (pyrlk_match.hh:32) */
  int32_t winsize;      /* square window side (odd, <= 15) */
  int32_t max_iter;     /* loop runs k = 0..max_iter inclusive (lucas_kanade.hpp:87) */
  int32_t grad_is_float;/* gradient pyramid element: 0 = vint2, 1 = vfloat2 */
  int32_t err_mode;     /* VPPB_LK_ERR_* */
  int32_t gate_on_max_err; /* 1: pyrlk_match.hh:37-41 (tr updated only if err < max_err); 0: lucas_kanade.hpp:177 */
  float min_ev;         /* reject if min |eig(G/cpt)| < min_ev */
  float delta;          /* convergence threshold on ||nk|| */
  float max_err;
  float factor;         /* pyramid factor (2) */
  float pred_div;       /* prediction divisor 2^nscales of lucas_kanade.hpp:163 */
} vppb_lk_params;
/* For each of n keypoints (device vppb_float2, (row,col) at level 0; `prediction` may be NULL):
 * coarse-to-fine LK; flow_out[i] = final tr, err_out[i] = final distance. u8 images. */
int vppb_lk_match_u8(const vppb_img* prev, const vppb_img* next, const vppb_img* grad,
                     const vppb_lk_params* params, const vppb_float2* kps, const vppb_float2* prediction,
                     int32_t n, vppb_float2* flow_out, float* err_out, void* stream);

/* oriented_lk_match_point_square_win<WS>::operator() (lk.hh:180-317) for n points of ONE level: template window rotated to dir1[i],
 * search window rotated to dir2[i] (unit vectors, (row, col)), steps clamped to max_step_norm, at most max_iter steps.
 * flow_out[i] = v - p or the reference's failure codes ((-1,-1) / (0,0) with err FLT_MAX); err = SAD / (cpt * MAD). */
int vppb_lk_match_oriented_u8(const vppb_img* a, const vppb_img* b, const vppb_img* grad, int32_t grad_is_float, int32_t winsize,
                              float min_ev, int32_t max_iter, float delta, float max_step_norm, const vppb_float2* kps,
                              const vppb_float2* prediction, const vppb_float2* dir1, const vppb_float2* dir2, int32_t n,
                              vppb_float2* flow_out, float* err_out, void* stream);

/* ---- semi-dense optical flow of video_extruder (semi_dense_optical_flow.hpp:46-214, gradient_descent.hh:10-89) --- */
typedef struct vppb_sdof_params {
  int32_t winsize;      /* SAD window side, 1..15 (reference default 7; video_extruder passes 9) */
  int32_t nscales;      /* pyramid levels, 1..8 */
  int32_t min_scale;    /* finest level processed, 0..nscales-1 */
  int32_t propagation;  /* number of neighbour-propagation sweeps per scale, >= 0 (even sweeps backward, odd forward) */
  int32_t patchsize;    /* cell side, >= 1 */
} vppb_sdof_params;
/* Workspace bytes of vppb_sdof_u8; the workspace must be 256-byte aligned (VPPB_E_ARG otherwise). */
int64_t vppb_sdof_workspace_bytes(int32_t nrows, int32_t ncols, const vppb_sdof_params* params);
/* pyr1 / pyr2: `nscales` u8 pyramid levels of the two frames (pyramid2d<uchar>(img, nscales, 2, _border >= winsize/2),
 * borders mirror-filled).  kps: n device (row, col) records.  For keypoint i, out_valid[i] tells whether the reference
 * would call match_callback(i, out_pos[i], out_dist[i]).  Serial semantics of the reference: the first keypoint (lowest
 * index) of a cell claims it; propagation sweeps are Gauss-Seidel in the reference's raster orders.  Schedules: with
 * propagation <= 30 the whole call is one cooperative launch that solves each sweep by relaxation; above 30, and under
 * VPPB_SDOF_SCHEDULE=dataflow, one persistent launch per sweep, which takes at most 255 sweeps per scale and
 * nscales * propagation <= 256 (VPPB_E_ARG otherwise, before anything is launched).  VPPB_SDOF_SCHEDULE=levels and
 * =antidiagonals take any number of sweeps. */
int vppb_sdof_u8(const vppb_img* pyr1, const vppb_img* pyr2, const vppb_sdof_params* params, const vppb_int2* kps, int32_t n,
                 void* workspace, int64_t workspace_bytes, vppb_int2* out_pos, int32_t* out_dist, unsigned char* out_valid,
                 void* stream);

/* ---- sparse optical flow (optical_flow.hh:52-73, optical_flow/sparse_optical_flow.hh:36-112; the reference body never compiled,
 * so these are this library's semantics, DESIGN §3.9) ------------------------------------------------------------------------------
 * K1 = fast9(i1, detector_th, _blockwise, _block_size) in its serial order (or the caller's DEVICE keypoints), K2 the same on i2;
 * D1 / D2 = extract_patches(K1 / K2, winsize) (vppb_extract_patches' layout and zero-row rule); (t, d) = vppb_match_local_sad of D1
 * (queries at K1) against D2 (trains at K2) with search_radius and cell_width.  One output entry per K1 keypoint: position K1[i],
 * flow, distance, valid.
 *   subpixelic = 0: valid where t >= 0 and K1[i] is inside the frame; flow = K2[t] - K1[i], distance = d.
 *   subpixelic = 1: lucas_kanade(i1, i2, _keypoints = K1, _niterations = lk_iterations, _winsize, _nscales) with the int-truncated
 *     min_ev / delta and the prediction K2[t] - K1[i] ((0, 0) without a match) divided by 2^nscales; every K1 keypoint inside the frame
 *     is valid, flow = LK's translation (failure codes (-1,-1) and (0,0) included), distance = SAD in int between row i of D1 and the
 *     winsize x winsize window of i2 centred on (int)(K1[i] + flow), truncated toward zero; a window leaving i2's domain plus border,
 *     or a non-finite position, counts as zeros.  winsize odd and 5..15, nscales 1..8 (VPPB_E_ARG).
 * An entry that is not valid has flow (0, 0) and distance INT32_MAX; a caller keypoint outside i1's domain is never valid.
 * i1 / i2: unsigned char, same domain (1..65535 per side), borders >= max(3, winsize / 2) read as they are (VPPB_E_BORDER).
 * keypoints: NULL = detect on i1, else n >= 0 device records.  Outputs: DEVICE arrays of `capacity` entries; *count_out (host) = |K1|;
 * |K1| > capacity gives VPPB_E_CAPACITY with the count filled in.  Nothing allocates: `workspace` (256-byte aligned, at least
 * vppb_sparse_flow_workspace_bytes(nrows, ncols, params, keypoints ? n : -1) bytes) holds every intermediate.  Every argument the host
 * can see is checked before anything is queued: a rejected call writes nothing.  The one host synchronisation is an 8-byte read of
 * the two keypoint counts after the detections. */
typedef struct vppb_sof_params {
  int32_t detector_th;   /* FAST threshold (sparse_optical_flow.hh:46: 5) */
  int32_t block_size;    /* blockwise FAST cell side >= 1 (:45: 5) */
  int32_t winsize;       /* patch / LK window side, 1..4096 (:49: 11) */
  int32_t search_radius; /* matcher radius R >= 0 (the body's _radius: 100) */
  int32_t cell_width;    /* matcher cell width s >= 1 (grid_index.hh:16: 300) */
  int32_t subpixelic;    /* 0: integer flows of the matches, 1: Lucas-Kanade refinement */
  int32_t lk_iterations; /* LK iterations >= 0 (:48: 5) */
  int32_t nscales;       /* LK pyramid levels 1..8 (lucas_kanade's default 3) */
} vppb_sof_params;
int64_t vppb_sparse_flow_workspace_bytes(int32_t nrows, int32_t ncols, const vppb_sof_params* params, int32_t nkeypoints);
int vppb_sparse_flow_u8(const vppb_img* i1, const vppb_img* i2, const vppb_sof_params* params, const vppb_int2* keypoints, int32_t n,
                        void* workspace, int64_t workspace_bytes, vppb_int2* pos_out, vppb_float2* flow_out, int32_t* dist_out,
                        unsigned char* valid_out, int32_t capacity, int32_t* count_out, void* stream);

/* ---- multi-GPU row tiles ------------------------------------------------------------------ */
/* Pack / unpack the `halo` edge rows of a row tile into/from a contiguous device staging buffer
 * (the payload of the one grouped NCCL neighbour exchange per frame).  which: 0 = top rows
 * [0,halo), 1 = bottom rows [nrows-halo, nrows) for pack; for unpack 0 = border rows
 * [-halo,0), 1 = border rows [nrows, nrows+halo).  Full buffer width (incl. column border). */
int64_t vppb_halo_bytes(const vppb_img* img, int32_t halo);
int vppb_halo_pack(const vppb_img* img, int32_t halo, int which, void* staging, void* stream);
int vppb_halo_unpack(const vppb_img* img, int32_t halo, int which, const void* staging, void* stream);
/* The same for n tiles of identical geometry in ONE launch (tile i at staging + i * vppb_halo_bytes): the
 * per-step cost of the halo exchange is then two small kernels + one grouped NCCL send/recv. */
int vppb_halo_pack_batch(const vppb_img* imgs, int32_t n, int32_t halo, int which, void* staging, void* stream);
int vppb_halo_unpack_batch(const vppb_img* imgs, int32_t n, int32_t halo, int which, const void* staging, void* stream);

/* ---- device-resident keypoint_container + trajectories (keypoint_container.hpp:22-200, keypoint_trajectory.hh:11-73) ---- */
/* The container of video_extruder_update (video_extruder.hpp:45-133) kept in HBM: every step of the update loop is a kernel
 * with the reference's serial semantics (see vpp_b200/csrc/kpc.cu); the host only keeps the entry count. */
int vppb_kpc_create(int32_t capacity, int32_t max_trajectory_length, void** handle);
int vppb_kpc_destroy(void* handle);
int32_t vppb_kpc_size(void* handle);                       /* entries, dead ones included (host copy) */
const vppb_int2* vppb_kpc_positions(void* handle);         /* DEVICE array of the entries' positions: the keypoints handed to vppb_sdof_u8 */
/* flow callback of :45-56: entry i moves to new_pos[i] (velocity, age + 1) if valid[i] and inside the frame, is removed if outside */
int vppb_kpc_flow_update(void* handle, const vppb_int2* new_pos, const unsigned char* valid, int32_t nrows, int32_t ncols, void* stream);
/* An entry outside the nrows x ncols frame (a caller's detection can put one there) is skipped the way vppb_fast9_scores skips an
 * out-of-frame keypoint: the merge gives it age 0 and leaves it out of the grid, the score filter gives it age 0 and the mask
 * gets nothing painted for it. */
/* :59-84 merge on the keypoint_spacing grid, the older entry of a cell survives */
int vppb_kpc_merge(void* handle, int32_t nrows, int32_t ncols, int32_t spacing, void* stream);
/* :87-91 remove entries whose fast9_score(img, th, position) < min_score (3 in the reference); img: u8, border >= 3 */
int vppb_kpc_score_filter(void* handle, const vppb_img* img, int32_t th, int32_t min_score, void* stream);
/* :97-109 detector mask: 1 everywhere (border included), 0 in [-spacing, spacing)^2 around every entry; mask: u8, border >= spacing */
int vppb_kpc_paint_mask(void* handle, const vppb_img* mask, int32_t spacing, void* stream);
/* :111-118 add(detections) + compact() + sync_attributes(trajectories, keypoint_trajectory(frame_id)); detections / count as
 * vppb_fast9_u8_async leaves them on the device.  Reads the new entry count back (the one host synchronisation of a frame).
 * The first min(*det_count_dev, max_detections, capacity - size) detections, in the detector's order, are appended and the rest
 * are dropped: a full container takes none, a negative count adds none, and no more than max_detections entries are ever read. */
int vppb_kpc_add_and_compact(void* handle, const vppb_int2* detections, const int32_t* det_count_dev, int32_t max_detections, int32_t frame_id, void* stream);
/* :122-133 alive entries push their position (oldest dropped beyond max_trajectory_length), dead entries' trajectories die */
int vppb_kpc_trajectories_update(void* handle, void* stream);
/* 6 ints per entry into a DEVICE buffer: row, col, age, trajectory start frame, trajectory length, trajectory alive */
int vppb_kpc_state_table(void* handle, int32_t* table_dev, void* stream);
/* into DEVICE buffers, either of which may be NULL: size velocities, and size x max_trajectory_length trajectory points
 * (row, col), newest first, NaN past the trajectory's length */
int vppb_kpc_history(void* handle, vppb_int2* velocity_dev, vppb_float2* history_dev, void* stream);

/* ---- multi-GPU row tiles, peer memory ----------------------------------------------------- */
/* Frames shard by contiguous row tiles, one tile per GPU (SURVEY 8e; the reference's only parallelism is OpenMP over
 * rows, vpp/core/pixel_wise.hpp:85-105).  A tile is an image2d whose border rows above / below are its halo.
 *
 * Fused form: the 5x5 box over n row tiles whose halo rows are NOT materialised: `ups[i]` / `downs[i]` describe the tiles
 * above / below tile i (base == NULL, or the whole array NULL: none - the tile's own, caller-filled border rows are
 * used, as for the outermost tiles).  A neighbour may live on a peer GPU (same process with peer access enabled, or
 * another process through vppb_ipc_open): the kernel pulls the 2 halo rows of every strip straight from the
 * neighbour's memory over NVLink with bulk copies inside its own load pipeline - no exchange step, no border writes.
 * All tiles of a call share one shape and layout (vppb_layout with the same border / align); the tile above must have
 * the same number of rows.  The caller orders the call after the neighbours' tiles are complete. */
int vppb_box5x5_u8c3_tiles(const vppb_img* ins, const vppb_img* ups, const vppb_img* downs, const vppb_img* outs, int32_t n, void* stream);
int vppb_box5x5_u8_tiles(const vppb_img* ins, const vppb_img* ups, const vppb_img* downs, const vppb_img* outs, int32_t n, void* stream);
/* CUDA IPC for one-process-per-GPU jobs: export an image that owns its allocation (vppb_alloc) as a 64-byte handle + the
 * offset of pixel (0,0); open it in another process (geometry = the exporter's descriptor; base / alloc are replaced by
 * the local mapping, peer access is enabled on demand); close unmaps. */
int vppb_ipc_export(const vppb_img* img, void* handle64, int64_t* offset_out);
int vppb_ipc_open(const void* handle64, int64_t offset, const vppb_img* geometry, vppb_img* out);
int vppb_ipc_close(vppb_img* img);
/* Materialised form: ONE grouped NCCL send/recv with both neighbours for n tiles (the `halo` top rows of every tile go to
 * rank - 1 and land in its bottom border rows, the bottom rows to rank + 1): what Scharr (1 row), FAST9 (3), the
 * pyramid (2 per level), LK windows and the semi-dense flow (64) use before their single-GPU kernels run on the tile.
 * comm: from vppb_comm_init (NCCL is loaded at run time; VPPB_E_NCCL if it is missing or fails).  The 128-byte id comes
 * from vppb_comm_unique_id on one rank and reaches the others by any means (MPI, torch.distributed, a file). */
int vppb_comm_unique_id(void* id128);
int vppb_comm_init(const void* id128, int32_t rank, int32_t nranks, void** comm_out);
int vppb_comm_destroy(void* comm);
int vppb_halo_exchange(void* comm, int32_t rank, int32_t nranks, const vppb_img* imgs, int32_t n, int32_t halo, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VPPB_H_ */
