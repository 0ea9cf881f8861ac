/*
 * igneous_b200.h -- C ABI of libigneous_b200.so
 *
 * H100 (sm_90a) implementation of the igneous per-chunk hot path.  Every
 * entry point replaces one call the reference (seung-lab/igneous @ 3b6e5b6)
 * makes into a third-party CPU library; the reference call site is cited
 * beside each declaration (paths relative to the igneous repo root).
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / numpy types.
 *   - all volumes are Fortran order: index = x + sx*(y + sy*z); a 4-D
 *     (x,y,z,c) array is passed as sz*sc slices.
 *   - every function returns IGN_OK (0) or a negative ign_status; the message
 *     is available from ign_last_error() (thread local).
 *   - functions without suffix take HOST buffers (pageable or pinned) and do
 *     H2D / D2H themselves; *_dev variants take DEVICE pointers obtained from
 *     ign_dev_alloc and run asynchronously on the context's stream.
 *   - one ign_ctx per process per GPU; a ctx is not thread safe.
 *   - there is no CPU fallback: without a usable CUDA device ign_init fails.
 */
#ifndef IGNEOUS_B200_H
#define IGNEOUS_B200_H

#include <stdint.h>

#if defined(__GNUC__)
#define IGN_API __attribute__((visibility("default")))
#else
#define IGN_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ign_ctx ign_ctx;
typedef struct ign_mesher ign_mesher;
typedef struct ign_group ign_group;

typedef enum {
  IGN_OK = 0,
  IGN_ERR_CUDA = -1,        /* CUDA runtime error (sticky errors kill the ctx) */
  IGN_ERR_INVALID = -2,     /* bad argument */
  IGN_ERR_UNSUPPORTED = -3, /* dtype / factor / option not implemented */
  IGN_ERR_NOMEM = -4,
  IGN_ERR_KEY = -5,         /* remap: label missing from the table (KeyError) */
  IGN_ERR_OVERFLOW = -6,    /* capacity exceeded (e.g. > 2^31-2 voxels per CCL call) */
  IGN_ERR_NCCL = -7
} ign_status;

typedef enum {
  IGN_U8 = 1,
  IGN_U16 = 2,
  IGN_U32 = 3,
  IGN_U64 = 4,
  IGN_F32 = 5
} ign_dtype;

/* averaging render rule (tinybrain parity is unpinned offline: SURVEY 8(c)) */
typedef enum { IGN_ROUND_FLOOR = 0, IGN_ROUND_HALF_UP = 1, IGN_ROUND_HALF_EVEN = 2 } ign_rounding;

/* ------------------------------------------------------------------ context */
IGN_API int ign_version(void);
IGN_API const char* ign_last_error(void);
IGN_API int ign_device_count(int* n);
IGN_API int ign_init(int device, ign_ctx** out);
IGN_API int ign_destroy(ign_ctx* ctx);
IGN_API int ign_sync(ign_ctx* ctx);
/* number of kernels this library launched on ctx since ign_init */
IGN_API int ign_launch_count(ign_ctx* ctx, uint64_t* n);
/* raw cudaStream_t of the context (for interop: events, NCCL, torch external stream) */
IGN_API int ign_stream(ign_ctx* ctx, void** stream);

/* device / pinned-host memory */
IGN_API int ign_dev_alloc(ign_ctx* ctx, uint64_t bytes, void** dptr);
IGN_API int ign_dev_free(ign_ctx* ctx, void* dptr);
IGN_API int ign_host_alloc(ign_ctx* ctx, uint64_t bytes, void** hptr); /* pinned */
IGN_API int ign_host_free(ign_ctx* ctx, void* hptr);
IGN_API int ign_h2d(ign_ctx* ctx, void* dst, const void* src, uint64_t bytes);  /* async on ctx stream */
IGN_API int ign_d2h(ign_ctx* ctx, void* dst, const void* src, uint64_t bytes);  /* async on ctx stream */
IGN_API int ign_d2d(ign_ctx* ctx, void* dst, const void* src, uint64_t bytes);
IGN_API int ign_memset(ign_ctx* ctx, void* dst, int byte, uint64_t bytes);

/* CUDA-event timers on the ctx stream: slot in [0,64) */
IGN_API int ign_timer_start(ign_ctx* ctx, int slot);
IGN_API int ign_timer_stop(ign_ctx* ctx, int slot);
IGN_API int ign_timer_ms(ign_ctx* ctx, int slot, float* ms); /* synchronises on the stop event */
/* cross-context ordering on one device: waiter's stream waits for the point where
 * producer last called ign_timer_start(producer, slot); no host synchronisation */
IGN_API int ign_stream_wait_mark(ign_ctx* waiter, ign_ctx* producer, int slot);
/* Re-creates the ctx stream (after synchronising it) with the device's greatest (high != 0) or least
 * stream priority.  Thread blocks of a higher-priority stream are dispatched first whenever an SM
 * frees up: a worker that runs short whole-volume passes (CCL: igneous/tasks/image/ccl.py:173) next to
 * long MeshTask streams (tasks/mesh/mesh.py:371-383) asks for high priority on the former. */
IGN_API int ign_stream_priority(ign_ctx* ctx, int high);

/* per-kernel-class CUDA-event profiling on the ctx stream (bench.py roofline):
 * classes 0 ccl_local, 1 ccl_merge, 2 ccl_label, 3 pool, 4 marching cubes */
IGN_API int ign_prof_enable(ign_ctx* ctx, int on);
IGN_API int ign_prof_read(ign_ctx* ctx, int cls, float* total_ms, uint64_t* launches);

/* strided 3-D sub-box copy between device volumes (task cutouts, +1 overlap) */
IGN_API int ign_copy_box_dev(ign_ctx* ctx, const void* src, int dtype, uint64_t sx, uint64_t sy,
                             uint64_t sz, uint64_t x0, uint64_t y0, uint64_t z0, uint64_t bx,
                             uint64_t by, uint64_t bz, void* dst);

/* ------------------------------------------------------------------ pooling
 * tinybrain.downsample_segmentation(img, factor=(2,2,1), num_mips, sparse)
 *   igneous/tasks/image/image.py:52-53 (bound) and :91 (called)
 * tinybrain.downsample_with_averaging(img, factor=(2,2,1), num_mips, sparse)
 *   igneous/tasks/image/image.py:50-51 and :91
 * outs[m] receives mip m+1, shape (ceil(sx/2^(m+1)), ceil(sy/2^(m+1)), sz).
 * Mode pooling is recursive per mip (COUNTLESS 2-D rule); averaging keeps
 * exact sums inside groups of four mips and renders with `rounding`.
 */
IGN_API int ign_pool_mode_2x2x1(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy,
                        uint64_t sz, int num_mips, int sparse, void* const* outs);
IGN_API int ign_pool_avg_2x2x1(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy,
                       uint64_t sz, int num_mips, int rounding, void* const* outs);
IGN_API int ign_pool_mode_2x2x1_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy,
                            uint64_t sz, int num_mips, int sparse, void* const* outs);
IGN_API int ign_pool_avg_2x2x1_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy,
                           uint64_t sz, int num_mips, int rounding, void* const* outs);

/* Block pooling with factors 1 or 2 per axis -- every tinybrain.downsample_* call other than
 * the (2,2,1) mode / average pyramids above:
 *   igneous/tasks/image/image.py:46-55 (downsample_method_to_fn: min / max / striding, and
 *   mode / average with a non-(2,2,1) factor such as (2,2,2) for --volumetric)
 * op: 0 min, 1 max, 2 striding (partial edge blocks reduce over the samples that exist);
 *     3 mode, 4 sparse mode (zeros ignored): a planar factor with four samples left uses the
 *       COUNTLESS 2-D pick, otherwise the highest count wins with ties to the earliest sample
 *       (x fastest); 5 / 6 / 7 average rendered with IGN_ROUND_FLOOR / HALF_UP / HALF_EVEN
 *       (the lone row / column / slice of an odd extent counts twice; u8, u16, u32, f32);
 *     8 / 9 / 10 sparse average = mean of the non-zero samples (0 if there are none), same
 *       roundings (tinybrain.downsample_with_averaging(sparse=True)).
 * Every mip is computed from the previous one.  Generic one-thread-per-output kernels.
 * [SURVEY 8(f) row 3, not on the headline path] */
IGN_API int ign_pool_select(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy,
                            uint64_t sz, uint32_t fx, uint32_t fy, uint32_t fz, int num_mips, int op,
                            void* const* outs);
IGN_API int ign_pool_select_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy,
                                uint64_t sz, uint32_t fx, uint32_t fy, uint32_t fz, int num_mips,
                                int op, void* const* outs);

/* ---------------------------------------------------------------------- CCL
 * cc3d.connected_components(labels, connectivity=6, out_dtype=np.uint64, return_N)
 *   igneous/tasks/image/ccl.py:173, :235-238, :339-342
 * 6-connected, multi-label (equal non-zero values connect), 0 = background.
 * Output ids 1..N in order of each component's first voxel in Fortran raster
 * order.  in_dtype U8 also serves bool input (threshold_image output).
 * out_dtype: IGN_U16 / IGN_U32 / IGN_U64 (overflow -> IGN_ERR_OVERFLOW); any other code ->
 * IGN_ERR_UNSUPPORTED before any launch, in every CCL call that writes labels.
 * Rows of up to 131,072 voxels (sx); longer rows -> IGN_ERR_OVERFLOW before any launch.  Rows
 * past 2048 voxels resolve in flatter tiles (tests/test_ccl_long_rows_gpu.py covers each height).
 */
IGN_API int ign_ccl6(ign_ctx* ctx, const void* in, int in_dtype, uint64_t sx, uint64_t sy, uint64_t sz,
             void* out, int out_dtype, uint64_t* n_components);
IGN_API int ign_ccl6_dev(ign_ctx* ctx, const void* in, int in_dtype, uint64_t sx, uint64_t sy,
                 uint64_t sz, void* out, int out_dtype, uint64_t* n_components);

/* Volumes that span several GPUs (one z-slab per rank).  This replaces the four
 * file-based passes of igneous/tasks/image/ccl.py (CCLFacesTask :126-194,
 * CCLEquivalancesTask :196-294, create_relabeling :358-420, RelabelCCLTask
 * :296-356) for data that is resident in HBM: every rank resolves its own volume
 * (begin), the outer z-planes are exchanged and compared (ign_ccl6_link_dev),
 * the equivalences are solved (ign_ccl6_solve, smaller id wins as ccl.py:70-73)
 * and every rank expands its labels once through the composed table (finish).
 * The result is bit-identical to one whole-volume ign_ccl6 call.
 *
 * ign_ccl6_volume_dev: one volume of up to 2^36 voxels in one call (no slabs: the
 * union-find runs over x-runs, not voxels).  ign_ccl6_dev is the same call. */
IGN_API int ign_ccl6_link_dev(ign_ctx* ctx, const uint64_t* values_a, const uint32_t* labels_a,
                              uint64_t offset_a, const uint64_t* values_b, const uint32_t* labels_b,
                              uint64_t offset_b, uint64_t n_plane, uint64_t* pairs_host,
                              uint64_t capacity, uint64_t* n_pairs);
IGN_API int ign_ccl6_solve(const uint64_t* pairs, uint64_t n_pairs, uint64_t total, uint32_t* lut,
                           uint64_t* n_global);
IGN_API int ign_ccl6_volume_dev(ign_ctx* ctx, const void* in, int in_dtype, uint64_t sx, uint64_t sy,
                                uint64_t sz, void* out, int out_dtype, uint64_t* n_components);
/* The same in two halves, so that several volumes (one per GPU) can be linked in
 * between: begin resolves the volume and fills its outer z-planes (voxel values
 * widened to u64 and volume-local ids 1..n_local; device buffers of sx*sy
 * entries, may be NULL); finish takes the caller's HOST table [n_local+1] from
 * volume-local to final ids (NULL = identity) and writes the labels. */
typedef struct ign_ccl_volume ign_ccl_volume;
IGN_API int ign_ccl6_volume_begin_dev(ign_ctx* ctx, const void* in, int in_dtype, uint64_t sx,
                                      uint64_t sy, uint64_t sz,
                                      uint64_t* first_values, uint32_t* first_labels,
                                      uint64_t* last_values, uint32_t* last_labels,
                                      ign_ccl_volume** out, uint64_t* n_local);
IGN_API int ign_ccl6_volume_finish_dev(ign_ccl_volume* v, const uint32_t* global_lut,
                                       uint64_t max_label, void* out, int out_dtype);
IGN_API int ign_ccl6_volume_abort(ign_ccl_volume* v);
/* The device-side finish of ign_ccl6_sharded_dev, for a volume from ign_ccl6_volume_begin_dev
 * that is slab `rank` of `nranks` z-slabs (slab r above slab r-1).  records_dev holds nranks
 * plane records of np = sx*sy entries each, back to back (record r at byte
 * r * (256 + 24*np), igneous_b200.multigpu.plane_record_bytes):
 *   bytes [0, 256)             header; u64 word 0 = n_local of slab r, the rest unused
 *   u64  first_values[np]      slab r's first z-plane, as begin writes it
 *   u64  last_values[np]       slab r's last z-plane
 *   u32  first_labels[np]
 *   u32  last_labels[np]
 * Links the nranks-1 boundaries, solves the dataset-wide union-find on the device (smaller id
 * wins), relabels the slab and expands it once into out; *n_global (may be NULL) = the
 * dataset's component count, the same on every rank.  Stitched together, the slabs' outputs are
 * bit-identical to one whole-volume ign_ccl6 call.  Consumes the volume, also on failure, except
 * when v is NULL or when volumes of the context are not ended in reverse order of begin.
 * IGN_ERR_INVALID: nranks < 1, rank outside [0, nranks), NULL records_dev or out, or record
 * `rank` whose n_local differs from the volume's.  IGN_ERR_OVERFLOW: the global count does not
 * fit out_dtype. */
IGN_API int ign_ccl6_volume_finish_gathered_dev(ign_ccl_volume* v, const void* records_dev, int nranks,
                                                int rank, void* out, int out_dtype, uint64_t* n_global);

/* cc3d.dust(labels, threshold, connectivity=6, in_place=True)
 *   igneous/tasks/image/ccl.py:169-172, :231-234, :335-338
 * zeroes (in place) every 6-connected component with < threshold voxels. */
IGN_API int ign_dust(ign_ctx* ctx, void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
             uint64_t threshold);
IGN_API int ign_dust_dev(ign_ctx* ctx, void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                 uint64_t threshold);

/* Fused CCLFacesTask body (igneous/tasks/image/ccl.py:166-175): optional
 * threshold (use_lte/use_gte), blackout_non_face_rails(shape), CCL,
 * += label_offset, background re-zeroed; out is u64. */
IGN_API int ign_ccl_task(ign_ctx* ctx, const void* in, int in_dtype, uint64_t sx, uint64_t sy,
                         uint64_t sz, int use_gte, double gte, int use_lte, double lte,
                         uint64_t rail_x, uint64_t rail_y, uint64_t rail_z, uint64_t dust_threshold,
                         uint64_t label_offset, uint64_t* out, uint64_t* n_components);
IGN_API int ign_ccl_task_dev(ign_ctx* ctx, const void* in, int in_dtype, uint64_t sx, uint64_t sy,
                     uint64_t sz, int use_gte, double gte, int use_lte, double lte,
                     uint64_t rail_x, uint64_t rail_y, uint64_t rail_z, uint64_t dust_threshold,
                     uint64_t label_offset, uint64_t* out, uint64_t* n_components);

/* ------------------------------------------------------------- hole filling
 * fastmorph.dilate(data, mode=multilabel, background_only=True)  igneous/tasks/mesh/mesh.py:211-218
 *   one pass: a 0 voxel with a non-zero voxel among its 26 in-box neighbours takes the most
 *   frequent non-zero neighbour label, ties to the smaller label; other voxels are copied.
 * fastmorph.fill_holes_v2(data, fix_borders, merge_threshold)   igneous/tasks/mesh/mesh.py:220-228
 *   the rule of DESIGN.md "Hole filling" (fastmorph parity unpinned): filled = every region
 *   replaced by the label of the non-zero region nearest the outside that encloses it; holes =
 *   input where it differs from filled and is non-zero, else 0.  merge_threshold_pct = 100 *
 *   merge_threshold (0..100, whole percent).  u8 / u16 / u32 / u64 (label 2^64-1 unsupported);
 *   out buffers of the input's dtype, not aliasing it.
 *   Not stream-ordered: the graph solve runs on the host, so ign_fill_holes_dev synchronises the
 *   ctx stream about four times per pass (one pass per face plane with fix_borders, six at most,
 *   then one for the volume) and returns with the results written.  ign_dilate_multilabel_dev is
 *   asynchronous like the other _dev calls.
 */
IGN_API int ign_dilate_multilabel(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                                  void* out);
IGN_API int ign_dilate_multilabel_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy,
                                      uint64_t sz, void* out);
IGN_API int ign_fill_holes(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                           int fix_borders, int merge_threshold_pct, void* filled, void* holes);
IGN_API int ign_fill_holes_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                               int fix_borders, int merge_threshold_pct, void* filled, void* holes);

/* ------------------------------------------------- contrast, CLAHE, quantize
 * The per-voxel rules are stated in DESIGN.md §5b.  u8 / u16 input only (IGN_ERR_UNSUPPORTED
 * otherwise).  Buffers must be aligned to their element size (IGN_ERR_INVALID otherwise).
 *
 * np.bincount(img2d) accumulated into levels   igneous/tasks/image/image.py:373-376
 *   hist[v] += number of voxels equal to v; hist has 256 (u8) or 65,536 (u16) entries (a DEVICE
 *   array for _dev, a HOST array otherwise) and is added into, not cleared.  n < 2^40.
 */
IGN_API int ign_histogram(ign_ctx* ctx, const void* in, int dtype, uint64_t n, uint64_t* hist);
IGN_API int ign_histogram_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t n, uint64_t* hist);
/* ContrastNormalizationTask.execute                 igneous/tasks/image/image.py:257-280
 *   (x, y, z, c) volume; slice z with lower[z] != upper[z] becomes
 *   (f32(v) - f32(lower)) * f32(maxval_t / (upper - lower)), maxval_t = 2^bits - 1 of in_dtype,
 *   every other slice keeps its values; then rint (half to even), clip to [minval, maxval] (in
 *   float32) and cast to out_dtype (u8, u16, u32 or f32).  lower / upper are HOST arrays of sz
 *   entries in both variants.  [f32(minval), f32(maxval)] outside out_dtype's range -> IGN_ERR_INVALID
 *   (for u32 output maxval may be at most 4294967040, the largest float32 below 2^32). */
IGN_API int ign_contrast_stretch(ign_ctx* ctx, const void* in, int in_dtype, uint64_t sx, uint64_t sy,
                                 uint64_t sz, uint64_t sc, const uint32_t* lower, const uint32_t* upper,
                                 double minval, double maxval, void* out, int out_dtype);
IGN_API int ign_contrast_stretch_dev(ign_ctx* ctx, const void* in, int in_dtype, uint64_t sx, uint64_t sy,
                                     uint64_t sz, uint64_t sc, const uint32_t* lower, const uint32_t* upper,
                                     double minval, double maxval, void* out, int out_dtype);
/* (image * 255.0).astype(np.uint8)                  igneous/tasks/image/image.py:158-159
 *   n float32 -> u8: trunc(v * 255) for products in [0, 256); below 0 -> 0, 256 and above -> 255,
 *   NaN -> 0 (numpy leaves those undefined).  Channel 0 of an F-order (x, y, z, c) array is its
 *   first sx*sy*sz elements. */
IGN_API int ign_quantize(ign_ctx* ctx, const float* in, uint64_t n, uint8_t* out);
IGN_API int ign_quantize_dev(ign_ctx* ctx, const float* in, uint64_t n, uint8_t* out);
/* cv2.createCLAHE(clipLimit, tileGridSize).apply(slice) on every z-slice
 *                                                   igneous/tasks/image/image.py:185, :201-202
 *   OpenCV 4.13 CLAHE::apply for CV_8UC1 / CV_16UC1 on each (sx, sy) slice of an (sx, sy, sz)
 *   stack, axis 0 (x) being OpenCV's rows: tiles_x tiles across y, tiles_y across x.  out may
 *   alias in.  The _dev variant takes the LUTs (sz * tiles_x * tiles_y * 256 or 65,536 entries of
 *   the dtype) from the scratch arena. */
IGN_API int ign_clahe(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                      double clip_limit, uint32_t tiles_x, uint32_t tiles_y, void* out);
IGN_API int ign_clahe_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                          double clip_limit, uint32_t tiles_x, uint32_t tiles_y, void* out);

/* ---------------------------------------------------------------- fastremap
 * fastremap.renumber(data, in_place=True)            igneous/tasks/mesh/mesh.py:206
 *   ids 1..K by first appearance in memory order, 0 kept.  out is u32;
 *   uniq[0..K) receives the original label of new id i+1.
 * fastremap.remap(arr, table, in_place=True)         igneous/tasks/image/ccl.py:346,
 *                                                    igneous/tasks/mesh/mesh.py:369
 *   preserve_missing=0 -> IGN_ERR_KEY when a label is not in keys[].
 * fastremap.unique(arr, return_counts=True)          igneous/tasks/mesh/mesh.py:318
 *   sorted ascending; call with uniq==NULL to get K only.
 * fastremap.mask / mask_except(arr, labels, in_place) igneous/tasks/mesh/mesh.py:201-204,320,368
 * fastremap.inverse_component_map(parents, components) igneous/tasks/image/ccl.py:280
 *   unique (parent, component) pairs sorted ascending; capacity in *n_pairs.
 */
IGN_API int ign_renumber(ign_ctx* ctx, const void* in, int dtype, uint64_t n, uint32_t* out,
                 uint64_t* uniq, uint64_t uniq_capacity, uint64_t* k);
IGN_API int ign_renumber_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t n, uint32_t* out,
                     uint64_t* uniq_dev, uint64_t uniq_capacity, uint64_t* k);
IGN_API int ign_remap(ign_ctx* ctx, void* arr, int dtype, uint64_t n, const uint64_t* keys,
              const uint64_t* vals, uint64_t n_keys, int preserve_missing);
IGN_API int ign_remap_dev(ign_ctx* ctx, void* arr, int dtype, uint64_t n, const uint64_t* keys_host,
                  const uint64_t* vals_host, uint64_t n_keys, int preserve_missing);
IGN_API int ign_unique(ign_ctx* ctx, const void* in, int dtype, uint64_t n, uint64_t* uniq,
               uint64_t* counts, uint64_t capacity, uint64_t* k);
IGN_API int ign_mask(ign_ctx* ctx, void* arr, int dtype, uint64_t n, const uint64_t* labels,
             uint64_t n_labels, int except, uint64_t value);
IGN_API int ign_inverse_component_map(ign_ctx* ctx, const void* parents, const void* components,
                              int dtype, uint64_t n, uint64_t* pairs, uint64_t* n_pairs);
/* widen/narrow unsigned integer arrays on the device */
IGN_API int ign_cast_dev(ign_ctx* ctx, const void* in, int in_dtype, void* out, int out_dtype, uint64_t n);

/* ---------------------------------------------------------- label statistics
 * scipy.ndimage.find_objects(labels)                 igneous/tasks/spatial_index.py:10-20, :56
 *   (sx, sy, sz) volume of u8 / u16 / u32 / u64 labels, each side below 2^31.
 *   *max_label == 0: the largest label is found on the device and written to *max_label
 *     (0 for an empty or all-zero volume); boxes is not touched.  The _dev variant
 *     synchronises the ctx stream in this case.
 *   *max_label == N > 0: boxes[N][6] (a DEVICE array for _dev, a HOST array otherwise)
 *     receives, for label l = 1..N in row l - 1, (min x, min y, min z, max x, max y, max z),
 *     maxima inclusive.  A label without voxels has mins 0xFFFFFFFF and maxima 0.  Label 0
 *     and labels above N are ignored.  The volume is read once.
 *   A given or found N of 2^32 or more -> IGN_ERR_UNSUPPORTED (renumber the labels first).
 */
IGN_API int ign_find_objects(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy,
                             uint64_t sz, uint64_t* max_label, uint32_t* boxes);
IGN_API int ign_find_objects_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy,
                                 uint64_t sz, uint64_t* max_label, uint32_t* boxes);

/* ------------------------------------------------------- distance transform
 * edt.edt / edt.edtsq(labels, anisotropy, black_border)  kimimaro.skeletonize's distance-to-boundary
 *   field (SkeletonTask, igneous/tasks/skeleton.py:54, :312); the rule of DESIGN.md §5d (edt parity
 *   unpinned): out[p] = 0 where labels[p] == 0, else the least sum_i (anisotropy[i] (p_i - q_i))^2 over
 *   voxels q whose label differs from labels[p] (labels compared for equality only), the one-voxel shell
 *   around the volume counting as label 0 when black_border != 0; +inf where there is no such q.
 *   squared == 0 writes sqrtf of that float32 value.
 *   (sx, sy, sz) volume of u8 / u16 / u32 / u64 labels, each side below 2^30; out is float32 of the
 *   same shape, not aliasing labels.  anisotropy[i] > 0 and finite; +inf is accepted on an axis of
 *   extent 1 and means the caller's array does not have that axis (a 1-D or 2-D input), so the shell
 *   is not applied along it.  Three separable passes (x, then y, then z); the y and z passes take
 *   their envelope stacks from the scratch arena (at most 1 GiB, or one line's worth if more). */
IGN_API int ign_edt(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                    const float anisotropy[3], int black_border, int squared, float* out);
IGN_API int ign_edt_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                        const float anisotropy[3], int black_border, int squared, float* out);

/* ------------------------------------------------ geodesic distances and parents
 * dijkstra3d.euclidean_distance_field / distance_field / parental_field, as kimimaro's TEASAR calls them
 *   once per label on a cutout (SkeletonTask, igneous/tasks/skeleton.py:54, :312): here for every label
 *   of an (sx, sy, sz) volume of u8 / u16 / u32 / u64 labels in the same launches.  The rule of DESIGN.md
 *   §5e (dijkstra3d parity unpinned): voxels p, q are joined when they are neighbours under `connectivity`
 *   (6, 18 or 26) and labels[p] == labels[q] != 0.  dist[source] = 0, every step is one float32 addition
 *   d[q] = fl32(d[p] + w(p -> q)), and dist[q] is the least such value over all paths from any source of
 *   q's label; +inf on label 0 and where no source reaches.  The result does not depend on the order of
 *   evaluation and equals a heap Dijkstra with the same additions, bit for bit.
 *   weights == NULL: w = fl32(sqrt(sum_i (anisotropy[i] * delta_i)^2)), computed once on the host in double
 *     (anisotropy[i] > 0 and finite).  weights != NULL: w(p -> q) = weights[q], a float32 array of the
 *     volume's shape, the cost of entering q; every entry must be finite and >= 0 (checked on the device
 *     in the first pass: IGN_ERR_INVALID), and anisotropy is not read.
 *   sources: n_sources linear indices x + sx * (y + sy * z) (a DEVICE array for _dev).  A source outside
 *     the volume or on label 0 -> IGN_ERR_INVALID.  Several sources may share a label.
 *   parents_out (may be NULL): uint32 of the volume's shape, the linear index + 1 of the chosen predecessor;
 *     0 for a source, an unreached voxel and label 0.  It is written in one pass over the converged
 *     distances: the first neighbour p, in (dz, dy, dx) raster order with dx fastest, with
 *     fl32(dist[p] + w(p -> q)) == dist[q] and (dist[p], p) < (dist[q], q) lexicographically.  The second
 *     condition keeps the parent graph acyclic where float32 addition stalls (dist[p] + w == dist[p]).  A
 *     reached voxel that is not a source and has no such neighbour (a plateau entered from a higher index)
 *     fails the call with IGN_ERR_INVALID (the message names one such voxel); a cycle is never written, and
 *     parents_out is then unspecified.  The refusal is of the whole call, every label of it.
 *     With parents_out the volume must have fewer than 2^32 - 1 voxels (IGN_ERR_OVERFLOW).
 *   Each side below 2^30; 64-bit indexing for the distances.  A label-correcting solver over bricks of
 *   32 x 8 x 8 voxels: not stream-ordered, the ctx stream is synchronised once per eight rounds to read
 *   the length of the device-side list of bricks still to relax, and once more for the parents.
 *   ign_geodesic_round_cap: the number of rounds after which a solve of that shape gives up with
 *   IGN_ERR_INVALID (one more than the voxel count, a bound no input reaches).
 *   ign_geodesic_last_stats: diagnostic only (tools/microbench_geodesic.py); thread-local counters of this
 *   thread's last solve, not part of any result: [0] rounds that relaxed a brick, [1] bricks relaxed over
 *   all rounds, [2] host synchronisations.
 */
IGN_API int ign_geodesic(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                         int connectivity, const float anisotropy[3], const float* weights,
                         const uint64_t* sources, uint64_t n_sources, float* dist_out, uint32_t* parents_out);
IGN_API int ign_geodesic_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                             int connectivity, const float anisotropy[3], const float* weights,
                             const uint64_t* sources, uint64_t n_sources, float* dist_out,
                             uint32_t* parents_out);
IGN_API int ign_geodesic_round_cap(uint64_t sx, uint64_t sy, uint64_t sz, uint64_t* cap);
IGN_API int ign_geodesic_last_stats(uint64_t stats[3]);
/* Per label l = 1..max_label of n voxels: index_out[l] = the voxel of greatest finite field value, ties
 *   to the lowest linear index, and value_out[l] = that value (2^64 - 1 and -inf for a label without a
 *   finite value; entry 0 likewise).  Both are DEVICE arrays of max_label + 1 entries.  Label 0 and labels
 *   above max_label are ignored; max_label of 2^32 or more -> IGN_ERR_UNSUPPORTED (renumber first).
 *   TEASAR's root (argmax of the first distance field) and the per-label maxima of its fields. */
IGN_API int ign_label_argmax_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t n, const float* field,
                                 uint64_t max_label, uint64_t* index_out, float* value_out);
/* TEASAR's penalty field (kimimaro's formula as recalled, parity unpinned; DESIGN.md §5e), float32,
 *   every operation rounded on its own:
 *     out[p] = scale * (1 - dbf[p] / (1.01f * dbf_max[l]))^exponent + daf[p] / daf_max[l],   l = labels[p]
 *   the power by exponent - 1 successive multiplications (exponent a whole number from 1 to 64), the
 *   second term 0 when daf_max[l] is 0; out[p] = 0 where l is 0 or above max_label or daf[p] is +inf.
 *   dbf_max, daf_max: DEVICE arrays of max_label + 1 entries, as ign_label_argmax_dev writes them. */
IGN_API int ign_teasar_pdrf_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t n, const float* dbf,
                                const float* daf, const float* dbf_max, const float* daf_max,
                                uint64_t max_label, float scale, int exponent, float* out);
/* TEASAR skeletons (kimimaro.skeletonize as recalled, parity unpinned; DESIGN.md §5f).  Every array is a
 * DEVICE array; volumes are (sx, sy, sz) F-order with fewer than 2^32 - 1 voxels.
 * kimimaro.skeletonize takes its objects from ign_label_parts_dev at connectivity 26, so a volume of 2^32 - 1
 *   voxels or more is refused there with IGN_ERR_UNSUPPORTED, before the solver's IGN_ERR_OVERFLOW.
 * ign_teasar_border_targets_dev: kimimaro's fix_borders targets (as recalled): for each face in the order
 *   x = 0, x = sx - 1, y = 0, y = sy - 1, z = 0, z = sz - 1, the 8-connected parts of each object in the
 *   face plane, ordered by first voxel in the plane's F order, and per part the voxel of greatest 2-D edt
 *   of the object plane (the plane's two anisotropies, black border), ties to the lowest plane index.
 *   targets_out: *count linear indices of the volume (at most capacity; the face areas summed suffice).
 * ign_teasar_last_target_dev: for each object with a target on it, roots[o] (n_objects + 1 entries) = its
 *   last target in the order given.  Targets on 0 are ignored; one outside the volume -> IGN_ERR_INVALID.
 * ign_teasar_paths_dev: the path loop for every object 1..n_objects at once.  dbf, daf, pdrf: the fields
 *   of ign_teasar_pdrf_dev on the objects; roots[o] the root of object o (n_objects + 1 entries).
 *   fix_branching: dist = the least cost from the roots where entering p costs pdrf[p]; it is lowered in
 *   place as paths join the skeleton, and parents is NULL.  Otherwise parents = the parent field under that
 *   cost (ign_geodesic_dev) and dist is NULL.  before / after: target voxels in the order given; the last
 *   before-target of an object must be its root and is not traced.  scale, cnst finite and >= 0;
 *   max_paths bounds the paths of the DAF loop of each object.  Out: *count skeleton voxels, skel_out
 *   their linear indices ascending, next_out the next voxel towards the root (the voxel itself at a root),
 *   radius_out dbf there; each of n entries at most.  A path voxel without a next voxel -> IGN_ERR_INVALID
 *   naming it.  The host synchronises once per round (plus the solver's own synchronisations).
 * ign_teasar_last_stats: diagnostic only; this thread's last paths call: [0] rounds, [1] paths, [2] box
 *   voxels visited by the invalidation, [3] host synchronisations. */
IGN_API int ign_teasar_border_targets_dev(ign_ctx* ctx, const uint32_t* objects, uint64_t sx, uint64_t sy,
                                          uint64_t sz, uint64_t n_objects, const float anisotropy[3],
                                          uint64_t* targets_out, uint64_t capacity, uint64_t* count);
IGN_API int ign_teasar_last_target_dev(ign_ctx* ctx, const uint32_t* objects, uint64_t n, uint64_t n_objects,
                                       const uint64_t* targets, uint64_t n_targets, uint64_t* roots);
IGN_API int ign_teasar_paths_dev(ign_ctx* ctx, const uint32_t* objects, uint64_t sx, uint64_t sy, uint64_t sz,
                                 uint64_t n_objects, const float anisotropy[3], const float* dbf, const float* daf,
                                 const float* pdrf, float* dist, const uint32_t* parents, const uint64_t* roots,
                                 const uint64_t* before, uint64_t n_before, const uint64_t* after,
                                 uint64_t n_after, float scale, float cnst, uint64_t max_paths,
                                 uint32_t* skel_out, uint32_t* next_out, float* radius_out, uint64_t* count);
IGN_API int ign_teasar_last_stats(uint64_t stats[4]);
/* Per-label export of a chunk's skeleton (SkeletonTask's vertex shift, spatial index and upload,
 * igneous/tasks/skeleton.py:229-236, :772-807, and kimimaro.skeletonize's split by label; DESIGN.md §5g).
 * Every array is a DEVICE array.
 * ign_skeleton_export_dev: labels u32 1..max_label (renumbered) of an (sx, sy, sz) F-order volume; skel, next,
 *   radius: the count entries of ign_teasar_paths_dev (skel ascending).  Out, for every label with a skeleton
 *   voxel, in ascending label order, *n_skeletons of them (at most min(max_label, count)):
 *     blobs_out  one neuroglancer precomputed skeleton per label, each starting on an 8-byte boundary (the
 *                padding between blobs is zeros and belongs to none): uint32 nv, uint32 ne,
 *                float32 vertices[nv][3], uint32 edges[ne][2], float32 radius[nv], and with vertex_types != 0
 *                uint8 vertex_types[nv], all 0.  *nbytes = the end of the last blob.
 *     table_out  uint64 [][4] rows (label, byte offset, nv, ne).
 *     boxes_out  float32 [][6] rows (min x, min y, min z, max x, max y, max z) of the label's vertices.
 *   A label's vertices are its skeleton voxels in ascending linear index; vertex i of voxel (x, y, z) is
 *   fl32((double)fl32(fl32(x) * anisotropy[0]) + offset[0]), and likewise for y and z.  Every voxel v with
 *   next(v) != v gives one edge (min, max) of the two local vertex indices; a label's edges are sorted by
 *   (min, max).  capacity (bytes) must be at least count * 25 + min(max_label, count) * 16
 *   (ign_skeleton_export_capacity), IGN_ERR_INVALID otherwise, before any launch.  A skeleton voxel outside
 *   the volume, not above the one before it or on label 0 or above max_label, and a next voxel that is not
 *   a skeleton voxel or lies on another label -> IGN_ERR_INVALID naming the lowest such voxel by linear
 *   index; no cross-label edge is ever written.  The skeleton voxels are checked before any pass that
 *   relies on them, the next voxels before any output is written.  The host synchronises three times.
 * ign_skeleton_export_capacity: that bound for count skeleton voxels (IGN_ERR_OVERFLOW from 2^31). */
IGN_API int ign_skeleton_export_dev(ign_ctx* ctx, const uint32_t* labels, uint64_t sx, uint64_t sy, uint64_t sz,
                                    uint64_t max_label, const uint32_t* skel, const uint32_t* next,
                                    const float* radius, uint64_t count, const float anisotropy[3],
                                    const double offset[3], int vertex_types, uint8_t* blobs_out, uint64_t capacity,
                                    uint64_t* table_out, float* boxes_out, uint64_t* n_skeletons, uint64_t* nbytes);
IGN_API int ign_skeleton_export_capacity(uint64_t count, uint64_t max_label, uint64_t* bytes);

/* ------------------------------------------------------------- skeleton merge
 * UnshardedSkeletonMergeTask's fuse and kimimaro.postprocess (igneous/tasks/skeleton.py:810-916) for a batch
 * of labels in one call; the rule is DESIGN.md §5h.  Every array is a DEVICE array.
 * ign_skeleton_merge_dev: n_labels labels; label l owns fragments [label_frag[l], label_frag[l + 1]), fragment f
 *   owns vertices [frag_vert[f], frag_vert[f + 1]) and edges [frag_edge[f], frag_edge[f + 1]) (label_frag,
 *   frag_vert and frag_edge ascend from 0 to n_frags, n_vertices and n_edges).  vertices float32 [][3],
 *   radius float32 [], vertex_types_in uint8 [] per vertex; edges uint32 [][2], indices local to their
 *   fragment; frag_box float64 [][6] (min xyz, max xyz) per fragment: a vertex outside it is cropped
 *   (-inf / +inf keeps all).  Each label is fused; unless its cable length exceeds max_cable_length (+inf:
 *   never) it is postprocessed with dust_threshold and tick_threshold (0 skips a step).  Out, one row per
 *   label in label order: blobs_out as ign_skeleton_export_dev's (radius, then vertex_types when
 *   vertex_types != 0, 8-byte aligned, an empty result is nv = ne = 0), table_out uint64 [][4] (label row,
 *   byte offset, nv, ne), *nbytes = the end of the last blob.  capacity (bytes) must be at least
 *   16 * n_labels + 25 * n_vertices + 8 * n_edges (ign_skeleton_merge_capacity).  Ranges that do not ascend,
 *   a non-finite vertex or an edge index outside its fragment -> IGN_ERR_INVALID before any output is
 *   written.  The host synchronises five times.
 * ign_skeleton_merge_capacity: that bound (IGN_ERR_OVERFLOW from 2^30 vertices or edges). */
IGN_API int ign_skeleton_merge_dev(ign_ctx* ctx, uint64_t n_labels, const uint64_t* label_frag, uint64_t n_frags,
                                   const uint64_t* frag_vert, const uint64_t* frag_edge, const double* frag_box,
                                   const float* vertices, const float* radius, const uint8_t* vertex_types_in,
                                   uint64_t n_vertices, const uint32_t* edges, uint64_t n_edges,
                                   double dust_threshold, double tick_threshold, double max_cable_length,
                                   int vertex_types, uint8_t* blobs_out, uint64_t capacity, uint64_t* table_out,
                                   uint64_t* nbytes);
IGN_API int ign_skeleton_merge_capacity(uint64_t n_labels, uint64_t n_vertices, uint64_t n_edges, uint64_t* bytes);

/* ------------------------------------------------------------- label shards
 * neuroglancer_uint64_sharded_v1 with the murmurhash3_x86_128 hash, for skeleton layers
 * (ShardedFromUnshardedSkeletonMergeTask, create_sharded_skeletons_from_unsharded_tasks,
 * igneous/tasks/skeleton.py:1074-1130); the rule is DESIGN.md §5l.  Every array is a DEVICE array unless
 * marked HOST.
 * ign_shard_hash_dev: h = MurmurHash3_x86_128 (seed 0) of the 8 little-endian bytes of label >> preshift_bits,
 *   low 64 bits; location = h & (2^(minishard_bits + shard_bits) - 1), that is (shard << minishard_bits) |
 *   minishard.  Out: labels_out the n labels sorted by (shard, minishard, label) (equal labels stay
 *   together), locations_out the location of each, and the runs of equal shards: *n_runs of them, run r
 *   starting at run_start_out[r] (run_start_out[*n_runs] = n) with shard run_shard_out[r].  run_start_out has
 *   room for min(n, 2^shard_bits) + 1 entries, run_shard_out for min(n, 2^shard_bits).  preshift_bits above 63
 *   or minishard_bits + shard_bits above 64 -> IGN_ERR_INVALID; n of 2^31 or more -> IGN_ERR_OVERFLOW.  The
 *   host synchronises once.
 * ign_skeleton_restrip_dev: n precomputed skeleton blobs packed in blobs, blob i the bytes
 *   [offsets[i], offsets[i + 1]).  attrs (HOST uint32 [n_attrs][2], n_attrs <= 32): the source's vertex
 *   attributes in blob order, each (bytes per vertex, keep).  Out: each blob with only the kept attribute
 *   sections, in the same order, blob i at out_offsets[i] of out (packed, no padding; out_offsets has n + 1
 *   entries), *nbytes = out_offsets[n].  A blob shorter than 8 bytes or whose length is not 8 + 12 nv + 8 ne +
 *   (sum of bytes per vertex) nv -> IGN_ERR_INVALID naming its row (the lowest), before anything is written
 *   to out; a capacity below the output -> IGN_ERR_INVALID.  The host synchronises once.
 * ign_shard_assemble_dev: the shard file of n payloads already at payload = shard + 16 * 2^minishard_bits,
 *   payload i at bytes [offsets[i], offsets[i + 1]) of it, rows in (minishard, label) order: locations
 *   the location of each row (its minishard = the low minishard_bits), labels its label.  Writes the shard
 *   index at shard[0..16 * 2^minishard_bits) and the raw minishard indices after the payloads; *nbytes = the
 *   file's length.  minishard_bits above 32 or a capacity below the file -> IGN_ERR_INVALID.  Rows out of
 *   (minishard, label) order are not detected.  The host synchronises once. */
IGN_API int ign_shard_hash_dev(ign_ctx* ctx, const uint64_t* labels, uint64_t n, int preshift_bits,
                               int minishard_bits, int shard_bits, uint64_t* labels_out, uint64_t* locations_out,
                               uint64_t* run_start_out, uint64_t* run_shard_out, uint64_t* n_runs);
IGN_API int ign_skeleton_restrip_dev(ign_ctx* ctx, const uint8_t* blobs, const uint64_t* offsets, uint64_t n,
                                     const uint32_t* attrs, int n_attrs, uint8_t* out, uint64_t capacity,
                                     uint64_t* out_offsets, uint64_t* nbytes);
IGN_API int ign_shard_assemble_dev(ign_ctx* ctx, const uint64_t* locations, const uint64_t* labels,
                                   const uint64_t* offsets, uint64_t n, int minishard_bits, uint8_t* shard,
                                   uint64_t capacity, uint64_t* nbytes);

/* ------------------------------------------------------- cross-sectional area
 * kimimaro.cross_sectional_area (igneous/tasks/skeleton.py:219-226, :400-475); the rule is DESIGN.md §5i.
 * ign_cross_section_normals: HOST arrays.  n_vertices vertices (below 2^32, else IGN_ERR_UNSUPPORTED) of any
 *   number of skeletons, voxels int64 [][3] the voxel of each; n_edges edges uint32 [][2] into the same list
 *   (an index >= n_vertices -> IGN_ERR_INVALID; self edges are ignored).  Per component of the edge graph: the
 *   root is the vertex farthest in hops from its lowest vertex, every vertex lies on the path from the shallowest
 *   leaf of its subtree to the root, and normals_out float64 [][3] is the sum of the voxel steps
 *   c_u - c_parent(u) over `window` (>= 1) path positions centred on it (numpy 'symmetric' padding at the ends),
 *   times anisotropy; its own step when that sum is zero; 0 for a vertex on no edge.  Host code only.
 * ign_cross_section_dev: DEVICE arrays, except anisotropy and stats.  labels (dtype u8/u16/u32/u64) of an
 *   (sx, sy, sz) F-order volume of fewer than 2^32 voxels (IGN_ERR_UNSUPPORTED otherwise); n_points points:
 *   voxel uint64 its linear index, label uint64 its skeleton's label, normal float64 [][3].  Out per point:
 *   area_out float32 the area of the section of the label through the voxel's centre across the normal (0 for
 *   a zero normal or a voxel of another label), contacts_out uint8 the faces of the volume it touches: bit 0
 *   x = 0, 1 x = sx - 1, 2 y = 0, 3 y = sy - 1, 4 z = 0, 5 z = sz - 1.  A voxel outside the volume or a
 *   non-finite normal -> IGN_ERR_INVALID naming the lowest such point.  stats: [0] voxels of every section,
 *   [1] points whose section outgrew the one-warp path, [2] voxels that path visited in them, [3] CTAs
 *   the large path ran with (each takes large points until none is left; at most one per SM, and fewer when
 *   their bitmaps and queues, 13 bytes per column of the largest projection each, would pass 512 MB).  The host
 *   synchronises once, twice when a section outgrows the one-warp path. */
IGN_API int ign_cross_section_normals(uint64_t n_vertices, const int64_t* voxels, uint64_t n_edges,
                                      const uint32_t* edges, const double anisotropy[3], uint64_t window,
                                      double* normals_out);
IGN_API int ign_cross_section_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                                  const uint64_t* voxel, const uint64_t* label, const double* normal,
                                  uint64_t n_points, const double anisotropy[3], float* area_out,
                                  uint8_t* contacts_out, uint64_t stats[4]);

/* --------------------------------------------------------------------- mesh
 * zmesh.Mesher(resolution).mesh(data, preserve_order=False)  igneous/tasks/mesh/mesh.py:151,245
 * Mesher.ids()                                                igneous/tasks/mesh/mesh.py:374
 * Mesher.get(id, reduction_factor, max_error, voxel_centered) igneous/tasks/mesh/mesh.py:376-381
 * Multi-label marching cubes over every 2x2x2 cube; per label a welded
 * (vertices f32 [nv,3], faces u32 [nf,3]) mesh in physical units:
 *   position = (half_voxel_coord/2 + (voxel_centered ? 0.5 : 0)) * resolution.
 * Vertices are ordered by (z,y,x), faces by cube raster order.
 * reduction_factor > 0 runs the quadric edge-collapse simplifier towards
 * nf/reduction_factor faces with error bound max_error (physical units).
 */
IGN_API int ign_mesh_begin(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy,
                   uint64_t sz, ign_mesher** out);
IGN_API int ign_mesh_begin_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy,
                       uint64_t sz, ign_mesher** out);
IGN_API int ign_mesh_num_ids(ign_mesher* m, uint64_t* n);
IGN_API int ign_mesh_ids(ign_mesher* m, uint64_t* ids, uint64_t capacity);
IGN_API int ign_mesh_counts(ign_mesher* m, uint64_t id, uint64_t* nv, uint64_t* nf);
IGN_API int ign_mesh_totals(ign_mesher* m, uint64_t* nv, uint64_t* nf);
IGN_API int ign_mesh_get(ign_mesher* m, uint64_t id, const float resolution[3], int reduction_factor,
                 float max_error, int voxel_centered, float* vertices, uint32_t* faces,
                 uint64_t* nv, uint64_t* nf);
/* Simplify every label of the mesher in place (round-based quadric edge collapse
 * towards nf/reduction_factor faces per label, collapse cost <= max_error^2 in
 * physical units, boundary vertices locked).  ign_mesh_get(reduction_factor>0)
 * calls it on first use; ign_mesh_export then returns the simplified meshes. */
IGN_API int ign_mesh_simplify(ign_mesher* m, const float resolution[3], int reduction_factor,
                              float max_error);
/* counters of the simplification that ran:
 * [0] most rounds of any label, [1] labels simplified in shared memory, [2] in global memory,
 * [3..5] labels simplified in the 1024-, 512- and 256-thread size classes (a label runs in the smallest
 *   CTA whose shared-memory budget holds it);
 * [6..8] labels which continued in the 1024-, 512- and 256-thread size class after migrating from the
 *   next larger one, once their alive faces and vertices fit it ([6] is always 0; a label that migrates
 *   twice counts in both smaller classes);
 * [9] label-rounds whose winners took more than one validation pass (more winners than the label's
 *   per-pass capacity), [10] winners rejected because an endpoint had more than 32 alive incident faces;
 * [11] half-edges costed before the first round, [12] half-edges re-costed after the collapse that moved
 *   an endpoint, [13] half-edges the key pass met without a cached cost (0 unless the simplifier is
 *   broken; such an edge posts no key);
 * [14..16] winners by the width of the lane group that validated, collapsed and re-costed them: 8 lanes
 *   (rings of at most 8 faces), 16 lanes, 32 lanes (rings over 16 faces, and those over 32 that are
 *   rejected); IGN_SIMP_GROUP=16 or 32 sets the narrowest width */
IGN_API int ign_mesh_simplify_counters(ign_mesher* m, uint32_t counters[17]);
/* bulk export of every label's mesh (simplified if ign_mesh_simplify ran) in ign_mesh_ids order:
 * vertices f32 [U,3], faces u32 [T,3] (label-local indices), offsets [n_ids+1] */
IGN_API int ign_mesh_export(ign_mesher* m, const float resolution[3], int voxel_centered,
                            float* vertices, uint32_t* faces, uint64_t* vert_offsets,
                            uint64_t* face_offsets);
IGN_API int ign_mesh_free(ign_mesher* m);

/* ------------------------------------------------- compressed_segmentation codec
 * The Precomputed `compressed_segmentation` chunk encoding that CloudVolume applies on the host
 * before uploading / after downloading a segmentation chunk around the hot path
 * (igneous/tasks/image/image.py:95-100 `vol[new_bounds] = mipped`, ccl.py:346-356 RelabelCCLTask's
 * output, igneous/task_creation/common.py:215-236 set_encoding).  labels: Fortran order [x,y,z,c],
 * uint32 / uint64; block (bx,by,bz) is (8,8,8) in every Precomputed layer.  The stream is the
 * uint32 word sequence of the file.  encode: *n_words = words of the stream; when they are more
 * than cap_words nothing is written and the call fails with IGN_ERR_OVERFLOW (*n_words still
 * reports the need).  One call = one chunk (24-bit table offsets). */
IGN_API int ign_cseg_encode(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                            uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz, uint32_t* out,
                            uint64_t cap_words, uint64_t* n_words);
IGN_API int ign_cseg_encode_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy,
                                uint64_t sz, uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz,
                                uint32_t* out, uint64_t cap_words, uint64_t* n_words);
IGN_API int ign_cseg_decode(ign_ctx* ctx, const uint32_t* in, uint64_t n_words, int dtype, uint64_t sx,
                            uint64_t sy, uint64_t sz, uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz,
                            void* out);
IGN_API int ign_cseg_decode_dev(ign_ctx* ctx, const uint32_t* in, uint64_t n_words, int dtype, uint64_t sx,
                                uint64_t sy, uint64_t sz, uint64_t sc, uint32_t bx, uint32_t by,
                                uint32_t bz, void* out);

/* Batches of chunks (the read and write paths of a layer, one call per cutout).  Chunk i is an F-order
 * [sx, sy, sz, sc] array, shapes[3*i .. 3*i+2] (host) = {sx, sy, sz}; chunks and decoded outputs are
 * packed back to back in the order given.
 * encode: writes the n files back to back into out (device); offsets (device, n + 1 words) delimit file
 * i as out[offsets[i] : offsets[i+1]] in words; *n_words = words of all files.  One size pass for the
 * whole batch; when the files need more than cap_words words nothing is written and the call fails
 * with IGN_ERR_OVERFLOW (*n_words still reports the need).  Every file is byte-identical to what
 * the CPU oracle's encoder (oracle/igneous_oracle.c::orc_cseg_encode_*) writes for that chunk alone.
 * decode: stream i is streams[word_offsets[i] : word_offsets[i+1]] (word_offsets on the host); a
 * malformed stream fails the call with IGN_ERR_INVALID, and the message names the first such index. */
IGN_API int ign_cseg_encode_batch_dev(ign_ctx* ctx, const void* chunks, int dtype, uint64_t n_chunks,
                                      const uint32_t* shapes, uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz,
                                      uint32_t* out, uint64_t cap_words, uint64_t* offsets, uint64_t* n_words);
IGN_API int ign_cseg_decode_batch_dev(ign_ctx* ctx, const uint32_t* streams, const uint64_t* word_offsets,
                                      uint64_t n_streams, int dtype, const uint32_t* shapes, uint64_t sc,
                                      uint32_t bx, uint32_t by, uint32_t bz, void* out);

/* ------------------------------------------------------------- chunk placement
 * The storage layer's cutouts stay on the device between decode, pooling and encode.
 * ign_chunks_place_dev: one launch copies many decoded chunks (packed, device) into one F-order
 * [X, Y, Z, nc] device cutout.  rows (host) holds n_rows rows of IGN_PLACE_ROW uint64 words:
 *   {sx, sy, sz, byte offset of the chunk in packed, x0, y0, z0, bx, by, bz, dx, dy, dz}
 * copying the chunk's sub-box [x0, x0+bx) x [y0, y0+by) x [z0, z0+bz) (every channel) to the cutout
 * at (dx, dy, dz).  Rows must write disjoint boxes; voxels no row covers keep their values.
 * ign_chunks_cut_dev: the reverse.  rows (host): n_rows rows of IGN_CUT_ROW words
 *   {x0, y0, z0, bx, by, bz, byte offset in packed}
 * box r of the cutout (every channel) is written F-order contiguous at its offset -- a `raw` chunk
 * file byte for byte; all_bg[r] (device) is non-zero when every value of the box equals `background`
 * (the value's bit pattern, zero-extended; float32 boxes compare as floats).
 * dtype: IGN_U8 / U16 / U32 / U64 / F32.  64-bit indexing throughout. */
#define IGN_PLACE_ROW 13
#define IGN_CUT_ROW 7
IGN_API int ign_chunks_place_dev(ign_ctx* ctx, const void* packed, int dtype, uint64_t nc, const uint64_t* rows,
                                 uint64_t n_rows, void* cutout, uint64_t X, uint64_t Y, uint64_t Z);
IGN_API int ign_chunks_cut_dev(ign_ctx* ctx, const void* cutout, int dtype, uint64_t X, uint64_t Y, uint64_t Z,
                               uint64_t nc, const uint64_t* rows, uint64_t n_rows, uint64_t background,
                               void* packed, uint32_t* all_bg);
/* ign_fill_box_dev: every voxel of the box [x0, x0+bx) x [y0, y0+by) x [z0, z0+bz), every channel, of an
 * F-order [X, Y, Z, nc] device cutout is set to `value` (the value's bit pattern, zero-extended, as for
 * ign_chunks_cut_dev's background).  BlackoutTask's write (igneous/tasks/image/image.py:124-135).
 * dtype: IGN_U8 / U16 / U32 / U64 / F32.  A box outside the cutout -> IGN_ERR_INVALID.  64-bit indexing. */
IGN_API int ign_fill_box_dev(ign_ctx* ctx, void* cutout, int dtype, uint64_t X, uint64_t Y, uint64_t Z, uint64_t nc,
                             uint64_t x0, uint64_t y0, uint64_t z0, uint64_t bx, uint64_t by, uint64_t bz,
                             uint64_t value);

/* ------------------------------------------------------- regions of interest
 * compute_rois (igneous/task_creation/image.py:1995-2058) per z slab of the top mip:
 *   np.greater(img, suppress_faint_voxels); cc3d.connected_components (26-connected); cc3d.dust;
 *   cc3d.statistics(...)["bounding_boxes"].
 * ign_threshold_dev: out[i] = in[i] > t (u8 0 / 1), n voxels, 64-bit indexing.  Integer dtypes
 *   (IGN_U8 / U16 / U32 / U64) compare as unsigned 64-bit integers, so every t >= 0 is exact; for
 *   IGN_F32 the low 32 bits of t are the float32 threshold's bit pattern (NaN is never greater).
 * ign_label_parts_dev: the connected parts of an F-order (sx, sy, sz) volume of labels (IGN_U8 / U16 / U32 /
 *   U64; any other dtype -> IGN_ERR_UNSUPPORTED) of fewer than 2^32 - 1 voxels (more -> IGN_ERR_UNSUPPORTED).
 *   Two neighbours under `connectivity` (6 / 18 / 26; anything else -> IGN_ERR_INVALID) join when they hold
 *   the same non-zero label.  Parts are numbered by first voxel in F order (cc3d's numbering); parts of fewer
 *   than dust_threshold voxels are dropped and the others keep their order.  *n = the number kept.
 *   parts_out (DEVICE, sx * sy * sz words, may be NULL): each voxel's kept part 1..*n, 0 on label 0 and dust.
 *   rows (HOST, capacity rows of IGN_BOX_ROW uint32 words; NULL only with capacity 0): when *n <= capacity,
 *   it receives per kept part
 *     {voxel count, min x, min y, min z, max x, max y, max z}   (maxima inclusive)
 *   in part order, copied from the device before the call returns; with *n > capacity it is not written.
 *   For a 0 / 1 mask at connectivity 26 a capacity of ceil(sx/2) * ceil(sy/2) * ceil(sz/2) rows always
 *   suffices (its parts cannot be denser).  The stream is synchronised for the part count, the kept count
 *   and, when rows are written, once more.  compute_rois uses it on a u8 mask at 26, kimimaro.skeletonize for its
 *   objects and ign_teasar_border_targets_dev for the parts of each face plane (18 on an extent-1 axis). */
#define IGN_BOX_ROW 7
IGN_API int ign_threshold_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t n, uint64_t t, uint8_t* out);
IGN_API int ign_label_parts_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy,
                                uint64_t sz, int connectivity, uint64_t dust_threshold, uint32_t* parts_out,
                                uint32_t* rows, uint64_t capacity, uint64_t* n);

/* ------------------------------------------------------------------ jpeg codec
 * The Precomputed `jpeg` chunk encoding of uint8 image layers, which CloudVolume applies on the host
 * around the image tasks (igneous/tasks/image/image.py:95-100 uploads; the CLI's image encoding,
 * igneous_cli/cli.py:64; `jpeg_quality` set by igneous/task_creation/common.py:215-236 set_encoding;
 * the png top mip of a sharded jpeg pyramid, task_creation/image.py:708-709).  A chunk [x,y,z] of
 * uint8 (one channel) is one grayscale JPEG of width sx and height sy*sz: image row y + sy*z, so the
 * Fortran-order chunk is the raster.  Each side of the image is at most 65535 pixels.
 * encode: byte-identical to libjpeg's defaults at the same quality (1..100) and restart interval:
 * JFIF APP0, the IJG-scaled Annex K table, SOF0, the Annex K Huffman tables, accurate integer DCT.
 * restart_interval: blocks between RSTn markers; 0 = no markers; < 0 = one block row of each chunk,
 * which lets ign_jpeg_decode give each row its own thread.
 * decode: pixel-identical to libjpeg's islow decode of any SOF0 / SOF1 8-bit grayscale stream
 * (any Huffman tables, APPn / COM, fill bytes, restart markers or none); progressive, arithmetic,
 * lossless, 12-bit, multi-component and DNL streams fail with IGN_ERR_UNSUPPORTED, malformed or
 * truncated ones and dimensions other than the chunk's with IGN_ERR_INVALID.
 * Batches: chunks / outputs are packed back to back; shapes are host arrays of n x {sx, sy, sz}.
 * encode: *n_bytes = bytes of all streams; nothing is written when out is NULL or cap is too small;
 * else offsets[0..n] (host) delimit stream c as out[offsets[c] : offsets[c+1]].
 * decode: stream c is streams[offsets[c] : offsets[c+1]] (offsets on the host). */
IGN_API int ign_jpeg_encode(ign_ctx* ctx, const uint8_t* chunks, uint64_t n_chunks, const uint32_t* shapes,
                            int quality, int64_t restart_interval, uint8_t* out, uint64_t cap, uint64_t* offsets,
                            uint64_t* n_bytes);
IGN_API int ign_jpeg_encode_dev(ign_ctx* ctx, const uint8_t* chunks, uint64_t n_chunks, const uint32_t* shapes,
                                int quality, int64_t restart_interval, uint8_t* out, uint64_t cap,
                                uint64_t* offsets, uint64_t* n_bytes);
IGN_API int ign_jpeg_decode(ign_ctx* ctx, const uint8_t* streams, const uint64_t* offsets, uint64_t n_streams,
                            const uint32_t* shapes, uint8_t* out);
IGN_API int ign_jpeg_decode_dev(ign_ctx* ctx, const uint8_t* streams, const uint64_t* offsets, uint64_t n_streams,
                                const uint32_t* shapes, uint8_t* out);

/* --------------------------------------------------- synthetic volumes (bench)
 * SURVEY.md 8(d): jittered-grid Voronoi segmentation / hash-byte image,
 * bit-identical to oracle.synth_seg / oracle.synth_image. */
IGN_API int ign_synth_seg_dev(ign_ctx* ctx, void* out, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                      int64_t ox, int64_t oy, int64_t oz, uint32_t pitch, uint64_t num_ids,
                      uint64_t seed, uint64_t id_base);
IGN_API int ign_synth_image_dev(ign_ctx* ctx, uint8_t* out, uint64_t sx, uint64_t sy, uint64_t sz,
                        int64_t ox, int64_t oy, int64_t oz, uint64_t seed);

/* ------------------------------------------------------- multi-GPU CCL merge
 * Replaces the file exchange of igneous/tasks/image/ccl.py:177-194 (faces),
 * :245-294 (equivalences) and :358-420 (create_relabeling) with one NCCL
 * all-gather of compacted (label_a,label_b) face-equivalence pairs.
 * One process per GPU; unique_id is ncclUniqueId bytes (128) created on rank 0
 * by ign_group_unique_id and broadcast by the host-side launcher.  NCCL is
 * dlopen()ed on first use (libnccl.so.2), so the library itself has no link-time
 * dependency on it.  Host orchestration: igneous_b200/multigpu.py. */
IGN_API int ign_group_unique_id(void* id128);
IGN_API int ign_group_init(ign_ctx* ctx, int rank, int nranks, const void* id128, ign_group** out);
IGN_API int ign_group_destroy(ign_group* g);
/* the single collective of the path: every rank contributes `bytes` bytes (its
 * component count + outer planes), everyone receives nranks*bytes */
IGN_API int ign_group_allgather(ign_group* g, const void* send_dev, uint64_t bytes, void* recv_dev);
/* SURVEY.md 8(b) `ign_ccl6_sharded`: this rank's z-slab of a dataset split over the group's ranks
 * (rank r above rank r-1).  Local CCL, ONE all-gather of [n_local | first plane | last plane],
 * then -- on the device, identically on every rank -- the N-1 boundaries are linked, the small
 * dataset-wide union-find is solved (smaller id wins, ccl.py:70-73) and the slab's labels are
 * expanded once with dataset-wide ids.  Bit-identical to one whole-volume ign_ccl6 call on the
 * stacked dataset.  Replaces ccl.py:177-194, :245-294, :358-420, :296-356.
 * It is ign_ccl6_volume_begin_dev + the all-gather + ign_ccl6_volume_finish_gathered_dev, so the
 * merge is tested on one device by emulating the ranks (tests/test_ccl_multirank_gpu.py). */
IGN_API int ign_ccl6_sharded_dev(ign_group* g, const void* in, int in_dtype, uint64_t sx, uint64_t sy,
                                 uint64_t sz, void* out, int out_dtype, uint64_t* n_global);

#ifdef __cplusplus
}
#endif
#endif /* IGNEOUS_B200_H */
