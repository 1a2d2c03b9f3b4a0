/*
 * psd_b200.h - C ABI of the H100-native (sm_90a) per-frame content-score engine for PySceneDetect.
 *
 * This is the drop-in boundary for the hot path named in BASELINE.json: the
 * process_frame() arithmetic of ContentDetector / AdaptiveDetector / ThresholdDetector /
 * HistogramDetector / HashDetector plus the cv2.resize pre-step SceneManager applies.  The reference is
 * pure Python over cv2/numpy and has no FFI of its own (SURVEY.md fact 5), so every entry
 * point below replaces a cv2/numpy call sequence at the reference line cited; the Python
 * host (pyscenedetect_b200/_capi.py) binds them with ctypes.
 *
 * Conventions: every call returns an int status (PSD_OK == 0, negative = error class);
 * no C++ exception crosses this boundary; output buffers are caller-allocated;
 * psd_last_error() returns a thread-local human-readable message for the last failure.
 * There is NO CPU fallback: without an sm_90 device psd_engine_create fails.
 */
#ifndef PSD_B200_H
#define PSD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PSD_ABI_VERSION 1

/* status codes */
#define PSD_OK 0
#define PSD_ERR_INVALID (-1) /* bad argument */
#define PSD_ERR_CUDA (-2)    /* CUDA runtime/driver failure (message has the cudaError) */
#define PSD_ERR_OOM (-3)     /* host or device allocation failed */
#define PSD_ERR_STATE (-4)   /* call not valid in the engine's current state */
#define PSD_ERR_NODEVICE (-5)/* no usable sm_90 device */

/* feature mask: which per-frame integer results the fused pass produces */
#define PSD_F_HSV 1u    /* SAD of H,S,V planes vs previous frame: content_detector.py:29-36,155,166-175 */
#define PSD_F_BGRSUM 2u /* sum of all B,G,R bytes: numpy.mean(frame_img), threshold_detector.py:127 */
#define PSD_F_YHIST 4u  /* 256-bin histogram of YUV-Y: histogram_detector.py:156-159 */
#define PSD_F_EDGES 8u  /* Canny+dilate edge-map SAD: content_detector.py:213-239 (implies HSV) */
#define PSD_F_HASH 16u  /* perceptual hash of every frame: hash_detector.py:124-158 */
#define PSD_HASH_WORDS 4 /* the hash stride for size <= 16: 4 x uint64 (size * size <= 256 bits) */
/* Per-frame stride (uint64 words) of every hash array of an engine or scan with HashDetector(size=...):
 * max(4, ceil(size * size / 64)), so 4 for size <= 16.  Bit u*size+v (word (u*size+v)/64, bit (u*size+v)%64) is
 * D[u][v] > median; the bits past size * size are 0. */
#define PSD_HASH_WORDS_FOR(size) ((size) * (size) <= 256 ? PSD_HASH_WORDS : ((size) * (size) + 63) / 64)

/* submit flags */
#define PSD_SUBMIT_PINNED 1u /* host buffer is page-locked (psd_host_alloc): DMA straight from it,
                                caller keeps it unchanged until psd_engine_sync() */

typedef struct psd_engine psd_engine;

/* Where the bytes of n frames of 8-bit B, G, R samples lie, in signed byte strides from a base pointer that
 * addresses channel B of pixel (0,0) of frame 0: channel c (0 = B, 1 = G, 2 = R) of pixel (x,y) of frame f is at
 * base + f*frame_stride + y*row_stride + x*pixel_stride + c*channel_stride.
 *   packed BGR24:          {H*3W, 3W, 3, 1}
 *   packed RGB24:          base = R byte + 2, {H*3W, 3W, 3, -1}
 *   planar RGB (NCHW):     base = B plane, {3HW, W, 1, -HW}
 * A crop is a base offset with the same strides, frame skipping multiplies frame_stride, and a zero stride
 * repeats a frame (a broadcast view). */
typedef struct psd_frame_layout {
    int64_t frame_stride, row_stride, pixel_stride, channel_stride;
} psd_frame_layout;

/* Engine configuration.  (src_width,src_height) is the size of the frames submitted;
 * (width,height) the size the detectors score at.  If they differ the engine applies the
 * exact cv2.resize(..., INTER_LINEAR) fixed-point bilinear of scene_manager.py:670-678. */
typedef struct psd_config {
    int32_t struct_size; /* sizeof(psd_config) */
    int32_t device;      /* CUDA ordinal */
    int32_t src_width, src_height;
    int32_t width, height;
    uint32_t features;        /* PSD_F_* */
    int32_t edge_kernel_size; /* dilate kernel k (odd >= 3); 0 = content_detector.py:39-46 estimate */
    int32_t max_batch;        /* frames per batch (staging and per-batch scratch are sized for it); an aligned
                                 device submission without resize, edges or hashes is scored in one batch */
    uint32_t flags;           /* reserved: no flags are defined, must be 0 */
    int32_t hash_size;        /* PSD_F_HASH: HashDetector(size=...) >= 1, 0 = 8 */
    int32_t hash_lowpass;     /* PSD_F_HASH: HashDetector(lowpass=...) >= 1, 0 = 2; the scored frame must be at
                                 least (size*lowpass) x (size*lowpass) */
    int32_t reserved[4];
} psd_config;

/* Per-frame integer results (device- and host-side layout, 64 bytes). */
typedef struct psd_frame_sums {
    uint64_t sad_hue;   /* sum |H_t - H_{t-1}|            */
    uint64_t sad_sat;   /* sum |S_t - S_{t-1}|            */
    uint64_t sad_lum;   /* sum |V_t - V_{t-1}|            */
    uint64_t sad_edges; /* sum |E_t - E_{t-1}|, E in {0,255} */
    uint64_t bgr_sum;   /* sum of all 3*W*H bytes          */
    uint64_t has_prev;  /* 0 for the first frame of a stream (content_detector.py:161-164) */
    uint64_t reserved[2];
} psd_frame_sums;

/* ---- library ---- */
int psd_abi_version(void);
const char* psd_version(void);
const char* psd_last_error(void);
int psd_device_count(void);
/* name_out may be NULL; fills compute capability, SM count and total memory. */
int psd_device_info(int device, char* name_out, size_t name_cap, int* cc_major, int* cc_minor,
                    int* sm_count, uint64_t* total_mem);
/* PCI bus id "0000:3b:00.0" of a device (lets a host place page-locked buffers on the GPU's NUMA node) */
int psd_device_pci_bus_id(int device, char* out, size_t cap);
/* total kernel launches issued by this library since load (for bench.py's gpu_launches). */
uint64_t psd_launch_count(void);

/* page-locked host memory for zero-staging submits */
int psd_host_alloc(size_t bytes, void** out);
int psd_host_free(void* p);
/* plain device memory + copies, so a torch-free host can keep batches resident in HBM */
int psd_device_alloc(int device, size_t bytes, void** out);
int psd_device_free(int device, void* p);
int psd_memcpy_h2d(int device, void* dst, const void* src, size_t bytes);
int psd_memcpy_d2h(int device, void* dst, const void* src, size_t bytes);

/* ---- engine: replaces the per-frame cv2/numpy work of detector.process_frame() ---- */
int psd_engine_create(const psd_config* cfg, psd_engine** out);
void psd_engine_destroy(psd_engine* e);
/* forget all frames and the carried previous frame (detector re-use on a new video) */
int psd_engine_reset(psd_engine* e);
/* Set the predecessor of the NEXT submitted frame (the one-frame halo of a time shard).
 * Source-size BGR24.  host variant copies before returning. */
int psd_engine_set_halo_host(psd_engine* e, const uint8_t* bgr, int64_t row_pitch);
int psd_engine_set_halo_device(psd_engine* e, const void* dptr);
/* Score n frames of host memory.  frame_stride / row_pitch in bytes (numpy strides:
 * the SceneManager crop view of scene_manager.py:666-668 is non-contiguous).  Without
 * PSD_SUBMIT_PINNED the bytes are copied to internal page-locked staging before return. */
int psd_engine_submit_host(psd_engine* e, const uint8_t* bgr, int64_t n_frames,
                           int64_t frame_stride, int64_t row_pitch, uint32_t flags);
/* Score n tightly packed frames already resident in HBM (row pitch = 3*src_width).
 * The memory must stay valid until psd_engine_sync(). */
int psd_engine_submit_device(psd_engine* e, const void* dptr, int64_t n_frames,
                             int64_t frame_stride);
/* Score n frames of device (or managed) memory on the engine's device in any layout (psd_frame_layout): packed
 * 16-byte-aligned BGR is read in place, a resizing engine reads the 2x2 taps of each output pixel straight from
 * the layout, anything else is first gathered to packed BGR (psd_gather_bgr) max_batch frames at a time.
 * PSD_ERR_INVALID for host memory or memory of another device.  The work is queued on the engine's compute
 * stream (psd_engine_compute_stream), which does not wait for any other stream: make it wait for the producer
 * of the frames first.  The memory must stay valid until psd_engine_sync(). */
int psd_engine_submit_device_layout(psd_engine* e, const void* base, int64_t n_frames,
                                    const psd_frame_layout* layout);
int psd_engine_sync(psd_engine* e);
/* the engine's compute stream (cudaStream_t): launch the psd_scan_* kernels (or record events)
 * on it to stay ordered after the engine's own kernels */
void* psd_engine_compute_stream(psd_engine* e);
int64_t psd_engine_frame_count(const psd_engine* e);
/* copy results for frames [first, first+n) to host (implies sync) */
int psd_engine_read_sums(psd_engine* e, int64_t first, int64_t n, psd_frame_sums* out);
int psd_engine_read_yhist(psd_engine* e, int64_t first, int64_t n, uint32_t* out /*[n][256]*/);
int psd_engine_read_hash(psd_engine* e, int64_t first, int64_t n,
                         uint64_t* out /*[n][PSD_HASH_WORDS_FOR(hash_size)]*/);
/* device pointers of the engine-owned result arrays (valid until destroy/reset) */
int psd_engine_device_results(psd_engine* e, const psd_frame_sums** sums, const uint32_t** yhist);
int psd_engine_device_hash(psd_engine* e, const uint64_t** hashes /* stream frame i at hashes + i*PSD_HASH_WORDS_FOR(
                                                                      hash_size); the halo frame's hash sits one
                                                                      stride before */);
/* CUDA-event time (ms) spent in the engine's kernels between the first launch after the last
 * psd_engine_timing_reset() and the last launch (on the engine's compute stream). */
int psd_engine_timing_reset(psd_engine* e);
int psd_engine_timing_ms(psd_engine* e, float* total_ms, float* score_kernel_ms,
                         uint64_t* score_kernel_launches);
/* effective dilate kernel size used for the edge component */
int psd_engine_edge_kernel_size(const psd_engine* e);

/* ---- slots: several ContentDetector kernel sizes and HashDetector geometries in one engine, as the reference's
 *      SceneManager runs any mix of detectors (scene_manager.py:337-352, each detector's process_frame on the same
 *      frame).  Every batch is uploaded, resized, scored by the fused pass and Canny-classified once; each edge
 *      slot adds a dilation and a SAD (content_detector.py:238), each hash slot its INTER_AREA taps, DCT and
 *      median (hash_detector.py:130-149) over the one gray pass.  Slot 0 is the psd_config's kernel size /
 *      geometry.  Slots can be added only while the engine holds no frames (after create or reset, before any
 *      submit or halo; PSD_ERR_STATE otherwise); a size / geometry already present returns its slot.  Each slot
 *      has its own carried predecessor and halo result. ---- */
/* content_detector.py:135-138 kernel_size of another detector (0 = the :39-46 estimate); needs PSD_F_EDGES */
int psd_engine_add_edge_kernel_size(psd_engine* e, int32_t kernel_size, int32_t* slot);
/* hash_detector.py:50-51 size / lowpass of another HashDetector (0 = 8 / 2); needs PSD_F_HASH */
int psd_engine_add_hash_geometry(psd_engine* e, int32_t size, int32_t lowpass, int32_t* slot);
/* effective kernel size of an edge slot, -1 if there is no such slot */
int psd_engine_edge_kernel_size_at(const psd_engine* e, int32_t slot);
/* device array of an edge slot's sad_edges (stream frame i at sad_edges[i], the halo frame's one before; valid until
 * destroy/reset); NULL for slot 0, whose SADs are psd_frame_sums.sad_edges */
int psd_engine_device_edge_sads(psd_engine* e, int32_t slot, const uint64_t** sad_edges);
/* psd_engine_device_hash / psd_engine_read_hash of a hash slot (stride PSD_HASH_WORDS_FOR(that slot's size)) */
int psd_engine_device_hash_at(psd_engine* e, int32_t slot, const uint64_t** hashes);
int psd_engine_read_hash_at(psd_engine* e, int32_t slot, int64_t first, int64_t n, uint64_t* out);
/* debug/test taps: copy intermediate planes of frame `index` of the LAST submitted batch.
 * which: 0 = scored-size BGR (after resize), 1 = V plane, 2 = Canny map (0/255), 3 = dilated edges (of the
 * last edge slot) */
int psd_engine_debug_plane(psd_engine* e, int which, int64_t index, uint8_t* out, size_t cap);

/* ---- trailing device scans over result arrays (all pointers are DEVICE pointers unless the
 *      name says host; `stream` is a cudaStream_t or NULL) ---- */
/* content_detector.py:166-180: components = sad / float(W*H); content_val = sum(c*w)/sum(|w|);
 * out_components[n][4], out_content_val[n]; frames with has_prev == 0 get 0.0 */
int psd_scan_content(const psd_frame_sums* sums, int64_t n, int64_t n_pixels, const double weights[4],
                     double weight_abs_sum /* sum(abs(w)) as the host computed it */,
                     double* out_components, double* out_content_val, void* stream);
/* psd_scan_content with the edge component's SAD read from sad_edges[n] (an edge slot's array,
 * psd_engine_device_edge_sads) when it is non-NULL: content_detector.py:166-180 for that kernel size */
int psd_scan_content_edges(const psd_frame_sums* sums, const uint64_t* sad_edges, int64_t n, int64_t n_pixels,
                           const double weights[4], double weight_abs_sum, double* out_components,
                           double* out_content_val, void* stream);
/* adaptive_detector.py:100-143: ratio for target i uses scores[i-w .. i+w]; out_ratio[i] is NaN
 * where the window is incomplete.  scores[] is the content_val array incl. frame 0's 0.0. */
int psd_scan_adaptive(const double* scores, int64_t n, int32_t window_width, double min_content_val,
                      double* out_ratio, void* stream);
/* threshold_detector.py:127: average_rgb = bgr_sum / (3*W*H) */
int psd_scan_average(const psd_frame_sums* sums, int64_t n, int64_t n_values, double* out_avg,
                     void* stream);
/* histogram_detector.py:98,159-163: rebin 256 -> bins, L2-normalise to float32 as cv2.normalize,
 * HISTCMP_CORREL in fp64 against the previous frame; out_correl[0] (no predecessor in the
 * array) uses prev_hist if non-NULL else is NaN. */
int psd_scan_hist_correl(const uint32_t* yhist, int64_t n, int32_t bins, const uint32_t* prev_hist,
                         double* out_correl, void* stream);
/* hash_detector.py:95-99: hash_dist = popcount(hash_t xor hash_{t-1}) / (size*size); out[0] uses prev_hash if
 * non-NULL else is NaN.  hashes and prev_hash have the stride PSD_HASH_WORDS_FOR(hash_size) */
int psd_scan_hash_dist(const uint64_t* hashes, int64_t n, int32_t hash_size, const uint64_t* prev_hash,
                       double* out_dist, void* stream);
/* >= / <= compare producing u8 flags (content_detector.py:210, histogram_detector.py:108) */
int psd_scan_compare(const double* values, int64_t n, double threshold, int32_t op /*0: >=, 1: <=, 2: <*/,
                     uint8_t* out_flags, void* stream);
/* ---- cut state machines on the device (SURVEY.md §8(f) N2).  Frame-number domain, constant frame
 *      rate: `min_frames` is the host's conversion of min_scene_len (common.py:480-486,627-638).
 *      cuts[cap] receives absolute frame numbers (first_frame + index), *count the number found
 *      (may exceed cap: only cap are stored).  All pointers are DEVICE pointers. ---- */
/* detector.py:160-224 FlashFilter over the `score >= threshold` flags; mode 0 = MERGE, 1 = SUPPRESS */
int psd_cuts_flash_filter(const uint8_t* above, int64_t n, int64_t first_frame, int64_t min_frames,
                          int32_t mode, int64_t* cuts, int32_t* count, int32_t cap, void* stream);
/* adaptive_detector.py:134-143 (ratio from psd_scan_adaptive, NaN where the window is incomplete) */
int psd_cuts_adaptive(const double* ratio, const double* score, int64_t n, int64_t first_frame,
                      int32_t window_width, double adaptive_threshold, double min_content_val,
                      int64_t min_frames, int64_t* cuts, int32_t* count, int32_t cap, void* stream);
/* histogram_detector.py:87-112: cut where correl <= threshold and min_frames since the last cut */
int psd_cuts_histogram(const double* correl, int64_t n, int64_t first_frame, double threshold,
                       int64_t min_frames, int64_t* cuts, int32_t* count, int32_t cap, void* stream);
/* hash_detector.py:104-109: cut where dist >= threshold and min_frames since the last cut (NaN = no predecessor) */
int psd_cuts_hash(const double* dist, int64_t n, int64_t first_frame, double threshold, int64_t min_frames,
                  int64_t* cuts, int32_t* count, int32_t cap, void* stream);
/* threshold_detector.py:113-191: fade in/out automaton incl. the post_process final cut */
int psd_cuts_threshold(const double* average, int64_t n, int64_t first_frame, double threshold,
                       int32_t method_ceiling, double fade_bias, int64_t min_frames, int32_t add_final_scene,
                       int64_t* cuts, int32_t* count, int32_t cap, void* stream);

/* ---- parameter sweep: every cell of a detector-parameter grid over one scored video ---- */
/* cell kinds: which automaton a cell runs, over which metric array(s) */
#define PSD_SWEEP_CONTENT 0   /* FlashFilter over content_val >= threshold (content_detector.py:210, detector.py:160-224) */
#define PSD_SWEEP_ADAPTIVE 1  /* adaptive_detector.py:134-143: metric = ratio, metric2 = content_val */
#define PSD_SWEEP_THRESHOLD 2 /* threshold_detector.py:113-191: metric = average_rgb */
#define PSD_SWEEP_HISTOGRAM 3 /* histogram_detector.py:87-112: metric = hist correl, threshold = 1 - t clamped */
#define PSD_SWEEP_HASH 4      /* hash_detector.py:79-109: metric = hash_dist (NaN = no predecessor) */
#define PSD_SWEEP_MAX_TOLERANCES 8
/* One grid cell (64 bytes): the arguments the matching psd_cuts_* call takes.  Metric arrays are DEVICE
 * pointers of n doubles (the psd_scan_* outputs); cells that share an array should be adjacent so that
 * the 32 cells of a warp read each frame's value with one broadcast load. */
typedef struct psd_sweep_cell {
    int32_t kind;             /* PSD_SWEEP_* */
    int32_t mode;             /* CONTENT: 0 = MERGE, 1 = SUPPRESS; THRESHOLD: 1 = Method.CEILING; else 0 */
    const double* metric;     /* see the kinds */
    const double* metric2;    /* ADAPTIVE: content_val; else NULL */
    double threshold;         /* CONTENT / THRESHOLD / HISTOGRAM / HASH threshold, ADAPTIVE adaptive_threshold */
    double min_content_val;   /* ADAPTIVE */
    double fade_bias;         /* THRESHOLD */
    int64_t min_frames;       /* min_scene_len in frames, as for psd_cuts_* */
    int32_t window;           /* ADAPTIVE window_width (>= 1) */
    int32_t add_final_scene;  /* THRESHOLD */
} psd_sweep_cell;
/* benchmark/sweep.py:142-187 runs one SceneManager + detector per cell; here one thread per cell walks
 * the metric arrays with the automaton psd_cuts_* runs.  cells is a HOST array (validated, then copied
 * on `stream`); cuts[n_cells][cap] and count[n_cells] are DEVICE arrays: cell k's cut frames
 * (first_frame + index, in emission order) and how many it found (may exceed cap: only cap are stored). */
int psd_sweep_cuts(const psd_sweep_cell* cells, int32_t n_cells, int64_t n, int64_t first_frame, int64_t* cuts,
                   int32_t* count, int32_t cap, void* stream);
/* benchmark/evaluator.py:227-331 (score_video) for every (cell, tolerance), on the cells' cut lists from
 * psd_sweep_cuts.  Each cell's list is first turned, in place, into the predicted list of
 * benchmark/sweep.py:169 (`scene[1]` of SceneManager.get_scene_list()): sorted unique cuts followed by
 * end_frame, or nothing when the cell has no cut; out_n_pred[cell] is its length (-1: count > cap, the
 * cell overflowed and is not scored).  Fade intervals ([n_fades][2], inclusive) match first-hit in the
 * order given; the remaining predictions match the strictly increasing gt_cuts greedily by distance.
 * out_hard[n_cells][n_tol][5] = matched, false_positives, missed, offset_sum, offset_count;
 * out_fades[n_cells][3] = matched, false_positives, missed.  tolerances is a HOST array (n_tol <=
 * PSD_SWEEP_MAX_TOLERANCES); every other pointer is a DEVICE pointer.  workspace holds the matching
 * bitmaps: n_cells * n_tol * 4 * (ceil((cap + 1) / 32) + ceil(n_gt / 32) + ceil(n_fades / 32)) bytes. */
int psd_sweep_eval(int64_t* cuts, const int32_t* count, int32_t n_cells, int32_t cap, int64_t end_frame,
                   const int64_t* gt_cuts, int32_t n_gt, const int64_t* fades, int32_t n_fades,
                   const int32_t* tolerances, int32_t n_tol, void* workspace, size_t workspace_bytes,
                   int32_t* out_n_pred, int64_t* out_hard, int64_t* out_fades, void* stream);

/* ---- many clips in one engine pass: clips scored back to back into one engine, then every clip's cuts ----
 * A clip table is a DEVICE int64[n_clips + 1]: offsets[0] = 0, non-decreasing, offsets[n_clips] = n; clip j is
 * frames [offsets[j], offsets[j+1]) of the pass. */
/* After the psd_scan_* that filled values[n] over the whole pass: for every clip [b, e), values[i] = fill for i in
 * [b, min(b + head, e)) and in [max(e - tail, b), e): CUDART_NAN (sign bit set) when fill_nan is 1, else `fill` as
 * given, bit for bit.  This gives each clip the entries a one-clip engine's scan has there, in the scan's own bits:
 * content_val head 1, 0.0 (content_detector.py:161-164); adaptive ratio head w, tail w, fill_nan, after the
 * content_val fix-up (adaptive_detector.py:111-115); hist correl head 1, fill_nan; hash dist head 1, fill = the NaN
 * with the sign bit clear that psd_scan_hash_dist writes (no predecessor); average_rgb none. */
int psd_clip_fill(double* values, int64_t n, const int64_t* clip_offsets, int32_t n_clips, int32_t head, int32_t tail,
                  int32_t fill_nan, double fill, void* stream);
/* Every (cell, clip) automaton in one pass: cell k over clip j's slice of its metric arrays, with frame numbers from
 * clip_first_frame[j] and min_frames[k * n_clips + j].  cells is a HOST array (validated as psd_sweep_cuts does,
 * then copied on `stream`); everything else is DEVICE memory.  cut_offsets[n_cells * n_clips + 1] receives the
 * exclusive offsets of the (cell, clip) cut lists, cell-major, and their total; cuts[cut_offsets[t] ..] the cuts
 * of (cell, clip) t in emission order.  When the total exceeds cuts_cap, the offsets and the total are written and
 * no cut is: grow the cut array and call again. */
int psd_clip_cuts(const psd_sweep_cell* cells, int32_t n_cells, const int64_t* clip_offsets,
                  const int64_t* clip_first_frame, int32_t n_clips, const int64_t* min_frames, int64_t* cuts,
                  int64_t cuts_cap, int64_t* cut_offsets, void* stream);
/* psd_clip_cuts for clips read with SceneManager.detect_scenes(frame_skip = frame_step - 1): the per-frame loop
 * processes every frame_step-th frame and reads the frames between them without processing them
 * (scene_manager.py:682-685), so element i of clip j's slice is frame clip_first_frame[j] + i * frame_step, and the
 * automata (detector.py:160-224, adaptive_detector.py:134-143, histogram_detector.py:87-112,
 * hash_detector.py:79-109, threshold_detector.py:113-168) compare those true frame numbers with min_frames, which
 * stays in frames.  ThresholdDetector's post_process (threshold_detector.py:170-191) gets the stream's position after
 * the loop (scene_manager.py:618-621), which is past the last processed frame when skipped frames were read behind
 * it: clip_end_frame[j] - 1, clip_end_frame being the DEVICE int64[n_clips] end frames psd_clip_eval takes (that
 * position + 1), or NULL for the last processed frame.  frame_step >= 1; frame_step 1 and a NULL clip_end_frame give
 * psd_clip_cuts' results bit for bit.  Same kernels and launches as psd_clip_cuts. */
int psd_clip_cuts_step(const psd_sweep_cell* cells, int32_t n_cells, const int64_t* clip_offsets,
                       const int64_t* clip_first_frame, int32_t n_clips, const int64_t* min_frames, int64_t* cuts,
                       int64_t cuts_cap, int64_t* cut_offsets, int64_t frame_step, const int64_t* clip_end_frame,
                       void* stream);
/* psd_clip_cuts_step for clips read with different frame skips, each clip through its own window of
 * SceneManager.detect_scenes(frame_skip = frame_step[j] - 1) (scene_manager.py:682-685): element i of clip j's slice
 * is frame clip_first_frame[j] + i * frame_step[j], and the automata compare those true frame numbers with
 * min_frames as psd_clip_cuts_step's do (detector.py:160-224, adaptive_detector.py:134-143,
 * histogram_detector.py:87-112, hash_detector.py:79-109, threshold_detector.py:113-168).  post_process
 * (threshold_detector.py:170-191) gets clip_end_frame[j] - 1, the stream's position after the loop
 * (scene_manager.py:618-621), or the last processed frame when clip_end_frame is NULL.  frame_step is a HOST
 * int64[n_clips], every entry >= 1 (validated, then copied on `stream` with the cells); the other arrays are as
 * psd_clip_cuts_step's.  With every frame_step[j] equal to s it gives psd_clip_cuts_step(frame_step = s)'s results
 * bit for bit.  Same kernels and launches as psd_clip_cuts. */
int psd_clip_cuts_steps(const psd_sweep_cell* cells, int32_t n_cells, const int64_t* clip_offsets,
                        const int64_t* clip_first_frame, int32_t n_clips, const int64_t* min_frames, int64_t* cuts,
                        int64_t cuts_cap, int64_t* cut_offsets, const int64_t* frame_step,
                        const int64_t* clip_end_frame, void* stream);
/* benchmark/evaluator.py:227-331 (score_video) for every (cell, clip, tolerance) on psd_clip_cuts' output, and the
 * counts summed over the clips (evaluator.py:167-186).  cuts / cut_offsets are psd_clip_cuts' arrays and cuts_total
 * its total cut_offsets[n_cells * n_clips]; each (cell, clip) list is first turned, in place, into the predicted list
 * of benchmark/sweep.py:169 (sorted unique cuts followed by clip_end_frame[clip], or nothing when there is no cut) and
 * out_n_pred[cell * n_clips + clip] is its length (-1: more than max_cuts cuts, not scored).  Clip j's ground truth
 * is gt_cuts[gt_offsets[j] .. gt_offsets[j+1]) (strictly increasing) and fades[fade_offsets[j] ..
 * fade_offsets[j+1])[2] (inclusive), matched as psd_sweep_eval matches.  Outputs:
 *   out_hard[n_cells][n_clips][n_tol][5]  matched, false_positives, missed, offset_sum, offset_count
 *   out_fades[n_cells][n_clips][3]        matched, false_positives, missed
 *   out_totals_hard[n_cells][n_tol][5], out_totals_fades[n_cells][3]: the same summed over the clips
 *   out_over[1]                           the lowest cell * n_clips + clip with more than max_cuts cuts, or -1
 * tolerances is a HOST array (n_tol <= PSD_SWEEP_MAX_TOLERANCES); every other pointer is a DEVICE pointer.
 * workspace holds the matching bitmaps: 4 * (n_tol * (n_cells * n_clips + ceil(cuts_total / 32))
 * + n_cells * n_tol * (2 * n_clips + ceil(n_gt / 32) + ceil(n_fades / 32))) bytes. */
int psd_clip_eval(int64_t* cuts, const int64_t* cut_offsets, int32_t n_cells, int32_t n_clips, int64_t cuts_total,
                  int64_t max_cuts, const int64_t* clip_end_frame, const int64_t* gt_offsets, const int64_t* gt_cuts,
                  int32_t n_gt, const int64_t* fade_offsets, const int64_t* fades, int32_t n_fades,
                  const int32_t* tolerances, int32_t n_tol, void* workspace, size_t workspace_bytes,
                  int32_t* out_n_pred, int64_t* out_hard, int64_t* out_fades, int64_t* out_totals_hard,
                  int64_t* out_totals_fades, int64_t* out_over, void* stream);
/* ---- several clip tables in one launch: the same clips scored under several settings (crop, downscale, frame
 * step), each setting's engine with its own pass layout ----
 * One table (32 bytes) describes how one setting's engine holds the clips: clip j is elements [offsets[j],
 * offsets[j+1]) of that setting's metric arrays, element i of it is frame first_frame[j] + i * frame_step, and
 * end_frame[j] is the clip's end (the stream's position after that setting's reads + 1).  Every pointer is DEVICE
 * memory; every table has the same n_clips.  psd_clip_cuts / psd_clip_cuts_step / psd_clip_eval are the one-table
 * calls of these entries' kernels. */
typedef struct psd_clip_table {
    const int64_t* offsets;     /* int64[n_clips + 1] */
    const int64_t* first_frame; /* int64[n_clips] (psd_clip_cuts_tables) */
    const int64_t* end_frame;   /* int64[n_clips]; NULL for psd_clip_cuts_tables: post_process gets the last element */
    int64_t frame_step;         /* >= 1 */
} psd_clip_table;
/* psd_clip_cuts_step with a table per cell: cell k runs over tables[cell_table[k]] (cell_table NULL: every cell over
 * tables[0]), reading its own metric arrays, with min_frames[k * n_clips + j].  tables[n_tables] and
 * cell_table[n_cells] are HOST arrays (validated, then copied on `stream` with the cells).  Output as psd_clip_cuts.
 * Same kernels and launches as psd_clip_cuts. */
int psd_clip_cuts_tables(const psd_sweep_cell* cells, int32_t n_cells, const psd_clip_table* tables, int32_t n_tables,
                         const int32_t* cell_table, int32_t n_clips, const int64_t* min_frames, int64_t* cuts,
                         int64_t cuts_cap, int64_t* cut_offsets, void* stream);
/* A psd_clip_table whose clips each step by their own frame_step (clips read with different frame skips, the same
 * step under every setting): element i of clip j is frame first_frame[j] + i * frame_step[j].  32 bytes, every pointer
 * DEVICE memory; end_frame sits where psd_clip_table's does, so psd_clip_eval_tables takes the same three arrays as a
 * psd_clip_table. */
typedef struct psd_clip_steps_table {
    const int64_t* offsets;     /* int64[n_clips + 1] */
    const int64_t* first_frame; /* int64[n_clips] */
    const int64_t* end_frame;   /* int64[n_clips]; NULL: post_process gets the last element */
    const int64_t* frame_step;  /* int64[n_clips], every entry >= 1 (device memory: not validated; a smaller step
                                   gives meaningless frame numbers and touches nothing outside the arrays) */
} psd_clip_steps_table;
/* psd_clip_cuts_tables with a step per (table, clip): cell k runs over tables[cell_table[k]] and clip j steps by that
 * table's frame_step[j], as psd_clip_cuts_steps steps it for one table.  tables and cell_table are HOST arrays
 * (validated, then copied on `stream` with the cells).  With every frame_step[j] of a table equal to s it gives
 * psd_clip_cuts_tables with that table's frame_step = s bit for bit.  Same kernels and launches as psd_clip_cuts. */
int psd_clip_cuts_tables_steps(const psd_sweep_cell* cells, int32_t n_cells, const psd_clip_steps_table* tables,
                               int32_t n_tables, const int32_t* cell_table, int32_t n_clips, const int64_t* min_frames,
                               int64_t* cuts, int64_t cuts_cap, int64_t* cut_offsets, void* stream);
/* psd_clip_eval with a table per cell: (cell k, clip j)'s predicted list ends at tables[cell_table[k]].end_frame[j]
 * (cell_table NULL: tables[0]); only end_frame is read.  tables and cell_table are HOST arrays, copied on `stream`.
 * Ground truth, outputs and workspace as psd_clip_eval: the ground truth is per clip, shared by every table.  Same
 * kernels and launches as psd_clip_eval. */
int psd_clip_eval_tables(int64_t* cuts, const int64_t* cut_offsets, int32_t n_cells, int32_t n_clips,
                         int64_t cuts_total, int64_t max_cuts, const psd_clip_table* tables, int32_t n_tables,
                         const int32_t* cell_table, const int64_t* gt_offsets, const int64_t* gt_cuts, int32_t n_gt,
                         const int64_t* fade_offsets, const int64_t* fades, int32_t n_fades, const int32_t* tolerances,
                         int32_t n_tol, void* workspace, size_t workspace_bytes, int32_t* out_n_pred,
                         int64_t* out_hard, int64_t* out_fades, int64_t* out_totals_hard, int64_t* out_totals_fades,
                         int64_t* out_over, void* stream);
/* ---- cells that are sets of detectors: one SceneManager with several detectors cuts at the sorted union of their
 * cuts (scene_manager.py:403-408) ---- */
#define PSD_SWEEP_MAX_MEMBERS 16 /* lists per cell of psd_clip_union */
/* Every (cell, clip) union of psd_clip_cuts' (list, clip) cut lists, in two calls with the same arguments.  cuts /
 * cut_offsets are psd_clip_cuts' output over n_lists cells (here: lists) and n_clips clips, cuts_total its total.
 * Cell k is the set of lists cell_lists[cell_offsets[k] .. cell_offsets[k + 1]): 1 to PSD_SWEEP_MAX_MEMBERS indices
 * in [0, n_lists), repeats allowed; cell_offsets[n_cells + 1] (cell_offsets[0] = 0) and cell_lists are HOST int32
 * arrays (validated, then copied on `stream`).  unique is a DEVICE int32[n_lists * n_clips] workspace kept between
 * the two calls; everything else but the cell table is DEVICE memory.
 *   Counting call (out_cuts NULL, out_cap 0; three launches): every list is sorted and de-duplicated in place (the
 *   lists are read by many cells) and its length stored in unique; a list with more than max_cuts cuts counts as
 *   empty and out_over[0] receives the lowest such list * n_clips + clip, or -1.  out_offsets[n_cells * n_clips + 1]
 *   receives the exclusive offsets of the (cell, clip) unions, cell-major, and their total.
 *   Writing call (out_cuts of out_cap entries; one launch): out_cuts[out_offsets[t] ..] receives the strictly
 *   increasing union of (cell, clip) t, from the lists, unique and out_offsets the counting call left; nothing when
 *   the total exceeds out_cap.  out_over is not written. */
int psd_clip_union(int64_t* cuts, const int64_t* cut_offsets, int32_t n_lists, int32_t n_clips, int64_t cuts_total,
                   int64_t max_cuts, const int32_t* cell_offsets, const int32_t* cell_lists, int32_t n_cells,
                   int32_t* unique, int64_t* out_cuts, int64_t out_cap, int64_t* out_offsets, int64_t* out_over,
                   void* stream);
/* One column of a StatsManager CSV (stats_manager.py:save_to_csv) over a pass: frame i's value is values[i * stride]
 * (a psd_scan_* output, stride 1, or one component of psd_scan_content's out_components, stride 4).  The first `head`
 * and the last `tail` frames of every clip have no value there: the cell prints None. */
typedef struct psd_stats_column {
    const double* values; /* DEVICE */
    int64_t stride;
    int32_t head;
    int32_t tail;
} psd_stats_column;
#define PSD_STATS_MAX_COLUMNS 64
/* Every clip's StatsManager CSV rows, without the header, in one pass: for each frame of clip j that some column has
 * a value for, `frame_num + 1,HH:MM:SS.nnn,` then every column's str(value) or None, comma-separated, and "\n"; frame_num
 * = clip_first_frame[j] + the frame's index in the clip, the timecode FrameTimecode(frame_num, rate).get_timecode()
 * with rate = clip_rate[j] (float(frame rate)).  columns is a HOST array in CSV order (validated, then copied on
 * `stream`); everything else is DEVICE memory.  n = clip_offsets[n_clips] frames; row_offsets[n + 1] is workspace.
 * out receives clip 0's rows, then clip 1's, ...; clip_bytes[n_clips + 1] their exclusive byte offsets and the total.
 * When the total exceeds out_cap, clip_bytes is written and the text is not: grow out and call again. */
int psd_clip_stats_csv(const psd_stats_column* columns, int32_t n_columns, const int64_t* clip_offsets,
                       const int64_t* clip_first_frame, const double* clip_rate, int32_t n_clips, int64_t n,
                       int64_t* row_offsets, char* out, int64_t out_cap, int64_t* clip_bytes, void* stream);

/* ---- JPEG scene images: scenedetect/output/image.py:317-319, cv2.imencode(".jpg", frame, [IMWRITE_JPEG_QUALITY, q])
 *      for every selected frame ---- */
/* One image: width x height pixels of 8-bit B, G, R at `base` in `layout` (frame_stride is not read). */
typedef struct psd_jpeg_image {
    const void* base; /* DEVICE (or managed) memory: channel B of pixel (0, 0) */
    psd_frame_layout layout;
    int32_t width, height; /* 1 to 65535 each */
} psd_jpeg_image;
/* The baseline JPEG file cv2.imencode writes for each image, byte for byte (libjpeg-turbo: jpeg_set_quality(quality,
 * force_baseline) after cv2's clamp of quality to [0, 100], JFIF 1.01, 4:2:0, the T.81 Annex K Huffman tables, no
 * restart interval).  images[n] is a HOST array; out, image_bytes[n + 1] are DEVICE memory.  out receives image 0's
 * file, then image 1's, ...; image_bytes their exclusive byte offsets and the total.  A file that would end past
 * out_cap is not written (the files are written in order, so those that are form a prefix): when image_bytes[n]
 * exceeds out_cap, grow out and call again.  The images are encoded in sub-batches whose workspace (allocated on
 * `stream`) stays within workspace_cap bytes (0: 512 MiB), each at least one image: about 65 350 bytes per tile of 32
 * MCUs of 16x16 pixels, i.e. about 510 bytes per 8x8 luma block (a 1920x1080 image is 255 tiles, 16.7 MB); eight
 * launches per sub-batch, queued on `stream` (a cudaStream_t or NULL), not waited for. */
int psd_jpeg_encode(int device, const psd_jpeg_image* images, int32_t n, int32_t quality, int64_t workspace_cap,
                    uint8_t* out, int64_t out_cap, int64_t* image_bytes, void* stream);

/* ---- JPEG image sequences: cv2.imread(path, IMREAD_COLOR) of every file, decoded on the device ---- */
/* Why psd_jpeg_probe refuses a file (refusal): */
#define PSD_JPEG_OK 0
#define PSD_JPEG_TRUNCATED 1    /* a marker segment or the scan runs past the end, or there is no EOI after the scan */
#define PSD_JPEG_NOT_JPEG 2     /* no SOI */
#define PSD_JPEG_PROCESS 3      /* progressive, lossless, hierarchical or arithmetic-coded (SOF2-SOF15) */
#define PSD_JPEG_PRECISION 4    /* not 8-bit samples */
#define PSD_JPEG_COMPONENTS 5   /* not 1 or 3 components, or 3 that libjpeg takes as RGB: no JFIF marker, and an
                                   Adobe transform of 0 or (no Adobe marker) component ids 'R', 'G', 'B' */
#define PSD_JPEG_SAMPLING 6     /* luma not 1x1, 2x1 or 2x2 over 1x1 chroma (4:1:1, 4:4:0, ...) */
#define PSD_JPEG_MULTI_SCAN 7   /* a scan that does not hold every component (non-interleaved), or a second frame */
#define PSD_JPEG_ORIENTATION 8  /* an EXIF orientation other than 1: imread would rotate the image */
#define PSD_JPEG_TABLES 9       /* a missing or malformed quantisation or Huffman table */
typedef struct psd_jpeg_info {
    int32_t width, height, components;
    int32_t h_samp, v_samp;        /* luma sampling factors (chroma is 1x1); 1, 1 for gray */
    int32_t restart_interval;      /* MCUs per restart interval, 0 for none */
    int32_t refusal;               /* PSD_JPEG_* */
    int32_t reserved;
    int64_t scan_begin, scan_end;  /* the entropy-coded data: bytes [scan_begin, scan_end), up to the last EOI */
} psd_jpeg_info;
/* Parses one file's markers up to its scan (host only: no CUDA call).  Returns PSD_OK and fills *info; info->refusal
 * says whether psd_jpeg_decode takes the file.  Baseline (SOF0) and extended-sequential Huffman (SOF1) 8-bit files
 * of 1 or 3 components in one interleaved scan, with 4:4:4, 4:2:2 or 4:2:0 sampling, any restart interval and any
 * (optimised) Huffman tables. */
int psd_jpeg_probe(const uint8_t* data, int64_t size, psd_jpeg_info* info);
/* One file: the same `size` bytes at `host` (its markers are parsed there) and at `device` (DEVICE memory, decoded). */
typedef struct psd_jpeg_source {
    const void* host;
    const void* device;
    int64_t size;
} psd_jpeg_source;
/* Decodes n files into images[n] (a HOST array; each image's base is DEVICE memory and its width and height must be
 * the file's), byte for byte what cv2.imread gives (libjpeg-turbo 3.1: jdhuff.c decode_mcu, jidctint.c
 * jpeg_idct_islow with IDCT_range_limit's & RANGE_MASK wrap, jdsample.c h2v1 / h2v2 fancy upsampling when the
 * downsampled width is above 2 and h2v1 / h2v2 replication otherwise (jinit_upsampler), jdmainct.c context rows
 * replicating the first and last chroma rows, jdcolor.c build_ycc_rgb_table / ycc_rgb_convert, gray replicated to
 * B, G, R).  A file psd_jpeg_probe refuses is PSD_ERR_INVALID, and nothing is queued.  error_flags[n] (DEVICE) is
 * set to 0 for a file that decodes and nonzero for one whose entropy-coded data does not (its image is then
 * unspecified): read it after `stream`.  The files are decoded in sub-batches whose workspace (allocated on `stream`)
 * stays within workspace_cap bytes (0: 512 MiB), each at least one file: about 1.2 times the file's bytes, 132 bytes
 * per 8x8 block and 64 per block of component samples (a 1920x1080 4:2:0 file of 500 KB takes about 11 MB); thirteen
 * launches per sub-batch, queued on `stream` (a cudaStream_t or NULL), not waited for. */
int psd_jpeg_decode(int device, const psd_jpeg_source* srcs, int32_t n, const psd_jpeg_image* images,
                    int64_t workspace_cap, int32_t* error_flags, void* stream);

/* host-convenience wrappers: engine-owned sums -> host arrays (numpy), implies sync */
int psd_engine_scan_content_host(psd_engine* e, int64_t first, int64_t n, const double weights[4],
                                 double weight_abs_sum, double* out_components,
                                 double* out_content_val);
int psd_engine_scan_adaptive_host(psd_engine* e, const double* scores_host, int64_t n,
                                  int32_t window_width, double min_content_val, double* out_ratio);
int psd_engine_scan_average_host(psd_engine* e, int64_t first, int64_t n, double* out_avg);
int psd_engine_scan_hist_correl_host(psd_engine* e, int64_t first, int64_t n, int32_t bins,
                                     double* out_correl);
int psd_engine_scan_hash_dist_host(psd_engine* e, int64_t first, int64_t n, double* out_dist);
/* the same over an edge slot's / a hash slot's results */
int psd_engine_scan_content_host_at(psd_engine* e, int32_t edge_slot, int64_t first, int64_t n,
                                    const double weights[4], double weight_abs_sum, double* out_components,
                                    double* out_content_val);
int psd_engine_scan_hash_dist_host_at(psd_engine* e, int32_t hash_slot, int64_t first, int64_t n, double* out_dist);

/* ---- synthetic input generator (bench.py / tests; pyscenedetect_b200/synth.py bit-exact twin) ---- */
/* params_host: [n][24] int32 rows of ScenePlan.params for frames first..first+n-1 */
int psd_synth_frames(int device, void* d_out, const int32_t* params_host, int64_t n, int32_t width,
                     int32_t height, int64_t frame_stride, void* stream);

/* ---- layout conversion ---- */
/* n frames of width x height in `layout` at device (or managed) memory `base` -> packed BGR24 at device memory
 * dst, dst_frame_stride bytes apart; queued on `stream` (a cudaStream_t or NULL), not waited for */
int psd_gather_bgr(int device, const void* base, const psd_frame_layout* layout, int64_t n, int32_t width,
                   int32_t height, void* dst, int64_t dst_frame_stride, void* stream);

/* ---- test hooks ---- */
/* device BGR (n pixels, a multiple of 16) -> H,S,V and Y planes with the device functions the fused pass uses */
int psd_test_hsv(int device, const uint8_t* bgr_host, int64_t n_pixels, uint8_t* h_out, uint8_t* s_out,
                 uint8_t* v_out, uint8_t* y_out);
/* The INTER_LINEAR tap tables the engine builds for resizing one axis from src to dst pixels: ofs[dst] (the first
 * source index; the second is ofs + 1, clamped to src - 1) and coef[dst][2] (11-bit coefficients).  Host only: no
 * CUDA call, so it runs without a device. */
int psd_test_resize_taps(int32_t src, int32_t dst, int32_t* ofs, int16_t* coef);
/* str() of n host doubles with the device formatter psd_clip_stats_csv prints values with: text_out[n][32], each
 * value's text followed by NUL bytes */
int psd_test_format_f64(int device, const double* values_host, int64_t n, char* text_out);
/* HashDetector's stages through the engine's hash kernels: n_frames packed BGR24 frames (width x height, frame_stride
 * bytes apart) in DEVICE memory of `device`, and n_geo (1 to 16) geometries {size, lowpass} in geometries[n_geo][2].
 * Builds each geometry's plan for n_frames frames and runs the hash pass once.  Host outputs, geometry g's block
 * after geometry g-1's, n = size * lowpass:
 *   rowbuf_out [n_frames][height][n] float32: the horizontal pass (raw uint32 column sums where width and height
 *              are multiples of n), or NULL
 *   hash_out   [n_frames][PSD_HASH_WORDS_FOR(size)]
 *   image_out  [n_frames][n][n] float64: the normalised image, or NULL
 *   low_out    [n_frames][size][size] float32: the low band of the DCT, or NULL
 * A non-NULL image_out or low_out keeps the finish kernel's working set in global memory for every geometry.  Any of
 * rowbuf_out, image_out, low_out needs n_frames to fit one sub-batch of every geometry (PSD_ERR_INVALID otherwise). */
int psd_test_hash_stages(int device, const void* frames, int64_t n_frames, int32_t width, int32_t height,
                         int64_t frame_stride, const int32_t* geometries, int32_t n_geo, float* rowbuf_out,
                         uint64_t* hash_out, double* image_out, float* low_out);

#ifdef __cplusplus
}
#endif
#endif /* PSD_B200_H */
