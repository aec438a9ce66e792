/* lav_b200 — C ABI of the H100-native LAV frame-path kernels (sm_90a).
 *
 * The reference (dotchen/LAV) has no FFI: its boundary is Python (torch modules).  A
 * reference-side maintainer binds these entry points with ctypes (see INTEGRATION.md);
 * lav_b200/capi.py is that binding.  Every pointer named d_* is a DEVICE pointer,
 * h_* is a HOST pointer read synchronously during the call.  `stream` is a
 * cudaStream_t passed as void* (0 = legacy default stream).  All functions return 0
 * on success and a non-zero code otherwise; lavb_last_error() gives the message
 * (thread-local).  No global mutable state; safe from several host threads
 * (nn.DataParallel-style) as long as each uses its own stream/workspace.
 *
 * Layouts: activations are NHWC ("channels last"); `*_cstride` is the number of
 * channels of the underlying buffer (pixel stride in elements) and `*_coff` the first
 * channel this call reads/writes, so concatenations are written in place.
 */
#ifndef LAV_B200_H
#define LAV_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LAVB_ABI_VERSION 3

int lavb_abi_version(void);
const char* lavb_last_error(void);
/* compute capability major*10+minor of the current device, or <0 when no device */
int lavb_device_cc(void);

/* ---------------------------------------------------------------- element types */
enum { LAVB_F32 = 0, LAVB_BF16 = 1, LAVB_F16 = 2 };
/* The 16-bit storage type of the tensor-core path ("h16" below) is fixed when the library is built: IEEE half (LAVB_F16) by
 * default — fp32 accumulation everywhere, every fp32 -> half conversion saturates at +-65504 — or bfloat16 with
 * -DLAVB_H16_BF16.  Entry points that take a dtype accept LAVB_F32 and this value only. */
int lavb_h16_dtype(void);

/* ---------------------------------------------------------------- point painting
 * replaces: InferModel.point_painting / forward_paint (team_code_v2/model_inference.py:44-50,75-93),
 *           CoordConverter.forward (model_inference.py:280-297),
 *           point_painting() (lav/utils/point_painting.py:46-66).
 * h_cams: ncam x 41 floats = K(3x3 row-major) | lidar_to_world(4x4) | world_to_cam(4x4).
 * sem element (cam,c,v,u) lives at d_sem[cam*s_cam + c*s_c + v*s_y + u*s_x].
 * mode 0: gather c_in channels as they are           -> c_in outputs
 * mode 1: d_sem holds softmax probabilities (c_in>=2) -> c_in-1 outputs p[1+j]*(1-p[0])
 * mode 2: d_sem holds logits; softmax over c_in then as mode 1
 * Row i of the output receives `copy_cols` leading columns of point i, then the painted
 * channels at column `out_col0`; later cameras overwrite earlier ones; unseen points get 0.
 * Projection, bit for bit (project_hit.cuh): per camera, k-sequential fp32 FMA chains lidar_to_world, world_to_cam, the axis
 *   swap (y, -z, x) and K; u = q0 / (1e-5f + q2), v = q1 / (1e-5f + q2) (IEEE division), each and q2 truncated toward zero to
 *   int64, where NaN, +-inf and |value| >= 2^63 give INT64_MIN; a camera sees the point when q2' >= 0, 0 <= u < w, 0 <= v < h.
 * Values: mode 0 copies the sem bits (NaN payloads included); mode 1 computes bg = 1 - p0 and p[k] * bg in fp32; mode 2 first
 *   p = expf(x - max) / sum in fp32 (fmaxf max, so a NaN logit is skipped by the max; sum in class order; IEEE division), so any
 *   NaN or +inf logit, or all logits -inf, gives NaN in every painted channel of that point.  Copied columns keep their bits.
 * Written: per row the copy_cols leading columns and the c_out channels at out_col0, nothing else (columns between them and
 *   past out_col0 + c_out keep their values).
 * Checked before any launch (a rejected call writes nothing): n >= 0, pt_stride >= 3, ncam 1..4, mode 0..2, c_in 1..8 (mode
 *   0) or 2..8, copy_cols <= pt_stride, copy_cols <= out_col0, out_col0 + c_out <= out_stride, frames 0..65535; then, unless n
 *   or frames is 0 (nothing written), non-null pointers and d_pts / d_sem / d_out 4-byte aligned.  h_cams must hold 41 * ncam
 *   floats.  Any alignment above that is optional: the point row is read as one 16-byte vector when pt_stride is 4 and every
 *   frame's rows are 16-byte aligned, and the copied columns stored as one when copy_cols is 4, out_col0 >= 4 and every output
 *   row is 16-byte aligned; other layouts are read and written element by element. */
int lavb_paint(const float* d_pts, int n, int pt_stride,
               const float* d_sem, int ncam, int c_in, int h, int w,
               long long s_cam, long long s_c, long long s_y, long long s_x,
               const float* h_cams, int mode,
               float* d_out, int out_stride, int out_col0, int copy_cols, void* stream);

/* the same for `frames` independent agents in one launch: frame f reads points at d_pts + f*pts_frame_stride (floats),
 * semantic maps at d_sem + f*s_frame, writes rows at d_out + f*out_frame_stride (floats). */
int lavb_paint_batched(const float* d_pts, int frames, int n, int pt_stride, long long pts_frame_stride,
                       const float* d_sem, int ncam, int c_in, int h, int w, long long s_frame, long long s_cam,
                       long long s_c, long long s_y, long long s_x, const float* h_cams, int mode, float* d_out,
                       int out_stride, long long out_frame_stride, int out_col0, int copy_cols, void* stream);

/* painting straight from the ERFNet decoder's last 16-channel feature map: the segmentation head's final layer
 * replaces: Decoder.output_conv = ConvTranspose2d(16, c_cls, 2, stride 2) (lav/models/erfnet.py:122-124,132) + torch.softmax
 *           (lav_agent_fast.py:264) + the background suppression and gather of forward_paint (model_inference.py:44-50,75-93),
 * evaluated for the hit pixel only, so the (h x w x c_cls) logit maps are never materialised.
 * d_feat: NHWC (frames*ncam, h/2, w/2, 16) fp32 or h16 = input of output_conv; d_deconv: 2*2*16*8 + 8 = 520 floats =
 * w[v%2][u%2][c_in][k] (k >= c_cls zero) | bias[8].  Output row as lavb_paint mode 2: copy_cols point columns, then c_cls-1
 * painted channels at out_col0.  The hit pixel (v, u) of camera c in frame f reads feature pixel (v/2, u/2) of image f*ncam + c;
 * logit k = bias[k], then fmaf(feat[ch], w[v&1][u&1][ch][k], .) over ch = 0..15 in order (h16 features widened exactly), then
 * lavb_paint's mode-2 softmax, NaN rule and suppression.  Projection, written columns and layout checks as lavb_paint; also
 * checked: c_cls 2..8, h and w even, feat_dtype LAVB_F32 or the 16-bit type, and (n, frames > 0) non-null pointers, d_feat 16-byte
 * (fp32) / 8-byte (h16) aligned, d_pts / d_deconv / d_out 4-byte aligned. */
int lavb_paint_deconv_batched(const float* d_pts, int frames, int n, int pt_stride, long long pts_frame_stride,
                              const void* d_feat, int feat_dtype, int ncam, int c_cls, int h, int w,
                              const float* d_deconv, const float* h_cams, float* d_out, int out_stride,
                              long long out_frame_stride, int out_col0, int copy_cols, void* stream);

/* ---------------------------------------------------------------- confusion counts of the segmentation model
 * stands behind: an evaluation of RGBSegmentationModel (lav/models/rgb.py:35-45) against the recorded semantic camera images
 *           (SegmentationDataset, lav/utils/datasets/seg_dataset.py:16-30, with filter_sem, lav/utils/__init__.py:3-8); the
 *           reference has none.  The ERFNet logits are never materialised.
 * One launch; one thread per feature pixel evaluates its 2 x 2 output pixels.  d_feat: NHWC (n, h/2, w/2, 16) fp32 or h16
 *   (feat_dtype) = the input of output_conv, contiguous; d_deconv: lavb_paint_deconv_batched's 520-float table; d_labels:
 *   uint8 (n, h, w) = the recorded CARLA tags; h_lut: HOST uint8[256] = the class of each tag (filter_sem as a table), read
 *   during the call.
 * Per output pixel (v, u): the logits of lavb_paint_deconv_batched before its softmax (bias[k], then fmaf over c = 0..15 in
 *   order, weight phase [v&1][u&1]); the predicted class is the first index of the largest logit (ties to the lower class);
 *   a pixel with a NaN logit counts as invalid and in no confusion entry.
 * d_out: int32 (n, c_cls * c_cls + 1) = per image confusion[gt][pred], then the invalid count; integer sums, so the counts do
 *   not depend on the schedule.  2 <= c_cls <= 8, h and w even, n <= 65535, every h_lut entry < c_cls; features 16-byte (fp32) /
 *   8-byte (h16) and labels 2-byte aligned.  Every element of the n rows is written; a rejected call writes nothing. */
int lavb_seg_confusion(const void* d_feat, int feat_dtype, const float* d_deconv, const uint8_t* d_labels, const uint8_t* h_lut,
                       int n, int c_cls, int h, int w, int* d_out, void* stream);

/* ---------------------------------------------------------------- confusion counts of the point painting
 * stands behind: the painting of the LiDAR points, online (lavb_paint_deconv_batched: InferModel.point_painting /
 *           forward_paint, model_inference.py:44-50,75-93) and offline (lav/data_paint.py:44-107, lidar_sem_%05d), scored
 *           against the recorded semantic cameras at the pixel each point hits; the reference has no such evaluation.
 * One launch, one thread per point, grid (ceil(n / 256), frames).  d_pts: fp32 (frames, n, 4) (x, y, z, intensity), NaN-padded;
 *   d_meta: NULL, or DEVICE int32 (frames, 2) = (rows of the frame, score its stored rows 0 / 1), rows clamped to 0..n (NULL:
 *   every row, stored rows scored); d_feat: NULL, or NHWC (frames * ncam, h/2, w/2, 16) fp32 / h16 (feat_dtype) = the input of
 *   output_conv, with d_deconv lavb_paint_deconv_batched's 520-float table; d_tags: uint8 (frames * ncam, h, w) = the recorded
 *   CARLA tags; h_lut: HOST uint8[256], the class of each tag (filter_sem as a table); d_stored: NULL, or fp32 (frames, n,
 *   c_cls - 1) = lidar_sem rows; h_cams as lavb_paint; the pillar grid window [min_x, max_x) x [min_y, max_y).  At least one of
 *   d_feat and d_stored.
 * Per row i < rows: a NaN x, y or z counts as nan and nowhere else.  Otherwise: roof = inside LAVAgent.preprocess's roof box
 *   (lavb_roof_filter's fp32 test); in window = not roof and inside the grid window as the voxeliser tests it; the hit camera and
 *   pixel (v, u) are lavb_paint's (the last camera whose truncated pixel lies inside h x w); a point no camera sees counts as
 *   not_visible (and not_visible_in_window) and is scored nowhere.  gt = h_lut[tag at (v, u) of the hit camera]; range bin of
 *   fp32 sqrt(x*x + y*y): [0, 10), [10, 20), [20, 40), [40, inf) m.  Online class: the logits of lavb_seg_confusion at (v, u),
 *   first index of the largest, a NaN logit -> invalid.  Stored class: the row s_k = p_k (1 - p_0) decoded in fp64 without
 *   contraction, q = sqrt(sum s_k), p_0 = 1 - q, p_k = s_k / q, first index of the largest of (p_0, p_1, ...); a row summing to 0
 *   is class 0; a NaN entering the decode -> stored_invalid.
 * d_out: int32 (frames, lavb_paint_confusion_ints(ncam, c_cls, online, stored)); per frame: 8 counters (points, nan, roof,
 *   in_window, not_visible, not_visible_in_window, invalid, stored_invalid), then per scored source (online first, then stored)
 *   confusion[cam][range][in window 0 / 1][gt][pred], then with both sources agreement[cam][online][stored] over the points both
 *   score.  Integer sums, so the counts do not depend on the schedule.
 * 2 <= c_cls <= 8, 1 <= ncam <= 4, h and w even, frames <= 65535, every h_lut entry < c_cls, min < max; points 16-byte,
 *   features 16-byte (fp32) / 8-byte (h16), the other buffers 4-byte aligned.  Every element of the frames rows is written; a
 *   rejected call writes nothing.  lavb_paint_confusion_ints returns -1 for arguments the kernel rejects. */
int lavb_paint_confusion_ints(int ncam, int c_cls, int online, int stored);
int lavb_paint_confusion(const float* d_pts, int frames, int n, const int* d_meta, const void* d_feat, int feat_dtype,
                         const float* d_deconv, const uint8_t* d_tags, const uint8_t* h_lut, const float* d_stored,
                         const float* h_cams, int ncam, int c_cls, int h, int w, float min_x, float max_x, float min_y,
                         float max_y, int* d_out, void* stream);

/* ---------------------------------------------------------------- sweep stacking
 * replaces: LAVAgent.get_stacked_lidar + move_lidar_points (team_code_v2/lav_agent_fast.py:363-383,547-565)
 * and the ego-roof filter LAVAgent.preprocess (lav_agent.py:448-457, roof_filter!=0 marks dropped rows x=NaN).
 * dst row = [xyz @ R + (dx,dy,0) | src cols 3..src_cols | one_hot(time_idx, n_time)];  h_R is 3x3 row-major (9 floats).
 * Arithmetic, bit for bit: x' = fp32(fmaf(z, R[6], fmaf(y, R[3], x * R[0])) + dx), y' likewise with R[1], R[4], R[7] and dy (real
 * adds: a -0 sum becomes +0), z' = fmaf(z, R[8], fmaf(y, R[5], x * R[2])) (no add: a -0 z' stays -0).  With roof_filter, x' of a
 * row inside lavb_roof_filter's box (tested on the input x, y, z) is the canonical NaN.  Copied columns keep their bits.  Every
 * element of the n dst rows is written, nothing else.
 * Checked before any launch (a rejected call writes nothing): n >= 0, src_cols >= 3, n_time >= 0, time_idx >= 0 and, when
 * n_time > 0, time_idx < n_time; then, unless n is 0, non-null pointers, d_src / d_dst 4-byte aligned and not overlapping. */
int lavb_stack_sweep(const float* d_src, int n, int src_cols, const float* h_R, float dx, float dy,
                     int time_idx, int n_time, int roof_filter, float* d_dst, void* stream);

/* Ego-roof filter as an order-preserving drop (np.delete semantics).
 * replaces: LAVAgent.preprocess (team_code_v2/lav_agent.py:448-457; applied to the raw sweep before painting at :236 and
 *           lav_agent_fast.py:247): rows with x in (-2.4,0), y in (-0.8,0.8), z in (-1.5,-1) are removed, the others keep their order.
 * `frames` independent sweeps of n rows x cols floats (frame f at d_src + f*src_frame_stride); the kept rows of frame f are written
 * to d_dst + f*dst_frame_stride, their number to d_counts[f] (may be NULL); with pad_nan the remaining rows [count, n) are filled
 * with NaN (the fixed-shape pipeline's padding — every kernel drops NaN rows).  The box test is the fp32 comparisons above on the
 * raw x, y, z, so a row with a NaN coordinate is kept; kept rows are copied bit for bit.  Written: the kept rows and, with
 * pad_nan, rows [count, n) of each frame (canonical NaN); without pad_nan those rows keep their values.
 * Checked before any launch (a rejected call writes nothing): frames, n >= 0, cols >= 3, src_frame_stride >= 0; then, unless
 * frames is 0, dst_frame_stride >= n * cols when frames > 1 (output frames must not overlap), non-null d_src / d_dst, 4-byte
 * aligned pointers, and the dst extent ((frames - 1) * dst_frame_stride + n * cols floats) not overlapping the src extent. */
int lavb_roof_filter(const float* d_src, int frames, int n, int cols, long long src_frame_stride, float* d_dst,
                     long long dst_frame_stride, int* d_counts, int pad_nan, void* stream);

/* table-driven variant: d_jobs is a DEVICE array of n_jobs 72-byte records
 *   { const float* src; float* dst; int n; int time_idx; float R[9]; float dx, dy; int pad; }
 * (one per (agent, sweep)); all jobs run in one launch and the table can be rewritten between replays of a captured
 * CUDA graph (new poses, new ring-buffer slots) without touching kernel arguments.  Each job is lavb_stack_sweep's row
 * arithmetic on its n rows (src_cols in, src_cols + n_time out); a time_idx outside [0, n_time) sets no one-hot column; a job
 * with n <= 0 writes nothing.  max_n only sizes the grid: a job longer than max_n is still done in full.  A job's src and dst
 * must be 4-byte aligned and not overlap; with src_cols 8, a 16-byte aligned src is read as two 16-byte vectors (the kernel
 * tests each job's src, since the table is device data the call never sees).
 * Checked before any launch (a rejected call writes nothing): 0 <= n_jobs <= 65535, max_n >= 0, src_cols >= 3, n_time >= 0,
 * src_cols + n_time <= 16; then, unless n_jobs or max_n is 0, d_jobs non-null and 8-byte aligned. */
int lavb_stack_jobs(const void* d_jobs, int n_jobs, int max_n, int src_cols, int n_time, int roof_filter, void* stream);

/* ---------------------------------------------------------------- temporal BEV training targets
 * replaces: TemporalLiDARPaintedDataset.load_bev_channels (lav/utils/datasets/temporal_lidar_painted_dataset.py:182-198) and
 *           its calls at :110-136: rotate_image (lidar_dataset.py:159-163, cv2.warpAffine INTER_LINEAR, zero border) by the
 *           ego yaw change, zero-pad by 32, crop shifted by (dx, dy), rotate_image by the sample's jitter, > 0.
 * One launch builds every (h, w) uint8 plane of a batch.  d_jobs is a DEVICE array of n_jobs 128-byte records
 *   { long long src; long long dst; double m1[6]; double m2[6]; int dx, dy; int pad[2]; }
 * src = plane index into d_src (planes of h*w bytes; < 0 writes a zero plane: a frame before the recording's start),
 * dst = plane index into d_out; m1 / m2 = the inverse affine matrices (row-major 2x3, computed on the host the way
 * cv::warpAffine inverts getRotationMatrix2D) of the first and second warp; dx shifts rows and dy columns.
 * The output is bit-identical to OpenCV's fixed-point 8-bit warp chain; every output byte is 0 or 1. */
int lavb_bev_targets(const void* d_jobs, int n_jobs, const uint8_t* d_src, uint8_t* d_out, int h, int w, void* stream);

/* ---------------------------------------------------------------- grayscale PNG maps of a recording
 * replaces: BasicDataset.load_bev's cv2.imdecode(..., cv2.IMREAD_GRAYSCALE) of each map_%d_%05d plane
 *           (lav/utils/datasets/basic_dataset.py:94,99).
 * One launch decodes n_jobs 8-bit grayscale, non-interlaced PNG images into (n_planes, h, w) uint8 planes at d_out.  The host
 * walks the chunks; d_src (src_bytes bytes) holds each image's IDAT payloads concatenated, i.e. its zlib stream.  d_jobs is a
 * DEVICE array of n_jobs 32-byte records
 *   { long long off, len; int dst, h, w, pad; }
 * stream = bytes [off, off + len) of d_src, dst = output plane, h / w = the IHDR size (must equal the launch's h / w).
 * d_status: DEVICE int32[n_jobs], 0 = decoded, bit-identical to libpng; otherwise the job's stream is malformed (zlib header,
 * deflate block, code lengths, symbol, distance, inflated size != h * (w + 1), Adler-32, filter byte > 4: the codes of
 * lavb_png::PngStatus in png_inflate.cuh).  Every read stays inside the job's stream and every write inside its plane, so a
 * malformed job leaves all other bytes, and the other jobs, untouched.  Jobs must name distinct planes. */
int lavb_png_decode_gray8(const uint8_t* d_src, long long src_bytes, const void* d_jobs, int n_jobs, uint8_t* d_out,
                          int n_planes, int h, int w, int* d_status, void* stream);

/* ---------------------------------------------------------------- LiDAR rows of a training batch
 * replaces: one GpuLidarStacker call per sample (lav_b200/data_pipeline.py; TemporalLiDARPaintedDataset.__getitem__,
 *           temporal_lidar_painted_dataset.py:13-91): roof filter, rotate_lidar(-angle), the camera-FOV re-mask of the painted
 *           columns, move_lidar_points + time one-hot, shuffle, truncation to max_lidar_points and zero padding.
 * d_raw: n_raw rows of 4 + c floats [x y z r | painted c], every sweep of the batch; sweep s owns rows [row0(s), row0(s+1)).
 * d_rows: DEVICE int32[n_rows], one entry per output row: the raw row it copies, or -1 for a zero row.  The host does the roof
 *   filter (the fp32 predicate of lavb_roof_filter), the per-sample permutation, the truncation and the padding on these
 *   indices, so output row b*P + i of sample b (P rows per sample) is kept row perm_b[i] of the sample's sweeps taken newest
 *   first, each in its recorded order — the row order of GpuLidarStacker for the same permutation.
 * d_sweeps: DEVICE array of n_sweeps 88-byte records, sorted by row0,
 *   { float R_aug[9]; float R_mv[9]; float dx, dy; int time_idx; int row0; }
 *   (3x3 row-major matrices).  Each output row = [xyz' @ R_mv + (dx, dy, 0) | r | painted * vis | one_hot(time_idx, n_time)] with
 *   xyz' = xyz @ R_aug + (0, 0, 0) (lavb_stack_sweep's arithmetic: x' and y' take a real fp32 add, so a -0 there becomes +0;
 *   z' has no add, so a -0 z' stays -0) and vis = 1 if lavb_paint's projection through the ncam
 *   cameras of h_cams (host, as lavb_paint) lands inside an h x w image, else 0, multiplied in as one fp32 multiply (NaN * 0 stays
 *   NaN).  Bit-identical to lavb_roof_filter + lavb_stack_sweep + lavb_paint (mode 0, a ones map) + multiply + lavb_stack_sweep.
 *   A row index outside [0, n_raw) or below the first row0 gives a zero row.
 *   The sweep of row src is the last one with row0 <= src.
 * d_out: n_rows x (4 + c + n_time) fp32, every element written.  4 + c + n_time <= 16, ncam 1..4.
 * Checked before any launch (a rejected call writes nothing): the sizes >= 0, n_raw < 2^31, fewer than 2^31 blocks of 256 rows,
 *   non-null h_cams, row table and output (n_rows > 0), raw rows and sweeps (n_raw > 0), every device pointer 4-byte aligned. */
int lavb_lidar_batch(const float* d_raw, long long n_raw, int c, const int* d_rows, long long n_rows, const void* d_sweeps,
                     int n_sweeps, const float* h_cams, int ncam, int h, int w, int n_time, float* d_out, void* stream);

/* ---------------------------------------------------------------- detection targets of a training batch
 * replaces: LiDARDataset.detections_to_heatmap (lav/utils/datasets/lidar_dataset.py:92-127), once per sample.
 * d_actors: DEVICE array of 24-byte records { float x, y, ori, bx, by, typ; } (ego-frame metres, radians, box extents, class:
 *   0 pedestrian, 1 vehicle, anything else ignored); sample i owns records [d_offsets[i], d_offsets[i+1]) (DEVICE int32[b+1]).
 * Output planes (b, 2, h, w) fp32 each, every element written: d_heat = per class the maximum over its actors of
 *   exp(-((x - cx) / r)^2) * exp(-((y - cy) / r)^2), cx = -x * ppm + cx0, cy = (-y * ppm + cy0) + cy1, the division done as a
 *   multiply by inv_radius; ties go to the first actor, a NaN wins.  Where class 0's value is > 0, and then where class 1's
 *   value is > class 0's (or > 0 without pedestrians), d_size = (bx, by) * ppm and d_ori = (cos, sin)(ori) of that winning
 *   actor; elsewhere 0.  A class without actors leaves its heat plane 0.  Every operation is the fp32 operation torch performs
 *   in lav_b200.data_pipeline.detections_to_heatmap, in its order.  b <= 65535. */
int lavb_det_heatmaps(const void* d_actors, const int* d_offsets, int b, int h, int w, float ppm, float cx0, float cy0, float cy1,
                      float inv_radius, float* d_heat, float* d_size, float* d_ori, void* stream);

/* ---------------------------------------------------------------- scores of an evaluation batch
 * replaces: the comparisons LAV.train_lidar draws for wandb (lav/lav_final_v2.py:226-258): predicted detections against gt_det,
 *           ego_plan_locs against the expert's ego_locs, pred_bev against the GT bev — as counts over every sample of a batch.
 * One block per sample (batches of more than 256 samples take one launch per 256).
 * BEV: d_seg (b, h, w, 3) NHWC sigmoid probabilities, fp32 or h16 (seg_dtype); d_gt (b, gt_planes, h, w) uint8, planes 0..2 the
 *   targets.  d_iou (b, 3, 2) int64 = per channel (|pred > 0.5 and gt != 0|, |pred > 0.5 or gt != 0|).  h * w % 4 == 0.
 * Detections: d_packed (b, 7, 2 * n_det) fp32 = lavb_det_peaks' output (class c in columns [c * n_det, (c + 1) * n_det)), the
 *   peak pixel (flat % w, flat / w).  A peak survives InferModel.decode_packed's filters: score > float32(min_score) compared
 *   in fp32 (as the reference's `s > min_score` on an fp32 tensor; a NaN score never survives), not (class 1 and both
 *   box sides < float32(0.1 * ppm)), and 2 < d < 30 * ppm pixels from (cx0, cy0 + cy1).  d_actors: lavb_det_heatmaps' table
 *   (24-byte records, n_actors rows), sample i owning rows [h_offsets[i], h_offsets[i+1]) (HOST int32[b+1], monotone, at most
 *   1024 rows per sample); an actor of class typ (0 / 1, others ignored) counts when its centre, placed as lavb_det_heatmaps
 *   places it, lies in the same window.  Per class and threshold t in {0.5, 1, 2, 4} m, the survivors in descending score (ties:
 *   lower flat index, then lower column) each take the nearest untaken actor of their class with squared pixel distance
 *   <= (t * ppm)^2 (fp64, ties: lower row).  d_ngt (b, 2) int32 = actors counted per class; d_score (b, 2 * n_det) fp32 = the
 *   packed scores; d_flags (b, 2 * n_det) int32 = bit 4 set for a survivor, bit k for a match at threshold k.
 * Plan: d_plan (b, n_plan, 2) fp32, d_ego_locs (b, n_plan + 1, 2) fp32 with entry 0 the origin; d_plan_err (b, 2) fp64 = (mean
 *   over the steps of |plan[t] - ego_locs[t+1]|, the error at the last step).  n_plan <= 32.
 * Every output element of the b samples is written; a rejected call writes nothing. */
int lavb_eval_batch(const void* d_seg, int seg_dtype, const uint8_t* d_gt, int gt_planes, int b, int h, int w, const float* d_packed,
                    int n_det, const void* d_actors, int n_actors, const int* h_offsets, float ppm, float cx0, float cy0, float cy1,
                    double min_score, const float* d_plan, const float* d_ego_locs, int n_plan, long long* d_iou, int* d_ngt,
                    float* d_score, int* d_flags, double* d_plan_err, void* stream);

/* ---------------------------------------------------------------- box scores of the decoded detections
 * stands behind: the boxes LAVAgent.visualize draws (lav_agent_fast.py:485-490) and UniPlanner.infer crops at; the reference
 *           scores detections by centre only.  Rotated-box IoU matches and the position, size and heading errors of the
 *           detections lavb_eval_batch matches at 2 m.
 * One block per sample (batches of more than 256 samples take one launch per 256).  d_packed (b, 7, 2 * n_det), w, d_actors /
 *   n_actors / h_offsets (at most 1024 rows per sample), ppm, cx0, cy0, cy1 and min_score exactly as lavb_eval_batch takes them;
 *   the survivors (its decode_packed filters), their rank order and the ground truth (class 0 / 1 in the window) are its own, and
 *   d_ngt (b, 2) int32 equals its d_ngt.
 * Boxes in map pixels, fp64.  A survivor in column j: centre (x, y) = its peak pixel, half extents (ww, hh) = packed rows 2, 3,
 *   heading (c, s) = packed rows 4, 5.  An actor: centre = (cx, cy) placed as lavb_det_heatmaps places it, half extents (bx * ppm,
 *   by * ppm) (exact in fp64), (c, s) = (cos, sin)(ori) in fp64.  Corners: u = (-(s * ww), c * ww), v = (-(c * hh), -(s * hh)),
 *   corner k = (x + (a_k * u.x + b_k * v.x), y + (a_k * u.y + b_k * v.y)) for (a, b) = (-1, -1), (-1, 1), (1, 1), (1, -1) (the
 *   reference's drawing without its int cast).  Area = |s| / 2 with s the shoelace sum over i ascending of (x_i * y_{i+1} -
 *   x_{i+1} * y_i).  A box is degenerate when an extent is not finite and > 0, c, s or the centre is not finite, or its area is 0.
 * IoU of survivor box P and actor box Q: 0 when either is degenerate or when the corner bounding boxes are apart (P's largest x <
 *   Q's smallest x, or the same the other way or in y); else P is clipped by each edge e = 0..3 of Q in turn (Sutherland-Hodgman):
 *   with (x0, y0) = corner e, (ex, ey) = corner e+1 - corner e, side(p) = ex * (p.y - y0) - ey * (p.x - x0), a vertex is inside
 *   when side <= 0; the vertices q in order, each with its predecessor p (the last vertex before the first): when exactly one of
 *   p, q is inside, p + t * (q - p) with t = side(p) / (side(p) - side(q)) is emitted, then q when inside (at most 16 vertices
 *   kept; a convex polygon has at most 8).  I = the area of the result (0 below 3 vertices), IoU = I / ((A + B) - I), 0 when
 *   that union is not > 0.  Every fp64 operation is correctly rounded and none is contracted.
 * IoU match, per class and threshold k (0.3, 0.5, 0.7): the survivors in rank order each take the actor of their class not yet
 *   taken at k with the highest IoU >= the threshold; equal IoUs go to the lower actor row.  2 m match: lavb_eval_batch's match at
 *   2 m (the same search, the same result).
 * Outputs per column, (b, 2 * n_det) row-major: d_score fp32 = the packed score; d_flags int32 = bit 4 survivor, bit k (0..2) IoU
 *   match at threshold k, bit 3 the 2 m match; d_actor (.., 4) int32 = the actor row within the sample of the matches at the three
 *   thresholds and at 2 m, -1 for none; d_err (.., 5) fp64, for a column with a 2 m match (NaN otherwise): the IoU of its box
 *   with the actor's; the translation error sqrt(d2) / ppm in metres; the scale error 1 - i / ((ww * hh + wa * ha) - i), i =
 *   min(ww, wa) * min(hh, ha), with (wa, ha) the actor's half extents (1 when an extent is not finite and > 0); the heading error
 *   min(r, 2 pi - r) with r = fmod(|atan2(s, c) - ori|, 2 pi) (NaN when the heading or ori is not finite); the actor's distance
 *   from the window centre in metres.  Every output element of the b samples is written; a rejected call writes nothing.
 *   1 <= n_det <= 64; err 8-byte aligned, the other arrays 4-byte aligned. */
int lavb_det_box_eval(const float* d_packed, int b, int w, int n_det, const void* d_actors, int n_actors, const int* h_offsets,
                      float ppm, float cx0, float cy0, float cy1, double min_score, float* d_score, int* d_flags, int* d_actor,
                      double* d_err, int* d_ngt, void* stream);

/* ---------------------------------------------------------------- scores of the planners' motion forecasts
 * replaces: the forecast terms of the planners' training losses (other_cast_loss, ego_cast_loss, cmd_loss in lav_b200.train) as
 *           displacement errors and branch choices per forecast row, for an evaluation over a recording.
 * One warp per row, one lane per command branch (batches of any k in one launch).
 * d_cast (k, c, t, 2) fp32 = the c command branches of each row's forecast; d_score (k, c) fp32 = the command scores;
 * d_target (k, t, 2) fp32 = the recorded future in the same frame; d_cmd (k,) int32 = the recorded command, or -1 for none.
 * Per branch j: ADE_j = (sum over steps i in ascending order of |cast[j, i] - target[i]|) / t, FDE_j = the error at step t - 1,
 * every error in fp64 with no contraction.  d_err (k, 6) fp64 = (min_j ADE_j, min_j FDE_j, ADE and FDE of the top branch,
 * ADE and FDE of branch cmd, NaN where cmd is outside [0, c)); d_branch (k, 2) int32 = (argmin_j ADE_j, top branch).  The
 * minima are taken independently, ties go to the lower branch and a NaN error never wins; the top branch has the highest
 * score, ties to the lower branch, a NaN score counting as lowest.  1 <= c <= 32, 1 <= t <= 32, k >= 0 (k = 0 does nothing).
 * cast / target / err 8-byte aligned.  Every output element of the k rows is written; a rejected call writes nothing. */
int lavb_forecast_eval(const float* d_cast, const float* d_score, const float* d_target, const int* d_cmd, int k, int c, int t,
                       double* d_err, int* d_branch, void* stream);

/* ---------------------------------------------------------------- match of the forecast detections to the recorded tracks
 * stands behind: the vehicles UniPlanner.infer forecasts (team_code_v2/models/uniplanner.py:186-247, the detections of
 *           InferModel.det_inference that lie more than 4 px from the crop centre) and that lav_agent_fast.py:plan_collide brakes
 *           on; the reference has no evaluation of them.  Pairs each such row with the recorded actor it forecasts, so
 *           lavb_forecast_eval can score the row's forecast against that actor's recorded future.
 * One block per sample.  Rows: sample i owns rows [h_row_offsets[i], h_row_offsets[i+1]) (HOST int32[b+1], h_row_offsets[0] = 0,
 *   monotone, at most n_det rows per sample); h_cols (HOST int32, one per row) = the row's column of d_packed (b, 7, 2 * n_det)
 *   fp32 (lavb_det_peaks' layout, flat index read as lavb_eval_batch reads it on a map of width w), ascending within a sample
 *   and in the class-1 half [n_det, 2 * n_det).  d_actors / h_actor_offsets: lavb_eval_batch's actor table (at most 1024 rows
 *   per sample); actor row a of sample i has a recorded track when a < h_num_objs[i] (HOST int32[b], 0..max_objs): its label
 *   slot a of d_locs (b, max_objs, t + 1, 2) fp32, with d_ego_locs (b, t + 1, 2) fp32.
 * Match, per sample: the actors of class 1 whose centre lies in lavb_eval_batch's window (tracked or not) are the candidates;
 *   the rows in descending score (ties: lower flat index, then lower column; a NaN score last) each take the nearest candidate
 *   not yet taken with squared pixel distance <= (match_m * ppm)^2 (fp64, no contraction, ties: lower actor row) - the search
 *   of lavb_eval_batch.  Per row: d_actor int32 = the actor row or -1; d_flag int32 = bit 0 matched, bit 1 matched to a tracked
 *   actor; d_dist fp64 = the match distance in metres (sqrt(d2) / ppm) or NaN; d_target (t, 2) fp32 = locs[i, a, 1 + s] -
 *   ego_locs[i, 0] for a row matched to a tracked actor a (the frame of UniPlanner.infer's other_cast_locs), NaN otherwise.
 *   d_ngt (b, 2) int32 = the candidates with and without a track.  1 <= n_det <= 64, 1 <= t <= 32; dist and target 8-byte
 *   aligned.  Every output element of the b samples is written; a rejected call writes nothing. */
int lavb_det_forecast_match(const float* d_packed, int b, int w, int n_det, const void* d_actors, int n_actors,
                            const int* h_actor_offsets, const int* h_row_offsets, const int* h_cols, const int* h_num_objs,
                            const float* d_locs, const float* d_ego_locs, int max_objs, int t, float ppm, float cx0, float cy0,
                            float cy1, double match_m, int* d_actor, int* d_flag, double* d_dist, float* d_target, int* d_ngt,
                            void* stream);

/* ---------------------------------------------------------------- collisions and road departures of planned ego trajectories
 * stands behind: the check lav_agent_fast.py:plan_collide makes before the agent drives a plan; the reference has no open-loop
 *           evaluation of the plan against the recorded traffic or the road.
 * One block per sample (batches of more than 512 samples take one launch per 512).  d_traj (b, n, t, 2) fp32 = n trajectories of t
 *   steps per sample in the label frame (entry 0 of ego_locs, the origin, precedes step 1).  Ego box at step s (1..t): centre
 *   p_s; heading d / sqrt(d . d) with d = p_s - p_{s-1} (fp64, correctly rounded), the previous heading kept when
 *   sqrt(d . d) < 0.1 m, (0, -1) before step 1; half extents d_ego_ext (b, 2) fp64 = the ego's (half length, half width).
 *   A step whose centre or heading is not finite is invalid: counted, never a collision or off-road.
 * Actors: d_actors is a DEVICE array of 56-byte records
 *   { double x, y, cos, sin, e1, e2; int typ, present; }
 *   sample i owning actor rows [h_offsets[i], h_offsets[i+1]) (HOST int32[b+1], monotone, any number of rows per sample), row a's
 *   record of step s at index a * t + s - 1: label-frame centre, cos / sin of the yaw relative to the ego (heading (sin, -cos),
 *   perpendicular (cos, sin)), half extents, class (1 vehicle, 0 pedestrian, others ignored), present != 0 when recorded.
 * Collision: a separating-axis test over both boxes' headings and perpendiculars n, separated when |(c_B - c_A) . n| >=
 *   r_A(n) + r_B(n), r(n) = e1 |u1 . n| + e2 |u2 . n|, in fp64 with no contraction; touching boxes do not collide.
 * Road: the four corners of a valid box go to map pixels (floor(x * ppm + cx0), floor((y * ppm + cy0) + cy1)) in fp64 (column,
 *   row; lavb_det_heatmaps' grid for label-frame, i.e. negated, coordinates); a corner outside the h x w plane is off the map,
 *   an in-map corner on a 0 byte of d_map (plane of sample i at d_map + i * map_stride bytes, row-major) is off the road.
 * d_out (b, n, 8) int32 per trajectory: first step colliding with a vehicle and its actor row (the lowest row at that step),
 *   first step colliding with a pedestrian and its row, first off-road step, steps with a corner off the map, invalid steps,
 *   first step colliding with either class; -1 for none.  1 <= n <= 8, 1 <= t <= 32; traj, actors and ego_ext 8-byte aligned.
 *   Every output element of the b samples is written; a rejected call writes nothing. */
int lavb_plan_safety(const float* d_traj, int b, int n, int t, const void* d_actors, int n_actors, const int* h_offsets,
                     const double* d_ego_ext, const uint8_t* d_map, long long map_stride, int h, int w, float ppm, float cx0,
                     float cy0, float cy1, int* d_out, void* stream);

/* ---------------------------------------------------------------- the agent's controls: collision brake, PIDs, brake rules
 * stands behind: lav_agent_fast.py:228-231 and 325-352 (the stop counter, the 4/5 plan swap, pid_control called twice, the
 *           brake model, plan_collide, the speed cap and the creep), pid_control :404-426, plan_collide :385-401 and
 *           team_code_v2/pid.py, for b agents in one launch per 512 agents (one warp per agent).
 * Per agent i, in the reference's order:
 *   stop counter += 1 when (double)speed < 0.1, else 0.  plan = d_cast when h_cmd[i] is 4 or 5, else d_plan (both (b, t, 2)
 *   fp32).  If the plan has no NaN, pid_control: w = plan * (float)ppm with y negated (fp32); desired = fp32 mean of the t-1
 *   step lengths |w[s+1] - w[s]| (fp32 norms, numpy's pairwise summation order); angle = degrees(pi/2 - atan2f(w_a.y, w_a.x))
 *   / 90 in fp64 with atan2f correctly rounded, a = aim_point[cmd]; delta = clip(desired * speed_ratio[cmd] - speed, 0,
 *   clip_delta) in fp64.  Each PID window (n values, starting as n zeros) receives its error twice; its output is
 *   kp * e + ki * mean(window) + kd * (w[-1] - w[-2]) in fp64 (mean in numpy's pairwise order; 0 and 0 when n == 1).
 *   steer = clip(turn, -1, 1); brake = desired < brake_speed * ppm; throttle = brake ? 0 : clip(speed pid, 0, max_throttle).
 *   A plan with a NaN gives (0, 0, 0) and steps no PID.
 *   plan_collide: a forecast row whose first point has y > 0.5 * ppm is skipped, a branch scoring < cmd_thresh is skipped;
 *   otherwise the branch collides when min_s |row[s] - plan[s]| < (its fp32 mean step length < brake_speed ? 1.0 : 2.5).  All
 *   norms fp32, every comparison in fp64; a NaN anywhere in the branch or the plan means no collision.
 *   Brake rules: (double)pred_bra > 0.1 or a collision -> throttle 0, brake 1; speed * 3.6 > max_speed -> throttle 0; stop
 *   counter >= 600 -> creep counter = 20; creep counter > 0 -> throttle = max(0.4, throttle), brake 0, creep counter -= 1.
 * Inputs: forecast rows d_other_locs (k, c, t, 2) fp32 and their scores d_other_cmds (k, c) fp32, agent i owning rows
 *   [h_offsets[i], h_offsets[i+1]) (HOST int32[b+1], monotone, within 0..k, any number per agent); d_pred_bra, d_speed (b,)
 *   fp32 (m/s); h_cmd (b,) HOST int32 in 0..c-1; *h_config read during the call.  2 <= t <= 32, 1 <= c <= 8, 1 <= turn_n,
 *   speed_n <= 64, 0 <= aim_point[j] < t.
 * State: d_state holds b records of lavb_agent_control_state_bytes(turn_n, speed_n) bytes (8-byte aligned):
 *   { int stop_counter, creep_counter, turn_head, speed_head; double turn_window[turn_n], speed_window[speed_n]; }
 *   a window's oldest value at index head, the others following cyclically.  All-zero bytes are the state of a new route.
 * Outputs: d_control (b, 3) fp32 = steer, throttle, brake; d_flags (b,) int32, LAVB_CTL_* bits.  Every output of the b agents
 *   is written; a rejected call writes nothing. */
#define LAVB_CTL_PLAN_INVALID 1  /* the plan has a NaN: no PID step, controls (0, 0, 0) before the brake rules */
#define LAVB_CTL_PID_BRAKE 2     /* pid_control's brake: the desired speed is below brake_speed * ppm */
#define LAVB_CTL_BRAKE_MODEL 4   /* pred_bra > 0.1 */
#define LAVB_CTL_COLLIDE 8       /* plan_collide, evaluated for every agent */
#define LAVB_CTL_SPEED_CAP 16    /* speed * 3.6 > max_speed */
#define LAVB_CTL_CREEP 32        /* the creep after 600 stopped ticks forced the throttle */
#define LAVB_CTL_MAX_CMDS 8

typedef struct lavb_control_config {
  int aim_point[LAVB_CTL_MAX_CMDS];
  double speed_ratio[LAVB_CTL_MAX_CMDS];
  double turn_kp, turn_ki, turn_kd;
  double speed_kp, speed_ki, speed_kd;
  int turn_n, speed_n;
  double brake_speed, clip_delta, max_throttle, max_speed, cmd_thresh, pixels_per_meter;
} lavb_control_config;

size_t lavb_agent_control_state_bytes(int turn_n, int speed_n);
int lavb_agent_control(const float* d_plan, const float* d_cast, int b, int t, int c, const float* d_other_locs,
                       const float* d_other_cmds, int k, const int* h_offsets, const float* d_pred_bra, const float* d_speed,
                       const int* h_cmd, const lavb_control_config* h_config, void* d_state, float* d_control, int* d_flags,
                       void* stream);
/* The same with the commands on the DEVICE (d_cmd (b,) int32, e.g. lavb_agent_nav_front's output), in the same launch shape.  An
 * agent whose command lies outside 0..c-1 gets NaN controls and flags LAVB_CTL_BAD_CMD, and its state is left as it was. */
#define LAVB_CTL_BAD_CMD 64
int lavb_agent_control_dcmd(const float* d_plan, const float* d_cast, int b, int t, int c, const float* d_other_locs,
                            const float* d_other_cmds, int k, const int* h_offsets, const float* d_pred_bra, const float* d_speed,
                            const int* d_cmd, const lavb_control_config* h_config, void* d_state, float* d_control, int* d_flags,
                            void* stream);

/* ---------------------------------------------------------------- agent localisation and route following
 * replaces: the head of LAVAgent.run_step (team_code_v2/lav_agent_fast.py:215-226, 280-308, 314) and its EKF step (:338), with
 *           EKF (team_code_v2/ekf.py), Waypointer (waypointer.py, pop_lane_change=True, pop_turning=False, default thresholds) and
 *           RoutePlanner (planner.py, default thresholds), for b agents, one thread per agent.
 * Routes: d_nodes (n_nodes, 2) fp64 holds every route's nodes as latlon_to_xy with the route's own scale cos(cos_0), cos_0 the mean
 *   of the route latitudes in radians; d_node_cmd (n_nodes,) int32 their RoadOption values (-1..6).  d_route (b, 2) int32 =
 *   (start, count) of agent i's route; an entry with start < 0, count < 1 or start + count > n_nodes is no route: the agent gets
 *   flags LAVB_NAV_NO_ROUTE, cmds 3, NaN nxps and poses, and its state is left as it was.  The route table is device data, so
 *   this check runs per agent in the kernel, not before the launch, and writes that agent's outputs; the node command values are
 *   not checked here (lav_b200.navigation.set_routes checks them on the host).
 * State: d_state holds b lavb_nav_state records (lavb_agent_nav_state_bytes() each, 8-byte aligned).  A new route is a record of
 *   zeros with route_scale = cos(cos_0), ekf_scale = cos(1) (the agent's EKF is built with cos0 = 1) and lane_changed = -1.
 * Front, per tick, before the planner (lavb_agent_nav_front): gnss (b, 2) fp64 = lat, lon; compass (b,) fp64 = imu[-1], raw.
 *   compass' = 0 when NaN; on the route's first frame EKF.init(lat, lon, compass' - pi/2); poses (b, 3) fp64 = the EKF state
 *   (x, y, theta).  The first frame stops there (flags LAVB_NAV_FIRST_FRAME, cmds 3, nxps 0), as run_step returns early.  On the
 *   second frame the Waypointer (checkpoint = this frame's position, LANEFOLLOW) and the RoutePlanner are built; then every frame
 *   runs Waypointer.tick and RoutePlanner.run_step in O(1), cmds = RoadOption value - 1 (VOID -> 3), the lane-change counter
 *   and rule (a 4 / 5 held for more than 300 ticks becomes 3), and nxps (b, 2) fp32 = -(R(-compass + pi/2) @ (wx, wy)) with the
 *   RAW compass, so a NaN compass gives NaN nxps.
 * Update, per tick, after the controls (lavb_agent_nav_update): EKF.step(speed, steer, lat, lon, compass' - pi/2) of every agent
 *   past its first frame; speed (b,) fp64 m/s, steer = d_control[3 i] (b, 3) fp32, lavb_agent_control's output.
 * Arithmetic: fp64, correctly rounded, in numpy's order; cos, sin, tan and atan are CUDA's (within 2 ulp).  Every output of the
 * b agents is written; a rejected call writes nothing. */
#define LAVB_NAV_FIRST_FRAME 1   /* the route's first frame: pose only, no command, target or EKF step */
#define LAVB_NAV_NO_ROUTE 2      /* d_route holds no route for the agent: nothing computed */
#define LAVB_NAV_LANE_HELD 4     /* a lane change held past 300 ticks was replaced by 3 */

typedef struct lavb_nav_state {
  double ekf_x[3];           /* EKF.x: x, y, theta */
  double ekf_p[3];           /* the diagonal of EKF.P (F = H = I, diagonal Q and R keep it diagonal) */
  double wp_x, wp_y;         /* Waypointer.checkpoint */
  double rp_x, rp_y;         /* RoutePlanner.checkpoint */
  double route_scale;        /* cos(cos_0) of the route's Waypointer and RoutePlanner */
  double ekf_scale;          /* cos(cos0) of the EKF, cos(1) */
  int frames;                /* frames since the route was set (saturates at 2^30) */
  int wp_idx, wp_cmd;        /* Waypointer.current_idx, the checkpoint's RoadOption value */
  int rp_idx;                /* RoutePlanner.current_idx */
  int lane_counter;          /* lane_change_counter */
  int lane_changed;          /* lane_changed, -1 = None */
  int pad[2];
} lavb_nav_state;

size_t lavb_agent_nav_state_bytes(void);
int lavb_agent_nav_front(int b, const double* d_nodes, const int* d_node_cmd, int n_nodes, const int* d_route, const double* d_gnss,
                         const double* d_compass, void* d_state, int* d_cmds, float* d_nxps, double* d_poses, int* d_flags,
                         void* stream);
int lavb_agent_nav_update(int b, const float* d_control, const double* d_speed, const double* d_gnss, const double* d_compass,
                          void* d_state, void* stream);

/* The pose fields (R, dx, dy) of lavb_stack_jobs' table, b agents x t sweeps (record (i, k) at d_jobs + (i * t + k) * 72), as
 * StaticFramePipeline._fill_jobs computes them on the host.  d_ring_pose (b, keep, 3) fp64 holds each agent's pose (x, y, ori)
 * per ring slot; when d_poses (b, 3) fp64 is given it is first written to slot tick % keep.  Job k reads slot
 * (tick - k * gap) mod keep: R = [[cos d, sin d, 0], [-sin d, cos d, 0], [0, 0, 1]] with d = ori_k - ori_0, (dx, dy) =
 * (dl.x cos ori_0 + dl.y sin ori_0, -dl.x sin ori_0 + dl.y cos ori_0) with dl = loc_k - loc_0, in fp64 rounded to fp32.  The
 * other fields are not touched. */
#define LAVB_STACK_JOB_BYTES 72
int lavb_stack_job_poses(void* d_jobs, int b, int t, int gap, int keep, long long tick, double* d_ring_pose, const double* d_poses,
                         void* stream);

/* ---------------------------------------------------------------- the agent's debug view
 * stands behind: LAVAgent.visualize (lav_agent_fast.py:459-518, lidar_to_bev :567-581) without its text, the frame run_step keeps
 * every tick, for b agents in one memset and four launches (the points launch once per 256 agents, the boxes launch once per
 * 96 drawn boxes).  Bit for bit with numpy and OpenCV's 8-bit arithmetic; oracle/view_ref.py states it.  Per agent i:
 *   1. the LiDAR view: np.histogramdd of the (x, y) of d_points' rows over linspace(-10, 71, 321) x linspace(-40, 41, 321) (fp64
 *      edges, a value on the last edge in the last bin, NaN / inf / outside rows dropped), clamped at 10, / 10 * 255 in fp64,
 *      truncated; rows flipped; grey to RGB.
 *   2. the drawing on it, later draws overwriting earlier ones: each plan point (d_cast when d_cmd[i] is 4 or 5, else d_plan) a
 *      radius-1 dot (255, 0, 0); each step of each forecast branch scoring >= cmd_thresh a radius-1 dot in jet[row], row the
 *      matplotlib Colormap row of the fp32 score (x 256, 256 -> 255, under 256, over 257, NaN 258); each box an outline of
 *      thickness 2 (255, 0, 0) as cv2.drawContours draws it; the target a radius-2 dot (0, 255, 0) at clip(ego + tgt * ppm,
 *      0, 255).  A point's pixel is (160, 280) + (float)(loc * (float)ppm) in fp64, truncated; a point or target that is NaN or
 *      outside int32 is not drawn, nor a box whose corners are.
 *   3. the predicted BEV: (255 * mean_c sigmoid(logit)) in fp32 (sigmoid = 1 / (1 + expf(-x)), channels summed in order,
 *      divided by c), truncated; NaN -> 0.
 *   4. cv2.resize INTER_LINEAR of the three cameras (288 x 768 -> 320 x 853) and of the tele view (192 x 480 -> 320 x 800),
 *      the canvas [cameras | tele | LiDAR view | BEV] (320 x 2293) and its resize to 160 x 1146.
 * Inputs: d_rgbs (b, 3, 288, 256, 3) uint8, the cameras in order; d_tels (b, 192, 480, 3) uint8; d_points (b, p, point_stride)
 *   fp32, x and y in columns 0 and 1 (NaN rows are padding); d_bev the logits (b, c, 320, 320) fp32 (LAVB_F32) or the 16-bit
 *   type, element strides h_bev_strides[4] = (b, c, y, x); d_plan / d_cast (b, t, 2) fp32; d_cmd (b,) int32; forecast rows
 *   d_other_locs (k, m, t, 2) / d_other_cmds (k, m) fp32, agent i owning rows [h_offsets[i], h_offsets[i+1]); boxes h_boxes
 *   (n_boxes, 6) HOST fp64 (x, y, w, h, cos, sin) in BEV pixels, agent i owning rows [h_box_offsets[i], h_box_offsets[i+1])
 *   (HOST int32[b+1], monotone); d_target (b, 2) fp32 = [-wx, -wy]; *h_config read during the call.  1 <= t <= 64, 1 <= m <= 8,
 *   1 <= c <= 64, b <= 65535; pixels_per_meter positive and exact in fp32.
 * d_scratch: lavb_agent_view_scratch_bytes(b) bytes, 8-byte aligned, overwritten.  d_out (b, 160, 1146, 3) uint8, every byte of
 * the b frames written.  A rejected call writes nothing.  The row offsets, the boxes' corners (computed here in fp64) and the
 * config travel as kernel arguments: a captured graph replays those of the capture. */
#define LAVB_VIEW_JET_ROWS 259
typedef struct lavb_view_config {
  double pixels_per_meter, cmd_thresh;
  unsigned char jet[LAVB_VIEW_JET_ROWS * 3];   /* (int(r * 255), int(g * 255), int(b * 255)) of matplotlib's jet: 256 colours,
                                                  then its under, over and bad rows */
} lavb_view_config;

size_t lavb_agent_view_scratch_bytes(int b);
int lavb_agent_view(const unsigned char* d_rgbs, const unsigned char* d_tels, const float* d_points, int b, long long p,
                    int point_stride, const void* d_bev, int bev_dtype, int bev_c, const long long* h_bev_strides, const float* d_plan,
                    const float* d_cast, const int* d_cmd, int t, const float* d_other_locs, const float* d_other_cmds, int k, int m,
                    const int* h_offsets, const double* h_boxes, int n_boxes, const int* h_box_offsets, const float* d_target,
                    const lavb_view_config* h_config, void* d_scratch, size_t scratch_bytes, unsigned char* d_out, void* stream);

/* ---------------------------------------------------------------- PointPillars voxeliser + pillar encoder
 * replaces: PointPillarNet.forward (lav/models/point_pillar.py:92-116) incl. grid_locations :70-79,
 *           pillar_generation/decorate :55-68,81-85, DynamicPointNet.forward :28-35 (torch_scatter
 *           scatter_mean/scatter_max), scatter_points :87-90.
 * Clouds: cloud b = rows [h_cloud_start[b], +h_cloud_count[b]) of d_pts (row stride pt_stride floats,
 * first `d` columns used).  MLP: Linear(d+5,h1) -> affine(s1,t1) -> ReLU -> Linear(h1,h2) -> affine -> ReLU
 * with d_w1 [h1][d+5], d_w2 [h2][h1] row-major (nn.Linear layout); the affine is BatchNorm1d expressed as
 * y*s+t (bias folded into t).  Output canvas NHWC [B][ny][nx][h2] (row = ny-1-xi, col = yi), fully written.
 * Workspace: lavb_pillar_workspace_bytes(B, nx, ny) bytes, contents irrelevant on entry.
 * Grid: a point is kept when min_x <= x < max_x and min_y <= y < max_y on the raw fp32 coordinates (NaN and +-inf are
 *   dropped); xi = trunc(fp32(fp32(x - min_x) * ppm)), yi likewise.  A pillar is (b, xi, yi) before any clamp; its cell is
 *   row = clamp(ny-1-xi, 0, ny-1), col = clamp(yi, 0, nx-1).  When two pillars clamp onto one cell (yi == nx by rounding, or
 *   a grid with nx != ny), the cell holds the per-channel max over the rows of both.  The decorated row is [pt(d) | xyz -
 *   centroid of its pillar | x - fp32(fp32(yi / ppm) + min_x) | y - fp32(fp32(xi / ppm) + min_y)].
 * Values: each ReLU is max(a, 0) with NaN -> 0.  A NaN in any decorated column of a point (a NaN z or feature, or an inf z,
 *   whose z - centroid is inf - inf) makes all its hidden units NaN, hence 0, so the point contributes relu(t2) to its
 *   cell; a NaN z makes the centroid NaN, so every point of its pillar contributes relu(t2).  lavb_pillar_forward computes
 *   in fp32 throughout: other infinities propagate as in IEEE arithmetic and may reach the canvas as +inf (never NaN).
 *   With finite inputs whose fp32 sums stay finite it is accurate to fp32.
 * The centroid sums are float atomics in an order that varies between calls, so neither encoder is bit-reproducible; results
 *   differ by the rounding of those sums.
 * Checked (a rejected call writes nothing): 1 <= batch <= 128, starts and counts >= 0, fewer than 2^31 points; d == 11,
 *   h1 == h2 == 64, pt_stride >= d; ppm finite and > 0; finite window bounds with min < max; nx, ny >= 1, and the grid holds
 *   the window: for v the largest fp32 below max_x (max_y), trunc(fp32(fp32(v - min) * ppm)) <= nx (ny); d_pts non-null
 *   (unless there are no points) and 4-byte aligned; weights, canvas and workspace non-null; w2 8-byte aligned, the other
 *   weights 4-byte aligned, the workspace 16-byte aligned; the fp32 canvas 4-byte aligned (lavb_pillar_forward) or the canvas
 *   16-byte aligned (lavb_pillar_forward_sorted).  Not checked: that each cloud lies inside d_pts. */
size_t lavb_pillar_workspace_bytes(int batch, int nx, int ny);
int lavb_pillar_forward(const float* d_pts, int pt_stride, int d,
                        const long long* h_cloud_start, const int* h_cloud_count, int batch,
                        float min_x, float max_x, float min_y, float max_y, float ppm, int nx, int ny,
                        const float* d_w1, const float* d_s1, const float* d_t1, int h1,
                        const float* d_w2, const float* d_s2, const float* d_t2, int h2,
                        void* d_canvas, int canvas_dtype, void* d_workspace, void* stream);

/* Sorted, atomic-free variant for the tensor-core pipeline (the product encoder): counting sort of the points by canvas cell,
 * layer 1 on hi/lo-split h16 operands (~ fp32), layer 2 on h16 operands with fp32 accumulation (mma.sync), one canvas row written
 * per pillar and the rows of empty cells zero-filled by the scan pass.  out_mode 0: fp32 canvas [B][ny][nx][h2]; 2: h16 canvas
 * [B][ny][nx][h2], saturating; any other out_mode is rejected.  Same semantics otherwise.
 * Precision: layer 1 splits each decorated value and each w1 weight into an h16 hi and lo part (saturating) and drops lo*lo;
 *   this is close to fp32 only while the decorated values stay inside the h16 range (|v| < 65504): beyond it the split loses
 *   the value silently (from 2 * 65504 on, v counts as +-131008), and an infinite decorated value that is not NaN saturates
 *   the same way instead of propagating.  Layer 2 reads w2 and the hidden activations (after affine and ReLU) rounded to h16, saturating.  The
 *   fp32 canvas is never NaN; the h16 canvas is the fp32 result rounded once, saturating, so it is always finite. */
size_t lavb_pillar_sorted_workspace_bytes(int batch, int nx, int ny, long long total_points);
int lavb_pillar_forward_sorted(const float* d_pts, int pt_stride, int d,
                               const long long* h_cloud_start, const int* h_cloud_count, int batch,
                               float min_x, float max_x, float min_y, float max_y, float ppm, int nx, int ny,
                               const float* d_w1, const float* d_s1, const float* d_t1, int h1,
                               const float* d_w2, const float* d_s2, const float* d_t2, int h2,
                               void* d_canvas, int out_mode, void* d_workspace, void* stream);

/* training-mode pieces (BatchNorm1d batch statistics over all in-window points, arg-routed backward).
 * stage 0: voxelise + decorate -> d_feat [M][d+5] (M = number of in-window points, returned in *h_m),
 *          d_cell [M] int32 canvas cell id (b*ny*nx + row*nx + col), -1 never appears.
 *          Rows come in input order: clouds in batch order, points in their order within the cloud (an order-preserving
 *          compaction of the in-window points).  A pillar is (b, xi, yi) before any clamp, so a y that rounds to yi == nx
 *          (SURVEY App. C.5) forms its own pillar for the centroid and cell-origin columns, while its cell clamps onto
 *          col nx-1 (an x that rounds up to the last index likewise clamps onto row 0).  pt_stride >= d, 1 <= batch <= 128,
 *          d == 11; the grid is checked as for lavb_pillar_forward.
 * The Linear/BN1d/ReLU stack then runs on d_feat with autograd; stage 1 max-pools rows into the canvas and
 * records the arg-max row per (cell, channel) for the backward:
 *   precondition: d_h >= 0 (post-ReLU) and 0 <= d_cell[r] < n_cells; m >= 0, c >= 1, n_cells >= 0.
 *   canvas[cell, ch] = max over the rows r of that cell of h[r, ch]; an empty cell holds 0.  When two pillars share a
 *   cell (the clamp above), the cell holds the per-channel max over the rows of both.
 *   argmax[cell, ch] = the SMALLEST row r of that cell with h[r, ch] == canvas[cell, ch] (ties, including channels
 *   whose rows are all 0, go to the smallest row); an empty cell holds 0x7f7f7f7f.  d_argmax may be null.
 * backward: gh[r, ch] = gcanvas[cell[r], ch] if argmax[cell[r], ch] == r else 0, so each (cell, channel) gradient
 *   reaches exactly one row. */
int lavb_pillar_decorate(const float* d_pts, int pt_stride, int d,
                         const long long* h_cloud_start, const int* h_cloud_count, int batch,
                         float min_x, float max_x, float min_y, float max_y, float ppm, int nx, int ny,
                         float* d_feat, int* d_cell, int* h_m, void* d_workspace, void* stream);
int lavb_pillar_scatter_max(const float* d_h, const int* d_cell, int m, int c, long long n_cells,
                            float* d_canvas, int* d_argmax, void* stream);
int lavb_pillar_scatter_max_bwd(const float* d_gcanvas, const int* d_argmax, const int* d_cell, int m, int c,
                                float* d_gh, void* stream);

/* ---------------------------------------------------------------- generic tap-list convolution (CUDA cores)
 * replaces: every nn.Conv2d / nn.ConvTranspose2d (+ the ReLU / BatchNorm / residual that follows it) of
 *           ERFNet (lav/models/erfnet.py:12-134), ConvBackbone and Head (lav/models/lidar.py:48-164).
 * out[n, oy*out_sy+out_oy, ox*out_sx+out_ox, out_coff+co] = epi( sum_t sum_ci
 *        in[n, oy*in_sy+dy[t], ox*in_sx+dx[t], in_coff+ci] * w[t][ci][co] )   (zero outside the input)
 * epi(a): a += bias[co]; if pre_relu a=max(a,0); a = a*scale[co]+shift[co]; a += res[...]; if post_relu
 *         a=max(a,0); if sigmoid a=1/(1+exp(-a)).   Null pointers skip a step.
 *         max(a,0) is fmaxf(a, 0.f): a NaN that reaches a ReLU leaves it as 0; without a ReLU a NaN accumulator stays NaN
 *         through every step.  Every body follows this rule.
 * d_w: [ntaps][cin][cout_pad] fp32 with cout_pad = cout rounded up to 16.
 * Accumulation is fp32.  One exception to "fp32 weights": a 16-bit input with cin == 16 and ntaps <= 9 runs on the
 * tensor cores (mma.sync), which round each weight to the 16-bit type (round to nearest, saturating) before use; the
 * same layer with 10..16 taps, or any fp32 input, multiplies by the fp32 weights.
 * A strided Conv2d uses in_s=stride, dy=ky*dil-pad; a ConvTranspose2d is issued once per output phase with
 * in_s=1, out_s=stride (lav_b200/layers.py builds the tap lists).
 * Writes exactly the channels [out_coff, out_coff+cout) of the output pixels (oy*out_sy+out_oy, ox*out_sx+out_ox) with
 * oy < hog, ox < wog that fall inside hout x wout, for the n images; nothing else.
 * Checked (a rejected call writes nothing): 1 <= ntaps <= 16; cin >= 4 and cin, in_coff, in_cstride multiples of 4;
 * 0 <= in_coff, in_coff+cin <= in_cstride; 0 <= out_coff, out_coff+cout <= out_cstride; with a residual 0 <= res_coff,
 * res_coff+cout <= res_cstride and res_dtype == out_dtype; n, hog, wog, cout >= 1; hin, win, hout, wout >= 1;
 * in_s, out_s >= 1, out_oy, out_ox >= 0; in, out, w non-null; scale and shift both or neither; in, out and res
 * 4-element aligned (16 bytes fp32, 8 bytes 16-bit), w 16-byte aligned, bias / scale / shift 4-byte aligned.
 * Not checked: that the buffers hold the extents the descriptor describes. */
typedef struct {
  const void* in; int in_dtype; int n, hin, win, cin, in_cstride, in_coff;
  void* out; int out_dtype; int hout, wout, cout, out_cstride, out_coff;
  int hog, wog;                 /* output-grid extent visited by this call */
  int in_sy, in_sx, out_sy, out_sx, out_oy, out_ox;
  int ntaps; int dy[16]; int dx[16];
  const float* w; const float* bias; const float* scale; const float* shift;
  const void* res; int res_dtype; int res_cstride, res_coff;
  int pre_relu, post_relu, sigmoid;
  /* lavb_conv_umma only: depth-to-space epilogue.  d2s_nout > 0 means the (<= 32) GEMM columns are 4 output positions
   * x d2s_nout channels: column j = pos*d2s_nout + k goes to pixel (2*gy + pos/2, 2*gx + pos%2), channel k of an fp32
   * NHWC tensor [n][hout][wout][d2s_nout] (out_s must be 2).  This is how a ConvTranspose2d(k3,s2,p1,op1) with a few
   * output channels runs as a 2x2-tap GEMM (the four detection heads' last layer). */
  int d2s_nout;
} lavb_conv_desc;
int lavb_conv_taps(const lavb_conv_desc* h_desc, void* stream);

/* grouped ConvTranspose2d(k3,s2,p1,op1) with <=4 output channels per group: the 4 head output layers in one launch.
 * replaces: Head.net[3] x4 (lav/models/lidar.py:155,159-164) incl. bias and the seg head's sigmoid.
 * d_in NHWC [n][h][w][in_cstride] (group g reads channels [g*cin_g,(g+1)*cin_g)); d_w fp32 [g][cin_g][9][4]
 * (tap = ky*3+kx, cout padded to 4); d_bias [g][4]; output g: fp32 NHWC [n][2h][2w][n_out[g]], every element written,
 * sigmoid applied when h_sigmoid[g] != 0.  dtype LAVB_F32 or the 16-bit type; fp32 weights and accumulation.
 * Checked (a rejected call writes nothing): 1 <= groups <= 8; cin_g a multiple of 8 in 8..64; in_cstride a multiple
 * of 8 with groups*cin_g <= in_cstride; n, h, w >= 0 (an empty map writes nothing); 1 <= n_out[g] <= 4; d_in 4-element
 * aligned (16 bytes fp32, 8 bytes 16-bit); d_w, d_bias and the outputs non-null and 4-byte aligned. */
int lavb_deconv3x3s2_small(const void* d_in, int dtype, int n, int h, int w, int in_cstride, int groups, int cin_g,
                           const float* d_w, const float* d_bias, const int* h_n_out, const int* h_sigmoid,
                           float* const* h_out_ptrs, void* stream);

/* 2x2/2 max-pool -> y*scale[c]+shift[c] -> ReLU into a channel slice (ERFNet DownsamplerBlock, erfnet.py:20-23).
 * out[n, y, x, out_coff+k] = fmaxf(fmaf(max of the 2x2 window of in[.., in_coff+k], scale[k], shift[k]), 0), k < c, in the
 * input dtype (LAVB_F32 or the 16-bit type); nothing else is written.  A vector body runs when c, the offsets and the
 * strides are multiples of 4, d_in / d_out are 4-element aligned and scale / shift 16-byte aligned; otherwise a scalar
 * body computes the same values.  Checked (a rejected call writes nothing): n, hin, win >= 0 and even hin, win; c >= 1;
 * 0 <= in_coff, in_coff+c <= in_cstride; 0 <= out_coff, out_coff+c <= out_cstride; when there is work, non-null
 * pointers aligned to their element size. */
int lavb_pool2_affine_relu(const void* d_in, int dtype, int n, int hin, int win, int c, int in_cstride, int in_coff,
                           const float* d_scale, const float* d_shift,
                           void* d_out, int out_cstride, int out_coff, void* stream);

/* RGB ingest: uint8 NHWC (n,h,w,3) or float NCHW (n,3,h,w) in 0..255 -> (x/255-.5)*2 as NHWC with 4 channels
 * (4th = 0).  replaces RGBSegmentationModel.normalize (lav/models/rgb.py:41).  Computed as fp32 (x / 255 - 0.5) * 2 with
 * three roundings, then stored in out_dtype (LAVB_F32 or the 16-bit type).  Checked: n, h, w >= 0 (an empty batch writes
 * nothing); otherwise non-null pointers, d_out 4-element aligned (16 bytes fp32, 8 bytes 16-bit), a float source 4-byte
 * aligned. */
int lavb_rgb_normalize(const void* d_rgb, int src_is_u8_nhwc, int n, int h, int w, void* d_out, int out_dtype,
                       void* stream);

/* ---------------------------------------------------------------- brake-model stem on raw camera bytes
 * replaces: Normalize + ResNet conv1(7x7,s2,p3,3->64) + bn1 + ReLU of RGBBrakePredictionModel (team_code_v2/models/rgb.py:66-70,
 * lav/models/resnet.py:178,235-238).  d_img: uint8 (batch, ncam, h, cam_w, 3) — the logical image is the ncam cameras side by
 * side (h x ncam*cam_w), ncam <= 4, cam_w % 4 == 0; d_w: BatchNorm-folded weights h16 [64][160] with
 * k = ky*22 + kx*3 + c (slot 21 of every window row and k >= 154 are zero); d_bias [64]; h_mean/h_std: the 3 ImageNet
 * constants; d_out: h16 NHWC (batch, (h-1)/2+1, (ncam*cam_w-1)/2+1, 64), every element written.
 * The staged operand is fmaf(u8, na, nb) in fp32 with na = 1.f / (255.f * std), nb = -mean / std computed in fp32 on the host,
 * then rounded to h16; products with the h16 weights are summed in fp32 on the tensor cores; then + bias, ReLU = fmaxf(a, 0)
 * and a saturating h16 store.  The fp32 operand differs from the reference's (x / 255 - mean) / std by at most a few fp32
 * ulps, so an h16 operand can land one h16 ulp away from the reference's rounding.
 * Checked before any launch (a rejected call writes nothing): batch >= 0 (0 writes nothing), 1 <= ncam <= 4, h >= 7,
 * cam_w >= 8 and a multiple of 4; the grid fits (batch * ceil(ho / 8) < 2^31, ceil(wo / 128) <= 65535); otherwise non-null
 * pointers, d_img / d_w / d_bias 4-byte and d_out 16-byte aligned, d_out not overlapping d_img, d_w or d_bias (every block
 * reads them first), and mean / std giving a finite na, nb with std != 0. */
int lavb_stem7x7s2_u8(const void* d_img, int batch, int ncam, int h, int cam_w, const void* d_w, const float* d_bias,
                      const float* h_mean, const float* h_std, void* d_out, void* stream);
/* replaces: ResNet.maxpool = MaxPool2d(3, 2, 1) (lav/models/resnet.py:181,238) on h16 NHWC (n, h, w, c), c % 8 == 0
 * -> (n, (h-1)/2+1, (w-1)/2+1, c), every element written.  The result is the window's maximum, exactly; pixels off the map
 * are skipped.  A NaN anywhere in the window gives a NaN, as MaxPool2d propagates NaN: the canonical 0x7FFF when the window
 * holds two or more pixels; on a 1 x 1 map, whose windows hold one pixel, that pixel is copied, NaN payload and sign
 * included.  One rule
 * departs from MaxPool2d: when the maximum is zero and the window holds both -0 and +0 the result is +0, where MaxPool2d
 * keeps whichever comes first in the window.
 * Checked before any launch (a rejected call writes nothing): n >= 0 (0 writes nothing), h, w >= 1, c a positive multiple
 * of 8, fewer than 2^31 blocks of 256 output vectors; otherwise non-null, 16-byte aligned d_in and d_out that do not
 * overlap. */
int lavb_maxpool3x3s2_nhwc(const void* d_in, int n, int h, int w, int c, void* d_out, void* stream);

/* ---------------------------------------------------------------- detection decode (device part)
 * replaces: extract_peak (team_code_v2/model_inference.py:189-202: sigmoid, 7x7 max-pool NMS, top-k) and the per-peak
 * map reads of det_inference (:100-112).  d_center: heat-map LOGITS fp32 NHWC [batch][h][w][ncls]; d_box / d_ori: size /
 * orientation maps fp32 NHWC [batch][h][w][2], shared by the classes.  Score s = 1 / (1 + expf(-logit)) in fp32, bit for bit
 * torch.sigmoid on the device.  A pixel is a peak when nothing in its 7x7 window (pixels off the map ignored) is larger
 * (equal neighbours are all peaks); a NaN in the window never suppresses, as in max_pool2d.  Candidates: the peaks with
 * s > min_score compared in fp32, plus every NaN pixel (torch.topk ranks NaN first, so a NaN takes one of the reference's
 * max_det slots; the host filter then drops it).  Anything else is dropped by the reference's host filter anyway.  Per
 * (frame, class) the max_det first candidates — NaN first, then descending s, ties (and NaNs among themselves) to the
 * lower flat index y * w + x — fill d_packed [batch][7][ncls*max_det] = s | flat index | w | h | cos | sin | W with the
 * box and orientation values at the peak; the columns past the last candidate are (-1e5, 0, 0, 0, 0, 0, W).  The output
 * depends on the maps alone: however many candidates a class has, the selection is exact.  1 <= ncls <= 8,
 * 1 <= max_det <= 64, h, w >= 1, h * w <= 2^24 (the flat index is stored as fp32); batch = 0 writes nothing.  A rejected
 * call writes nothing.  d_workspace: lavb_det_peaks_workspace_bytes(batch, ncls) bytes. */
size_t lavb_det_peaks_workspace_bytes(int batch, int ncls);
int lavb_det_peaks(const float* d_center, const float* d_box, const float* d_ori, int batch, int h, int w, int ncls,
                   float min_score, int max_det, float* d_packed, void* d_workspace, void* stream);

/* ---------------------------------------------------------------- rotated bilinear crop
 * replaces: UniPlanner.crop_feature (team_code_v2/models/uniplanner.py:303-340; model_inference.py:204-238) =
 *           F.affine_grid(theta, align_corners=True) + F.grid_sample(bilinear, zeros padding, align_corners=True).
 * d_feat NHWC [b][h][w][c]; crop k samples frame d_frame_idx[k] with the 2x3 affine d_theta[k]; out NHWC
 * [k][crop][crop][c] in the feature dtype.  d_frame_idx: int32 [k]; d_theta: fp32 [k][2][3].
 * dtype LAVB_F32 (c a positive multiple of 4) or the library's 16-bit type (c a positive multiple of 8): a thread moves
 * 16 bytes of channels, so d_feat and d_out must be 16-byte aligned.  b, h, w >= 1 (maps one pixel wide or high included),
 * crop >= 2, 0 <= k <= 65535; k = 0 launches nothing and writes nothing.  Frame indices outside [0, b) are clamped to the
 * nearest frame.  Every element of d_out is written (zeros where a sample leaves the map).  Accumulation is fp32 in the same
 * fmaf order for both dtypes; the 16-bit output is the fp32 result rounded once to nearest. */
int lavb_crop_bilinear(const void* d_feat, int dtype, int b, int h, int w, int c, const int* d_frame_idx,
                       const float* d_theta, int k, int crop, void* d_out, void* stream);
/* the same crop from a uint8 PLANAR map (the ground-truth BEV): d_map [b][c][h][w] uint8 -> d_out NCHW [k][c][crop][crop] fp32.
 * replaces: BEVPlanner.forward's `bev.float()`, `bev.expand(N,...).permute(...).contiguous()[typs]`, F.affine_grid and
 *           F.grid_sample (lav/models/bev_planner_v2.py:92,104,146,222-264).
 * Bit-identical to lavb_crop_bilinear (fp32) on the float copy of the map.  Frame indices outside [0, b) are clamped to the
 * nearest frame, as in lavb_crop_bilinear.  Every output element is written (zeros where a sample leaves the map).
 * c >= 1, crop >= 2, k <= 65535; no backward (the map is data). */
int lavb_crop_bilinear_u8(const uint8_t* d_map, int b, int c, int h, int w, const int* d_frame_idx, const float* d_theta,
                          int k, int crop, float* d_out, void* stream);
/* gradient of lavb_crop_bilinear with respect to d_feat (fp32 NHWC; training, lav/models/uniplanner.py:56-151 through F.grid_sample):
 * replaces cudnn_grid_sampler_backward + the index_put of `features[frame]`.  A gather over the crops of each frame — no
 * atomics, fixed summation order, EVERY element of d_gfeat [b][h][w][c] is written (zeros where no crop samples, and for
 * every frame when k = 0).  d_gout fp32 NHWC [k][crop][crop][c]; d_frame_idx, d_theta as in lavb_crop_bilinear, frame
 * indices clamped the same way.  c a positive multiple of 4, d_gout and d_gfeat 16-byte aligned, 1 <= b <= 65535,
 * h, w >= 1, crop >= 2, k >= 0.  Any theta is accepted; one with no usable inverse (a map one pixel wide or high, a
 * rank-deficient theta) is handled exactly, at the cost of visiting every crop pixel for each feature pixel. */
int lavb_crop_bilinear_bwd(const float* d_gout, int b, int h, int w, int c, const int* d_frame_idx, const float* d_theta,
                           int k, int crop, float* d_gfeat, void* stream);

/* dtype / layout helpers
 * lavb_convert: count elements fp32 -> 16-bit (round to nearest, saturating to the finite range; NaN stays NaN) or 16-bit
 * -> fp32 (exact).  count >= 0; pointers non-null and aligned to their element size.  Both 4-element aligned take the
 * vector body, otherwise every element is converted one at a time; the results are the same. */
int lavb_convert(const void* d_src, int src_dtype, void* d_dst, int dst_dtype, long long count, void* stream);

/* ---------------------------------------------------------------- wgmma implicit-GEMM tap-list convolution
 * replaces (h16 path): the Conv2d -> ReLU -> BatchNorm2d layers of ConvBackbone (lidar.py:57-131), the fused 4-head
 *           384->256 conv (lidar.py:152-154) and the 64/128-channel factorised convs of ERFNet (erfnet.py:31-61).
 * Same descriptor and epilogue semantics as lavb_conv_taps, with these differences: input is h16 NHWC, cin % 64 == 0,
 * cout % 32 == 0 and <= 256, channel offsets/strides multiples of 8; d->w points to h16 weights laid out
 * [ntaps][cout][cin] (K contiguous).  Tiles are 8 x 16 output-grid pixels; operands are fetched by TMA
 * (cuTensorMapEncodeTiled through cudaGetDriverEntryPoint), accumulators live in registers. */
int lavb_conv_umma(const lavb_conv_desc* h_desc, void* stream);

/* ---------------------------------------------------------------- planner embedder stem
 * replaces: conv1 (7x7, s2, p3, cin -> 64) + bn1 + ReLU of UniPlanner's crop embedder resnet18(num_channels=384)
 * (team_code_v2/models/uniplanner.py:36-40, lav/models/resnet.py:178,235-238) on the h16 path.  d_in: h16 NHWC (n, h, w, cin),
 * cin % 64 == 0, h, w >= 7; d_w: BatchNorm-folded h16 weights laid out [49 taps (ky*7 + kx)][64 cout][cin]; d_bias: fp32 [64];
 * d_out: h16 NHWC (n, (h-1)/2+1, (w-1)/2+1, 64) = relu(conv + bias), saturating.  wgmma implicit GEMM with output channels
 * in M and 16 x 16 output-pixel tiles in N; operands fetched by TMA, whose out-of-bounds zero fill is the padding. */
int lavb_conv7x7s2_umma(const void* d_in, int n, int h, int w, int cin, const void* d_w, const float* d_bias, void* d_out,
                        void* stream);

/* ---------------------------------------------------------------- 3x3 convolution, output channels in M
 * replaces (h16 path): the stride-1 and stride-2 Conv2d -> ReLU -> BatchNorm2d layers of ConvBackbone (lidar.py:57-131) and the
 * fused 4-head 384->256 conv (lidar.py:152-154) where LiDARModel routes them here (layers.py).  The kernel of
 * lavb_conv7x7s2_umma with a 3x3 / pad-1 tap set: 16 x 16 output-pixel tiles, one TMA box per kernel row (stride 1) or per
 * kernel row and column parity (stride 2).
 *   d_in : h16 NHWC (n, h, w, cin), dense; cin in {64, 128, 384}; h, w >= 1
 *   d_w  : h16 [9 taps (ky*3 + kx)][cout][cin] (the lavb_conv_umma packing); cout in {64, 128, 256}; stride in {1, 2}
 *   d_out: h16 NHWC (n, (h-1)/stride+1, (w-1)/stride+1, cout), dense, saturating:
 *          out = max(conv + bias, 0) * scale + shift with pre_relu, (conv + bias) * scale + shift without it; d_bias,
 *          d_scale / d_shift (fp32 [cout]) may be NULL (0, 1 / 0; scale and shift come together).  The fp32 operations are
 *          those of lavb_conv_umma's epilogue; with cin <= 128 at stride 1, and cin = 64 at stride 2, the MMA order is too, so
 *          the output equals lavb_conv_umma's bit for bit. */
int lavb_conv3x3_umma(const void* d_in, int n, int h, int w, int cin, int stride, const void* d_w, int cout, const float* d_bias,
                      const float* d_scale, const float* d_shift, int pre_relu, void* d_out, void* stream);

/* ---------------------------------------------------------------- fused (3x1 -> 1x3) convolution pair
 * replaces: conv3x1_k -> ReLU -> conv1x3_k -> bn_k [-> + input] -> ReLU of non_bottleneck_1d (lav/models/erfnet.py:37-63) in
 * one wgmma kernel; the intermediate activation stays in shared memory.
 *   mid = relu(conv3x1_dil(in) + bias1);  out = [relu](conv1x3_dil(mid) + shift2 [+ res])
 * The BatchNorm affine (conv + b2) * s + t is folded by the caller: w2 <- w2 * s per output channel, shift2 <- b2 * s + t.
 * bias1 / shift2 (fp32 [c]) are added to the register accumulators in the epilogues, which then pack, clamp and add the residual
 * (16-bit packed arithmetic: the residual add rounds once more than an fp32 add would, and its sum saturates at +-65504).
 * in / out / res: h16 NHWC (n, h, w, c) contiguous, c in {64, 128}, w in {32, 64, 128}; w1 / w2: h16 [3 taps][c out][c in];
 * res may be NULL.  out must not overlap in or res (rejected): the kernel reads a tile's residual while earlier tiles are
 * still being stored. */
typedef struct lavb_conv_pair_desc {
  const void* in; void* out; const void* res;
  int n, h, w, c, dil, post_relu;
  const void* w1; const float* bias1;
  const void* w2; const float* shift2;
} lavb_conv_pair_desc;
int lavb_conv_pair_umma(const lavb_conv_pair_desc* h_desc, void* stream);
/* profiling aid: while d_buf is non-NULL every lavb_conv_pair_umma launch writes clock64 stamps of its pipeline events,
 * d_buf[cta][tile iteration < tiles_per_cta][8] int64 (conv_pair_umma.cu: PAIR_STAMP).  NULL switches it off (the default). */
int lavb_conv_pair_set_trace(void* d_buf, int tiles_per_cta);

/* ---------------------------------------------------------------- fused ERFNet entry block on the raw camera bytes
 * replaces: RGBSegmentationModel.normalize ((x/255 - .5) * 2, lav/models/rgb.py:41-45) + Encoder.initial_block =
 * DownsamplerBlock(3, 16): relu(bn(cat[conv3x3 s2 p1 (13 ch), maxpool2x2 (3 ch)])) (lav/models/erfnet.py:12-23,67).
 * d_rgb_u8: uint8 NHWC (n, h, w, 3); h_w27x16: host fp32 [(ky*3+kx)*3+c][16] conv weights (columns >= 13 zero); h_scale16 /
 * h_shift16: host fp32 [16], epi(a) = relu(a * scale + shift) with the conv bias folded into the first 13 shifts; d_out: NHWC
 * (n, h/2, w/2, 16) fp32 or h16, every element written.  Arithmetic: the normalised value is the fp32 (v / 255 - .5) * 2 of
 * the reference (three roundings); each conv channel is a 27-term fp32 fmaf chain in (ky, kx, c) order over the zero-padded
 * normalised image, then relu(fmaf(acc, scale, shift)); the pooled channels are relu(fmaf(max of 4, scale, shift)); the h16
 * output is that fp32 value rounded once, saturating.  Weight columns 13..15 are never read.  ReLU is fmaxf(a, 0), so a NaN
 * that reaches one (a NaN weight, scale or shift) comes out as 0.
 * Checked before any launch (a rejected call writes nothing): n >= 0 (0 writes nothing), h, w even and >= 2, out_dtype
 * LAVB_F32 or the 16-bit type, fewer than 2^31 blocks of 8 x 32 output pixels; otherwise non-null pointers, d_out 16-byte
 * (fp32) or 8-byte (h16) aligned and not overlapping d_rgb_u8. */
int lavb_erf_stem(const void* d_rgb_u8, int n, int h, int w, const float* h_w27x16, const float* h_scale16,
                  const float* h_shift16, void* d_out, int out_dtype, void* stream);

/* ---------------------------------------------------------------- fused DownsamplerBlock(16, 64)
 * replaces: Encoder.layers[0] = DownsamplerBlock(16, 64) (lav/models/erfnet.py:12-23,71): relu(bn(cat[conv3x3 s2 p1 (16 -> 48),
 * maxpool2x2 (16)])).  d_in: h16 NHWC (n, h, w, 16), h and w even, w <= 128; d_out: h16 NHWC (n, h/2, w/2, 64); d_w9: fp32
 * [9 taps (ky*3+kx)][16 cin][48 cout]; d_st: fp32 [64][2] = (scale, shift), epi(a) = relu(a * scale + shift) with the conv bias
 * folded into the first 48 shifts (the last 16 apply to the pooled channels, after the max).  Every output element is written.
 * Arithmetic: the weights are rounded to h16; the conv channels sum the 144 products in fp32 on the tensor cores, then
 * relu(fmaf(acc, scale, shift)) and a saturating h16 store; the pooled channels take the exact max of the four h16 inputs.
 * NaN rules: ReLU is fmaxf(a, 0), so a conv channel whose window holds a NaN comes out as 0.  The pool starts from -inf and
 * uses fmaxf, so it skips a NaN; a window of four NaNs gives -inf, which the affine and ReLU turn into 0 (scale > 0) or
 * +inf, stored as 65504 (scale < 0).
 * Checked before any launch (a rejected call writes nothing): n >= 0 (0 writes nothing), h, w even and >= 2, w <= 128,
 * n * ceil(h / 8) < 2^31; otherwise non-null pointers, d_in / d_out 16-byte and d_w9 / d_st 4-byte aligned, d_out not
 * overlapping d_in, d_w9 or d_st. */
int lavb_erf_down16(const void* d_in, void* d_out, int n, int h, int w, const float* d_w9, const float* d_st, void* stream);

/* ---------------------------------------------------------------- fused 16-channel non_bottleneck_1d block
 * replaces: non_bottleneck_1d(16, dropprob, dilated=1) of the ERFNet decoder (lav/models/erfnet.py:37-63, Decoder layers 4 and 5) —
 * conv3x1 -> ReLU -> conv1x3 -> bn1 -> ReLU -> conv3x1 -> ReLU -> conv1x3 -> bn2 -> (+ input) -> ReLU — in one kernel, all four
 * intermediates in shared memory.  d_in / d_out: h16 NHWC (n, h, w, 16), w % 16 == 0; d_w4: fp32
 * [4 convs][3 taps][16 cin][16 cout]; d_st: fp32 [4 convs][16 cout][2] = (scale, shift) with epi(a) = relu(a * scale + shift)
 * (conv bias folded into shift; scale = 1 for the two convs that have no BatchNorm).  Every output element is written.
 * Arithmetic: the weights are rounded to h16; each conv sums its 48 products in fp32 on the tensor cores, then fmaf(acc,
 * scale, shift), [+ the input x for the last conv, one fp32 add], ReLU, and each intermediate is stored as saturating h16.
 * NaN rule: every ReLU is fmaxf(a, 0), so a NaN that reaches one comes out as 0; an output is never NaN.
 * Checked before any launch (a rejected call writes nothing): n >= 0 (0 writes nothing), h >= 1, 16 <= w <= 256,
 * n * ceil(h / 8) < 2^31; otherwise non-null pointers, d_in / d_out 16-byte, d_w4 4-byte and d_st 8-byte aligned, and
 * d_out not overlapping d_in (halo rows of neighbouring tiles are re-read), d_w4 or d_st (every block reads them first). */
int lavb_erf_nb16(const void* d_in, void* d_out, int n, int h, int w, const float* d_w4, const float* d_st, void* stream);

/* ---------------------------------------------------------------- motion-forecast ("cast") heads in one launch
 * replaces: UniPlanner.cast / BEVPlanner.cast (team_code_v2/models/uniplanner.py:286-301, lav/models/bev_planner_v2.py:226-236):
 * for each of ncmd branches, nn.GRU(512, 64, batch_first=True) over the embedding repeated `steps` times, nn.Linear(64, 2) and the
 * cumulative sum over the steps — 6 x (GRU + Linear + cumsum) calls in the reference.  fp32 FFMA.
 * d_embd (n, 512); d_wih_t (ncmd, 512, 192) = weight_ih_l0 TRANSPOSED; d_whh_t (ncmd, 64, 192) = weight_hh_l0 transposed;
 * d_bih / d_bhh (ncmd, 192); d_wmlp (ncmd, 2, 64); d_bmlp (ncmd, 2); d_out (n, ncmd, steps, 2) fp32. */
int lavb_cast_gru(const float* d_embd, int n, const float* d_wih_t, const float* d_whh_t, const float* d_bih, const float* d_bhh,
                  const float* d_wmlp, const float* d_bmlp, int ncmd, int steps, float* d_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LAV_B200_H */
