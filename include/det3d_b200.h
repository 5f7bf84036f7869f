/*
 * det3d_b200 -- C ABI of the H100-native (sm_90a) point-cloud inference hot path.
 *
 * Every entry point is `extern "C"`, takes plain pointers / sizes / a CUDA
 * stream (as void*), returns an int status (0 = D3B_OK), never calls exit(),
 * never allocates device memory and never synchronises the host: the caller
 * owns every buffer (sizes come from the *_workspace_bytes() queries) and the
 * data-dependent row counts stay in device memory (`int*` count arguments).
 *
 * The reference (V2AI/Det3D) has no C/FFI plugin boundary for this path; its
 * operator API is Python.  Each entry point below names the reference
 * interface it stands behind (paths relative to the Det3D repository root).
 * INTEGRATION.md shows the ctypes binding a Det3D maintainer would add.
 */
#ifndef DET3D_B200_H_
#define DET3D_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes ------------------------------------------------------- */
#define D3B_OK 0
#define D3B_ERR_INVALID_ARG 1   /* null pointer, negative size, unsupported shape */
#define D3B_ERR_CUDA 2          /* a CUDA runtime call failed: see d3b_last_error() */
#define D3B_ERR_UNSUPPORTED 3   /* channel count / kernel size not built          */
#define D3B_ERR_WORKSPACE 4     /* workspace too small                            */

/* Human-readable text of the last error raised on the calling thread. */
const char* d3b_last_error(void);
/* ABI version; bumped whenever a signature changes. */
int d3b_abi_version(void);
/* Number of kernels this library has launched since load (process-wide);
 * bench.py reports the delta over the timed region as "gpu_launches". */
unsigned long long d3b_launch_count(void);
/* Programmatic dependent launch between consecutive convolution kernels of a stream (default on): the next kernel's
 * launch latency and prologue overlap the previous kernel's tail; results are unaffected. 0 = plain stream order. */
void d3b_set_pdl(int on);
/* Schedule of d3b_bev_conv16 for 3x3 stride-1 layers whose output blocks are 128 channels wide (the RPN blocks of
 * necks/rpn.py:124-142): 0 = pixel-stationary (two 128-pixel halves per 16 x 16 pixel tile), 2 = automatic (default:
 * the pipelined kernel -- 16 x 8 pixel tiles, one m64n128 chain per kernel offset, two partials in flight -- for such
 * layers whose C_in is a multiple of 64, the pixel-stationary kernel otherwise; measured the fastest on the H100).  Any
 * other value selects 2.  Same products in the same order: the results are bit-identical. */
void d3b_set_bev_variant(int variant);
int d3b_get_bev_variant(void);

/* ========================================================================= *
 * 1. Voxelizer
 *    replaces det3d/ops/point_cloud/point_cloud_ops.py:112-184
 *    (points_to_voxel) + :7-55 (_points_to_voxel_reverse_kernel), the
 *    batch-index prepend of det3d/torchie/parallel/collate.py:130-137 and the
 *    per-voxel mean of det3d/models/readers/voxel_encoder.py:206-211.
 * ========================================================================= */
typedef struct {
  float voxel_size[3];   /* x, y, z                                      */
  float range_min[3];    /* x, y, z lower bound of point_cloud_range     */
  int32_t grid[3];       /* x, y, z cells = round((hi - lo) / voxel_size) */
  int32_t ndim;          /* floats per point (>= 3)                      */
  int32_t max_points;    /* max points kept per voxel                    */
  int32_t max_voxels;    /* max voxels per cloud (the reference `break`) */
} d3b_voxel_cfg;

/* Bytes of scratch needed to voxelize `batch` clouds holding n_points_total
 * points in one call. */
size_t d3b_voxelize_workspace_bytes(const d3b_voxel_cfg* cfg, int32_t n_points_total,
                                    int32_t batch);

/* Voxelizes `batch` clouds in one call, with the cloud offsets in DEVICE memory, so one captured CUDA graph serves clouds
 * of any size up to point_capacity.
 * points            [point_capacity, ndim] f32 device, clouds concatenated; rows at or past off[batch] are never read
 * cloud_offsets_dev [batch + 1] i32 DEVICE: cloud b owns points [off[b], off[b+1])
 * voxels            [batch*max_voxels, max_points, ndim] f32 device, or NULL
 * coors             [batch*max_voxels, 4] i32 device (batch, z, y, x)
 * num_points        [batch*max_voxels] i32 device
 * mean_feats        [batch*max_voxels, ndim] f32 device, or NULL
 * voxel_counts      [batch + 1] i32 device: [b] = voxels of cloud b, [batch] = total.
 * status            [1] i32 device or NULL: set to 1 if the offsets were not 0 = off[0] <= ... <= off[batch] <= point_capacity;
 *                   they are then clamped into that shape before any point index is formed (0 when they were)
 * workspace: d3b_voxelize_workspace_bytes(cfg, point_capacity, batch); point lists: d3b_voxelize_point_lists(cfg, point_capacity, batch, ws)
 * Rows of all clouds are written back to back (cloud 0 first); only the first voxel_counts[batch] rows of each output
 * are defined.  The outputs are the same bits for any capacity >= off[batch]. */
int d3b_voxelize_dev(const d3b_voxel_cfg* cfg, const float* points, int32_t point_capacity,
                     const int32_t* cloud_offsets_dev, int32_t batch, float* voxels, int32_t* coors,
                     int32_t* num_points, float* mean_feats, int32_t* voxel_counts, int32_t* status,
                     void* workspace, size_t workspace_bytes, void* stream);

/* Multi-sweep ingest (nuScenes) for a batch of samples: each sample's raw sweeps -> one cloud [n, n_feat + 1] =
 * (x, y, z, .., time lag), with the sweep table in DEVICE memory, for graph replay over sweeps of any size.
 * replaces read_file / remove_close / read_sweep and the NuScenes branch of LoadPointCloudFromFile.__call__,
 * det3d/datasets/pipelines/loading.py:17-64,98-124.  Runs three kernels, whatever the batch (no host sync).
 * S = sweep_capacity, 1 <= batch <= 64, 1 <= S <= D3B_INGEST_MAX_SWEEPS * batch.
 * raw            [raw_capacity, raw_stride] f32 device: the sweeps' file contents, each sample's key frame first; rows no
 *                sweep covers are never read
 * sweep_offsets  [S + 1] i32 DEVICE: the logical prefix of the sweeps' lengths, len_s = sweep_offsets[s + 1] -
 *                sweep_offsets[s]; it drives the chunking, the scan and cloud_offsets
 * sweep_src      [S] i32 DEVICE or NULL: sweep s is rows [sweep_src[s], sweep_src[s] + len_s) of raw (e.g. a ring of
 *                per-stream history slots that stay on the device from one frame to the next).  NULL: sweep s is rows
 *                [sweep_offsets[s], sweep_offsets[s + 1]), the sweeps back to back; the same as sweep_src[s] =
 *                sweep_offsets[s], bit for bit
 * sample_sweeps  [batch + 1] i32 DEVICE: sample b owns sweeps [sample_sweeps[b], sample_sweeps[b + 1])
 * transforms     [S, 16] f64 DEVICE row-major 4x4, time_lag [S] f32 DEVICE
 * flags          [S] u8 DEVICE: bit 0 = has_transform, bit 1 = filter_close (drop points with |x| < radius and
 *                |y| < radius before the transform: remove_close); a key frame has neither
 * out            [raw_capacity, n_feat + 1] f32 device: the samples' clouds back to back, each in input order
 * cloud_offsets  [batch + 1] i32 device: sample b's cloud is rows [cloud_offsets[b], cloud_offsets[b + 1]) of `out` --
 *                the form d3b_voxelize_dev takes
 * status         [1] i32 device or NULL.  Bit 0 (value 1) is set if the tables were not 0 = sweep_offsets[0] <= ... <=
 *                sweep_offsets[S] <= raw_capacity and 0 = sample_sweeps[0] <= ... <= sample_sweeps[batch] <= S; they are
 *                then clamped into that shape as t[i] = min(max(0, t[1..i]), bound) before any point index is formed.
 *                After that, each sweep_src[s] is clamped into [0, raw_capacity - len_s], identically in every CTA,
 *                and bit 1 (value 2) is set when that changed anything.  0 when nothing was clamped.
 * workspace: d3b_ingest_dev_workspace_bytes(raw_capacity, S).  Each sample's rows are the bits it gives as a batch of
 * one. */
#define D3B_INGEST_MAX_SWEEPS 16
size_t d3b_ingest_dev_workspace_bytes(int32_t raw_capacity, int32_t sweep_capacity);
int d3b_ingest_sweeps_dev(const float* raw, int32_t raw_capacity, int32_t raw_stride, int32_t n_feat,
                          const int32_t* sweep_offsets, const int32_t* sweep_src, const int32_t* sample_sweeps,
                          const double* transforms, const float* time_lag, const uint8_t* flags,
                          int32_t sweep_capacity, int32_t batch, float radius, float* out, int32_t* cloud_offsets,
                          int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* KITTI camera-frustum crop for a batch of raw scans, with the cloud offsets and the planes in DEVICE memory, for graph
 * replay over scans of any size.  replaces box_np_ops.remove_outside_points (det3d/core/bbox/box_np_ops.py:941-952;
 * the point test of core/bbox/geometry.py:241-276) as called by Preprocess (datasets/pipelines/preprocess.py:111-116).
 * 1 <= batch <= 64, 3 <= ndim <= 16.
 * points            [point_capacity, ndim] f32 device: the scans back to back; rows at or past cloud_offsets_in[batch]
 *                   are never read
 * cloud_offsets_in  [batch + 1] i32 DEVICE: scan b is rows [off[b], off[b + 1])
 * planes            [batch][6][4] f64 DEVICE: scan b's frustum planes (n0, n1, n2, d), in the reference's order
 *                   (det3d_b200.core.bbox.box_np_ops.camera_frustum_planes).  A point is kept when every plane gives
 *                   s = ((x*n0 + y*n1) + z*n2) + d < 0, x, y, z promoted to f64, each operation rounded on its own (no
 *                   FMA); a NaN coordinate fails every s >= 0 test and is kept, as in the reference
 * out               [point_capacity, ndim] f32 device: the kept rows of every scan (all ndim columns), scan after scan,
 *                   each in input order
 * cloud_offsets_out [batch + 1] i32 device: scan b's kept rows are [cloud_offsets_out[b], cloud_offsets_out[b + 1]) of
 *                   `out` -- the form d3b_voxelize_dev takes
 * status            [1] i32 device or NULL: set to 1 if the offsets were not 0 = off[0] <= ... <= off[batch] <=
 *                   point_capacity; they are then clamped into that shape as off[i] = min(max(0, off[1..i]),
 *                   point_capacity) before any point index is formed (0 when they were)
 * workspace: d3b_frustum_crop_workspace_bytes(point_capacity, batch) (0 for arguments out of range).  Runs three kernels
 * (count, scan, emit), no host sync; each scan's rows are bit-identical to that scan cropped alone. */
size_t d3b_frustum_crop_workspace_bytes(int32_t point_capacity, int32_t batch);
int d3b_frustum_crop_dev(const float* points, int32_t point_capacity, int32_t ndim, const int32_t* cloud_offsets_in,
                         const double* planes, int32_t batch, float* out, int32_t* cloud_offsets_out, int32_t* status,
                         void* workspace, size_t workspace_bytes, void* stream);

/* KITTI result rows from predict's packed detections, for graph replay.  replaces the per-box loop of
 * KittiDataset.convert_detection_to_kitti_annos (det3d/datasets/kitti/kitti.py:78-158): limit_period and the z shift in
 * f32, box_lidar_to_camera, center_to_corner_box3d (origin (0.5, 1, 0.5), axis 1) and project_to_image (with its column
 * of ZEROS, so P2's translation never enters) in f64, the strict in-image test, the clip, alpha.
 * 1 <= batch <= 64, 0 <= max_det <= 2^20, nd 7 or 9 (D3B_ERR_UNSUPPORTED otherwise).
 * detections [batch][max_det][nd + 3] f32 device: box, score, label, valid (a row counts when valid > 0.5)
 * calib      [batch][32] f64 DEVICE: M = rect @ Trv2c row-major [0, 16), P2 rows 0..2 row-major [16, 28), image
 *            height [28] and width [29]; [30, 32) unused
 * results    [batch][max_det][14] f64 device: per kept detection, in predict's order, bbox (x0, y0, x1, y1) clipped,
 *            alpha, dimensions (l, h, w), location (camera frame, bottom centre), rotation_y, score, label; rows at or
 *            past counts[b] are written as zeros
 * counts     [batch] i32 device: kept detections of each sample
 * Every f64 product, sum and quotient is rounded on its own in a fixed order (no FMA contraction); sin / cos / atan2 are
 * the CUDA math library's.  One kernel, one CTA per sample, no host sync, no workspace. */
int d3b_kitti_results_dev(const float* detections, const double* calib, int32_t batch, int32_t max_det, int32_t nd,
                          double* results, int32_t* counts, void* stream);

/* nuScenes result rows from predict's packed detections, for graph replay.  replaces the per-box loop of
 * NuScenesDataset.evaluation (det3d/datasets/nuscenes/nuscenes.py:219-259) with _second_det_to_nusc_box and
 * _lidar_nusc_box_to_global (det3d/datasets/nuscenes/nusc_common.py:222-265): yaw' = -r - pi/2 in f32, the orientation
 * quaternion about z, then the sensor -> ego -> global rotation and translation of the centre, the velocity and the
 * orientation in f64, and the reference's speed test (> 0.2 m/s in f64) that picks the attribute.
 * 1 <= batch <= 64, 0 <= max_det <= 2^20, nd 9 (x, y, z, w, l, h, vx, vy, r; D3B_ERR_UNSUPPORTED otherwise).
 * detections [batch][max_det][12] f32 device: box, score, label, valid (a row counts when valid > 0.5)
 * poses      [batch][32] f64 DEVICE: the key frame's calibrated_sensor rotation matrix Rc (row-major) [0, 9) and
 *            translation tc [9, 12), its ego_pose rotation matrix Rp [12, 21) and translation tp [21, 24), the two
 *            rotations as unit quaternions (w, x, y, z) qc [24, 28) and qp [28, 32)
 * results    [batch][max_det][15] f64 device: per valid detection, in predict's order, translation 3 (global), size 3
 *            (w, l, h), rotation 4 (w, x, y, z), velocity 2 (global x, y), score, label, moving (1 or 0); rows at or
 *            past counts[b] are written as zeros
 * counts     [batch] i32 device: valid detections of each sample
 * Every f64 product and sum is rounded on its own in a fixed order (no FMA contraction); sin / cos are the CUDA math
 * library's.  One kernel, one CTA per sample, no host sync, no workspace. */
int d3b_nusc_results_dev(const float* detections, const double* poses, int32_t batch, int32_t max_det, int32_t nd,
                         double* results, int32_t* counts, void* stream);

/* ========================================================================= *
 * 2. Rulebook (sparse-convolution index maps)
 *    replaces spconv v1.x `get_indice_pairs` as called by SubMConv3d /
 *    SparseConv3d at det3d/models/backbones/scn.py:106-157,323-355
 *    (spconv is an un-vendored dependency of the reference).
 *
 *    The map is output-stationary: nbr[k * row_cap + o] is the input row
 *    feeding output row o through kernel offset k, or -1.  k enumerates
 *    (kz, ky, kx) row-major.  tile_mask[o / 128] has bit k set when any of
 *    the 128 rows of that tile has a neighbour at offset k.
 * ========================================================================= */
typedef struct {
  int32_t spatial[3];   /* D, H, W of the level                              */
  int32_t batch;
  /* level-0 index: open-addressing hash (key -> row)                         */
  uint64_t* hash_keys;  /* [hash_cap] , NULL when the level uses the bitmap   */
  int32_t* hash_vals;   /* [hash_cap]                                         */
  int32_t hash_cap;     /* power of two                                       */
  /* strided-level index: occupancy bitmap + exclusive popcount prefix        */
  uint32_t* bitmap;     /* [n_words]                                          */
  int32_t* word_prefix; /* [n_words]                                          */
  int64_t n_words;
} d3b_site_index;

size_t d3b_rulebook_workspace_bytes(int64_t n_words);

/* Build the level-0 hash index of `coors` ([n,4] b,z,y,x; n read from *n_rows). */
int d3b_index_build_hash(const int32_t* coors, const int32_t* n_rows, int32_t row_cap,
                         d3b_site_index* index, void* stream);

/* Submanifold rulebook: outputs == inputs (same rows, same order).  Fills nbr and tile_mask. */
int d3b_rulebook_subm(const int32_t* coors, const int32_t* n_rows, int32_t row_cap,
                      const d3b_site_index* index, const int32_t ksize[3],
                      int32_t* nbr, uint32_t* tile_mask, void* stream);

/* Strided sparse conv rulebook.  Output sites = every site reachable from an
 * active input, in ascending linear index ((b*D+z)*H+y)*W+x.  Fills
 * out_index (bitmap form), out_coors [out_cap,4], *n_out, nbr, tile_mask. */
int d3b_rulebook_conv(const int32_t* in_coors, const int32_t* n_in, int32_t in_cap,
                      const d3b_site_index* in_index, const int32_t ksize[3],
                      const int32_t stride[3], const int32_t padding[3],
                      d3b_site_index* out_index, int32_t* out_coors, int32_t* n_out,
                      int32_t out_cap, int32_t* nbr, uint32_t* tile_mask, void* workspace,
                      size_t workspace_bytes, void* stream);

/* ========================================================================= *
 * 3. Sparse convolution (gather -> contraction -> fused epilogue)
 *    replaces spconv v1.x `indice_conv` (gather, torch.mm, scatter-add) plus
 *    the BatchNorm1d(eval) / ReLU / residual that follow it in
 *    det3d/models/backbones/scn.py:73-89,106-157.
 *
 *    out[o,:] = act( (sum_k in[nbr[k][o],:] . W[k] + bias) * scale + shift
 *                    + residual[o,:] )
 * ========================================================================= */
#define D3B_ALGO_SIMT 0     /* fp32 FFMA, output-stationary                              */
#define D3B_ALGO_TC 1       /* wgmma 3xTF32 (fp32-equivalent), output-stationary tiles    */

typedef struct {
  int32_t c_in, c_out, k_vol;    /* k_vol = kd*kh*kw                          */
  const float* weight;           /* [k_vol, c_in, c_out] f32 (spconv layout)  */
  const float* weight_packed;    /* D3B_ALGO_TC operand image, see below      */
  const float* bias;             /* [c_out] or NULL                           */
  const float* scale;            /* [c_out] or NULL (folded BN)               */
  const float* shift;            /* [c_out] or NULL                           */
  const float* residual;         /* [n_out, c_out] or NULL                    */
  int32_t relu;
  int32_t algo;                  /* D3B_ALGO_SIMT or D3B_ALGO_TC; any other value: D3B_ERR_INVALID_ARG */
} d3b_conv_params;

/* Size in floats / fill of the tensor-core weight image (hi/lo TF32 split,
 * K-major 128B-swizzled tiles).  Done once per layer at model load. */
size_t d3b_conv_packed_weight_floats(int32_t c_in, int32_t c_out, int32_t k_vol);
int d3b_conv_pack_weight(const float* weight_dev, int32_t c_in, int32_t c_out, int32_t k_vol,
                         float* packed_dev, void* stream);

int d3b_sparse_conv(const float* feat_in, const int32_t* nbr, const uint32_t* tile_mask,
                    const int32_t* n_out, int32_t out_cap, const d3b_conv_params* p,
                    float* feat_out, void* stream);

/* PillarFeatureNet, eval mode, one PFN layer (every Det3D PointPillars config): decoration
 * (x,y,z,.. | xyz - pillar mean | xy - pillar centre), Linear(ndim+5 -> units, no bias), BatchNorm1d folded
 * to scale/shift, ReLU, max over the max_points slots -- padded slots count as all-zero features, as the
 * reference's mask makes them.  replaces det3d/models/readers/pillar_encoder.py:115-155 (+ PFNLayer :33-47).
 * voxels [row_cap, max_points, ndim] f32, num_points [row_cap] i32, coors [row_cap, 4] i32 (b,z,y,x),
 * n_rows device i32 (live rows; the rest of `out` is zero-filled), weight [units, ndim+5] (nn.Linear
 * layout), out [row_cap, units].  x_offset = vx/2 + range_min_x (likewise y).
 * D3B_ERR_UNSUPPORTED unless 3 <= ndim <= 11 and units in {32, 64, 96, 128}. */
int d3b_pillar_features(const float* voxels, const int32_t* num_points, const int32_t* coors,
                        const int32_t* n_rows, int32_t row_cap, int32_t max_points, int32_t ndim,
                        int32_t units, const float* weight, const float* scale, const float* shift,
                        float vx, float vy, float x_offset, float y_offset, float* out, void* stream);

/* The same reader fused with the voxelizer (SURVEY 8f.3): the pillar's points are fetched through the voxelizer's
 * per-voxel point-index lists, so the [rows, max_points, ndim] voxel tensor is never materialised (call d3b_voxelize_dev
 * with voxels = NULL).  `lists` = d3b_voxelize_point_lists(...) of the workspace that d3b_voxelize_dev just filled:
 * [batch][max_voxels][max_points] int32 indices into `points`, >= 0x7f000000 = empty slot; valid until that workspace is
 * used again.  voxel_counts = d3b_voxelize_dev's per-cloud counts.  Everything else as d3b_pillar_features. */
const int32_t* d3b_voxelize_point_lists(const d3b_voxel_cfg* cfg, int32_t n_points_total, int32_t batch, void* workspace);
int d3b_pillar_features_lists(const float* points, const int32_t* lists, const int32_t* voxel_counts, int32_t batch,
                              int32_t max_voxels, const int32_t* num_points, const int32_t* coors, const int32_t* n_rows,
                              int32_t row_cap, int32_t max_points, int32_t ndim, int32_t units, const float* weight,
                              const float* scale, const float* shift, float vx, float vy, float x_offset, float y_offset,
                              float* out, void* stream);

/* .dense(): rows -> zero-initialised [B, C, D, H, W] (caller zero-fills `out`).
 * replaces SparseConvTensor.dense() at scn.py:192,365. */
int d3b_sparse_to_dense(const float* feat, const int32_t* coors, const int32_t* n_rows,
                        int32_t row_cap, int32_t channels, const int32_t spatial[3],
                        int32_t batch, float* out, void* stream);

/* rows -> zero-initialised channels-last BEV rows [B*H*W, C*D], channel = c*D + z: the same
 * values as .dense().view(B, C*D, H, W) (scn.py:192-195), laid out for the NHWC dense path. */
int d3b_sparse_to_bev_rows(const float* feat, const int32_t* coors, const int32_t* n_rows,
                           int32_t row_cap, int32_t channels, const int32_t spatial[3],
                           int32_t batch, float* out_rows, void* stream);

/* Static rulebook of a dense stride-1 2-D convolution over a [B, H, W] grid (row = (b*H+y)*W+x):
 * nbr[k*n + row] = row of (y + ky - pad_y, x + kx - pad_x) or -1; k = ky*kw + kx.  Lets the
 * dense RPN (det3d/models/necks/rpn.py:124-159) and head 1x1 convs (mg_head.py:198-230) run
 * through d3b_sparse_conv in channels-last layout.  n = B*H*W is also written to n_rows[0..1]. */
int d3b_rulebook_dense2d(int32_t batch, int32_t height, int32_t width, const int32_t ksize[2],
                         const int32_t padding[2], int32_t* nbr, uint32_t* tile_mask,
                         int32_t* n_rows, void* stream);

/* ========================================================================= *
 * 3b. Split-f16 ("FP16x3") convolutions: fp32-equivalent accuracy on the f16 tensor pipe, deterministic.
 *
 *     Activations are carried as TWO f16 planes of the same shape, hi = f16(x) and lo = f16(x - hi) (x = hi + lo
 *     to 22 significant bits, |x| < 65504); weights are split the same way after an exact power-of-two scaling
 *     2^w_exp (undone by `acc_scale` = 2^-w_exp in the epilogue).  The kernels compute hi.hi + hi.lo + lo.hi with
 *     fp32 accumulation.  A result outside the f16 range cannot be carried: the kernels then OR 1 into `*overflow`
 *     (device int, may be NULL) and the caller must fall back to the tf32 path -- nothing saturates silently.
 *     Same reference call sites as section 3 (scn.py:106-157,323-355; necks/rpn.py:82-159; mg_head.py:198-230).
 *
 *     Single-pass FP16 (opt-in, not fp32-equivalent): a NULL lo plane selects it.  An activation is then the hi plane
 *     alone, hi = f16(x), and the kernels compute hi.hi only (one MMA per product) from the same packed weight image;
 *     the f16-range guard is the same.  The lo pointers of one call must all be given or all be NULL:
 *       d3b_sparse_conv16 / d3b_bev_conv16: in_lo, out_lo (when out_hi is given) and residual_lo (when residual_hi is
 *       given) -- e.g. in_lo set with out_lo NULL returns D3B_ERR_INVALID_ARG, with a message, before any CUDA call;
 *       d3b_sparse_to_bev16: in_lo (with plane rows) and out_lo; d3b_split16 / d3b_merge16: lo.
 *     A lo plane without its hi plane is rejected the same way.
 * ========================================================================= */
typedef struct {
  int32_t c_in, c_out, k_vol;
  const void* in_hi;             /* f16 [rows, c_in] (c_in % 8 == 0)                                          */
  const void* in_lo;
  const float* in_f32;           /* first layer only: fp32 rows [rows, c_in <= 16] (then in_hi = in_lo = NULL)  */
  const float* weight;           /* fp32 [k_vol, c_in, c_out]: used by the fp32-input first layer only          */
  const void* weight_packed;     /* d3b_conv16_pack_weight image                                                */
  float acc_scale;               /* 2^-w_exp (1 for the fp32-input layer)                                       */
  const float* bias;             /* [c_out] or NULL                                                             */
  const float* scale;            /* folded BatchNorm [c_out] or NULL (with shift)                               */
  const float* shift;
  const void* residual_hi;       /* f16 [rows, c_out] planes added before the ReLU, or NULL                     */
  const void* residual_lo;
  int32_t relu;
  void* out_hi;                  /* f16 [rows, c_out] planes (out_lo NULL: single-pass FP16, see above)         */
  void* out_lo;
  float* out_f32;                /* optional fp32 copy of the result [rows, c_out]                              */
  int32_t* overflow;             /* device flag, may be NULL                                                    */
  int32_t in_f32_ld;             /* row stride of in_f32 in floats (>= c_in), 0 = c_in: the first layer can read the
                                    leading c_in columns of wider rows, e.g. 3 of the voxelizer's 4-column means    */
} d3b_conv16_params;

/* Size in halves / fill of the f16 weight image: packed[k][kb][hi|lo][n][64 channels, 128B-swizzled].
 * 0 if the shape is not built (c_out in {16,32,64,128}, c_in <= 512, k_vol <= 32). */
size_t d3b_conv16_packed_weight_halves(int32_t c_in, int32_t c_out, int32_t k_vol);
int d3b_conv16_pack_weight(const float* weight_dev, int32_t c_in, int32_t c_out, int32_t k_vol, int32_t w_exp,
                           void* packed_dev, void* stream);

/* Output-stationary sparse convolution over a rulebook (nbr / tile_mask as in d3b_sparse_conv): no atomics, fixed
 * summation order -> bit-identical results run to run. */
int d3b_sparse_conv16(const int32_t* nbr, const uint32_t* tile_mask, const int32_t* n_out, int32_t out_cap,
                      const d3b_conv16_params* p, void* stream);

/* fp32 <-> plane conversions (API boundaries) and the sparse -> dense NHWC scatter on planes
 * (channel = c*D + z, as d3b_sparse_to_bev_rows; rows given as planes OR as fp32).  Every launch that splits fp32
 * values into planes ORs 1 into `*overflow` (may be NULL) when one of them has |x| >= 65504 or is NaN: d3b_split16
 * and d3b_sparse_to_bev16 with fp32 rows.  Plane rows are copied as they are (their writer checked them). */
int d3b_split16(const float* x, int64_t n, void* hi, void* lo, int32_t* overflow, void* stream);
int d3b_merge16(const void* hi, const void* lo, int64_t n, float* x, void* stream);
int d3b_sparse_to_bev16(const void* in_hi, const void* in_lo, const float* in_f32, const int32_t* coors,
                        const int32_t* n_rows, int32_t row_cap, int32_t channels, const int32_t spatial[3],
                        int32_t batch, void* out_hi, void* out_lo, int32_t* overflow, void* stream);

/* Dense NHWC convolution on planes [batch, h_in, w_in, c_in] through TMA tensor maps: 3x3 (stride 1 or 2) or 1x1
 * with zero padding `pad` (<= ksize / 2 + 1), or ksize == stride == s for s in {2, 3, 4} with pad 0 (the Conv2d
 * deblock of an up-sampling stride 1/s, necks/rpn.py:96-102; trailing rows / columns of an h_in or w_in that is not
 * a multiple of s are not read, as in torch); other (ksize, stride, pad) return D3B_ERR_INVALID_ARG.
 * `groups` weight blocks of c_out (32/64/128) channels each in one launch:
 *   group g -> channel block cg = g % cgroups, sub-pixel ug = g / cgroups, (uy, ux) = (ug / up, ug % up);
 *   conv output pixel (y, x) of group g is written to pixel (y*up + uy, x*up + ux) of the output tensor
 *   [batch, h_out*up, w_out*up, out_channels], channels [out_c0 + cg*c_out, out_c0 + (cg+1)*c_out).
 * cgroups > 1 tiles a wide C_out; up > 1 (with ksize 1) is ConvTranspose2d(kernel = stride = up)
 * (necks/rpn.py:108-122).  weight_packed = the groups' d3b_conv16_pack_weight images back to back;
 * bias / scale / shift hold groups * c_out entries, group-major. */
typedef struct {
  int32_t batch, h_in, w_in, c_in;
  int32_t c_out;                 /* per group */
  int32_t ksize, stride, pad;
  int32_t groups, cgroups, up;
  const void* in_hi;
  const void* in_lo;
  const void* weight_packed;
  float acc_scale;
  const float* bias;
  const float* scale;
  const float* shift;
  int32_t relu;
  int32_t out_channels, out_c0;
  void* out_hi;
  void* out_lo;
  float* out_f32;
  int32_t* overflow;
} d3b_bev16_params;

int d3b_bev_conv16(const d3b_bev16_params* p, void* stream);

/* A chain of n_layers (1..8) 3x3 stride-1 layers over one grid, run as ONE persistent launch that hands out the tiles
 * of every layer in order: a tile of layer k starts as soon as the <= 9 tiles of layer k - 1 it reads are written,
 * so the tail of one layer overlaps the head of the next.  Every layer must be one d3b_bev_conv16 would run on the
 * pipelined kernel (ksize 3, stride 1, pad 1, c_out 128 per group, c_in % 64 == 0, up 1) and write whole output planes
 * (out_hi set, out_c0 0, out_channels = cgroups * 128); layer k's in_hi / in_lo must be layer k - 1's out_hi / out_lo,
 * no layer may write its own input, and all layers share layer 0's overflow flag.  Layer k may write the planes layer
 * k - 1 read (the ping-pong of an RPN block).  `workspace` holds the launch's tile counters: at least
 * d3b_bev_conv16_chain_workspace_bytes(batch, h_in, w_in, n_layers) bytes, zero before the first call; every call
 * leaves it zero again, so a captured graph replays with no host action.  Results are bit-identical to the layers run
 * one by one.  Under d3b_set_bev_variant(0) the layers run one by one through d3b_bev_conv16.  Argument errors
 * return D3B_ERR_INVALID_ARG before any CUDA call. */
int64_t d3b_bev_conv16_chain_workspace_bytes(int32_t batch, int32_t h, int32_t w, int32_t n_layers);
int d3b_bev_conv16_chain(const d3b_bev16_params* layers, int32_t n_layers, void* workspace, int64_t workspace_bytes,
                         void* stream);

/* ========================================================================= *
 * 4. Rotated-box BEV IoU / NMS
 * ========================================================================= */
#define D3B_BOX_XYXYR 0   /* [x1,y1,x2,y2,ry]: det3d/ops/iou3d/src/iou3d_kernel.cu:108-221 */
#define D3B_BOX_XYWLR 1   /* [cx,cy,w,l,r]  : det3d/ops/nms/nms_cpu.py:34-45 + nms_cpu.h:73-169 */
#define D3B_BOX_XYWLR_RRPN 2 /* [cx,cy,w,l,r]: numba RRPN routine, det3d/ops/nms/nms_gpu.py:180-470 */

/* Pairwise rotated IoU (mode 0) or overlap area (mode 1) of [x1,y1,x2,y2,ry] boxes, out [na, nb].
 * replaces boxes_iou_bev_gpu / boxes_overlap_bev_gpu, det3d/ops/iou3d/src/iou3d.cpp:31-71
 * mode 2: the overlap D3B_BOX_XYWLR NMS thresholds, for [cx,cy,w,l,r] boxes (rotate_nms_cc): 0 when the fp32
 *         IoU of the axis-aligned hulls is <= 0, when the intersection area is not > 0 or the union is not > 0,
 *         else (float)(inter / union).  The same device function makes the NMS decisions (suppress when
 *         out >= thresh), so the matrix shows exactly the values the NMS compares.
 * Any other mode is an invalid argument. */
int d3b_boxes_iou_bev(const float* boxes_a, int32_t na, const float* boxes_b, int32_t nb,
                      int32_t mode, float* out, void* stream);

/* RRPN rotated IoU matrix, out[n, k] = f(query[k], boxes[n]); criterion -1: IoU, 0: inter / area(query),
 * 1: inter / area(box), other: intersection area.  replaces rotate_iou_gpu / rotate_iou_gpu_eval,
 * det3d/ops/nms/nms_gpu.py:499-669 (numba.cuda). */
int d3b_rotate_iou_rrpn(const float* boxes, int32_t n, const float* query_boxes, int32_t k,
                        int32_t criterion, float* out, void* stream);

size_t d3b_nms_workspace_bytes(int32_t n_cap);

/* Greedy NMS over boxes already sorted by descending score.
 * fmt = D3B_BOX_XYXYR: suppress when iou >  thresh   (iou3d.cpp:73-120, nms_gpu)
 * fmt = D3B_BOX_XYWLR: suppress when iou >= thresh and the axis-aligned hulls
 *                      overlap                         (nms_cpu.h:73-169)
 * fmt = D3B_BOX_XYWLR_RRPN: suppress when iou > thresh (rotate_nms_gpu, nms_gpu.py:411-496)
 * n_boxes may be a device count (n_boxes_dev != NULL, bounded by n_cap).
 * keep_idx [min(n_cap, max_keep)] i64 device receives kept positions in
 * ascending order, keep_count [1] i32 device their number (<= max_keep). */
int d3b_rotate_nms(const float* boxes, int32_t n_cap, const int32_t* n_boxes_dev, int32_t fmt,
                   float thresh, int32_t max_keep, int64_t* keep_idx, int32_t* keep_count,
                   void* workspace, size_t workspace_bytes, void* stream);

/* Axis-aligned variants, boxes [n,5] = (x1, y1, x2, y2, ignored), suppress when iou > thresh.
 * mode = D3B_AA_IOU3D: plain extents       -- nms_normal_gpu, iou3d.cpp:123-170 / iou3d_kernel.cu:295-303
 * mode = D3B_AA_PIXEL: "+1" pixel extents  -- numba nms_gpu behind box_torch_ops.nms
 *                      (det3d/ops/nms/nms_gpu.py:22-33,129-166, core/bbox/box_torch_ops.py:506-525) */
#define D3B_AA_IOU3D 0
#define D3B_AA_PIXEL 1
int d3b_normal_nms(const float* boxes, int32_t n_cap, const int32_t* n_boxes_dev, int32_t mode, float thresh,
                   int32_t max_keep, int64_t* keep_idx, int32_t* keep_count, void* workspace,
                   size_t workspace_bytes, void* stream);

/* ========================================================================= *
 * 5. Detection post-processing of one task head (whole batch, fixed shapes)
 *    replaces MultiGroupHead.get_task_detections, det3d/models/bbox_heads/mg_head.py:805-1085
 *    (use_multi_class_nms = False), incl. second_box_decode (core/bbox/box_torch_ops.py:80-148)
 *    and rotate_nms (:528-549).  Head tensors are addressed as rows: element (b, cell, j) lives
 *    at ptr[(b*hw + cell) * row_stride + col0 + j], so both NHWC-permuted tensors and column
 *    slices of a fused [B*H*W, 32] row buffer work without a copy.
 * ========================================================================= */
typedef struct {
  const float* cls;  int32_t cls_row_stride, cls_col0;   /* logits, na*n_cls per cell          */
  const float* box;  int32_t box_row_stride, box_col0;   /* encodings, na*code per cell        */
  const float* dir;  int32_t dir_row_stride, dir_col0;   /* direction logits, na*2, or NULL     */
  const float* anchors;                                   /* [hw*na, nd], shared by the batch    */
  int32_t batch, hw, na, n_cls, code, nd;
  int32_t vec_encode, smooth_dim, norm_velo;              /* box coder flags                     */
  int32_t use_rotate_nms, pre_max, post_max;              /* test_cfg.nms                        */
  float nms_iou_threshold, score_threshold, direction_offset;
  float post_center_range[6]; int32_t has_range;
  int32_t label_offset;                                   /* added to the class index            */
} d3b_predict_params;

size_t d3b_predict_workspace_bytes(const d3b_predict_params* p);

/* packed [batch, packed_rows_per_sample, nd+3] f32: rows [row_offset, row_offset+post_max) of every
 * sample receive box[nd], score, label, valid(0/1); rows beyond the kept count are zero.
 * keep_counts [batch] i32 (optional) = boxes surviving NMS (before the range mask). */
int d3b_predict_task(const d3b_predict_params* p, float* packed, int32_t packed_rows_per_sample,
                     int32_t row_offset, int32_t* keep_counts, void* workspace,
                     size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DET3D_B200_H_ */
