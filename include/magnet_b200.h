/*
 * magnet_b200.h — C ABI of the H100-native multi-view matching hot path of MaGNet.
 *
 * The reference (baegwangbin/MaGNet) has no FFI layer: its boundary is two Python
 * module-level functions and two inlined blocks (SURVEY §8 b).  Every entry point
 * below names the reference interface it replaces.  A maintainer binds these with
 * ctypes / cffi / pybind (see INTEGRATION.md); magnet_b200/_lib.py is such a binding.
 *
 * Conventions
 *   - plain C, no torch types; every pointer is a DEVICE pointer unless the field says
 *     "host"; all tensors are fp32, dense, in the layout stated per field (the one exception:
 *     the fp16 / bf16 input of magnet_repack_half16);
 *   - caller owns all memory; no entry point allocates, frees or synchronises; every
 *     launch goes to the cudaStream_t passed as `stream` (NULL = legacy default
 *     stream), so calls are CUDA-graph capturable;
 *   - re-entrant and stateless (one-time cudaFuncSetAttribute calls are idempotent);
 *   - return value: MAGNET_OK (0) or a negative magnet_status; never throws.
 */
#ifndef MAGNET_B200_H_
#define MAGNET_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MAGNET_ABI_VERSION 4
#define MAGNET_MAX_PLANES 256   /* max depth hypotheses / planes per call (D) */

typedef enum magnet_status {
  MAGNET_OK = 0,
  MAGNET_ERR_NULL = -1,        /* a required pointer is NULL */
  MAGNET_ERR_SHAPE = -2,       /* a dimension is <= 0 or inconsistent */
  MAGNET_ERR_UNSUPPORTED = -3, /* C, D, layout or variant not supported by this build */
  MAGNET_ERR_CUDA = -4,        /* a CUDA runtime call failed (see magnet_last_cuda_error) */
  MAGNET_ERR_ALIGN = -5        /* a pointer violates the required 16-byte alignment */
} magnet_status;

/* Where the per-pixel depth hypotheses come from. */
typedef enum magnet_depth_mode {
  MAGNET_DEPTH_VOLUME = 0, /* read d_volume (B,D,H,W): drop-in for est_costvolume_CW         */
  MAGNET_DEPTH_GAUSS = 1,  /* d_j = mu + sigma*k_j from ref_gmm + k: sampler fused            */
  MAGNET_DEPTH_PLANES = 2  /* d_j = k_j for every pixel: fronto-parallel planes (est_costvolume_F) */
} magnet_depth_mode;

/* Memory layout of the source-view feature maps. */
typedef enum magnet_src_layout {
  MAGNET_SRC_NCHW = 0,   /* (V*B, C, H, W), the reference layout                               */
  MAGNET_SRC_TILED32 = 1, /* (V*B, H, ceil(W/32), C/4, 32, 4): per row, tiles of 32 pixels; inside a tile
                            the C/4 channel quads are 512 B apart and the 32 pixels of one quad are
                            contiguous (see magnet_repack_tiled32_f32).  Pixels x >= W are padding. */
  MAGNET_SRC_PIXC = 2,    /* (V*B, H, W, C+4): pixel-major, per pixel the C channels followed by the source
                            Gaussian (mu, sigma) and two zeros (see magnet_repack_pixc_f32): the layout the
                            TMA-staged CUDA-core kernel fetches its windows from.  With this layout
                            magnet_cost_args.src_gmm is ignored (the Gaussians travel inside src_feat). */
  MAGNET_SRC_SPLIT16 = 3, /* tensor-core layout (C == 64): a 256-byte header (power-of-two scale s), two fp16 planes
                            (V*B, 2, H, W, 64) with x*s = hi + lo, and a (V*B, H, W+1, 4) table whose entry x+1 holds (mu, sigma) of
                            pixel x and of pixel x+1 (zeros outside the row); see
                            magnet_repack_split16_f32 / magnet_split16_bytes.  With this layout ref_feat must ALSO
                            point to a split buffer (of the B reference feature maps, Gaussians NULL) and src_gmm is
                            ignored. */
  MAGNET_SRC_HALF16 = 4   /* tensor-core layout for fp16 / bf16 feature maps (C == 64): SPLIT16's header and table around
                            ONE fp16 plane (V*B, 1, H, W, 64) holding fp16(x*s), s from the same rule (x*s is then
                            itself an fp16 number; DESIGN §3.7); see magnet_repack_half16 / magnet_half16_bytes.
                            Accepted wherever SPLIT16 is, with the same rules: ref_feat must ALSO point to a HALF16
                            buffer, src_gmm is ignored.  The ABI cannot tell the two kinds of buffer apart: the caller
                            names the right one. */
} magnet_src_layout;

/* Element type of the input of magnet_repack_half16. */
typedef enum magnet_dtype {
  MAGNET_DTYPE_F16 = 0,   /* IEEE binary16 */
  MAGNET_DTYPE_BF16 = 1   /* bfloat16 */
} magnet_dtype;

/* Kernel selection (for parity cross-checks and profiling). */
typedef enum magnet_variant {
  MAGNET_VARIANT_AUTO = 0,   /* production choice: MMA for MAGNET_SRC_SPLIT16 / HALF16, TMA for MAGNET_SRC_PIXC, CELLS for
                                MAGNET_SRC_TILED32, DIRECT otherwise                           */
  MAGNET_VARIANT_DIRECT = 1, /* one thread per output, 4 taps x C channels per hypothesis,
                                reference operation order, fp64 view accumulation             */
  MAGNET_VARIANT_CELLS = 2,  /* tap-sharing kernel: per-lane bilinear-cell records             */
  MAGNET_VARIANT_CELLS_NOREUSE = 3, /* diagnostic: as CELLS, but every cell gathers all 4 taps
                                       (MAGNET_DEPTH_GAUSS only)                               */
  MAGNET_VARIANT_TMA = 4,    /* CUDA-core tap-sharing kernel, 4 lanes per pixel, the CTA's source window
                                staged in shared memory by TMA (MAGNET_SRC_PIXC only)          */
  MAGNET_VARIANT_MMA = 5     /* tensor-core kernel: all (reference pixel, window cell) channel dot products of an
                                8x8 tile by wgmma tensor-core MMA (MAGNET_SRC_SPLIT16 / HALF16 only) */
} magnet_variant;

/* Per (batch element, view) camera constants, 16 floats, produced by magnet_pack_cameras_f32.
 * index = b*V + v.  Replaces the per-pair matmuls at homography.py:98-102. */
typedef struct magnet_camera {
  float valid;  /* 1.0f when is_valid[b,v] == 1, else 0.0f (homography.py:97)                  */
  float a[3];   /* K_b * t_bv          ('term1_pix', homography.py:101)                        */
  float A[9];   /* K_b * R_bv row-major; A*ray = 'term2_pix' (homography.py:102).  Row 2 equals
                   R_bv[2,:] and a[2] equals t_bv[2], i.e. the z rows of 'term1_cam/term2_cam' */
  float pad[3];
} magnet_camera;

/*
 * Arguments of the fused warp + bilinear sample + consistency weight + view fusion kernel.
 * Replaces models/submodules/homography.py:79-161 (est_costvolume_CW + _compute_cost_CW) and,
 * with consistency == 0, homography.py:10-75 (est_costvolume_F + _compute_cost_F);
 * with depth_mode == MAGNET_DEPTH_GAUSS it also absorbs the sampler of models/MAGNET.py:154-156.
 */
typedef struct magnet_cost_args {
  int32_t B, V, D, C, H, W;
  int32_t depth_mode;      /* magnet_depth_mode                                                 */
  int32_t src_layout;      /* magnet_src_layout                                                 */
  int32_t consistency;     /* 1: CW weighting |z - mu~| < kappa*sigma~ ; 0: plain plane sweep   */
  int32_t softmax;         /* 1: softmax over the D planes after the 1/V mean (est_costvolume_F)*/
  int32_t variant;         /* magnet_variant                                                    */
  float kappa;             /* 'thres' of est_costvolume_CW (float(int))                         */
  const float* ref_feat;   /* (B, C, H, W) NCHW; a split buffer with MAGNET_SRC_SPLIT16           */
  const float* src_feat;   /* (V*B, ...) view-major, layout = src_layout                        */
  const float* src_gmm;    /* (V*B, 2, H, W) [mu, sigma]; required when consistency == 1        */
  const float* rays;       /* (B, 3, H*W) 'unit_ray_array_2D'                                   */
  const magnet_camera* cams; /* (B*V)                                                           */
  const float* d_volume;   /* (B, D, H, W); MAGNET_DEPTH_VOLUME only                            */
  const float* ref_gmm;    /* (B, 2, H, W) [mu, sigma]; MAGNET_DEPTH_GAUSS only                 */
  const float* k_host;     /* HOST pointer, D floats: k_j (GAUSS) or plane depths (PLANES)      */
  float* out;              /* (B, D, H, W)                                                      */
} magnet_cost_args;

int magnet_abi_version(void);
const char* magnet_strerror(int status);
/* Text of the last CUDA error seen by this library on the calling thread ("" if none). */
const char* magnet_last_cuda_error(void);
/* Number of kernels this library has launched so far in this process (all entry points). */
uint64_t magnet_launch_count(void);

/* Bytes of dynamic shared memory and threads per CTA the selected variant will use (for reports). */
int magnet_cost_launch_info(const magnet_cost_args* args, int* grid_ctas, int* block_threads, int* smem_bytes);

/* Cost volume, forward.  Replaces homography.est_costvolume_CW / est_costvolume_F (see above). */
int magnet_cost_volume_f32(const magnet_cost_args* args, void* stream);

/*
 * Cost volume, forward, with the source views read through a frame table (sequence evaluation, where consecutive
 * references share most of their neighbours: each distinct frame is repacked once).  Everything is as in
 * magnet_cost_volume_f32, except that args->src_feat (and args->src_gmm, and the Gaussians inside PIXC / SPLIT16 /
 * HALF16 buffers) hold n_src source images in any order, and view (b, v) reads image src_index[b*V + v] instead of
 * v*B + b.  The cameras stay per (b, v) and the reference operands per b.
 *   src_index: DEVICE int32 array (B, V), b*V + v order.  Every entry, also those of views with is_valid == 0, must lie
 *              in [0, n_src): the kernels do not check them (the Python layer does, on the host before any launch,
 *              or on the device with magnet_check_src_index while torch.compile traces).
 *   n_src:     images in src_feat, >= 1; a SPLIT16 / HALF16 buffer is magnet_split16_bytes(n_src, H, W) /
 *              magnet_half16_bytes(n_src, H, W) bytes.
 * MAGNET_ERR_NULL for a NULL src_index, MAGNET_ERR_SHAPE for n_src < 1, MAGNET_ERR_ALIGN for a misaligned src_index.
 * Forward only: the backward entry points read view-major buffers.
 */
int magnet_cost_volume_indexed_f32(const magnet_cost_args* args, const int32_t* src_index, int32_t n_src, void* stream);
/* magnet_cost_launch_info for magnet_cost_volume_indexed_f32 (the same kernels and grid; the arguments checked alike). */
int magnet_cost_indexed_launch_info(const magnet_cost_args* args, const int32_t* src_index, int32_t n_src,
                                    int* grid_ctas, int* block_threads, int* smem_bytes);

/* Element type of the frame table magnet_check_src_index reads. */
typedef enum magnet_index_dtype {
  MAGNET_INDEX_I32 = 0,   /* int32_t */
  MAGNET_INDEX_I64 = 1    /* int64_t, read as 64-bit: an entry >= 2^31 is out of range, never wrapped */
} magnet_index_dtype;

/*
 * The range check of a frame table on the device, for callers that cannot read the table back (a CUDA graph, a
 * torch.compile graph).  src_index: DEVICE (B, V) array, b*V + v order, of element type `dtype` (magnet_index_dtype).
 *   index_out: DEVICE int32 (B, V), the table magnet_cost_volume_indexed_f32 may read: each entry in [0, n_src) copied,
 *              every other entry replaced by 0.
 *   bad:       DEVICE int32 (B,), nonzero for each b with at least one entry outside [0, n_src) (views with
 *              is_valid == 0 count too), 0 otherwise.
 * One kernel launch, no allocation, no host synchronisation.  MAGNET_ERR_NULL for a NULL pointer, MAGNET_ERR_SHAPE for
 * B < 1, V < 1, n_src < 1 or B*V >= 2^31, MAGNET_ERR_UNSUPPORTED for an unknown dtype, MAGNET_ERR_ALIGN for a pointer
 * not aligned to its element size.
 */
int magnet_check_src_index(const void* src_index, int32_t dtype, int32_t B, int32_t V, int32_t n_src,
                           int32_t* index_out, int32_t* bad, void* stream);

/*
 * Backward of the plane-sweep volume (est_costvolume_F) w.r.t. both feature maps — what autograd derives for
 * homography.py:10-75 during F-Net training (train_FNet.py:95-114): through the softmax, the 1/V mean, the channel
 * dot product and grid_sample's bilinear gather (scatter-add into the source features).
 * Geometry fields of `fwd` as in the forward call (consistency must be 0, depth_mode MAGNET_DEPTH_PLANES); `fwd->out` is
 * ignored.  Two forms:
 *   - src_layout MAGNET_SRC_NCHW, C in {8,16,32,64}: ref_feat / src_feat are the NCHW feature maps (CUDA-core kernel);
 *   - src_layout MAGNET_SRC_SPLIT16, variant AUTO or MMA, C == 64, V <= 16: ref_feat / src_feat are the split buffers
 *     the forward read (tensor-core kernel: both gradients as GEMMs on the fp16 hi/lo planes).  MAGNET_SRC_HALF16 in
 *     the same way, on HALF16 buffers.
 * grad_src is accumulated with atomics in either form, so results are not bit-deterministic from run to run.
 */
typedef struct magnet_cost_f_bwd_args {
  const magnet_cost_args* fwd;
  const float* prob;      /* (B,D,H,W) forward output; used when fwd->softmax == 1                          */
  const float* grad_out;  /* (B,D,H,W) gradient w.r.t. the forward output                                   */
  float* workspace;       /* (B,D,H,W) scratch (gradient w.r.t. the pre-softmax scores)                     */
  float* grad_ref;        /* (B,C,H,W)   written                                                            */
  float* grad_src;        /* (V*B,C,H,W) NCHW, ACCUMULATED with atomics: the caller zeroes it               */
} magnet_cost_f_bwd_args;
int magnet_cost_volume_f_bwd_f32(const magnet_cost_f_bwd_args* args, void* stream);

/*
 * Backward of the cost volume with per-pixel depths (est_costvolume_CW, homography.py:79-161; consistency 0 or 1) w.r.t.
 * both feature maps and the depth hypotheses — what autograd derives for the reference, through the 1/V mean, the
 * consistency mask (piecewise constant: the source Gaussians get no gradient), the channel dot product and
 * grid_sample's bilinear gather, including its derivative in the sample position.
 * `fwd` is the forward call (depth_mode MAGNET_DEPTH_VOLUME or MAGNET_DEPTH_GAUSS); its src_layout and variant name the
 * forward kernel, whose consistency mask the backward reproduces bit for bit.  Two forms:
 *   - src_layout MAGNET_SRC_SPLIT16 or MAGNET_SRC_HALF16, variant AUTO or MMA (C == 64, V <= 16): fwd->ref_feat /
 *     fwd->src_feat are the SPLIT16 / HALF16 buffers the forward read; grad_ref and grad_src come from the tensor-core kernel (two GEMMs on the fp16 hi/lo
 *     planes).  The NCHW maps below are needed only for grad_depth.  With fwd->ref_feat and fwd->src_feat both NULL,
 *     every gradient comes from the CUDA-core kernel on the NCHW maps, still with the tensor-core forward's mask;
 *   - variant MAGNET_VARIANT_DIRECT (src_layout NCHW or TILED32): everything from the NCHW maps below, C <= 64.
 * Other forward kernels (CELLS, TMA) are rejected with MAGNET_ERR_UNSUPPORTED.  The depth gradient always comes from
 * the CUDA-core kernel; fwd->out is ignored.  Each of grad_ref, grad_src and grad_depth may be NULL when it is not wanted.
 * grad_src is accumulated with atomics, so results are not bit-deterministic from run to run.
 */
typedef struct magnet_cost_bwd_args {
  const magnet_cost_args* fwd;
  const float* ref_feat;  /* (B,C,H,W) NCHW                                                                       */
  const float* src_feat;  /* (V*B,C,H,W) NCHW, view-major                                                         */
  const float* src_gmm;   /* (V*B,2,H,W) [mu, sigma]; required when fwd->consistency == 1                         */
  const float* grad_out;  /* (B,D,H,W) gradient w.r.t. the forward output                                         */
  float* workspace;       /* (B,D,H,W) scratch                                                                    */
  float* grad_ref;        /* (B,C,H,W)   written, or NULL                                                         */
  float* grad_src;        /* (V*B,C,H,W) ACCUMULATED with atomics (the caller zeroes it), or NULL                 */
  float* grad_depth;      /* VOLUME: (B,D,H,W) w.r.t. d_volume; GAUSS: (B,2,H,W) w.r.t. ref_gmm; written, or NULL */
} magnet_cost_bwd_args;
int magnet_cost_volume_bwd_f32(const magnet_cost_bwd_args* args, void* stream);

/*
 * Gradients of either cost volume w.r.t. the cameras (DESIGN §3.11) — what autograd derives for the reference's
 * term1_pix = K t and term2_pix = (K R) Ray through grid_sample's position derivative; the consistency mask passes none.
 * `fwd` is the forward call:
 *   - depth_mode MAGNET_DEPTH_VOLUME or MAGNET_DEPTH_GAUSS, consistency 0 or 1, softmax 0: src_layout and variant name the
 *     forward kernel whose mask is reproduced, as for magnet_cost_volume_bwd_f32 (SPLIT16 / HALF16 with AUTO or MMA, or
 *     DIRECT with NCHW / TILED32; CELLS and TMA forwards are rejected);
 *   - depth_mode MAGNET_DEPTH_PLANES, consistency 0, softmax 0 or 1 (the F volume): any forward kernel; the positions
 *     are those of the tensor-core forward.
 * fwd->ref_feat / src_feat / out are ignored: the kernel reads the NCHW fp32 maps below.  Feature gradients are not
 * computed here (magnet_cost_volume_bwd_f32 / magnet_cost_volume_f_bwd_f32).  Requires C <= 64.  No atomics: the
 * results are bit-identical from run to run.  Three launches, no allocation, no synchronisation.
 */
typedef struct magnet_cost_geom_bwd_args {
  const magnet_cost_args* fwd;
  const float* ref_feat;  /* (B,C,H,W) NCHW                                                                       */
  const float* src_feat;  /* (V*B,C,H,W) NCHW, view-major                                                         */
  const float* src_gmm;   /* (V*B,2,H,W) [mu, sigma]; required when fwd->consistency == 1                         */
  const float* grad_out;  /* (B,D,H,W) gradient w.r.t. the forward output                                         */
  const float* prob;      /* (B,D,H,W) forward output; required when fwd->softmax == 1                            */
  float* score;           /* (B,D,H,W) scratch                                                                    */
  void* workspace;        /* magnet_cost_geom_workspace_bytes(B, V, H, W) bytes, 16-byte aligned, scratch         */
  float* grad_cams;       /* (B*V, 12) written: d/dA (K R, row-major), then d/da (K t); zero for an invalid view   */
  float* grad_rays;       /* (B,3,H*W) written, or NULL                                                           */
  float* grad_depth;      /* VOLUME (B,D,H,W) / GAUSS (B,2,H,W) written, or NULL; must be NULL for PLANES         */
} magnet_cost_geom_bwd_args;
/* Bytes of the workspace of magnet_cost_volume_geom_bwd_f32 (0 for a non-positive dimension). */
size_t magnet_cost_geom_workspace_bytes(int32_t B, int32_t V, int32_t H, int32_t W);
int magnet_cost_volume_geom_bwd_f32(const magnet_cost_geom_bwd_args* args, void* stream);

/*
 * Camera constants.  Replaces homography.py:89,98-102 (IntM/R/t products, done there per pair per
 * iteration).  intM (B,3,3) dense; R and t are addressed with element strides so that the
 * non-contiguous views nghbr_poses[:,:,:3,:3] / [:,:,:3,3] of MAGNET.py:147-148 can be passed as is:
 *   R[b,v,i,j] = R[b*r_sb + v*r_sv + i*r_si + j*r_sj],  t[b,v,i] = t[b*t_sb + v*t_sv + i*t_si].
 * is_valid (B,V) int32 on the device.
 */
int magnet_pack_cameras_f32(const float* intM, const float* R, int64_t r_sb, int64_t r_sv, int64_t r_si,
                            int64_t r_sj, const float* t, int64_t t_sb, int64_t t_sv, int64_t t_si,
                            const int32_t* is_valid, int32_t B, int32_t V, magnet_camera* cams_out,
                            void* stream);

/* Source repack (N, C, H, W) features [+ (N, 2, H, W) Gaussians, may be NULL -> zeros] -> MAGNET_SRC_PIXC
 * (N, H, W, C+4); C in {16, 32, 64}, dst 16-byte aligned.  Once per forward (the features do not change across the
 * N_iter iterations, MAGNET.py:150-169). */
int magnet_repack_pixc_f32(const float* src_nchw, const float* src_gmm, float* dst, int32_t N, int32_t C, int32_t H,
                           int32_t W, void* stream);

/* Feature split (N, 64, H, W) features [+ (N, 2, H, W) Gaussians, may be NULL -> zeros] -> MAGNET_SRC_SPLIT16 buffer of
 * magnet_split16_bytes(N, H, W) bytes; src and dst 16-byte aligned.  Three stream operations (header memset, max |x|
 * reduction, split).  Once per forward for the source views and once for the reference features. */
size_t magnet_split16_bytes(int32_t N, int32_t H, int32_t W);
int magnet_repack_split16_f32(const float* src_nchw, const float* src_gmm, void* dst, int32_t N, int32_t C, int32_t H,
                              int32_t W, void* stream);

/* Half-precision feature maps (N, 64, H, W) of element type `dtype` (magnet_dtype) [+ fp32 (N, 2, H, W) Gaussians, may
 * be NULL -> zeros] -> MAGNET_SRC_HALF16 buffer of magnet_half16_bytes(N, H, W) bytes; src and dst 16-byte aligned.
 * The scale and the table are those magnet_repack_split16_f32 gives for the fp32 upcast of src, the plane is its hi
 * plane.  C != 64 or an unknown dtype -> MAGNET_ERR_UNSUPPORTED.  Three stream operations, as the fp32 split. */
size_t magnet_half16_bytes(int32_t N, int32_t H, int32_t W);
int magnet_repack_half16(const void* src_nchw, int32_t dtype, const float* src_gmm, void* dst, int32_t N, int32_t C,
                         int32_t H, int32_t W, void* stream);

/* Source-feature repack (N, C, H, W) -> MAGNET_SRC_TILED32 (N, H, ceil(W/32), C/4, 32, 4);
 * C % 4 == 0, dst 16-byte aligned, padding pixels are written as zeros. */
int magnet_repack_tiled32_f32(const float* src_nchw, float* dst, int32_t N, int32_t C, int32_t H, int32_t W,
                            void* stream);

/*
 * Depth-candidate sampler alone.  Replaces models/MAGNET.py:154-156:
 *   d_volume[b,j,y,x] = mu[b,y,x] + sigma[b,y,x] * k_j   (separate multiply and add).
 * gmm (B,2,H,W); k_host: HOST pointer, D floats; d_volume (B,D,H,W).
 */
int magnet_sample_depths_f32(const float* gmm, const float* k_host, int32_t B, int32_t D, int32_t HW,
                             float* d_volume, void* stream);

/*
 * Gaussian update, forward.  Replaces models/MAGNET.py:60,65-69 (inside GNET.forward):
 *   mu' = mu0 + mu1*sigma0 ; sigma' = (elu(sigma1) + 1 + 1e-10) * sigma0.
 * d_output (B,2,H,W) = G-Net raw output (mu1, sigma1); ref_gmm (B,2,H,W); out (B,2,H,W).
 */
int magnet_gaussian_update_fwd_f32(const float* d_output, const float* ref_gmm, int32_t B, int32_t HW,
                                   float* out, void* stream);
/* Backward of the update w.r.t. d_output (ref_gmm is detached in the reference, MAGNET.py:168):
 *   g_mu1 = g_mu' * sigma0 ; g_sigma1 = g_sigma' * sigma0 * (sigma1 > 0 ? 1 : exp(sigma1)). */
int magnet_gaussian_update_bwd_f32(const float* grad_out, const float* d_output, const float* ref_gmm,
                                   int32_t B, int32_t HW, float* grad_d_output, void* stream);

/*
 * G-Net head of inference, fused — replaces one iteration's G-Net and update of models/MAGNET.py:167-168 when the
 * x_d3 half of the first convolution is hoisted out of the loop (GNET.invariant_part):
 *   h0 = ReLU(conv3x3(cost, W0[:, :D]) + invariant),  h1 = ReLU(W1 h0 + b1),  h2 = ReLU(W2 h1 + b2),
 *   (mu1, sigma1) = W3 h2 + b3,  then the Gaussian update of magnet_gaussian_update_fwd_f32 on prev_gmm.
 * One kernel on the fp16 tensor cores with fp32 accuracy (SPLIT16 products, DESIGN §3.8); no 128-channel map is
 * written.  Forward only (inference); no atomics, so results are bit-identical from run to run.
 *
 * magnet_gnet_pack_weights_f32 writes the weights in the kernel's layout into `packed` (magnet_gnet_weights_bytes(D)
 * bytes, 16-byte aligned): w0_cost (128, D, 3, 3) dense = the cost-volume slice of the first convolution's weight,
 * w1 / w2 (128, 128), b1 / b2 (128), w3 (2, 128), b3 (2).  Two kernels; once per forward (the weights do not change
 * across the iterations).  magnet_gnet_weights_bytes returns 0 for D outside 1..MAGNET_MAX_PLANES.
 *
 * magnet_gnet_update_f32: a memset of scratch, the cost volume's max |x| and the fused kernel.
 * D > MAGNET_MAX_PLANES -> MAGNET_ERR_UNSUPPORTED; cost, invariant and packed_weights 16-byte aligned.
 */
#define MAGNET_HIDDEN_CHANNELS 128
#define MAGNET_GNET_SCRATCH_BYTES 16
typedef struct magnet_gnet_args {
  int32_t B, D, H, W;
  const float* cost;           /* (B, D, H, W) cost volume                                                      */
  const float* invariant;      /* (B, 128, H, W) = conv3x3(x_d3, W0[:, D:]) + b0                                */
  const void* packed_weights;  /* magnet_gnet_pack_weights_f32 output for this D                                */
  const float* prev_gmm;       /* (B, 2, H, W) [mu0, sigma0]                                                    */
  void* scratch;               /* MAGNET_GNET_SCRATCH_BYTES of device scratch (the cost volume's scale)         */
  float* out;                  /* (B, 2, H, W) updated [mu, sigma]; must not overlap the inputs                 */
} magnet_gnet_args;
size_t magnet_gnet_weights_bytes(int32_t D);
int magnet_gnet_pack_weights_f32(const float* w0_cost, const float* w1, const float* b1, const float* w2,
                                 const float* b2, const float* w3, const float* b3, int32_t D, void* packed,
                                 void* stream);
int magnet_gnet_update_f32(const magnet_gnet_args* args, void* stream);

/*
 * G-Net head of training, fused — replaces one iteration's G-Net and update of models/MAGNET.py:47-70,167-168 (split
 * data flow, detached cost volume) and their autograd backward into the head's weights (DESIGN §3.10).
 *
 * magnet_gnet_pack_train_weights_f32: the inference pack of magnet_gnet_pack_weights_f32 followed by W1^T and W2^T for
 * the backward, magnet_gnet_train_weights_bytes(D) bytes (0 for D outside 1..MAGNET_MAX_PLANES).  Two kernels.
 *
 * magnet_gnet_train_fwd_f32: the inference kernel's arithmetic (out is bit-identical to magnet_gnet_update_f32 on the
 * same inputs) plus stores of h0, h1, h2 (B,128,H,W each) and the raw (mu1, sigma1) (B,2,H,W) into `saved`
 * (magnet_gnet_saved_bytes(B,H,W) bytes).  Reads cost, invariant, packed_weights, prev_gmm; writes scratch, out, saved.
 *
 * magnet_gnet_bwd_f32: given grad_out = dL/d out, writes
 *   grad_invariant (B,128,H,W) = dL/d(pre-activation of h0), which is also the gradient of conv3x3(x_d3, W0[:, D:]) + b0;
 *   grad_w0_cost (128,D,3,3), grad_w1 / grad_w2 (128,128), grad_b1 / grad_b2 (128), grad_w3 (2,128), grad_b3 (2);
 *   grad_prev (B,2,H,W) when not NULL.
 * Weight / bias gradient pointers may be NULL (not computed).  No gradient into the cost volume.  Reads cost, prev_gmm,
 * packed_weights, saved (the forward's); uses `workspace` (magnet_gnet_bwd_workspace_bytes(B,D,H,W) bytes).  Weight
 * gradients are sums over pixels of per-CTA partials in a fixed order: bit-identical from run to run.
 * Both calls: D > MAGNET_MAX_PLANES -> MAGNET_ERR_UNSUPPORTED; B*H*W < 2^31; cost, invariant, packed_weights, saved and
 * workspace 16-byte aligned.
 */
typedef struct magnet_gnet_train_args {
  int32_t B, D, H, W;
  const float* cost;           /* (B, D, H, W) cost volume                                                      */
  const float* invariant;      /* (B, 128, H, W), forward only                                                  */
  const void* packed_weights;  /* magnet_gnet_pack_train_weights_f32 output for this D                          */
  const float* prev_gmm;       /* (B, 2, H, W) [mu0, sigma0]                                                    */
  void* scratch;               /* MAGNET_GNET_SCRATCH_BYTES, forward only                                       */
  float* out;                  /* (B, 2, H, W) updated [mu, sigma], forward only                                */
  float* saved;                /* magnet_gnet_saved_bytes(B, H, W): written by the forward, read by the backward  */
  const float* grad_out;       /* (B, 2, H, W), backward only                                                   */
  void* workspace;             /* magnet_gnet_bwd_workspace_bytes(B, D, H, W), backward only                    */
  float* grad_invariant;       /* (B, 128, H, W), backward only                                                 */
  float* grad_w0_cost;         /* (128, D, 3, 3) or NULL                                                        */
  float* grad_w1;              /* (128, 128) or NULL                                                            */
  float* grad_b1;              /* (128) or NULL                                                                 */
  float* grad_w2;              /* (128, 128) or NULL                                                            */
  float* grad_b2;              /* (128) or NULL                                                                 */
  float* grad_w3;              /* (2, 128) or NULL                                                              */
  float* grad_b3;              /* (2) or NULL                                                                   */
  float* grad_prev;            /* (B, 2, H, W) or NULL                                                          */
} magnet_gnet_train_args;
size_t magnet_gnet_train_weights_bytes(int32_t D);
size_t magnet_gnet_saved_bytes(int32_t B, int32_t H, int32_t W);
size_t magnet_gnet_bwd_workspace_bytes(int32_t B, int32_t D, int32_t H, int32_t W);
int magnet_gnet_pack_train_weights_f32(const float* w0_cost, const float* w1, const float* b1, const float* w2,
                                       const float* b2, const float* w3, const float* b3, int32_t D, void* packed,
                                       void* stream);
int magnet_gnet_train_fwd_f32(const magnet_gnet_train_args* args, void* stream);
int magnet_gnet_bwd_f32(const magnet_gnet_train_args* args, void* stream);

/*
 * Mask head and learned upsampling of inference, fused (DESIGN §3.12) — replaces, after the reference's first mask-head
 * convolution, the rest of mask_head (models/MAGNET.py:111-118) and upsample_depth_via_mask (MAGNET.py:15-27,172-173)
 * of every prediction:
 *   h0 = ReLU(pre0),  h1 = ReLU(W1 h0 + b1),  h2 = ReLU(W2 h1 + b2),  mask = W3 h2 + b3 (144 = 9 x k x k channels),
 *   out[p] = the convex upsampling of pred[p] by the mask, for p < P.
 * One kernel on the fp16 tensor cores with fp32 accuracy (SPLIT16 products, as the G-Net head); neither the hidden
 * maps nor the mask are written.  For equal mask logits the upsampling is bit-identical to
 * magnet_convex_upsample_fwd_f32.  Forward only; no atomics, so results are bit-identical from run to run.
 *
 * magnet_mask_pack_weights_f32 writes the weights in the kernel's layout into `packed` (magnet_mask_weights_bytes(4)
 * bytes, 16-byte aligned): w1 / w2 (128, 128), b1 / b2 (128), w3 (144, 128), b3 (144).  Two kernels.
 * magnet_mask_weights_bytes returns 0 for any k other than 4 (the only factor the kernel takes).
 *
 * magnet_mask_upsample_f32: one kernel.  P outside 1..MAGNET_MASK_MAX_PRED or k != 4 -> MAGNET_ERR_UNSUPPORTED;
 * B*H*W < 2^31; pre0, packed_weights and every pred / out pointer 16-byte aligned.
 */
#define MAGNET_MASK_MAX_PRED 8
typedef struct magnet_mask_upsample_args {
  int32_t P, B, H, W;        /* predictions, images, quarter-resolution size                                        */
  int32_t k;                 /* upsampling factor: 4                                                                */
  const float* pre0;         /* (B, 128, H, W) the first mask-head convolution's output, before its ReLU             */
  const void* packed_weights;/* magnet_mask_pack_weights_f32 output                                                 */
  const float* const* pred;  /* HOST array of P DEVICE pointers, each (B, 2, H, W) [mu, sigma]                      */
  float* const* out;         /* HOST array of P DEVICE pointers, each (B, 2, k*H, k*W); must not overlap the inputs  */
} magnet_mask_upsample_args;
size_t magnet_mask_weights_bytes(int32_t k);
int magnet_mask_pack_weights_f32(const float* w1, const float* b1, const float* w2, const float* b2, const float* w3,
                                 const float* b3, void* packed, void* stream);
int magnet_mask_upsample_f32(const magnet_mask_upsample_args* args, void* stream);

/*
 * Mask head, learned upsampling and Gaussian NLL of training, fused (DESIGN §3.13) — replaces, after the first mask-head
 * convolution, mask_head (models/MAGNET.py:111-118), upsample_depth_via_mask (MAGNET.py:15-27,172-173) and MagnetLoss
 * (utils/losses.py:34-50) of every prediction, and their autograd backward:
 *   loss = sum_p gamma_p mean_{gt_mask} nll(upsample(pred[p], mask)),  nll = (mu-gt)^2 / (2 var) + 0.5 log(var),
 *   var = max(sigma^2, 1e-10), mask as magnet_mask_upsample_f32 computes it (the logits are that kernel's bits).
 *
 * magnet_mask_pack_train_weights_f32: the inference pack of magnet_mask_pack_weights_f32 followed by W3^T, W2^T and W1^T
 * for the backward, magnet_mask_train_weights_bytes(4) bytes (0 for any other k).  Two kernels.
 *
 * magnet_mask_train_fwd_f32: partial[magnet_mask_train_partials(B,H,W) x P] receives, per 8x16 tile and prediction,
 * the tile's sum of nll over its supervised full-resolution pixels (row-major [tile][p]; the caller adds them in a
 * fixed order, divides by the number of supervised pixels and weights them).  pred_scale[p] (HOST) = gamma_p / count,
 * the scale of prediction p's gradient at unit upstream gradient.  With save_maps the forward stores h0, h1, h2 and the
 * logits' gradient into `saved` (needed by any weight or pre0 gradient); with pred_grad it accumulates the prediction
 * gradients there (needed by grad_pred).  `saved` holds magnet_mask_saved_bytes(P,B,H,W) bytes: the P prediction
 * gradients (B,2,H,W) first, then h0, h1, h2 (B,128,H,W) and the logits' gradient (B,128,H,W) + (B,16,H,W); a forward
 * without save_maps uses only the first 2*P*B*H*W floats, so the caller may pass a buffer of that size.  No upsampled
 * prediction and no mask is written.  Loss partials and saved maps are bit-identical from run to run; the prediction
 * gradients are sums of atomic adds.  One memset (pred_grad) and one kernel.
 *
 * magnet_mask_bwd_f32: given grad_scale = dL/d loss (a DEVICE float), writes grad_pre0 (B,128,H,W) = dL/d pre0,
 * grad_w1 / grad_w2 (128,128), grad_b1 / grad_b2 (128), grad_w3 (144,128), grad_b3 (144) and grad_pred[p] (B,2,H,W);
 * each may be NULL (not computed), as may grad_pred itself.  Each output is its unit-gradient value times grad_scale
 * (one rounding; exact for 1.0).  Weight gradients are fixed-order sums: bit-identical from run to run.  Uses
 * `workspace` (magnet_mask_bwd_workspace_bytes(B,H,W) bytes).  Asking for a weight or pre0 gradient after a forward
 * without save_maps, or for a prediction gradient after one without pred_grad, reads unwritten memory.
 *
 * Both calls: P outside 1..MAGNET_MASK_MAX_PRED or k != 4 -> MAGNET_ERR_UNSUPPORTED; B*H*W < 2^31; pre0,
 * packed_weights, saved, workspace and every pred pointer 16-byte aligned.
 */
typedef struct magnet_mask_train_args {
  int32_t P, B, H, W;        /* predictions, images, quarter-resolution size                                        */
  int32_t k;                 /* upsampling factor: 4                                                                */
  const float* pre0;         /* (B, 128, H, W) the first mask-head convolution's output, before its ReLU; forward    */
  const void* packed_weights;/* magnet_mask_pack_train_weights_f32 output                                           */
  const float* const* pred;  /* HOST array of P DEVICE pointers, each (B, 2, H, W) [mu, sigma]; forward             */
  const float* gt;           /* (B, 1, k*H, k*W) ground-truth depth; forward                                         */
  const uint8_t* gt_mask;    /* (B, 1, k*H, k*W) nonzero = supervised; forward                                       */
  const float* pred_scale;   /* HOST array of P floats: gamma_p / number of supervised pixels; forward              */
  int32_t save_maps;         /* forward: nonzero = store what the weight and pre0 gradients need                     */
  int32_t pred_grad;         /* forward: nonzero = accumulate the prediction gradients                               */
  float* partial;            /* forward: magnet_mask_train_partials(B, H, W) x P floats                              */
  float* saved;              /* magnet_mask_saved_bytes(P, B, H, W): written by the forward, read by the backward    */
  const float* grad_scale;   /* DEVICE float, the loss's upstream gradient; backward                                */
  void* workspace;           /* magnet_mask_bwd_workspace_bytes(B, H, W); backward                                  */
  float* grad_pre0;          /* (B, 128, H, W) or NULL                                                              */
  float* grad_w1;            /* (128, 128) or NULL                                                                  */
  float* grad_b1;            /* (128) or NULL                                                                       */
  float* grad_w2;            /* (128, 128) or NULL                                                                  */
  float* grad_b2;            /* (128) or NULL                                                                       */
  float* grad_w3;            /* (144, 128) or NULL                                                                  */
  float* grad_b3;            /* (144) or NULL                                                                       */
  float* const* grad_pred;   /* HOST array of P DEVICE pointers (entries may be NULL), or NULL; backward            */
} magnet_mask_train_args;
size_t magnet_mask_train_weights_bytes(int32_t k);
size_t magnet_mask_saved_bytes(int32_t P, int32_t B, int32_t H, int32_t W);
size_t magnet_mask_bwd_workspace_bytes(int32_t B, int32_t H, int32_t W);
int magnet_mask_train_partials(int32_t B, int32_t H, int32_t W);
int magnet_mask_pack_train_weights_f32(const float* w1, const float* b1, const float* w2, const float* b2,
                                       const float* w3, const float* b3, void* packed, void* stream);
int magnet_mask_train_fwd_f32(const magnet_mask_train_args* args, void* stream);
/* magnet_mask_train_fwd_f32 with the P prediction scales read from the DEVICE array pred_scale (args->pred_scale is not
 * read) when the kernel runs, so that a captured CUDA graph takes them from memory.  Same arithmetic otherwise. */
int magnet_mask_train_fwd_dev_f32(const magnet_mask_train_args* args, const float* pred_scale, void* stream);
int magnet_mask_bwd_f32(const magnet_mask_train_args* args, void* stream);

/*
 * D-Net heads of inference, fused (DESIGN §3.15) — replace, after the reference's first depth-head and mask-head
 * convolutions, the rest of Decoder.depth_head / mask_head (models/submodules/D_dense_depth.py:148-160,187-192),
 * upsample_depth_via_mask (D_dense_depth.py:86-100) and DNET's activations (models/DNET.py:56-67):
 *   depth:    h0 = ReLU(pre_d),  h1 = ReLU(W1 h0 + b1),  [mu, v] = W2 h1 + b2 (2 channels);
 *   upsample: g0 = ReLU(pre_m),  g1 = ReLU(M1 g0 + c1),  mask = M3 g1 + c3 (144 = 9 x k x k channels),
 *             [mu, v'] = convex upsampling of the raw [mu, v] by the mask,  var = (elu(v') + 1) + 1e-10.
 * The 128 -> 128 layers and the 128 -> 144 layer run on the fp16 tensor cores with fp32 accuracy (SPLIT16, as the G-Net
 * and mask heads), the 128 -> 2 layer on the CUDA cores; no hidden map and no mask is written.  elu is x <= 0 ?
 * expm1f(x) : x and every add is one fp32 rounding, in torch's order.  Forward only; no atomics, so results are
 * bit-identical from run to run.
 *
 * magnet_dnet_pack_weights_f32 writes both heads in the kernels' layout into `packed` (magnet_dnet_weights_bytes(k)
 * bytes, 16-byte aligned): depth head d_w1 (128, 128), d_b1 (128), d_w2 (2, 128), d_b2 (2); with k == 4 also the mask
 * head m_w1 (128, 128), m_b1 (128), m_w3 (144, 128), m_b3 (144); with k == 0 the m_* pointers are not read (may be
 * NULL).  Two kernels.  magnet_dnet_weights_bytes: k == 0 the depth head alone, k == 4 both
 * heads, 0 for any other k.
 *
 * magnet_dnet_depth_f32: pre_d (B, 128, H, W) the first depth-head convolution's output before its ReLU -> out
 * (B, 2, H, W): with sigma == 0 the raw [mu, v] (what magnet_dnet_upsample_f32 reads), else [mu, sqrt(var)]
 * (activation_G_magnet: D-Net's mono_gmms inside MaGNet).  One kernel.
 * magnet_dnet_upsample_f32: pre_m (B, 128, H, W) the first mask-head convolution's output before its ReLU, raw (B, 2, H,
 * W) from magnet_dnet_depth_f32 with sigma == 0, a k == 4 pack -> out (B, 2, k*H, k*W) [mu, var] (activation_G: what
 * DNET(args) returns).  One kernel.  k != 4 -> MAGNET_ERR_UNSUPPORTED.
 * Both: B*H*W < 2^31; every pointer 16-byte aligned; out must not overlap the inputs.
 */
size_t magnet_dnet_weights_bytes(int32_t k);
int magnet_dnet_pack_weights_f32(const float* d_w1, const float* d_b1, const float* d_w2, const float* d_b2,
                                 const float* m_w1, const float* m_b1, const float* m_w3, const float* m_b3, int32_t k,
                                 void* packed, void* stream);
int magnet_dnet_depth_f32(const float* pre_d, const void* packed, int32_t B, int32_t H, int32_t W, int32_t sigma,
                          float* out, void* stream);
int magnet_dnet_upsample_f32(const float* pre_m, const void* packed, const float* raw, int32_t B, int32_t H, int32_t W,
                             int32_t k, float* out, void* stream);

/*
 * Caller-side camera preparation on the device (SURVEY §8 f-4).
 * magnet_relative_poses_f32 replaces utils/utils.py:72-98 (data_preprocess): poses_out[b,v] = ext_nghbr[v,b] *
 * inv(ext_ref[b]) (ref-camera -> source-camera), is_valid_out[b,v] = 0 when either extrinsic or the product holds a
 * NaN (the pose is then all zeros).  ext_ref (B,4,4); ext_nghbr (V,B,4,4) view-major; poses_out (B,V,4,4).
 */
int magnet_relative_poses_f32(const float* ext_ref, const float* ext_nghbr, int32_t B, int32_t V, float* poses_out,
                              int32_t* is_valid_out, void* stream);
/*
 * magnet_camera_rays_f32 replaces get_ray_array + get_cam_intrinsics (data/dataloader_scannet.py:113-153 and the
 * crop-margin variant data/dataloader_kitti.py:94-127): raw_intrinsics (B,8) float64 on the device =
 * fx, fy, cx, cy of the raw image; img_W, img_H = size of the (cropped) image the grid spans; left_margin, top_margin
 * = crop offsets in raw pixels (ScanNet: the raw size and 0, 0; KITTI: 1216, 352, (raw_W-1216)/2, raw_H-352).
 * intM_out (B,3,3) = intrinsics of the H x W grid; rays_out (B,3,H*W) = K_raw^-1 (pixel centre), z = 1.
 * Evaluated in fp64 and rounded once, bit-identical to the numpy originals.
 */
int magnet_camera_rays_f32(const double* raw_intrinsics, int32_t B, int32_t H, int32_t W, float* intM_out,
                           float* rays_out, void* stream);

/*
 * Learned convex upsampling.  Replaces upsample_depth_via_mask (models/MAGNET.py:15-27): softmax over the 9
 * neighbours of up_mask (B, 9*k*k, H, W) viewed (B,1,9,k,k,H,W), weighted sum of the zero-padded 3x3
 * neighbourhood of depth (B,CH,H,W), pixel shuffle -> out (B,CH,k*H,k*W).  CH in {1,2}.
 */
int magnet_convex_upsample_fwd_f32(const float* depth, const float* up_mask, int32_t B, int32_t CH, int32_t H,
                                   int32_t W, int32_t k, float* out, void* stream);
/* Backward: grad_mask (B,9*k*k,H,W) is written; grad_depth (B,CH,H,W) is ACCUMULATED (caller zeroes it). */
int magnet_convex_upsample_bwd_f32(const float* grad_out, const float* depth, const float* up_mask, int32_t B,
                                   int32_t CH, int32_t H, int32_t W, int32_t k, float* grad_depth, float* grad_mask,
                                   void* stream);

/*
 * Convex upsampling fused with the Gaussian negative log-likelihood — replaces, per prediction of pred_list,
 * upsample_depth_via_mask (models/MAGNET.py:15-27,172-173) followed by MagnetLoss's term (utils/losses.py:39-49):
 *   nll = (mu - gt)^2 / (2 var) + 0.5 log(var),  var = max(sigma^2, 1e-10),  over the pixels where gt_mask != 0.
 * depth (B,2,H,W) quarter-resolution [mu, sigma]; up_mask (B,9*k*k,H,W); gt (B,1,k*H,k*W); gt_mask (B,1,k*H,k*W)
 * uint8.  The (B,2,k*H,k*W) prediction is never materialised.
 * forward: partial[magnet_upsample_nll_partials(B,H,W,k)] receives one partial sum of nll per CTA (the caller adds
 *   them — deterministic — and divides by the number of supervised pixels).
 * backward: scale = upstream gradient * gamma^(n-i-1) / number of supervised pixels; grad_depth (B,2,H,W) is
 *   ACCUMULATED (the caller zeroes it), grad_mask (B,9*k*k,H,W) is written.
 */
int magnet_upsample_nll_partials(int32_t B, int32_t H, int32_t W, int32_t k);
int magnet_upsample_nll_fwd_f32(const float* depth, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                int32_t B, int32_t H, int32_t W, int32_t k, float* partial, void* stream);
int magnet_upsample_nll_bwd_f32(const float* depth, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                float scale, int32_t B, int32_t H, int32_t W, int32_t k, float* grad_depth,
                                float* grad_mask, void* stream);
/* magnet_upsample_nll_bwd_f32 with the scale read from the DEVICE float *scale when the kernel runs (for CUDA graphs). */
int magnet_upsample_nll_bwd_dev_f32(const float* depth, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                    const float* scale, int32_t B, int32_t H, int32_t W, int32_t k, float* grad_depth,
                                    float* grad_mask, void* stream);

/*
 * D-Net's training loss, fused — replaces, on the output of D-Net's depth and mask heads, upsample_depth_via_mask
 * (models/submodules/D_dense_depth.py:86-100), activation_G (models/DNET.py:56-60) and DnetLoss (utils/losses.py:13-22):
 *   var = elu(v_up) + 1 + 1e-10, var[var < 1e-10] = 1e-10, nll = (mu - gt)^2 / (2 var) + 0.5 log(var),
 * with [mu, v_up] the convex upsampling of the RAW depth-head output raw (B,2,H,W) [mu, v], over the pixels where
 * gt_mask != 0.  The clamp never fires for a non-NaN v (elu(v) + 1 >= 0).  Arguments, outputs, partial sums and their
 * count (magnet_upsample_nll_partials) as the magnet_upsample_nll_* trio, with raw in place of depth and grad_raw
 * (B,2,H,W, ACCUMULATED: the caller zeroes it) in place of grad_depth; scale = upstream gradient / number of supervised
 * pixels.  The _dev form reads the scale from the DEVICE float *scale when the kernel runs (for CUDA graphs).  One
 * kernel each.
 */
int magnet_dnet_nll_fwd_f32(const float* raw, const float* up_mask, const float* gt, const uint8_t* gt_mask, int32_t B,
                            int32_t H, int32_t W, int32_t k, float* partial, void* stream);
int magnet_dnet_nll_bwd_f32(const float* raw, const float* up_mask, const float* gt, const uint8_t* gt_mask, float scale,
                            int32_t B, int32_t H, int32_t W, int32_t k, float* grad_raw, float* grad_mask, void* stream);
int magnet_dnet_nll_bwd_dev_f32(const float* raw, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                const float* scale, int32_t B, int32_t H, int32_t W, int32_t k, float* grad_raw,
                                float* grad_mask, void* stream);

/*
 * F-Net training loss, fused — replaces train_FNet.py:96-108 on the 1/V-averaged scores of the plane-sweep volume
 * (magnet_cost_volume_f32 with softmax == 0, depth_mode MAGNET_DEPTH_PLANES):
 *   prob = softmax over the D planes, pred = sum_j prob_j * planes_host[j], l1 = |pred - gt| where mask != 0.
 * scores (B,D,H,W); planes_host: HOST pointer, D floats; gt (B,1,H,W) quarter-resolution depth; mask (B,1,H,W) uint8.
 * Neither the probability volume nor the prediction is materialised.
 * forward: partial[magnet_fnet_l1_partials(B,H,W)] receives one partial sum of l1 per CTA (the caller adds them and
 *   divides by the number of supervised pixels).
 * backward: grad_scores (B,D,H,W) is WRITTEN with prob_j (d_j - pred) sign(pred - gt) mask scale, sign(0) = 0;
 *   scale = upstream gradient / number of supervised pixels, multiplied by *grad_scale (a DEVICE scalar) when
 *   grad_scale is not NULL, so that a captured CUDA graph can take the upstream gradient from memory.
 */
int magnet_fnet_l1_partials(int32_t B, int32_t H, int32_t W);
int magnet_fnet_l1_fwd_f32(const float* scores, const float* planes_host, const float* gt, const uint8_t* mask, int32_t B,
                           int32_t D, int32_t H, int32_t W, float* partial, void* stream);
int magnet_fnet_l1_bwd_f32(const float* scores, const float* planes_host, const float* gt, const uint8_t* mask,
                           float scale, const float* grad_scale, int32_t B, int32_t D, int32_t H, int32_t W,
                           float* grad_scores, void* stream);

/*
 * Depth evaluation — replaces the metric block of validate() (test_MaGNet.py:52-79, train_MaGNet.py:153-180) with
 * utils.compute_depth_errors (utils/utils.py:106-144), for every image of the batch and up to MAGNET_METRICS_MAX_PRED
 * predictions that share the GT (e.g. every prediction of pred_list).  Per image: gt > max_depth -> 0;
 * valid = min_depth < gt < max_depth inside the evaluation box; mu clamped to [min_depth, max_depth], inf -> max,
 * NaN -> min; var = max(sigma^2, 1e-6); per-pixel terms in float32, sums and the NLL in float64 (DESIGN §3.6).
 * Two forms: k == 0, pred[p] is the full-resolution (B,2,H,W) [mu, sigma]; k >= 1, pred[p] is the quarter-resolution
 * (B,2,H/k,W/k) [mu, sigma] and up_mask (B,9*k*k,H/k,W/k) the upsampling mask (upsample_depth_via_mask fused in, the
 * full-resolution prediction is never written).
 * out (P,B,13) float64: n, then a1 a2 a3 abs_diff abs_rel sq_rel rmse log_10 irmse rmse_log silog nll (NaN when n == 0).
 * Two kernels, no atomics: results are bit-identical from run to run.
 */
#define MAGNET_METRICS_MAX_PRED 8
#define MAGNET_METRICS_COLS 13
typedef struct magnet_depth_metrics_args {
  int32_t P, B, H, W;             /* predictions (1..MAGNET_METRICS_MAX_PRED), images, full-resolution GT size      */
  int32_t k;                      /* 0: full-resolution predictions; >= 1: upsampling factor (H % k == W % k == 0)  */
  int32_t row0, row1, col0, col1; /* evaluation box [row0,row1) x [col0,col1) (no crop: 0, H, 0, W)                 */
  float min_depth, max_depth;     /* compared in float32                                                            */
  const float* const* pred;       /* HOST array of P DEVICE pointers, each (B,2,H,W) or (B,2,H/k,W/k)               */
  const float* up_mask;           /* (B,9*k*k,H/k,W/k) when k >= 1, else ignored                                    */
  const float* gt;                /* (B,1,H,W) raw GT (values above max_depth are treated as 0)                     */
  double* workspace;              /* magnet_depth_metrics_workspace(args) doubles of scratch                        */
  double* out;                    /* (P,B,MAGNET_METRICS_COLS)                                                      */
} magnet_depth_metrics_args;
/* Doubles of workspace the call needs (shape fields and box of args only), or a negative magnet_status. */
int64_t magnet_depth_metrics_workspace(const magnet_depth_metrics_args* args);
int magnet_depth_metrics_f32(const magnet_depth_metrics_args* args, void* stream);

/*
 * F-Net depth map — the soft-argmin prediction of train_FNet.py:96 / :180, sum_j prob_j * planes_host[j], without the
 * probability volume.  volume (B,D,H,W); planes_host: HOST pointer, D floats; out (B,1,H,W).
 *   scores != 0: volume holds the 1/V-averaged scores of magnet_cost_volume_f32 with softmax == 0 (depth_mode
 *     MAGNET_DEPTH_PLANES); the softmax over the planes is fused in, with the same code as magnet_fnet_l1_fwd_f32, so
 *     the prediction is bit for bit the one the training loss supervises.
 *   scores == 0: volume holds the probabilities (the output of est_costvolume_F / MAGNET_F.forward).
 * A row with a NaN or an infinite maximum gives NaN, as torch.softmax does.  One kernel.
 * D outside 1..MAGNET_MAX_PLANES: D <= 0 -> MAGNET_ERR_SHAPE, D > MAGNET_MAX_PLANES -> MAGNET_ERR_UNSUPPORTED.
 */
int magnet_plane_depth_f32(const float* volume, const float* planes_host, int32_t B, int32_t D, int32_t H, int32_t W,
                           int32_t scores, float* out, void* stream);

/*
 * Depth evaluation of F-Net — replaces the metric block of train_FNet.py validate() (:165-193): the (B,1,h,w)
 * predictions are upsampled to the GT size with F.interpolate(..., size=(H, W), mode='nearest') inside the kernel,
 * source row min(floor(Y * (float)h / H), h - 1) in float32 (likewise for columns), any h <= H and w <= W.  Masking,
 * per-pixel terms and sums as magnet_depth_metrics_f32.  There is no variance: the nll column is 0.0 for every image,
 * also one without a valid pixel (compute_depth_errors(..., var=None)), while the other columns are NaN there.
 * out (P,B,MAGNET_METRICS_COLS) float64 as magnet_depth_metrics_f32.  Two kernels, no atomics.
 */
typedef struct magnet_depth_metrics_nearest_args {
  int32_t P, B, H, W;             /* predictions (1..MAGNET_METRICS_MAX_PRED), images, full-resolution GT size      */
  int32_t h, w;                   /* prediction grid, 1 <= h <= H, 1 <= w <= W                                      */
  int32_t row0, row1, col0, col1; /* evaluation box [row0,row1) x [col0,col1) of the GT (no crop: 0, H, 0, W)      */
  float min_depth, max_depth;     /* compared in float32                                                            */
  const float* const* pred;       /* HOST array of P DEVICE pointers, each (B,1,h,w)                                */
  const float* gt;                /* (B,1,H,W) raw GT (values above max_depth are treated as 0)                     */
  double* workspace;              /* magnet_depth_metrics_nearest_workspace(args) doubles of scratch                */
  double* out;                    /* (P,B,MAGNET_METRICS_COLS)                                                      */
} magnet_depth_metrics_nearest_args;
/* Doubles of workspace the call needs (shape fields and box of args only), or a negative magnet_status. */
int64_t magnet_depth_metrics_nearest_workspace(const magnet_depth_metrics_nearest_args* args);
int magnet_depth_metrics_nearest_f32(const magnet_depth_metrics_nearest_args* args, void* stream);

/*
 * Depth evaluation of D-Net — replaces the metric block of test_DNet.py validate() (:40-71): the full-resolution
 * prediction's channel 1 is the variance D-Net returns (activation_G), passed to compute_depth_errors as var, so
 * var = max(channel 1, 1e-6) on the float32 value instead of max(sigma^2, 1e-6).  Everything else as
 * magnet_depth_metrics_f32 with k == 0: the same args (k must be 0, up_mask is ignored), the same workspace
 * (magnet_depth_metrics_workspace), out (P,B,MAGNET_METRICS_COLS).  k != 0 -> MAGNET_ERR_UNSUPPORTED.  Two kernels.
 */
int magnet_depth_metrics_var_f32(const magnet_depth_metrics_args* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MAGNET_B200_H_ */
