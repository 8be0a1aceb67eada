// C-ABI entry points declared in include/magnet_b200.h: argument validation + dispatch only.
#include <atomic>
#include <cstdlib>
#include <cstdio>
#include <cstring>

#include "common.cuh"
#include "launchers.h"

namespace {
std::atomic<uint64_t> g_launches{0};
thread_local char g_cuda_err[256] = "";

bool misaligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 != 0; }
bool misaligned4(const void* p) { return reinterpret_cast<uintptr_t>(p) % 4 != 0; }

// The end of every launching entry point: a CUDA error is recorded for magnet_last_cuda_error, a success adds the
// kernels it enqueued to magnet_launch_count.
int finish(cudaError_t e, int launches) {
  if (e != cudaSuccess) {
    snprintf(g_cuda_err, sizeof(g_cuda_err), "%s: %s", cudaGetErrorName(e), cudaGetErrorString(e));
    return MAGNET_ERR_CUDA;
  }
  g_launches += launches;
  return MAGNET_OK;
}

// B, H, W positive and B*H*W pixels indexable with an int32
bool pixels_ok(int32_t B, int32_t H, int32_t W) {
  return B > 0 && H > 0 && W > 0 && (int64_t)B * H * W < ((int64_t)1 << 31);
}

// ---- pieces of the checks of a magnet_cost_args description, shared by the forward and the three backwards ----

// the tensor-core layouts: a header + fp16 plane(s) + (mu, sigma) table per buffer, ref_feat included
bool packed_layout(int layout) { return layout == MAGNET_SRC_SPLIT16 || layout == MAGNET_SRC_HALF16; }

bool cost_dims_ok(const magnet_cost_args* a) {
  return a->B > 0 && a->V > 0 && a->D > 0 && a->C > 0 && a->H > 0 && a->W > 0;
}

// The depth source's pointers, for a depth_mode in `modes` (a set of 1 << magnet_depth_mode bits).
int check_depth_source(const magnet_cost_args* a, unsigned modes) {
  if (a->depth_mode < MAGNET_DEPTH_VOLUME || a->depth_mode > MAGNET_DEPTH_PLANES || !(modes & (1u << a->depth_mode)))
    return MAGNET_ERR_UNSUPPORTED;
  switch (a->depth_mode) {
    case MAGNET_DEPTH_VOLUME: return a->d_volume ? MAGNET_OK : MAGNET_ERR_NULL;
    case MAGNET_DEPTH_GAUSS: return a->ref_gmm && a->k_host ? MAGNET_OK : MAGNET_ERR_NULL;
    default: return a->k_host ? MAGNET_OK : MAGNET_ERR_NULL;
  }
}
constexpr unsigned kAnyDepth = (1u << MAGNET_DEPTH_VOLUME) | (1u << MAGNET_DEPTH_GAUSS) | (1u << MAGNET_DEPTH_PLANES);
constexpr unsigned kPixelDepth = (1u << MAGNET_DEPTH_VOLUME) | (1u << MAGNET_DEPTH_GAUSS);

bool tc_variant(const magnet_cost_args* a) {
  return a->variant == MAGNET_VARIANT_AUTO || a->variant == MAGNET_VARIANT_MMA;
}
bool split_misaligned(const magnet_cost_args* a) { return misaligned16(a->src_feat) || misaligned16(a->ref_feat); }

// A backward of a tensor-core forward: an AUTO / MMA variant and shapes the kernels take (`supports`), then, with
// `split`, 16-byte aligned ref / src buffers.
int tensor_core_gate(const magnet_cost_args* a, bool supports, bool split) {
  if (!tc_variant(a) || !supports) return MAGNET_ERR_UNSUPPORTED;
  if (split && split_misaligned(a)) return MAGNET_ERR_ALIGN;
  return MAGNET_OK;
}

// The host plane array: k_j for GAUSS / PLANES, zeros for VOLUME and past D.
void fill_planes(float k[MAGNET_MAX_PLANES], const magnet_cost_args* a) {
  for (int j = 0; j < MAGNET_MAX_PLANES; ++j)
    k[j] = (a->depth_mode != MAGNET_DEPTH_VOLUME && j < a->D) ? a->k_host[j] : 0.0f;
}

// The geometry fields every cost-volume kernel parameter block has.
template <class Params>
void fill_geometry(Params& p, const magnet_cost_args* a) {
  p.B = a->B; p.V = a->V; p.D = a->D; p.H = a->H; p.W = a->W; p.HW = a->H * a->W;
  p.rays = a->rays; p.cams = a->cams;
  fill_planes(p.k, a);
}

// The CUDA-core CW / geometry backwards' parameters: the forward's description with these maps and gradients.
magnet::CwBwdParams cw_bwd_params(const magnet_cost_args* a, const float* ref_feat, const float* src_feat,
                                  const float* src_gmm, const float* g_score, float* grad_ref, float* grad_src,
                                  float* grad_depth) {
  magnet::CwBwdParams p;
  fill_geometry(p, a);
  p.cw = a->consistency != 0;
  p.kappa = a->kappa;
  p.ref_feat = ref_feat; p.src_feat = src_feat; p.src_gmm = src_gmm;
  p.d_volume = a->d_volume; p.ref_gmm = a->ref_gmm;
  p.g_score = g_score;
  p.grad_ref = grad_ref; p.grad_src = grad_src; p.grad_depth = grad_depth;
  return p;
}

int validate_cost(const magnet_cost_args* a) {
  if (!a) return MAGNET_ERR_NULL;
  if (!cost_dims_ok(a)) return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if ((int64_t)a->H * a->W > (1 << 26)) return MAGNET_ERR_SHAPE;
  if (!a->ref_feat || !a->src_feat || !a->rays || !a->cams || !a->out) return MAGNET_ERR_NULL;
  if (a->consistency && !a->src_gmm && a->src_layout != MAGNET_SRC_PIXC && !packed_layout(a->src_layout))
    return MAGNET_ERR_NULL;
  if (a->consistency && a->softmax) return MAGNET_ERR_UNSUPPORTED;
  const int st = check_depth_source(a, kAnyDepth);
  if (st != MAGNET_OK) return st;
  if (a->src_layout == MAGNET_SRC_TILED32) {
    if (a->C % 4 != 0) return MAGNET_ERR_UNSUPPORTED;
    if (misaligned16(a->src_feat)) return MAGNET_ERR_ALIGN;
  } else if (a->src_layout == MAGNET_SRC_PIXC) {
    if (!magnet::tma_supports(a->C, a->D, a->V, a->src_layout)) return MAGNET_ERR_UNSUPPORTED;
    if (misaligned16(a->src_feat)) return MAGNET_ERR_ALIGN;
    if (a->variant != MAGNET_VARIANT_AUTO && a->variant != MAGNET_VARIANT_TMA) return MAGNET_ERR_UNSUPPORTED;
  } else if (packed_layout(a->src_layout)) {
    // not tensor_core_gate: the forward reports misaligned buffers before a variant the layout does not run
    if (!magnet::mma_supports(a->C, a->D, a->V, a->src_layout)) return MAGNET_ERR_UNSUPPORTED;
    if (split_misaligned(a)) return MAGNET_ERR_ALIGN;
    if (!tc_variant(a)) return MAGNET_ERR_UNSUPPORTED;
  } else if (a->src_layout != MAGNET_SRC_NCHW) {
    return MAGNET_ERR_UNSUPPORTED;
  }
  if (a->variant < MAGNET_VARIANT_AUTO || a->variant > MAGNET_VARIANT_MMA) return MAGNET_ERR_UNSUPPORTED;
  if (a->variant == MAGNET_VARIANT_MMA && !magnet::mma_supports(a->C, a->D, a->V, a->src_layout))
    return MAGNET_ERR_UNSUPPORTED;
  if (a->variant == MAGNET_VARIANT_TMA && !magnet::tma_supports(a->C, a->D, a->V, a->src_layout))
    return MAGNET_ERR_UNSUPPORTED;
  if ((a->variant == MAGNET_VARIANT_CELLS || a->variant == MAGNET_VARIANT_CELLS_NOREUSE) &&
      !magnet::cells_supports(a->C, a->D, a->src_layout))
    return MAGNET_ERR_UNSUPPORTED;
  if (a->variant == MAGNET_VARIANT_CELLS_NOREUSE && a->depth_mode != MAGNET_DEPTH_GAUSS) return MAGNET_ERR_UNSUPPORTED;
  return MAGNET_OK;
}

bool use_cells(const magnet_cost_args* a) {
  if (a->variant == MAGNET_VARIANT_DIRECT || a->variant == MAGNET_VARIANT_TMA || a->variant == MAGNET_VARIANT_MMA)
    return false;
  return magnet::cells_supports(a->C, a->D, a->src_layout);
}

bool use_tma(const magnet_cost_args* a) {                  // the PIXC layout is served by the TMA kernel only
  return a->src_layout == MAGNET_SRC_PIXC && magnet::tma_supports(a->C, a->D, a->V, a->src_layout);
}

bool use_mma(const magnet_cost_args* a) {                  // SPLIT16 / HALF16 are served by the tensor-core kernel only
  return packed_layout(a->src_layout) && magnet::mma_supports(a->C, a->D, a->V, a->src_layout);
}

// The frame table of an indexed forward: a (B, V) device array over n_src >= 1 source images.  Its entries are read
// by the kernels only; the caller guarantees that each lies in [0, n_src).
int validate_index(const int32_t* src_index, int32_t n_src) {
  if (!src_index) return MAGNET_ERR_NULL;
  if (n_src < 1) return MAGNET_ERR_SHAPE;
  if (misaligned4(src_index)) return MAGNET_ERR_ALIGN;
  return MAGNET_OK;
}

int launch_info(const magnet_cost_args* a, int* grid_ctas, int* block_threads, int* smem_bytes) {
  if (!grid_ctas || !block_threads || !smem_bytes) return MAGNET_ERR_NULL;
  if (use_mma(a)) {
    magnet::mma_launch_info(a->B, a->H, a->W, a->D, grid_ctas, block_threads, smem_bytes);
  } else if (use_tma(a)) {
    magnet::tma_launch_info(a->B, a->H, a->W, a->D, grid_ctas, block_threads, smem_bytes);
  } else if (use_cells(a)) {
    magnet::cells_launch_info(a->B, a->H, a->W, a->D, grid_ctas, block_threads, smem_bytes);
  } else {
    *grid_ctas = ((a->H * a->W + 127) / 128) * a->D * a->B;
    *block_threads = 128;
    *smem_bytes = 0;
  }
  return MAGNET_OK;
}

// One cost-volume forward of validated arguments: view (b, v) reads source image v*B + b (src_index NULL) or
// src_index[b*V + v] of n_src images.
int run_cost(const magnet_cost_args* a, const int32_t* src_index, int n_src, void* stream) {
  magnet::CostParams p;
  fill_geometry(p, a);
  p.kappa = a->kappa;
  p.vf = (float)a->V;
  p.inv_v_exact = ((a->V & (a->V - 1)) == 0) ? 1.0f / (float)a->V : 0.0f;
  p.ref_feat = a->ref_feat; p.src_feat = a->src_feat; p.src_gmm = a->src_gmm;
  p.d_volume = a->d_volume; p.ref_gmm = a->ref_gmm; p.out = a->out;
  p.k_sorted = 1;
  for (int j = 1; j < a->D; ++j)
    if (!(p.k[j] >= p.k[j - 1])) p.k_sorted = 0;
  int launches = 0;
  cudaError_t e;
  const cudaStream_t st = (cudaStream_t)stream;
  const bool cw = a->consistency != 0;
  if (use_mma(a))
    e = magnet::launch_cost_mma(p, a->depth_mode, cw, a->src_layout, src_index, n_src, st, &launches);
  else if (use_tma(a))
    e = magnet::launch_cost_tma(p, a->depth_mode, a->C, cw, src_index, n_src, st, &launches);
  else if (use_cells(a))
    e = magnet::launch_cost_cells(p, a->depth_mode, a->C, cw, a->variant != MAGNET_VARIANT_CELLS_NOREUSE, src_index, st,
                                  &launches);
  else
    e = magnet::launch_cost_direct(p, a->depth_mode, a->src_layout, a->C, cw, src_index, st, &launches);
  if (e == cudaSuccess && a->softmax) {            // homography.py:46, in place on the 1/V-averaged scores
    e = magnet::launch_softmax_planes(a->out, a->B, a->D, a->H * a->W, st);
    ++launches;
  }
  return finish(e, launches);
}

// Shape fields and box of a depth-metrics call (the sizing calls need no pointers).
int validate_box(int32_t H, int32_t W, int32_t row0, int32_t row1, int32_t col0, int32_t col1) {
  if (row0 < 0 || row0 > row1 || row1 > H) return MAGNET_ERR_SHAPE;
  if (col0 < 0 || col0 > col1 || col1 > W) return MAGNET_ERR_SHAPE;
  return MAGNET_OK;
}

int validate_depth_metrics_shape(const magnet_depth_metrics_args* a) {
  if (!a) return MAGNET_ERR_NULL;
  if (a->P <= 0 || a->B <= 0 || a->H <= 0 || a->W <= 0 || a->k < 0) return MAGNET_ERR_SHAPE;
  if (a->P > MAGNET_METRICS_MAX_PRED) return MAGNET_ERR_UNSUPPORTED;
  if ((int64_t)a->P * a->B > 65535 || (int64_t)a->H * a->W > (1 << 28)) return MAGNET_ERR_SHAPE;
  if (a->k > 0 && (a->H % a->k != 0 || a->W % a->k != 0)) return MAGNET_ERR_SHAPE;
  return validate_box(a->H, a->W, a->row0, a->row1, a->col0, a->col1);
}

int validate_depth_metrics_nearest_shape(const magnet_depth_metrics_nearest_args* a) {
  if (!a) return MAGNET_ERR_NULL;
  if (a->P <= 0 || a->B <= 0 || a->H <= 0 || a->W <= 0 || a->h <= 0 || a->w <= 0) return MAGNET_ERR_SHAPE;
  if (a->P > MAGNET_METRICS_MAX_PRED) return MAGNET_ERR_UNSUPPORTED;
  if ((int64_t)a->P * a->B > 65535 || (int64_t)a->H * a->W > (1 << 28)) return MAGNET_ERR_SHAPE;
  if (a->h > a->H || a->w > a->W) return MAGNET_ERR_SHAPE;
  return validate_box(a->H, a->W, a->row0, a->row1, a->col0, a->col1);
}

// The upsample + NLL losses (magnet_upsample_nll_* with MagnetLoss's variance, magnet_dnet_nll_* with DnetLoss's):
// one launch each, checked the same way.  Grid: W*k / 128 x H*k x B.
bool upsample_nll_shape_ok(int32_t B, int32_t H, int32_t W, int32_t k) {
  return B > 0 && H > 0 && W > 0 && k > 0 && B <= 65535 && (int64_t)H * k <= 65535;
}

int upsample_nll_fwd(bool dnet, const float* depth, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                     int32_t B, int32_t H, int32_t W, int32_t k, float* partial, void* stream) {
  if (!depth || !up_mask || !gt || !gt_mask || !partial) return MAGNET_ERR_NULL;
  if (!upsample_nll_shape_ok(B, H, W, k)) return MAGNET_ERR_SHAPE;
  return finish(magnet::launch_upsample_nll_fwd(dnet, depth, up_mask, gt, gt_mask, B, H, W, k, partial,
                                                (cudaStream_t)stream), 1);
}

// scale_dev (on_device): a DEVICE float read in place of `scale` when the kernel runs; det: the fixed-order form,
// which needs `workspace` (magnet_upsample_nll_bwd_det_workspace_bytes)
int upsample_nll_bwd(bool dnet, bool det, const float* depth, const float* up_mask, const float* gt,
                     const uint8_t* gt_mask, float scale, const float* scale_dev, bool on_device, int32_t B, int32_t H,
                     int32_t W, int32_t k, float* workspace, float* grad_depth, float* grad_mask, void* stream) {
  if (!depth || !up_mask || !gt || !gt_mask || (on_device && !scale_dev) || !grad_depth || !grad_mask)
    return MAGNET_ERR_NULL;
  if (det && !workspace) return MAGNET_ERR_NULL;
  if (!upsample_nll_shape_ok(B, H, W, k)) return MAGNET_ERR_SHAPE;
  if (det && misaligned4(workspace)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_upsample_nll_bwd(dnet, det, depth, up_mask, gt, gt_mask, scale, scale_dev, B, H, W, k,
                                                workspace, grad_depth, grad_mask, (cudaStream_t)stream), det ? 2 : 1);
}

int convex_upsample_bwd(bool det, const float* grad_out, const float* depth, const float* up_mask, int32_t B, int32_t CH,
                        int32_t H, int32_t W, int32_t k, float* grad_depth, float* grad_mask, void* stream) {
  if (!grad_out || !depth || !up_mask || !grad_depth || !grad_mask) return MAGNET_ERR_NULL;
  if (B <= 0 || H <= 0 || W <= 0 || k <= 0 || B > 65535 || H * k > 65535) return MAGNET_ERR_SHAPE;
  if (CH != 1 && CH != 2) return MAGNET_ERR_UNSUPPORTED;
  return finish(magnet::launch_upsample_bwd(grad_out, depth, up_mask, B, CH, H, W, k, det, grad_depth, grad_mask,
                                            (cudaStream_t)stream), det ? 2 : 1);
}

// P prediction pointers, none NULL
bool preds_null(const float* const* pred, int P) {
  for (int p = 0; p < P; ++p)
    if (!pred[p]) return true;
  return false;
}

// a plane volume (B, D, H, W) with D host plane depths: F-Net's L1 loss and soft-argmin depth
int validate_planes_shape(int32_t B, int32_t D, int32_t H, int32_t W) {
  if (B <= 0 || D <= 0 || H <= 0 || W <= 0 || B > 65535) return MAGNET_ERR_SHAPE;
  if ((int64_t)H * W > (1 << 26)) return MAGNET_ERR_SHAPE;
  if (D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  return MAGNET_OK;
}

// shape and the pointers both G-Net training calls read
int validate_gnet_train(const magnet_gnet_train_args* a) {
  if (!a) return MAGNET_ERR_NULL;
  if (!pixels_ok(a->B, a->H, a->W) || a->D <= 0 || (int64_t)a->H * a->W > (1 << 26)) return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if (!a->cost || !a->packed_weights || !a->prev_gmm || !a->saved) return MAGNET_ERR_NULL;
  if (misaligned16(a->cost) || misaligned16(a->packed_weights) || misaligned16(a->saved)) return MAGNET_ERR_ALIGN;
  return MAGNET_OK;
}

// shape, factor, prediction count and the pointers both mask training calls read
int validate_mask_train(const magnet_mask_train_args* a) {
  if (!a) return MAGNET_ERR_NULL;
  if (!pixels_ok(a->B, a->H, a->W)) return MAGNET_ERR_SHAPE;
  if (a->P < 1 || a->P > MAGNET_MASK_MAX_PRED || a->k != 4) return MAGNET_ERR_UNSUPPORTED;
  if (!a->packed_weights || !a->saved) return MAGNET_ERR_NULL;
  if (misaligned16(a->packed_weights) || misaligned16(a->saved)) return MAGNET_ERR_ALIGN;
  return MAGNET_OK;
}
}  // namespace

extern "C" {

int magnet_abi_version(void) { return MAGNET_ABI_VERSION; }

const char* magnet_strerror(int status) {
  switch (status) {
    case MAGNET_OK: return "ok";
    case MAGNET_ERR_NULL: return "required pointer is NULL";
    case MAGNET_ERR_SHAPE: return "bad or inconsistent dimension";
    case MAGNET_ERR_UNSUPPORTED: return "unsupported C / D / layout / mode / variant";
    case MAGNET_ERR_CUDA: return "CUDA runtime error (see magnet_last_cuda_error)";
    case MAGNET_ERR_ALIGN: return "pointer not 16-byte aligned";
    default: return "unknown status";
  }
}

const char* magnet_last_cuda_error(void) { return g_cuda_err; }

uint64_t magnet_launch_count(void) { return g_launches.load(); }

int magnet_cost_launch_info(const magnet_cost_args* a, int* grid_ctas, int* block_threads, int* smem_bytes) {
  const int st = validate_cost(a);
  if (st != MAGNET_OK) return st;
  return launch_info(a, grid_ctas, block_threads, smem_bytes);
}

int magnet_cost_volume_f32(const magnet_cost_args* a, void* stream) {
  const int st = validate_cost(a);
  if (st != MAGNET_OK) return st;
  return run_cost(a, nullptr, 0, stream);
}

int magnet_cost_indexed_launch_info(const magnet_cost_args* a, const int32_t* src_index, int32_t n_src, int* grid_ctas,
                                    int* block_threads, int* smem_bytes) {
  int st = validate_cost(a);
  if (st == MAGNET_OK) st = validate_index(src_index, n_src);
  if (st != MAGNET_OK) return st;
  return launch_info(a, grid_ctas, block_threads, smem_bytes);
}

int magnet_cost_volume_indexed_f32(const magnet_cost_args* a, const int32_t* src_index, int32_t n_src, void* stream) {
  int st = validate_cost(a);
  if (st == MAGNET_OK) st = validate_index(src_index, n_src);
  if (st != MAGNET_OK) return st;
  return run_cost(a, src_index, n_src, stream);
}

int magnet_check_src_index(const void* src_index, int32_t dtype, int32_t B, int32_t V, int32_t n_src,
                           int32_t* index_out, int32_t* bad, void* stream) {
  if (!src_index || !bad) return MAGNET_ERR_NULL;
  int st = validate_index(index_out, n_src);       // the table the indexed forward will read
  if (st != MAGNET_OK) return st;
  if (B < 1 || V < 1 || (int64_t)B * V >= ((int64_t)1 << 31)) return MAGNET_ERR_SHAPE;
  if (dtype != MAGNET_INDEX_I32 && dtype != MAGNET_INDEX_I64) return MAGNET_ERR_UNSUPPORTED;
  const bool wide = dtype == MAGNET_INDEX_I64;
  if (reinterpret_cast<uintptr_t>(src_index) % (wide ? 8 : 4) != 0 || misaligned4(bad)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_check_src_index(src_index, wide, B, V, n_src, index_out, bad, (cudaStream_t)stream), 1);
}

int magnet_cost_volume_f_bwd_f32(const magnet_cost_f_bwd_args* b, void* stream) {
  if (!b || !b->fwd) return MAGNET_ERR_NULL;
  const magnet_cost_args* a = b->fwd;
  if (!cost_dims_ok(a)) return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if (!a->ref_feat || !a->src_feat || !a->rays || !a->cams || !a->k_host) return MAGNET_ERR_NULL;
  if (!b->grad_out || !b->workspace || !b->grad_ref || !b->grad_src) return MAGNET_ERR_NULL;
  if (a->softmax && !b->prob) return MAGNET_ERR_NULL;
  if (a->consistency || a->depth_mode != MAGNET_DEPTH_PLANES) return MAGNET_ERR_UNSUPPORTED;
  const bool mma = packed_layout(a->src_layout);
  if (mma) {                                   // tensor-core backward on the forward's SPLIT16 / HALF16 buffers
    const int st = tensor_core_gate(a, magnet::f_bwd_mma_supports(a->C, a->V), true);
    if (st != MAGNET_OK) return st;
  } else {
    if (a->src_layout != MAGNET_SRC_NCHW) return MAGNET_ERR_UNSUPPORTED;
    if (a->C != 8 && a->C != 16 && a->C != 32 && a->C != 64) return MAGNET_ERR_UNSUPPORTED;
  }
  magnet::BwdParams p;
  fill_geometry(p, a);
  p.C = a->C;
  p.softmax = a->softmax != 0;
  p.vf = (float)a->V;
  p.ref_feat = a->ref_feat; p.src_feat = a->src_feat;
  p.prob = b->prob; p.grad_out = b->grad_out; p.g_score = b->workspace; p.grad_ref = b->grad_ref; p.grad_src = b->grad_src;
  int launches = 0;
  const cudaError_t e = mma ? magnet::launch_cost_f_bwd_mma(p, a->src_layout, (cudaStream_t)stream, &launches)
                            : magnet::launch_cost_f_bwd(p, (cudaStream_t)stream, &launches);
  return finish(e, launches);
}

int magnet_cost_volume_bwd_f32(const magnet_cost_bwd_args* b, void* stream) {
  if (!b || !b->fwd) return MAGNET_ERR_NULL;
  const magnet_cost_args* a = b->fwd;
  if (!cost_dims_ok(a)) return MAGNET_ERR_SHAPE;
  if ((int64_t)a->H * a->W > (1 << 26) || a->B > 65535) return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if (!a->rays || !a->cams || !b->grad_out || !b->workspace) return MAGNET_ERR_NULL;
  if (a->softmax) return MAGNET_ERR_UNSUPPORTED;
  int st = check_depth_source(a, kPixelDepth);
  if (st != MAGNET_OK) return st;
  const bool mask_mma = packed_layout(a->src_layout);   // the tensor-core forward's mask
  // its split buffers given: feature gradients on the tensor cores; both NULL: everything on the CUDA cores
  const bool split = mask_mma && (a->ref_feat || a->src_feat);
  if (mask_mma) {
    st = tensor_core_gate(a, magnet::mma_supports(a->C, a->D, a->V, a->src_layout) &&
                             magnet::f_bwd_mma_supports(a->C, a->V), false);
    if (st != MAGNET_OK) return st;
  }
  if (split) {
    if (!a->ref_feat || !a->src_feat) return MAGNET_ERR_NULL;
    if (split_misaligned(a)) return MAGNET_ERR_ALIGN;
  } else if (!mask_mma && (a->variant != MAGNET_VARIANT_DIRECT ||
             (a->src_layout != MAGNET_SRC_NCHW && a->src_layout != MAGNET_SRC_TILED32))) {
    return MAGNET_ERR_UNSUPPORTED;                 // only the tensor-core and DIRECT forwards' masks are reproduced
  }
  // the CUDA-core kernel reads the NCHW maps: for every gradient without split buffers, for the depth gradient always
  const bool nchw = !split || b->grad_depth != nullptr;
  if (nchw) {
    if (!b->ref_feat || !b->src_feat) return MAGNET_ERR_NULL;
    if (a->consistency && !b->src_gmm) return MAGNET_ERR_NULL;
    if (!magnet::cw_bwd_supports(a->C)) return MAGNET_ERR_UNSUPPORTED;
  }
  const magnet::CwBwdParams p = cw_bwd_params(a, b->ref_feat, b->src_feat, b->src_gmm, b->workspace, b->grad_ref,
                                              b->grad_src, b->grad_depth);
  magnet::CwBwdParams ps = p;
  ps.ref_feat = a->ref_feat; ps.src_feat = a->src_feat; ps.src_gmm = nullptr; ps.grad_depth = nullptr;
  int launches = 0;
  const cudaError_t e = magnet::launch_cost_cw_bwd(p, split ? &ps : nullptr, a->src_layout, a->C, a->depth_mode,
                                                   mask_mma, b->grad_out, (cudaStream_t)stream, &launches);
  return finish(e, launches);
}

size_t magnet_cost_geom_workspace_bytes(int32_t B, int32_t V, int32_t H, int32_t W) {
  if (B <= 0 || V <= 0 || H <= 0 || W <= 0) return 0;
  return magnet::geom_workspace_bytes(B, V, H, W);
}

int magnet_cost_volume_geom_bwd_f32(const magnet_cost_geom_bwd_args* b, void* stream) {
  if (!b || !b->fwd) return MAGNET_ERR_NULL;
  const magnet_cost_args* a = b->fwd;
  if (!cost_dims_ok(a)) return MAGNET_ERR_SHAPE;
  if ((int64_t)a->H * a->W > (1 << 26) || a->B > 65535 || (int64_t)a->B * a->V > (1 << 30)) return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES || !magnet::cw_bwd_supports(a->C)) return MAGNET_ERR_UNSUPPORTED;
  if (!a->rays || !a->cams || !b->ref_feat || !b->src_feat || !b->grad_out || !b->score || !b->workspace ||
      !b->grad_cams)
    return MAGNET_ERR_NULL;
  int st = check_depth_source(a, kAnyDepth);
  if (st != MAGNET_OK) return st;
  bool mask_mma = false;
  if (a->depth_mode == MAGNET_DEPTH_PLANES) {      // the F volume: no mask, the tensor-core forward's positions
    if (a->consistency || b->grad_depth) return MAGNET_ERR_UNSUPPORTED;
    if (a->softmax && !b->prob) return MAGNET_ERR_NULL;
  } else {
    if (a->softmax) return MAGNET_ERR_UNSUPPORTED;
    mask_mma = packed_layout(a->src_layout);     // the tensor-core forward's mask, else the DIRECT forward's
    if (mask_mma) {
      st = tensor_core_gate(a, magnet::mma_supports(a->C, a->D, a->V, a->src_layout), false);
      if (st != MAGNET_OK) return st;
    } else if (a->variant != MAGNET_VARIANT_DIRECT ||
               (a->src_layout != MAGNET_SRC_NCHW && a->src_layout != MAGNET_SRC_TILED32)) {
      return MAGNET_ERR_UNSUPPORTED;
    }
    if (a->consistency && !b->src_gmm) return MAGNET_ERR_NULL;
  }
  if (misaligned16(b->workspace)) return MAGNET_ERR_ALIGN;
  const magnet::CwBwdParams p = cw_bwd_params(a, b->ref_feat, b->src_feat, b->src_gmm, b->score, nullptr, nullptr,
                                              b->grad_depth);
  int launches = 0;
  const cudaError_t e = magnet::launch_cost_geom_bwd(p, a->C, a->depth_mode, mask_mma, a->softmax != 0, b->prob,
                                                     b->grad_out, static_cast<float*>(b->workspace), b->grad_rays,
                                                     b->grad_cams, (cudaStream_t)stream, &launches);
  return finish(e, launches);
}

int magnet_pack_cameras_f32(const float* intM, const float* R, int64_t r_sb, int64_t r_sv, int64_t r_si,
                            int64_t r_sj, const float* t, int64_t t_sb, int64_t t_sv, int64_t t_si,
                            const int32_t* is_valid, int32_t B, int32_t V, magnet_camera* cams_out,
                            void* stream) {
  if (!intM || !R || !t || !is_valid || !cams_out) return MAGNET_ERR_NULL;
  if (B <= 0 || V <= 0) return MAGNET_ERR_SHAPE;
  return finish(magnet::launch_pack_cameras(intM, R, r_sb, r_sv, r_si, r_sj, t, t_sb, t_sv, t_si, is_valid, B, V,
                                            cams_out, (cudaStream_t)stream), 1);
}

int magnet_repack_tiled32_f32(const float* src_nchw, float* dst, int32_t N, int32_t C, int32_t H, int32_t W,
                            void* stream) {
  if (!src_nchw || !dst) return MAGNET_ERR_NULL;
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0) return MAGNET_ERR_SHAPE;
  if (C % 4 != 0 || C / 4 > 65535 || N > 65535) return MAGNET_ERR_UNSUPPORTED;
  if (misaligned16(dst)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_repack(src_nchw, dst, N, C, H, W, (cudaStream_t)stream), 1);
}

int magnet_repack_pixc_f32(const float* src_nchw, const float* src_gmm, float* dst, int32_t N, int32_t C, int32_t H,
                           int32_t W, void* stream) {
  if (!src_nchw || !dst) return MAGNET_ERR_NULL;
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0 || N > 65535) return MAGNET_ERR_SHAPE;
  if (C != 16 && C != 32 && C != 64) return MAGNET_ERR_UNSUPPORTED;
  if (misaligned16(dst)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_repack_pixc(src_nchw, src_gmm, dst, N, C, H, W, (cudaStream_t)stream), 1);
}

size_t magnet_split16_bytes(int32_t N, int32_t H, int32_t W) {
  if (N <= 0 || H <= 0 || W <= 0) return 0;
  return magnet::split16_buffer_bytes(N, H, W);
}

int magnet_repack_split16_f32(const float* src_nchw, const float* src_gmm, void* dst, int32_t N, int32_t C, int32_t H,
                              int32_t W, void* stream) {
  if (!src_nchw || !dst) return MAGNET_ERR_NULL;
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0 || N > 65535) return MAGNET_ERR_SHAPE;
  if (C != 64) return MAGNET_ERR_UNSUPPORTED;
  if (misaligned16(dst) || misaligned16(src_nchw)) return MAGNET_ERR_ALIGN;
  int launches = 0;
  const cudaError_t e =
      magnet::launch_repack_split16(src_nchw, src_gmm, dst, N, C, H, W, (cudaStream_t)stream, &launches);
  return finish(e, launches);
}

size_t magnet_half16_bytes(int32_t N, int32_t H, int32_t W) {
  if (N <= 0 || H <= 0 || W <= 0) return 0;
  return magnet::half16_buffer_bytes(N, H, W);
}

int magnet_repack_half16(const void* src_nchw, int32_t dtype, const float* src_gmm, void* dst, int32_t N, int32_t C,
                         int32_t H, int32_t W, void* stream) {
  if (!src_nchw || !dst) return MAGNET_ERR_NULL;
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0 || N > 65535) return MAGNET_ERR_SHAPE;
  if (C != 64 || (dtype != MAGNET_DTYPE_F16 && dtype != MAGNET_DTYPE_BF16)) return MAGNET_ERR_UNSUPPORTED;
  if (misaligned16(dst) || misaligned16(src_nchw)) return MAGNET_ERR_ALIGN;
  int launches = 0;
  const cudaError_t e =
      magnet::launch_repack_half16(src_nchw, dtype, src_gmm, dst, N, C, H, W, (cudaStream_t)stream, &launches);
  return finish(e, launches);
}

#if defined(MAGNET_MMA_DEBUG) || defined(MAGNET_MMA_PROFILE)
// MAGNET_MMA_PROFILE builds: the buffer receives the per-stage clock64() totals of cost_mma_kernel (uint64[8])
void magnet_mma_debug_buffer(float* p) { magnet::mma_set_debug_buffer(p); }
#endif
#ifdef MAGNET_MMA_DEBUG
void magnet_f_bwd_mma_debug_buffer(float* p) { magnet::f_bwd_mma_set_debug_buffer(p); }
#endif

int magnet_sample_depths_f32(const float* gmm, const float* k_host, int32_t B, int32_t D, int32_t HW,
                             float* d_volume, void* stream) {
  if (!gmm || !k_host || !d_volume) return MAGNET_ERR_NULL;
  if (B <= 0 || D <= 0 || HW <= 0) return MAGNET_ERR_SHAPE;
  if (D > MAGNET_MAX_PLANES || B > 65535) return MAGNET_ERR_UNSUPPORTED;
  return finish(magnet::launch_sample(gmm, k_host, B, D, HW, d_volume, (cudaStream_t)stream), 1);
}

int magnet_gaussian_update_fwd_f32(const float* d_output, const float* ref_gmm, int32_t B, int32_t HW,
                                   float* out, void* stream) {
  if (!d_output || !ref_gmm || !out) return MAGNET_ERR_NULL;
  if (B <= 0 || HW <= 0 || B > 65535) return MAGNET_ERR_SHAPE;
  return finish(magnet::launch_update_fwd(d_output, ref_gmm, B, HW, out, (cudaStream_t)stream), 1);
}

int magnet_gaussian_update_bwd_f32(const float* grad_out, const float* d_output, const float* ref_gmm,
                                   int32_t B, int32_t HW, float* grad_d_output, void* stream) {
  if (!grad_out || !d_output || !ref_gmm || !grad_d_output) return MAGNET_ERR_NULL;
  if (B <= 0 || HW <= 0 || B > 65535) return MAGNET_ERR_SHAPE;
  return finish(magnet::launch_update_bwd(grad_out, d_output, ref_gmm, B, HW, grad_d_output, (cudaStream_t)stream), 1);
}

int magnet_relative_poses_f32(const float* ext_ref, const float* ext_nghbr, int32_t B, int32_t V, float* poses_out,
                              int32_t* is_valid_out, void* stream) {
  if (!ext_ref || !ext_nghbr || !poses_out || !is_valid_out) return MAGNET_ERR_NULL;
  if (B <= 0 || V <= 0) return MAGNET_ERR_SHAPE;
  return finish(magnet::launch_relative_poses(ext_ref, ext_nghbr, B, V, poses_out, is_valid_out, (cudaStream_t)stream),
                1);
}

int magnet_camera_rays_f32(const double* raw_intrinsics, int32_t B, int32_t H, int32_t W, float* intM_out,
                           float* rays_out, void* stream) {
  if (!raw_intrinsics || !intM_out || !rays_out) return MAGNET_ERR_NULL;
  if (B <= 0 || H <= 0 || W <= 0 || B > 65535) return MAGNET_ERR_SHAPE;
  return finish(magnet::launch_camera_rays(raw_intrinsics, B, H, W, intM_out, rays_out, (cudaStream_t)stream), 1);
}

int magnet_convex_upsample_fwd_f32(const float* depth, const float* up_mask, int32_t B, int32_t CH, int32_t H,
                                   int32_t W, int32_t k, float* out, void* stream) {
  if (!depth || !up_mask || !out) return MAGNET_ERR_NULL;
  if (B <= 0 || H <= 0 || W <= 0 || k <= 0 || B > 65535 || H * k > 65535) return MAGNET_ERR_SHAPE;
  if (CH != 1 && CH != 2) return MAGNET_ERR_UNSUPPORTED;
  return finish(magnet::launch_upsample_fwd(depth, up_mask, B, CH, H, W, k, out, (cudaStream_t)stream), 1);
}

int magnet_convex_upsample_bwd_f32(const float* grad_out, const float* depth, const float* up_mask, int32_t B,
                                   int32_t CH, int32_t H, int32_t W, int32_t k, float* grad_depth, float* grad_mask,
                                   void* stream) {
  return convex_upsample_bwd(false, grad_out, depth, up_mask, B, CH, H, W, k, grad_depth, grad_mask, stream);
}

int magnet_convex_upsample_bwd_det_f32(const float* grad_out, const float* depth, const float* up_mask, int32_t B,
                                       int32_t CH, int32_t H, int32_t W, int32_t k, float* grad_depth,
                                       float* grad_mask, void* stream) {
  return convex_upsample_bwd(true, grad_out, depth, up_mask, B, CH, H, W, k, grad_depth, grad_mask, stream);
}

int magnet_upsample_nll_partials(int32_t B, int32_t H, int32_t W, int32_t k) {
  if (B <= 0 || H <= 0 || W <= 0 || k <= 0) return MAGNET_ERR_SHAPE;
  return B * H * k * ((W * k + 127) / 128);
}

int magnet_upsample_nll_fwd_f32(const float* depth, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                int32_t B, int32_t H, int32_t W, int32_t k, float* partial, void* stream) {
  return upsample_nll_fwd(false, depth, up_mask, gt, gt_mask, B, H, W, k, partial, stream);
}

int magnet_upsample_nll_bwd_f32(const float* depth, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                float scale, int32_t B, int32_t H, int32_t W, int32_t k, float* grad_depth,
                                float* grad_mask, void* stream) {
  return upsample_nll_bwd(false, false, depth, up_mask, gt, gt_mask, scale, nullptr, false, B, H, W, k, nullptr,
                          grad_depth, grad_mask, stream);
}

int magnet_upsample_nll_bwd_dev_f32(const float* depth, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                    const float* scale, int32_t B, int32_t H, int32_t W, int32_t k, float* grad_depth,
                                    float* grad_mask, void* stream) {
  return upsample_nll_bwd(false, false, depth, up_mask, gt, gt_mask, 0.0f, scale, true, B, H, W, k, nullptr,
                          grad_depth, grad_mask, stream);
}

size_t magnet_upsample_nll_bwd_det_workspace_bytes(int32_t B, int32_t H, int32_t W, int32_t k) {
  if (!upsample_nll_shape_ok(B, H, W, k)) return 0;
  return (size_t)B * 2 * H * W * k * k * 4;
}

int magnet_upsample_nll_bwd_det_f32(const float* depth, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                    float scale, int32_t B, int32_t H, int32_t W, int32_t k, float* workspace,
                                    float* grad_depth, float* grad_mask, void* stream) {
  return upsample_nll_bwd(false, true, depth, up_mask, gt, gt_mask, scale, nullptr, false, B, H, W, k, workspace,
                          grad_depth, grad_mask, stream);
}

int magnet_upsample_nll_bwd_dev_det_f32(const float* depth, const float* up_mask, const float* gt,
                                        const uint8_t* gt_mask, const float* scale, int32_t B, int32_t H, int32_t W,
                                        int32_t k, float* workspace, float* grad_depth, float* grad_mask,
                                        void* stream) {
  return upsample_nll_bwd(false, true, depth, up_mask, gt, gt_mask, 0.0f, scale, true, B, H, W, k, workspace,
                          grad_depth, grad_mask, stream);
}

int magnet_dnet_nll_fwd_f32(const float* raw, const float* up_mask, const float* gt, const uint8_t* gt_mask, int32_t B,
                            int32_t H, int32_t W, int32_t k, float* partial, void* stream) {
  return upsample_nll_fwd(true, raw, up_mask, gt, gt_mask, B, H, W, k, partial, stream);
}

int magnet_dnet_nll_bwd_f32(const float* raw, const float* up_mask, const float* gt, const uint8_t* gt_mask, float scale,
                            int32_t B, int32_t H, int32_t W, int32_t k, float* grad_raw, float* grad_mask, void* stream) {
  return upsample_nll_bwd(true, false, raw, up_mask, gt, gt_mask, scale, nullptr, false, B, H, W, k, nullptr, grad_raw,
                          grad_mask, stream);
}

int magnet_dnet_nll_bwd_dev_f32(const float* raw, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                const float* scale, int32_t B, int32_t H, int32_t W, int32_t k, float* grad_raw,
                                float* grad_mask, void* stream) {
  return upsample_nll_bwd(true, false, raw, up_mask, gt, gt_mask, 0.0f, scale, true, B, H, W, k, nullptr, grad_raw,
                          grad_mask, stream);
}

int magnet_dnet_nll_bwd_det_f32(const float* raw, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                float scale, int32_t B, int32_t H, int32_t W, int32_t k, float* workspace,
                                float* grad_raw, float* grad_mask, void* stream) {
  return upsample_nll_bwd(true, true, raw, up_mask, gt, gt_mask, scale, nullptr, false, B, H, W, k, workspace, grad_raw,
                          grad_mask, stream);
}

int magnet_dnet_nll_bwd_dev_det_f32(const float* raw, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                    const float* scale, int32_t B, int32_t H, int32_t W, int32_t k, float* workspace,
                                    float* grad_raw, float* grad_mask, void* stream) {
  return upsample_nll_bwd(true, true, raw, up_mask, gt, gt_mask, 0.0f, scale, true, B, H, W, k, workspace, grad_raw,
                          grad_mask, stream);
}

int magnet_fnet_l1_partials(int32_t B, int32_t H, int32_t W) {
  if (B <= 0 || H <= 0 || W <= 0) return MAGNET_ERR_SHAPE;
  return magnet::fnet_l1_partials(B, H * W);
}

int magnet_fnet_l1_fwd_f32(const float* scores, const float* planes_host, const float* gt, const uint8_t* mask, int32_t B,
                           int32_t D, int32_t H, int32_t W, float* partial, void* stream) {
  if (!scores || !planes_host || !gt || !mask) return MAGNET_ERR_NULL;
  const int st = validate_planes_shape(B, D, H, W);
  if (st != MAGNET_OK) return st;
  if (!partial) return MAGNET_ERR_NULL;
  return finish(magnet::launch_fnet_l1_fwd(scores, planes_host, gt, mask, B, D, H * W, partial, (cudaStream_t)stream), 1);
}

int magnet_fnet_l1_bwd_f32(const float* scores, const float* planes_host, const float* gt, const uint8_t* mask,
                           float scale, const float* grad_scale, int32_t B, int32_t D, int32_t H, int32_t W,
                           float* grad_scores, void* stream) {
  if (!scores || !planes_host || !gt || !mask) return MAGNET_ERR_NULL;
  const int st = validate_planes_shape(B, D, H, W);
  if (st != MAGNET_OK) return st;
  if (!grad_scores) return MAGNET_ERR_NULL;
  return finish(magnet::launch_fnet_l1_bwd(scores, planes_host, gt, mask, scale, grad_scale, B, D, H * W, grad_scores,
                                           (cudaStream_t)stream), 1);
}

size_t magnet_gnet_weights_bytes(int32_t D) {
  if (D <= 0 || D > MAGNET_MAX_PLANES) return 0;
  return magnet::gnet_weights_bytes(D);
}

int magnet_gnet_pack_weights_f32(const float* w0_cost, const float* w1, const float* b1, const float* w2,
                                 const float* b2, const float* w3, const float* b3, int32_t D, void* packed,
                                 void* stream) {
  if (!w0_cost || !w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !packed) return MAGNET_ERR_NULL;
  if (D <= 0) return MAGNET_ERR_SHAPE;
  if (D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if (misaligned16(packed)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_gnet_pack(w0_cost, w1, b1, w2, b2, w3, b3, D, packed, (cudaStream_t)stream), 2);
}

int magnet_gnet_update_f32(const magnet_gnet_args* a, void* stream) {
  if (!a) return MAGNET_ERR_NULL;
  if (a->B <= 0 || a->D <= 0 || a->H <= 0 || a->W <= 0) return MAGNET_ERR_SHAPE;
  if ((int64_t)a->H * a->W > (1 << 26) || (int64_t)a->B * ((a->H + 7) / 8) * ((a->W + 15) / 16) > (1 << 30))
    return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if (!a->cost || !a->invariant || !a->packed_weights || !a->prev_gmm || !a->scratch || !a->out) return MAGNET_ERR_NULL;
  if (misaligned16(a->cost) || misaligned16(a->invariant) || misaligned16(a->packed_weights) || misaligned4(a->scratch))
    return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_gnet_update(a->B, a->D, a->H, a->W, a->cost, a->invariant, a->packed_weights,
                                           a->prev_gmm, static_cast<unsigned*>(a->scratch), a->out,
                                           (cudaStream_t)stream), 2);
}

size_t magnet_gnet_train_weights_bytes(int32_t D) {
  if (D <= 0 || D > MAGNET_MAX_PLANES) return 0;
  return magnet::gnet_train_weights_bytes(D);
}

size_t magnet_gnet_saved_bytes(int32_t B, int32_t H, int32_t W) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  return magnet::gnet_saved_bytes(B, H, W);
}

size_t magnet_gnet_bwd_workspace_bytes(int32_t B, int32_t D, int32_t H, int32_t W) {
  if (B <= 0 || H <= 0 || W <= 0 || D <= 0 || D > MAGNET_MAX_PLANES) return 0;
  return magnet::gnet_bwd_workspace_bytes(B, D, H, W);
}

int magnet_gnet_pack_train_weights_f32(const float* w0_cost, const float* w1, const float* b1, const float* w2,
                                       const float* b2, const float* w3, const float* b3, int32_t D, void* packed,
                                       void* stream) {
  if (!w0_cost || !w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !packed) return MAGNET_ERR_NULL;
  if (D <= 0) return MAGNET_ERR_SHAPE;
  if (D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if (misaligned16(packed)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_gnet_pack_train(w0_cost, w1, b1, w2, b2, w3, b3, D, packed, (cudaStream_t)stream), 2);
}

int magnet_gnet_train_fwd_f32(const magnet_gnet_train_args* a, void* stream) {
  const int st = validate_gnet_train(a);
  if (st != MAGNET_OK) return st;
  if (!a->invariant || !a->scratch || !a->out) return MAGNET_ERR_NULL;
  if (misaligned16(a->invariant) || misaligned4(a->scratch)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_gnet_train_fwd(a->B, a->D, a->H, a->W, a->cost, a->invariant, a->packed_weights,
                                              a->prev_gmm, static_cast<unsigned*>(a->scratch), a->out, a->saved,
                                              (cudaStream_t)stream), 2);
}

int magnet_gnet_bwd_f32(const magnet_gnet_train_args* a, void* stream) {
  const int st = validate_gnet_train(a);
  if (st != MAGNET_OK) return st;
  if (!a->grad_out || !a->workspace || !a->grad_invariant) return MAGNET_ERR_NULL;
  if (misaligned16(a->workspace)) return MAGNET_ERR_ALIGN;
  int launches = 0;
  const cudaError_t e = magnet::launch_gnet_bwd(a->B, a->D, a->H, a->W, a->cost, a->prev_gmm, a->packed_weights,
                                                a->saved, a->grad_out, a->workspace, a->grad_invariant,
                                                a->grad_w0_cost, a->grad_w1, a->grad_b1, a->grad_w2, a->grad_b2,
                                                a->grad_w3, a->grad_b3, a->grad_prev, (cudaStream_t)stream, &launches);
  return finish(e, launches);
}

size_t magnet_mask_weights_bytes(int32_t k) { return k == 4 ? magnet::mask_weights_bytes() : 0; }

int magnet_mask_pack_weights_f32(const float* w1, const float* b1, const float* w2, const float* b2, const float* w3,
                                 const float* b3, void* packed, void* stream) {
  if (!w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !packed) return MAGNET_ERR_NULL;
  if (misaligned16(packed)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_mask_pack(w1, b1, w2, b2, w3, b3, packed, (cudaStream_t)stream), 2);
}

int magnet_mask_upsample_f32(const magnet_mask_upsample_args* a, void* stream) {
  if (!a) return MAGNET_ERR_NULL;
  if (!pixels_ok(a->B, a->H, a->W)) return MAGNET_ERR_SHAPE;
  if (a->P < 1 || a->P > MAGNET_MASK_MAX_PRED || a->k != 4) return MAGNET_ERR_UNSUPPORTED;
  if (!a->pre0 || !a->packed_weights || !a->pred || !a->out) return MAGNET_ERR_NULL;
  for (int p = 0; p < a->P; ++p)
    if (!a->pred[p] || !a->out[p]) return MAGNET_ERR_NULL;
  if (misaligned16(a->pre0) || misaligned16(a->packed_weights)) return MAGNET_ERR_ALIGN;
  for (int p = 0; p < a->P; ++p)
    if (misaligned16(a->pred[p]) || misaligned16(a->out[p])) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_mask_upsample(a->P, a->B, a->H, a->W, a->pre0, a->packed_weights, a->pred, a->out,
                                             (cudaStream_t)stream), 1);
}

size_t magnet_mask_train_weights_bytes(int32_t k) { return k == 4 ? magnet::mask_train_weights_bytes() : 0; }

size_t magnet_mask_saved_bytes(int32_t P, int32_t B, int32_t H, int32_t W) {
  if (P < 1 || P > MAGNET_MASK_MAX_PRED || !pixels_ok(B, H, W)) return 0;
  return magnet::mask_saved_bytes(P, B, H, W);
}

size_t magnet_mask_bwd_workspace_bytes(int32_t B, int32_t H, int32_t W) {
  if (!pixels_ok(B, H, W)) return 0;
  return magnet::mask_bwd_workspace_bytes(B, H, W);
}

size_t magnet_mask_train_det_workspace_bytes(int32_t P, int32_t B, int32_t H, int32_t W) {
  if (P < 1 || P > MAGNET_MASK_MAX_PRED || !pixels_ok(B, H, W) || (int64_t)P * B > 65535) return 0;
  return magnet::mask_train_det_workspace_bytes(P, B, H, W);
}

int magnet_mask_train_partials(int32_t B, int32_t H, int32_t W) {
  if (!pixels_ok(B, H, W)) return MAGNET_ERR_SHAPE;
  return magnet::mask_train_partials(B, H, W);
}

int magnet_mask_pack_train_weights_f32(const float* w1, const float* b1, const float* w2, const float* b2,
                                       const float* w3, const float* b3, void* packed, void* stream) {
  if (!w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !packed) return MAGNET_ERR_NULL;
  if (misaligned16(packed)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_mask_pack_train(w1, b1, w2, b2, w3, b3, packed, (cudaStream_t)stream), 2);
}

// the fused mask-loss forward with its prediction scales from `scale` (host or device, `on_device`); det: the prediction
// gradients in a fixed order through a->workspace (magnet_mask_train_det_workspace_bytes) when a->pred_grad is set
static int mask_train_fwd(const magnet_mask_train_args* a, const float* scale, bool on_device, bool det, void* stream) {
  const int st = validate_mask_train(a);
  if (st != MAGNET_OK) return st;
  if (!a->pre0 || !a->pred || !a->gt || !a->gt_mask || !scale || !a->partial) return MAGNET_ERR_NULL;
  if (preds_null(a->pred, a->P)) return MAGNET_ERR_NULL;
  const bool det_pg = det && a->pred_grad != 0;
  if (det_pg && !a->workspace) return MAGNET_ERR_NULL;
  if (det_pg && (int64_t)a->P * a->B > 65535) return MAGNET_ERR_SHAPE;
  if (misaligned16(a->pre0)) return MAGNET_ERR_ALIGN;
  for (int p = 0; p < a->P; ++p)
    if (misaligned16(a->pred[p])) return MAGNET_ERR_ALIGN;
  if (det_pg && misaligned16(a->workspace)) return MAGNET_ERR_ALIGN;
  int launches = 0;
  const cudaError_t e = magnet::launch_mask_train_fwd(a->P, a->B, a->H, a->W, a->pre0, a->packed_weights, a->pred,
                                                      a->gt, a->gt_mask, scale, on_device, a->save_maps != 0,
                                                      a->pred_grad != 0, a->partial, a->saved,
                                                      det_pg ? static_cast<float*>(a->workspace) : nullptr,
                                                      (cudaStream_t)stream, &launches);
  return finish(e, launches);
}

int magnet_mask_train_fwd_f32(const magnet_mask_train_args* a, void* stream) {
  return mask_train_fwd(a, a ? a->pred_scale : nullptr, false, false, stream);
}

int magnet_mask_train_fwd_dev_f32(const magnet_mask_train_args* a, const float* pred_scale, void* stream) {
  return mask_train_fwd(a, pred_scale, true, false, stream);
}

int magnet_mask_train_fwd_det_f32(const magnet_mask_train_args* a, void* stream) {
  return mask_train_fwd(a, a ? a->pred_scale : nullptr, false, true, stream);
}

int magnet_mask_train_fwd_dev_det_f32(const magnet_mask_train_args* a, const float* pred_scale, void* stream) {
  return mask_train_fwd(a, pred_scale, true, true, stream);
}

int magnet_mask_bwd_f32(const magnet_mask_train_args* a, void* stream) {
  const int st = validate_mask_train(a);
  if (st != MAGNET_OK) return st;
  if (!a->grad_scale || !a->workspace) return MAGNET_ERR_NULL;
  if (misaligned16(a->workspace)) return MAGNET_ERR_ALIGN;
  int launches = 0;
  const cudaError_t e = magnet::launch_mask_bwd(a->P, a->B, a->H, a->W, a->packed_weights, a->saved, a->grad_scale,
                                                a->workspace, a->grad_pre0, a->grad_w1, a->grad_b1, a->grad_w2,
                                                a->grad_b2, a->grad_w3, a->grad_b3, a->grad_pred, (cudaStream_t)stream,
                                                &launches);
  return finish(e, launches);
}

int64_t magnet_depth_metrics_workspace(const magnet_depth_metrics_args* a) {
  const int st = validate_depth_metrics_shape(a);
  if (st != MAGNET_OK) return st;
  return (int64_t)magnet::depth_metrics_workspace(a->P, a->B, a->row1 - a->row0, a->col1 - a->col0);
}

int magnet_depth_metrics_f32(const magnet_depth_metrics_args* a, void* stream) {
  const int st = validate_depth_metrics_shape(a);
  if (st != MAGNET_OK) return st;
  if (!a->pred || !a->gt || !a->workspace || !a->out || (a->k > 0 && !a->up_mask)) return MAGNET_ERR_NULL;
  if (preds_null(a->pred, a->P)) return MAGNET_ERR_NULL;
  return finish(magnet::launch_depth_metrics(a->pred, a->P, a->k > 0 ? a->up_mask : nullptr, a->gt, a->B, a->H, a->W,
                                             a->k, 0, 0, false, a->row0, a->row1, a->col0, a->col1, a->min_depth,
                                             a->max_depth, a->workspace, a->out, (cudaStream_t)stream), 2);
}

int magnet_depth_metrics_var_f32(const magnet_depth_metrics_args* a, void* stream) {
  const int st = validate_depth_metrics_shape(a);
  if (st != MAGNET_OK) return st;
  if (a->k != 0) return MAGNET_ERR_UNSUPPORTED;
  if (!a->pred || !a->gt || !a->workspace || !a->out) return MAGNET_ERR_NULL;
  if (preds_null(a->pred, a->P)) return MAGNET_ERR_NULL;
  return finish(magnet::launch_depth_metrics(a->pred, a->P, nullptr, a->gt, a->B, a->H, a->W, 0, 0, 0, true, a->row0,
                                             a->row1, a->col0, a->col1, a->min_depth, a->max_depth, a->workspace,
                                             a->out, (cudaStream_t)stream), 2);
}

size_t magnet_dnet_weights_bytes(int32_t k) {
  return k == 0 || k == 4 ? magnet::dnet_weights_bytes(k == 4) : 0;
}

int magnet_dnet_pack_weights_f32(const float* d_w1, const float* d_b1, const float* d_w2, const float* d_b2,
                                 const float* m_w1, const float* m_b1, const float* m_w3, const float* m_b3, int32_t k,
                                 void* packed, void* stream) {
  if (k != 0 && k != 4) return MAGNET_ERR_UNSUPPORTED;
  if (!d_w1 || !d_b1 || !d_w2 || !d_b2 || !packed) return MAGNET_ERR_NULL;
  if (k == 4 && (!m_w1 || !m_b1 || !m_w3 || !m_b3)) return MAGNET_ERR_NULL;
  if (misaligned16(packed)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_dnet_pack(d_w1, d_b1, d_w2, d_b2, m_w1, m_b1, m_w3, m_b3, k == 4, packed,
                                         (cudaStream_t)stream), 2);
}

int magnet_dnet_depth_f32(const float* pre_d, const void* packed, int32_t B, int32_t H, int32_t W, int32_t sigma,
                          float* out, void* stream) {
  if (!pixels_ok(B, H, W)) return MAGNET_ERR_SHAPE;
  if (!pre_d || !packed || !out) return MAGNET_ERR_NULL;
  if (misaligned16(pre_d) || misaligned16(packed) || misaligned16(out)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_dnet_depth(B, H, W, pre_d, packed, sigma != 0, out, (cudaStream_t)stream), 1);
}

int magnet_dnet_upsample_f32(const float* pre_m, const void* packed, const float* raw, int32_t B, int32_t H, int32_t W,
                             int32_t k, float* out, void* stream) {
  if (!pixels_ok(B, H, W)) return MAGNET_ERR_SHAPE;
  if (k != 4) return MAGNET_ERR_UNSUPPORTED;
  if (!pre_m || !packed || !raw || !out) return MAGNET_ERR_NULL;
  if (misaligned16(pre_m) || misaligned16(packed) || misaligned16(raw) || misaligned16(out)) return MAGNET_ERR_ALIGN;
  return finish(magnet::launch_dnet_upsample_packed(B, H, W, pre_m, packed, raw, out, (cudaStream_t)stream), 1);
}

int magnet_plane_depth_f32(const float* volume, const float* planes_host, int32_t B, int32_t D, int32_t H, int32_t W,
                           int32_t scores, float* out, void* stream) {
  if (!volume || !planes_host || !out) return MAGNET_ERR_NULL;
  const int st = validate_planes_shape(B, D, H, W);
  if (st != MAGNET_OK) return st;
  return finish(magnet::launch_plane_depth(volume, planes_host, B, D, H * W, scores != 0, out, (cudaStream_t)stream), 1);
}

int64_t magnet_depth_metrics_nearest_workspace(const magnet_depth_metrics_nearest_args* a) {
  const int st = validate_depth_metrics_nearest_shape(a);
  if (st != MAGNET_OK) return st;
  return (int64_t)magnet::depth_metrics_workspace(a->P, a->B, a->row1 - a->row0, a->col1 - a->col0);
}

int magnet_depth_metrics_nearest_f32(const magnet_depth_metrics_nearest_args* a, void* stream) {
  const int st = validate_depth_metrics_nearest_shape(a);
  if (st != MAGNET_OK) return st;
  if (!a->pred || !a->gt || !a->workspace || !a->out) return MAGNET_ERR_NULL;
  if (preds_null(a->pred, a->P)) return MAGNET_ERR_NULL;
  return finish(magnet::launch_depth_metrics(a->pred, a->P, nullptr, a->gt, a->B, a->H, a->W, 0, a->h, a->w, false,
                                             a->row0, a->row1, a->col0, a->col1, a->min_depth, a->max_depth,
                                             a->workspace, a->out, (cudaStream_t)stream), 2);
}

}  // extern "C"
