// C-ABI entry points declared in include/magnet_b200.h: argument validation + dispatch only.
#include <atomic>
#include <cstdlib>
#include <cstdio>
#include <cstring>

#include "common.cuh"

namespace magnet {
cudaError_t launch_cost_direct(const CostParams& p, int depth_mode, int src_layout, int C, bool cw,
                               bool softmax, cudaStream_t st, int* launches);
cudaError_t launch_cost_cells(const CostParams& p, int mode, int C, bool cw, bool reuse, cudaStream_t st);
cudaError_t launch_softmax_planes(float* vol, int B, int D, int HW, cudaStream_t st);
bool cells_supports(int C, int D, int layout);
cudaError_t launch_cost_tma(const CostParams& p, int mode, int C, bool cw, cudaStream_t st);
bool tma_supports(int C, int D, int V, int layout);
void tma_launch_info(int B, int H, int W, int D, int* grid, int* block, int* smem);
cudaError_t launch_cost_mma(const CostParams& p, int mode, bool cw, int layout, cudaStream_t st);
bool mma_supports(int C, int D, int V, int layout);
void mma_launch_info(int B, int H, int W, int D, int* grid, int* block, int* smem);
size_t split16_buffer_bytes(int N, int H, int W);
size_t half16_buffer_bytes(int N, int H, int W);
cudaError_t launch_repack_split16(const float* src, const float* gmm, void* dst, int N, int C, int H, int W,
                                  cudaStream_t st, int* launches);
cudaError_t launch_repack_half16(const void* src, int dtype, const float* gmm, void* dst, int N, int C, int H, int W,
                                 cudaStream_t st, int* launches);
#if defined(MAGNET_MMA_DEBUG) || defined(MAGNET_MMA_PROFILE)
void mma_set_debug_buffer(float* p);
#endif
cudaError_t launch_repack_pixc(const float* src, const float* gmm, float* dst, int N, int C, int H, int W,
                               cudaStream_t st);
void cells_launch_info(int B, int H, int W, int D, int* grid, int* block, int* smem);
cudaError_t launch_pack_cameras(const float* intM, const float* R, int64_t r_sb, int64_t r_sv, int64_t r_si,
                                int64_t r_sj, const float* t, int64_t t_sb, int64_t t_sv, int64_t t_si,
                                const int32_t* is_valid, int B, int V, magnet_camera* out, cudaStream_t st);
cudaError_t launch_repack(const float* src, float* dst, int N, int C, int H, int W, cudaStream_t st);
cudaError_t launch_sample(const float* gmm, const float* k_host, int B, int D, int HW, float* dvol,
                          cudaStream_t st);
cudaError_t launch_update_fwd(const float* dout, const float* gmm0, int B, int HW, float* out, cudaStream_t st);
cudaError_t launch_update_bwd(const float* gout, const float* dout, const float* gmm0, int B, int HW, float* gin,
                              cudaStream_t st);
cudaError_t launch_relative_poses(const float* ext_ref, const float* ext_nghbr, int B, int V, float* poses,
                                  int32_t* valid, cudaStream_t st);
cudaError_t launch_camera_rays(const double* raw, int B, int H, int W, float* intM, float* rays, cudaStream_t st);
cudaError_t launch_upsample_fwd(const float* depth, const float* mask, int B, int CH, int H, int W, int k, float* out,
                                cudaStream_t st);
cudaError_t launch_upsample_bwd(const float* gout, const float* depth, const float* mask, int B, int CH, int H, int W,
                                int k, float* gdepth, float* gmask, cudaStream_t st);
cudaError_t launch_cost_f_bwd(const BwdParams& p, cudaStream_t st, int* launches);
cudaError_t launch_cost_f_bwd_mma(const BwdParams& p, int layout, cudaStream_t st, int* launches);
bool f_bwd_mma_supports(int C, int V);
cudaError_t launch_cost_cw_bwd(const CwBwdParams& p, const CwBwdParams* split, int split_layout, int C, int mode,
                               bool mask_mma, const float* grad_out, cudaStream_t st, int* launches);
bool cw_bwd_supports(int C);
size_t geom_workspace_bytes(int B, int V, int H, int W);
cudaError_t launch_cost_geom_bwd(const CwBwdParams& p, int C, int mode, bool mask_mma, int softmax, const float* prob,
                                 const float* grad_out, float* partials, float* grad_rays, float* grad_cams,
                                 cudaStream_t st, int* launches);
#ifdef MAGNET_MMA_DEBUG
void f_bwd_mma_set_debug_buffer(float* p);
#endif
int fnet_l1_partials(int B, int HW);
cudaError_t launch_fnet_l1_fwd(const float* scores, const float* planes, const float* gt, const uint8_t* mask, int B,
                               int D, int HW, float* partial, cudaStream_t st);
cudaError_t launch_fnet_l1_bwd(const float* scores, const float* planes, const float* gt, const uint8_t* mask,
                               float scale, const float* grad_scale, int B, int D, int HW, float* grad_scores,
                               cudaStream_t st);
cudaError_t launch_upsample_nll_fwd(const float* depth, const float* mask, const float* gt, const uint8_t* gtm, int B,
                                    int H, int W, int k, float* partial, cudaStream_t st);
cudaError_t launch_upsample_nll_bwd(const float* depth, const float* mask, const float* gt, const uint8_t* gtm, float scale,
                                    int B, int H, int W, int k, float* gdepth, float* gmask, cudaStream_t st);
cudaError_t launch_plane_depth(const float* vol, const float* planes, int B, int D, int HW, bool scores, float* out,
                               cudaStream_t st);
size_t depth_metrics_workspace(int P, int B, int rows, int cols);
cudaError_t launch_depth_metrics(const float* const* preds, int P, const float* up_mask, const float* gt, int B, int H,
                                 int W, int k, int h, int w, bool variance, int r0, int r1, int c0, int c1, float min_d,
                                 float max_d, double* partial, double* out, cudaStream_t st);
size_t dnet_weights_bytes(bool with_mask);
cudaError_t launch_dnet_pack(const float* dw1, const float* db1, const float* dw2, const float* db2, const float* mw1,
                             const float* mb1, const float* mw3, const float* mb3, bool with_mask, void* dst,
                             cudaStream_t st, int* launches);
cudaError_t launch_dnet_depth(int B, int H, int W, const float* pre_d, const void* weights, bool sigma, float* out,
                              cudaStream_t st);
cudaError_t launch_dnet_upsample_packed(int B, int H, int W, const float* pre_m, const void* weights, const float* raw,
                                        float* out, cudaStream_t st);
size_t gnet_weights_bytes(int D);
cudaError_t launch_gnet_pack(const float* w0, const float* w1, const float* b1, const float* w2, const float* b2,
                             const float* w3, const float* b3, int D, void* dst, cudaStream_t st);
cudaError_t launch_gnet_update(int B, int D, int H, int W, const float* cost, const float* inv, const void* weights,
                               const float* prev, unsigned* scratch, float* out, cudaStream_t st);
size_t gnet_train_weights_bytes(int D);
size_t mask_weights_bytes();
cudaError_t launch_mask_pack(const float* w1, const float* b1, const float* w2, const float* b2, const float* w3,
                             const float* b3, void* dst, cudaStream_t st);
cudaError_t launch_mask_upsample(int P, int B, int H, int W, const float* pre0, const void* weights,
                                 const float* const* pred, float* const* out, cudaStream_t st);
size_t mask_train_weights_bytes();
int mask_train_partials(int B, int H, int W);
size_t mask_saved_bytes(int P, int B, int H, int W);
size_t mask_bwd_workspace_bytes(int B, int H, int W);
cudaError_t launch_mask_pack_train(const float* w1, const float* b1, const float* w2, const float* b2, const float* w3,
                                   const float* b3, void* dst, cudaStream_t st);
cudaError_t launch_mask_train_fwd(int P, int B, int H, int W, const float* pre0, const void* weights,
                                  const float* const* pred, const float* gt, const unsigned char* gtm,
                                  const float* scale, bool save_maps, bool pred_grad, float* partial, float* saved,
                                  cudaStream_t st, int* launches);
cudaError_t launch_mask_bwd(int P, int B, int H, int W, const void* weights, const float* saved, const float* gscale,
                            void* workspace, float* grad_pre0, float* gw1, float* gb1, float* gw2, float* gb2,
                            float* gw3, float* gb3, float* const* grad_pred, cudaStream_t st, int* launches);
size_t gnet_saved_bytes(int B, int H, int W);
size_t gnet_bwd_workspace_bytes(int B, int D, int H, int W);
cudaError_t launch_gnet_pack_train(const float* w0, const float* w1, const float* b1, const float* w2, const float* b2,
                                   const float* w3, const float* b3, int D, void* dst, cudaStream_t st);
cudaError_t launch_gnet_train_fwd(int B, int D, int H, int W, const float* cost, const float* inv, const void* weights,
                                  const float* prev, unsigned* scratch, float* out, float* saved, cudaStream_t st);
cudaError_t launch_gnet_bwd(int B, int D, int H, int W, const float* cost, const float* prev, const void* weights,
                            const float* saved, const float* grad, void* workspace, float* grad_inv, float* gw0,
                            float* gw1, float* gb1, float* gw2, float* gb2, float* gw3, float* gb3, float* grad_prev,
                            cudaStream_t st, int* launches);
}  // namespace magnet

namespace {
std::atomic<uint64_t> g_launches{0};
thread_local char g_cuda_err[256] = "";

// the tensor-core layouts: a header + fp16 plane(s) + (mu, sigma) table per buffer, ref_feat included
bool packed_layout(int layout) { return layout == MAGNET_SRC_SPLIT16 || layout == MAGNET_SRC_HALF16; }

int cuda_fail(cudaError_t e) {
  snprintf(g_cuda_err, sizeof(g_cuda_err), "%s: %s", cudaGetErrorName(e), cudaGetErrorString(e));
  return MAGNET_ERR_CUDA;
}

int validate_cost(const magnet_cost_args* a) {
  if (!a) return MAGNET_ERR_NULL;
  if (a->B <= 0 || a->V <= 0 || a->D <= 0 || a->C <= 0 || a->H <= 0 || a->W <= 0) return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if ((int64_t)a->H * a->W > (1 << 26)) return MAGNET_ERR_SHAPE;
  if (!a->ref_feat || !a->src_feat || !a->rays || !a->cams || !a->out) return MAGNET_ERR_NULL;
  if (a->consistency && !a->src_gmm && a->src_layout != MAGNET_SRC_PIXC && !packed_layout(a->src_layout))
    return MAGNET_ERR_NULL;
  if (a->consistency && a->softmax) return MAGNET_ERR_UNSUPPORTED;
  switch (a->depth_mode) {
    case MAGNET_DEPTH_VOLUME: if (!a->d_volume) return MAGNET_ERR_NULL; break;
    case MAGNET_DEPTH_GAUSS: if (!a->ref_gmm || !a->k_host) return MAGNET_ERR_NULL; break;
    case MAGNET_DEPTH_PLANES: if (!a->k_host) return MAGNET_ERR_NULL; break;
    default: return MAGNET_ERR_UNSUPPORTED;
  }
  if (a->src_layout == MAGNET_SRC_TILED32) {
    if (a->C % 4 != 0) return MAGNET_ERR_UNSUPPORTED;
    if (reinterpret_cast<uintptr_t>(a->src_feat) % 16 != 0) return MAGNET_ERR_ALIGN;
  } else if (a->src_layout == MAGNET_SRC_PIXC) {
    if (!magnet::tma_supports(a->C, a->D, a->V, a->src_layout)) return MAGNET_ERR_UNSUPPORTED;
    if (reinterpret_cast<uintptr_t>(a->src_feat) % 16 != 0) return MAGNET_ERR_ALIGN;
    if (a->variant != MAGNET_VARIANT_AUTO && a->variant != MAGNET_VARIANT_TMA) return MAGNET_ERR_UNSUPPORTED;
  } else if (packed_layout(a->src_layout)) {
    if (!magnet::mma_supports(a->C, a->D, a->V, a->src_layout)) return MAGNET_ERR_UNSUPPORTED;
    if (reinterpret_cast<uintptr_t>(a->src_feat) % 16 != 0 || reinterpret_cast<uintptr_t>(a->ref_feat) % 16 != 0)
      return MAGNET_ERR_ALIGN;
    if (a->variant != MAGNET_VARIANT_AUTO && a->variant != MAGNET_VARIANT_MMA) return MAGNET_ERR_UNSUPPORTED;
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

int magnet_cost_volume_f32(const magnet_cost_args* a, void* stream) {
  const int st = validate_cost(a);
  if (st != MAGNET_OK) return st;
  magnet::CostParams p;
  p.B = a->B; p.V = a->V; p.D = a->D; p.H = a->H; p.W = a->W; p.HW = a->H * a->W;
  p.kappa = a->kappa;
  p.vf = (float)a->V;
  p.inv_v_exact = ((a->V & (a->V - 1)) == 0) ? 1.0f / (float)a->V : 0.0f;
  p.ref_feat = a->ref_feat; p.src_feat = a->src_feat; p.src_gmm = a->src_gmm; p.rays = a->rays;
  p.cams = a->cams; p.d_volume = a->d_volume; p.ref_gmm = a->ref_gmm; p.out = a->out;
  for (int j = 0; j < MAGNET_MAX_PLANES; ++j)
    p.k[j] = (a->depth_mode != MAGNET_DEPTH_VOLUME && j < a->D) ? a->k_host[j] : 0.0f;
  p.k_sorted = 1;
  for (int j = 1; j < a->D; ++j)
    if (!(p.k[j] >= p.k[j - 1])) p.k_sorted = 0;
  int launches = 0;
  cudaError_t e;
  if (use_mma(a) || use_tma(a) || use_cells(a)) {
    if (use_mma(a))
      e = magnet::launch_cost_mma(p, a->depth_mode, a->consistency != 0, a->src_layout, (cudaStream_t)stream);
    else if (use_tma(a))
      e = magnet::launch_cost_tma(p, a->depth_mode, a->C, a->consistency != 0, (cudaStream_t)stream);
    else
      e = magnet::launch_cost_cells(p, a->depth_mode, a->C, a->consistency != 0,
                                    a->variant != MAGNET_VARIANT_CELLS_NOREUSE, (cudaStream_t)stream);
    launches = 1;
    if (e == cudaSuccess && a->softmax) {          // homography.py:46, in place on the 1/V-averaged scores
      e = magnet::launch_softmax_planes(a->out, a->B, a->D, a->H * a->W, (cudaStream_t)stream);
      launches = 2;
    }
  } else {
    e = magnet::launch_cost_direct(p, a->depth_mode, a->src_layout, a->C, a->consistency != 0, a->softmax != 0,
                                   (cudaStream_t)stream, &launches);
  }
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += launches;
  return MAGNET_OK;
}

int magnet_cost_volume_f_bwd_f32(const magnet_cost_f_bwd_args* b, void* stream) {
  if (!b || !b->fwd) return MAGNET_ERR_NULL;
  const magnet_cost_args* a = b->fwd;
  if (a->B <= 0 || a->V <= 0 || a->D <= 0 || a->C <= 0 || a->H <= 0 || a->W <= 0) return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if (!a->ref_feat || !a->src_feat || !a->rays || !a->cams || !a->k_host) return MAGNET_ERR_NULL;
  if (!b->grad_out || !b->workspace || !b->grad_ref || !b->grad_src) return MAGNET_ERR_NULL;
  if (a->softmax && !b->prob) return MAGNET_ERR_NULL;
  if (a->consistency || a->depth_mode != MAGNET_DEPTH_PLANES) return MAGNET_ERR_UNSUPPORTED;
  const bool mma = packed_layout(a->src_layout);
  if (mma) {                                   // tensor-core backward on the forward's SPLIT16 / HALF16 buffers
    if (a->variant != MAGNET_VARIANT_AUTO && a->variant != MAGNET_VARIANT_MMA) return MAGNET_ERR_UNSUPPORTED;
    if (!magnet::f_bwd_mma_supports(a->C, a->V)) return MAGNET_ERR_UNSUPPORTED;
    if (reinterpret_cast<uintptr_t>(a->src_feat) % 16 != 0 || reinterpret_cast<uintptr_t>(a->ref_feat) % 16 != 0)
      return MAGNET_ERR_ALIGN;
  } else {
    if (a->src_layout != MAGNET_SRC_NCHW) return MAGNET_ERR_UNSUPPORTED;
    if (a->C != 8 && a->C != 16 && a->C != 32 && a->C != 64) return MAGNET_ERR_UNSUPPORTED;
  }
  magnet::BwdParams p;
  p.B = a->B; p.V = a->V; p.D = a->D; p.C = a->C; p.H = a->H; p.W = a->W; p.HW = a->H * a->W;
  p.softmax = a->softmax != 0;
  p.vf = (float)a->V;
  p.ref_feat = a->ref_feat; p.src_feat = a->src_feat; p.rays = a->rays; p.cams = a->cams;
  p.prob = b->prob; p.grad_out = b->grad_out; p.g_score = b->workspace; p.grad_ref = b->grad_ref; p.grad_src = b->grad_src;
  for (int j = 0; j < MAGNET_MAX_PLANES; ++j) p.k[j] = j < a->D ? a->k_host[j] : 0.0f;
  int launches = 0;
  cudaError_t e = mma ? magnet::launch_cost_f_bwd_mma(p, a->src_layout, (cudaStream_t)stream, &launches)
                      : magnet::launch_cost_f_bwd(p, (cudaStream_t)stream, &launches);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += launches;
  return MAGNET_OK;
}

int magnet_cost_volume_bwd_f32(const magnet_cost_bwd_args* b, void* stream) {
  if (!b || !b->fwd) return MAGNET_ERR_NULL;
  const magnet_cost_args* a = b->fwd;
  if (a->B <= 0 || a->V <= 0 || a->D <= 0 || a->C <= 0 || a->H <= 0 || a->W <= 0) return MAGNET_ERR_SHAPE;
  if ((int64_t)a->H * a->W > (1 << 26) || a->B > 65535) return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if (!a->rays || !a->cams || !b->grad_out || !b->workspace) return MAGNET_ERR_NULL;
  if (a->softmax) return MAGNET_ERR_UNSUPPORTED;
  switch (a->depth_mode) {
    case MAGNET_DEPTH_VOLUME: if (!a->d_volume) return MAGNET_ERR_NULL; break;
    case MAGNET_DEPTH_GAUSS: if (!a->ref_gmm || !a->k_host) return MAGNET_ERR_NULL; break;
    default: return MAGNET_ERR_UNSUPPORTED;
  }
  const bool mask_mma = packed_layout(a->src_layout);   // the tensor-core forward's mask
  // its split buffers given: feature gradients on the tensor cores; both NULL: everything on the CUDA cores
  const bool split = mask_mma && (a->ref_feat || a->src_feat);
  if (mask_mma) {
    if (a->variant != MAGNET_VARIANT_AUTO && a->variant != MAGNET_VARIANT_MMA) return MAGNET_ERR_UNSUPPORTED;
    if (!magnet::mma_supports(a->C, a->D, a->V, a->src_layout) || !magnet::f_bwd_mma_supports(a->C, a->V))
      return MAGNET_ERR_UNSUPPORTED;
  }
  if (split) {
    if (!a->ref_feat || !a->src_feat) return MAGNET_ERR_NULL;
    if (reinterpret_cast<uintptr_t>(a->src_feat) % 16 != 0 || reinterpret_cast<uintptr_t>(a->ref_feat) % 16 != 0)
      return MAGNET_ERR_ALIGN;
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
  magnet::CwBwdParams p;
  p.B = a->B; p.V = a->V; p.D = a->D; p.H = a->H; p.W = a->W; p.HW = a->H * a->W;
  p.cw = a->consistency != 0;
  p.kappa = a->kappa;
  p.ref_feat = b->ref_feat; p.src_feat = b->src_feat; p.src_gmm = b->src_gmm; p.rays = a->rays; p.cams = a->cams;
  p.d_volume = a->d_volume; p.ref_gmm = a->ref_gmm;
  p.g_score = b->workspace;
  p.grad_ref = b->grad_ref; p.grad_src = b->grad_src; p.grad_depth = b->grad_depth;
  for (int j = 0; j < MAGNET_MAX_PLANES; ++j)
    p.k[j] = (a->depth_mode == MAGNET_DEPTH_GAUSS && j < a->D) ? a->k_host[j] : 0.0f;
  magnet::CwBwdParams ps = p;
  ps.ref_feat = a->ref_feat; ps.src_feat = a->src_feat; ps.src_gmm = nullptr; ps.grad_depth = nullptr;
  int launches = 0;
  cudaError_t e = magnet::launch_cost_cw_bwd(p, split ? &ps : nullptr, a->src_layout, a->C, a->depth_mode, mask_mma,
                                             b->grad_out, (cudaStream_t)stream, &launches);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += launches;
  return MAGNET_OK;
}

size_t magnet_cost_geom_workspace_bytes(int32_t B, int32_t V, int32_t H, int32_t W) {
  if (B <= 0 || V <= 0 || H <= 0 || W <= 0) return 0;
  return magnet::geom_workspace_bytes(B, V, H, W);
}

int magnet_cost_volume_geom_bwd_f32(const magnet_cost_geom_bwd_args* b, void* stream) {
  if (!b || !b->fwd) return MAGNET_ERR_NULL;
  const magnet_cost_args* a = b->fwd;
  if (a->B <= 0 || a->V <= 0 || a->D <= 0 || a->C <= 0 || a->H <= 0 || a->W <= 0) return MAGNET_ERR_SHAPE;
  if ((int64_t)a->H * a->W > (1 << 26) || a->B > 65535 || (int64_t)a->B * a->V > (1 << 30)) return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES || !magnet::cw_bwd_supports(a->C)) return MAGNET_ERR_UNSUPPORTED;
  if (!a->rays || !a->cams || !b->ref_feat || !b->src_feat || !b->grad_out || !b->score || !b->workspace ||
      !b->grad_cams)
    return MAGNET_ERR_NULL;
  bool mask_mma = false;
  switch (a->depth_mode) {
    case MAGNET_DEPTH_VOLUME: if (!a->d_volume) return MAGNET_ERR_NULL; break;
    case MAGNET_DEPTH_GAUSS: if (!a->ref_gmm || !a->k_host) return MAGNET_ERR_NULL; break;
    case MAGNET_DEPTH_PLANES: if (!a->k_host) return MAGNET_ERR_NULL; break;
    default: return MAGNET_ERR_UNSUPPORTED;
  }
  if (a->depth_mode == MAGNET_DEPTH_PLANES) {      // the F volume: no mask, the tensor-core forward's positions
    if (a->consistency || b->grad_depth) return MAGNET_ERR_UNSUPPORTED;
    if (a->softmax && !b->prob) return MAGNET_ERR_NULL;
  } else {
    if (a->softmax) return MAGNET_ERR_UNSUPPORTED;
    mask_mma = packed_layout(a->src_layout);     // the tensor-core forward's mask, else the DIRECT forward's
    if (mask_mma) {
      if (a->variant != MAGNET_VARIANT_AUTO && a->variant != MAGNET_VARIANT_MMA) return MAGNET_ERR_UNSUPPORTED;
      if (!magnet::mma_supports(a->C, a->D, a->V, a->src_layout)) return MAGNET_ERR_UNSUPPORTED;
    } else if (a->variant != MAGNET_VARIANT_DIRECT ||
               (a->src_layout != MAGNET_SRC_NCHW && a->src_layout != MAGNET_SRC_TILED32)) {
      return MAGNET_ERR_UNSUPPORTED;
    }
    if (a->consistency && !b->src_gmm) return MAGNET_ERR_NULL;
  }
  if (reinterpret_cast<uintptr_t>(b->workspace) % 16 != 0) return MAGNET_ERR_ALIGN;
  magnet::CwBwdParams p;
  p.B = a->B; p.V = a->V; p.D = a->D; p.H = a->H; p.W = a->W; p.HW = a->H * a->W;
  p.cw = a->consistency != 0;
  p.kappa = a->kappa;
  p.ref_feat = b->ref_feat; p.src_feat = b->src_feat; p.src_gmm = b->src_gmm; p.rays = a->rays; p.cams = a->cams;
  p.d_volume = a->d_volume; p.ref_gmm = a->ref_gmm;
  p.g_score = b->score;
  p.grad_ref = p.grad_src = nullptr;
  p.grad_depth = b->grad_depth;
  for (int j = 0; j < MAGNET_MAX_PLANES; ++j)
    p.k[j] = (a->depth_mode != MAGNET_DEPTH_VOLUME && j < a->D) ? a->k_host[j] : 0.0f;
  int launches = 0;
  cudaError_t e = magnet::launch_cost_geom_bwd(p, a->C, a->depth_mode, mask_mma, a->softmax != 0, b->prob, b->grad_out,
                                               static_cast<float*>(b->workspace), b->grad_rays, b->grad_cams,
                                               (cudaStream_t)stream, &launches);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += launches;
  return MAGNET_OK;
}

int magnet_pack_cameras_f32(const float* intM, const float* R, int64_t r_sb, int64_t r_sv, int64_t r_si,
                            int64_t r_sj, const float* t, int64_t t_sb, int64_t t_sv, int64_t t_si,
                            const int32_t* is_valid, int32_t B, int32_t V, magnet_camera* cams_out,
                            void* stream) {
  if (!intM || !R || !t || !is_valid || !cams_out) return MAGNET_ERR_NULL;
  if (B <= 0 || V <= 0) return MAGNET_ERR_SHAPE;
  cudaError_t e = magnet::launch_pack_cameras(intM, R, r_sb, r_sv, r_si, r_sj, t, t_sb, t_sv, t_si, is_valid, B, V,
                                              cams_out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_repack_tiled32_f32(const float* src_nchw, float* dst, int32_t N, int32_t C, int32_t H, int32_t W,
                            void* stream) {
  if (!src_nchw || !dst) return MAGNET_ERR_NULL;
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0) return MAGNET_ERR_SHAPE;
  if (C % 4 != 0 || C / 4 > 65535 || N > 65535) return MAGNET_ERR_UNSUPPORTED;
  if (reinterpret_cast<uintptr_t>(dst) % 16 != 0) return MAGNET_ERR_ALIGN;
  cudaError_t e = magnet::launch_repack(src_nchw, dst, N, C, H, W, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_repack_pixc_f32(const float* src_nchw, const float* src_gmm, float* dst, int32_t N, int32_t C, int32_t H,
                           int32_t W, void* stream) {
  if (!src_nchw || !dst) return MAGNET_ERR_NULL;
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0 || N > 65535) return MAGNET_ERR_SHAPE;
  if (C != 16 && C != 32 && C != 64) return MAGNET_ERR_UNSUPPORTED;
  if (reinterpret_cast<uintptr_t>(dst) % 16 != 0) return MAGNET_ERR_ALIGN;
  cudaError_t e = magnet::launch_repack_pixc(src_nchw, src_gmm, dst, N, C, H, W, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
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
  if (reinterpret_cast<uintptr_t>(dst) % 16 != 0 || reinterpret_cast<uintptr_t>(src_nchw) % 16 != 0) return MAGNET_ERR_ALIGN;
  int launches = 0;
  cudaError_t e = magnet::launch_repack_split16(src_nchw, src_gmm, dst, N, C, H, W, (cudaStream_t)stream, &launches);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += launches;
  return MAGNET_OK;
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
  if (reinterpret_cast<uintptr_t>(dst) % 16 != 0 || reinterpret_cast<uintptr_t>(src_nchw) % 16 != 0) return MAGNET_ERR_ALIGN;
  int launches = 0;
  cudaError_t e = magnet::launch_repack_half16(src_nchw, dtype, src_gmm, dst, N, C, H, W, (cudaStream_t)stream, &launches);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += launches;
  return MAGNET_OK;
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
  cudaError_t e = magnet::launch_sample(gmm, k_host, B, D, HW, d_volume, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_gaussian_update_fwd_f32(const float* d_output, const float* ref_gmm, int32_t B, int32_t HW,
                                   float* out, void* stream) {
  if (!d_output || !ref_gmm || !out) return MAGNET_ERR_NULL;
  if (B <= 0 || HW <= 0 || B > 65535) return MAGNET_ERR_SHAPE;
  cudaError_t e = magnet::launch_update_fwd(d_output, ref_gmm, B, HW, out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_gaussian_update_bwd_f32(const float* grad_out, const float* d_output, const float* ref_gmm,
                                   int32_t B, int32_t HW, float* grad_d_output, void* stream) {
  if (!grad_out || !d_output || !ref_gmm || !grad_d_output) return MAGNET_ERR_NULL;
  if (B <= 0 || HW <= 0 || B > 65535) return MAGNET_ERR_SHAPE;
  cudaError_t e = magnet::launch_update_bwd(grad_out, d_output, ref_gmm, B, HW, grad_d_output, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_relative_poses_f32(const float* ext_ref, const float* ext_nghbr, int32_t B, int32_t V, float* poses_out,
                              int32_t* is_valid_out, void* stream) {
  if (!ext_ref || !ext_nghbr || !poses_out || !is_valid_out) return MAGNET_ERR_NULL;
  if (B <= 0 || V <= 0) return MAGNET_ERR_SHAPE;
  cudaError_t e = magnet::launch_relative_poses(ext_ref, ext_nghbr, B, V, poses_out, is_valid_out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_camera_rays_f32(const double* raw_intrinsics, int32_t B, int32_t H, int32_t W, float* intM_out,
                           float* rays_out, void* stream) {
  if (!raw_intrinsics || !intM_out || !rays_out) return MAGNET_ERR_NULL;
  if (B <= 0 || H <= 0 || W <= 0 || B > 65535) return MAGNET_ERR_SHAPE;
  cudaError_t e = magnet::launch_camera_rays(raw_intrinsics, B, H, W, intM_out, rays_out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_convex_upsample_fwd_f32(const float* depth, const float* up_mask, int32_t B, int32_t CH, int32_t H,
                                   int32_t W, int32_t k, float* out, void* stream) {
  if (!depth || !up_mask || !out) return MAGNET_ERR_NULL;
  if (B <= 0 || H <= 0 || W <= 0 || k <= 0 || B > 65535 || H * k > 65535) return MAGNET_ERR_SHAPE;
  if (CH != 1 && CH != 2) return MAGNET_ERR_UNSUPPORTED;
  cudaError_t e = magnet::launch_upsample_fwd(depth, up_mask, B, CH, H, W, k, out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_convex_upsample_bwd_f32(const float* grad_out, const float* depth, const float* up_mask, int32_t B,
                                   int32_t CH, int32_t H, int32_t W, int32_t k, float* grad_depth, float* grad_mask,
                                   void* stream) {
  if (!grad_out || !depth || !up_mask || !grad_depth || !grad_mask) return MAGNET_ERR_NULL;
  if (B <= 0 || H <= 0 || W <= 0 || k <= 0 || B > 65535 || H * k > 65535) return MAGNET_ERR_SHAPE;
  if (CH != 1 && CH != 2) return MAGNET_ERR_UNSUPPORTED;
  cudaError_t e = magnet::launch_upsample_bwd(grad_out, depth, up_mask, B, CH, H, W, k, grad_depth, grad_mask,
                                              (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_upsample_nll_partials(int32_t B, int32_t H, int32_t W, int32_t k) {
  if (B <= 0 || H <= 0 || W <= 0 || k <= 0) return MAGNET_ERR_SHAPE;
  return B * H * k * ((W * k + 127) / 128);
}

int magnet_upsample_nll_fwd_f32(const float* depth, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                int32_t B, int32_t H, int32_t W, int32_t k, float* partial, void* stream) {
  if (!depth || !up_mask || !gt || !gt_mask || !partial) return MAGNET_ERR_NULL;
  if (B <= 0 || H <= 0 || W <= 0 || k <= 0 || B > 65535 || H * k > 65535) return MAGNET_ERR_SHAPE;
  cudaError_t e = magnet::launch_upsample_nll_fwd(depth, up_mask, gt, gt_mask, B, H, W, k, partial, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_upsample_nll_bwd_f32(const float* depth, const float* up_mask, const float* gt, const uint8_t* gt_mask,
                                float scale, int32_t B, int32_t H, int32_t W, int32_t k, float* grad_depth,
                                float* grad_mask, void* stream) {
  if (!depth || !up_mask || !gt || !gt_mask || !grad_depth || !grad_mask) return MAGNET_ERR_NULL;
  if (B <= 0 || H <= 0 || W <= 0 || k <= 0 || B > 65535 || H * k > 65535) return MAGNET_ERR_SHAPE;
  cudaError_t e = magnet::launch_upsample_nll_bwd(depth, up_mask, gt, gt_mask, scale, B, H, W, k, grad_depth, grad_mask,
                                                  (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_fnet_l1_partials(int32_t B, int32_t H, int32_t W) {
  if (B <= 0 || H <= 0 || W <= 0) return MAGNET_ERR_SHAPE;
  return magnet::fnet_l1_partials(B, H * W);
}

namespace {
int validate_fnet_l1(const float* scores, const float* planes_host, const float* gt, const uint8_t* mask, int32_t B,
                     int32_t D, int32_t H, int32_t W) {
  if (!scores || !planes_host || !gt || !mask) return MAGNET_ERR_NULL;
  if (B <= 0 || D <= 0 || H <= 0 || W <= 0 || B > 65535) return MAGNET_ERR_SHAPE;
  if ((int64_t)H * W > (1 << 26)) return MAGNET_ERR_SHAPE;
  if (D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  return MAGNET_OK;
}
}  // namespace

int magnet_fnet_l1_fwd_f32(const float* scores, const float* planes_host, const float* gt, const uint8_t* mask, int32_t B,
                           int32_t D, int32_t H, int32_t W, float* partial, void* stream) {
  const int st = validate_fnet_l1(scores, planes_host, gt, mask, B, D, H, W);
  if (st != MAGNET_OK) return st;
  if (!partial) return MAGNET_ERR_NULL;
  cudaError_t e = magnet::launch_fnet_l1_fwd(scores, planes_host, gt, mask, B, D, H * W, partial, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_fnet_l1_bwd_f32(const float* scores, const float* planes_host, const float* gt, const uint8_t* mask,
                           float scale, const float* grad_scale, int32_t B, int32_t D, int32_t H, int32_t W,
                           float* grad_scores, void* stream) {
  const int st = validate_fnet_l1(scores, planes_host, gt, mask, B, D, H, W);
  if (st != MAGNET_OK) return st;
  if (!grad_scores) return MAGNET_ERR_NULL;
  cudaError_t e = magnet::launch_fnet_l1_bwd(scores, planes_host, gt, mask, scale, grad_scale, B, D, H * W, grad_scores,
                                             (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

namespace {
// Shape fields and box only (the sizing call needs no pointers).
int validate_depth_metrics_shape(const magnet_depth_metrics_args* a) {
  if (!a) return MAGNET_ERR_NULL;
  if (a->P <= 0 || a->B <= 0 || a->H <= 0 || a->W <= 0 || a->k < 0) return MAGNET_ERR_SHAPE;
  if (a->P > MAGNET_METRICS_MAX_PRED) return MAGNET_ERR_UNSUPPORTED;
  if ((int64_t)a->P * a->B > 65535 || (int64_t)a->H * a->W > (1 << 28)) return MAGNET_ERR_SHAPE;
  if (a->k > 0 && (a->H % a->k != 0 || a->W % a->k != 0)) return MAGNET_ERR_SHAPE;
  if (a->row0 < 0 || a->row0 > a->row1 || a->row1 > a->H) return MAGNET_ERR_SHAPE;
  if (a->col0 < 0 || a->col0 > a->col1 || a->col1 > a->W) return MAGNET_ERR_SHAPE;
  return MAGNET_OK;
}
}  // namespace

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
  if (reinterpret_cast<uintptr_t>(packed) % 16 != 0) return MAGNET_ERR_ALIGN;
  cudaError_t e = magnet::launch_gnet_pack(w0_cost, w1, b1, w2, b2, w3, b3, D, packed, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 2;
  return MAGNET_OK;
}

int magnet_gnet_update_f32(const magnet_gnet_args* a, void* stream) {
  if (!a) return MAGNET_ERR_NULL;
  if (a->B <= 0 || a->D <= 0 || a->H <= 0 || a->W <= 0) return MAGNET_ERR_SHAPE;
  if ((int64_t)a->H * a->W > (1 << 26) || (int64_t)a->B * ((a->H + 7) / 8) * ((a->W + 15) / 16) > (1 << 30))
    return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if (!a->cost || !a->invariant || !a->packed_weights || !a->prev_gmm || !a->scratch || !a->out) return MAGNET_ERR_NULL;
  if (reinterpret_cast<uintptr_t>(a->cost) % 16 != 0 || reinterpret_cast<uintptr_t>(a->invariant) % 16 != 0 ||
      reinterpret_cast<uintptr_t>(a->packed_weights) % 16 != 0 || reinterpret_cast<uintptr_t>(a->scratch) % 4 != 0)
    return MAGNET_ERR_ALIGN;
  cudaError_t e = magnet::launch_gnet_update(a->B, a->D, a->H, a->W, a->cost, a->invariant, a->packed_weights,
                                             a->prev_gmm, static_cast<unsigned*>(a->scratch), a->out,
                                             (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 2;
  return MAGNET_OK;
}

namespace {
bool misaligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 != 0; }

// shape and the pointers both training calls read
int validate_gnet_train(const magnet_gnet_train_args* a) {
  if (!a) return MAGNET_ERR_NULL;
  if (a->B <= 0 || a->D <= 0 || a->H <= 0 || a->W <= 0) return MAGNET_ERR_SHAPE;
  if ((int64_t)a->H * a->W > (1 << 26) || (int64_t)a->B * a->H * a->W >= ((int64_t)1 << 31)) return MAGNET_ERR_SHAPE;
  if (a->D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  if (!a->cost || !a->packed_weights || !a->prev_gmm || !a->saved) return MAGNET_ERR_NULL;
  if (misaligned16(a->cost) || misaligned16(a->packed_weights) || misaligned16(a->saved)) return MAGNET_ERR_ALIGN;
  return MAGNET_OK;
}
}  // namespace

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
  cudaError_t e = magnet::launch_gnet_pack_train(w0_cost, w1, b1, w2, b2, w3, b3, D, packed, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 3;
  return MAGNET_OK;
}

int magnet_gnet_train_fwd_f32(const magnet_gnet_train_args* a, void* stream) {
  const int st = validate_gnet_train(a);
  if (st != MAGNET_OK) return st;
  if (!a->invariant || !a->scratch || !a->out) return MAGNET_ERR_NULL;
  if (misaligned16(a->invariant) || reinterpret_cast<uintptr_t>(a->scratch) % 4 != 0) return MAGNET_ERR_ALIGN;
  cudaError_t e = magnet::launch_gnet_train_fwd(a->B, a->D, a->H, a->W, a->cost, a->invariant, a->packed_weights,
                                                a->prev_gmm, static_cast<unsigned*>(a->scratch), a->out, a->saved,
                                                (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 2;
  return MAGNET_OK;
}

int magnet_gnet_bwd_f32(const magnet_gnet_train_args* a, void* stream) {
  const int st = validate_gnet_train(a);
  if (st != MAGNET_OK) return st;
  if (!a->grad_out || !a->workspace || !a->grad_invariant) return MAGNET_ERR_NULL;
  if (misaligned16(a->workspace)) return MAGNET_ERR_ALIGN;
  int launches = 0;
  cudaError_t e = magnet::launch_gnet_bwd(a->B, a->D, a->H, a->W, a->cost, a->prev_gmm, a->packed_weights, a->saved,
                                          a->grad_out, a->workspace, a->grad_invariant, a->grad_w0_cost, a->grad_w1,
                                          a->grad_b1, a->grad_w2, a->grad_b2, a->grad_w3, a->grad_b3, a->grad_prev,
                                          (cudaStream_t)stream, &launches);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += launches;
  return MAGNET_OK;
}

size_t magnet_mask_weights_bytes(int32_t k) { return k == 4 ? magnet::mask_weights_bytes() : 0; }

int magnet_mask_pack_weights_f32(const float* w1, const float* b1, const float* w2, const float* b2, const float* w3,
                                 const float* b3, void* packed, void* stream) {
  if (!w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !packed) return MAGNET_ERR_NULL;
  if (misaligned16(packed)) return MAGNET_ERR_ALIGN;
  cudaError_t e = magnet::launch_mask_pack(w1, b1, w2, b2, w3, b3, packed, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 2;
  return MAGNET_OK;
}

int magnet_mask_upsample_f32(const magnet_mask_upsample_args* a, void* stream) {
  if (!a) return MAGNET_ERR_NULL;
  if (a->B <= 0 || a->H <= 0 || a->W <= 0) return MAGNET_ERR_SHAPE;
  if ((int64_t)a->B * a->H * a->W >= ((int64_t)1 << 31)) return MAGNET_ERR_SHAPE;
  if (a->P < 1 || a->P > MAGNET_MASK_MAX_PRED || a->k != 4) return MAGNET_ERR_UNSUPPORTED;
  if (!a->pre0 || !a->packed_weights || !a->pred || !a->out) return MAGNET_ERR_NULL;
  for (int p = 0; p < a->P; ++p)
    if (!a->pred[p] || !a->out[p]) return MAGNET_ERR_NULL;
  if (misaligned16(a->pre0) || misaligned16(a->packed_weights)) return MAGNET_ERR_ALIGN;
  for (int p = 0; p < a->P; ++p)
    if (misaligned16(a->pred[p]) || misaligned16(a->out[p])) return MAGNET_ERR_ALIGN;
  cudaError_t e = magnet::launch_mask_upsample(a->P, a->B, a->H, a->W, a->pre0, a->packed_weights, a->pred, a->out,
                                               (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

namespace {
bool mask_train_shape_ok(int32_t B, int32_t H, int32_t W) {
  return B > 0 && H > 0 && W > 0 && (int64_t)B * H * W < ((int64_t)1 << 31);
}

// shape, factor, prediction count and the pointers both training calls read
int validate_mask_train(const magnet_mask_train_args* a) {
  if (!a) return MAGNET_ERR_NULL;
  if (!mask_train_shape_ok(a->B, a->H, a->W)) return MAGNET_ERR_SHAPE;
  if (a->P < 1 || a->P > MAGNET_MASK_MAX_PRED || a->k != 4) return MAGNET_ERR_UNSUPPORTED;
  if (!a->packed_weights || !a->saved) return MAGNET_ERR_NULL;
  if (misaligned16(a->packed_weights) || misaligned16(a->saved)) return MAGNET_ERR_ALIGN;
  return MAGNET_OK;
}
}  // namespace

size_t magnet_mask_train_weights_bytes(int32_t k) { return k == 4 ? magnet::mask_train_weights_bytes() : 0; }

size_t magnet_mask_saved_bytes(int32_t P, int32_t B, int32_t H, int32_t W) {
  if (P < 1 || P > MAGNET_MASK_MAX_PRED || !mask_train_shape_ok(B, H, W)) return 0;
  return magnet::mask_saved_bytes(P, B, H, W);
}

size_t magnet_mask_bwd_workspace_bytes(int32_t B, int32_t H, int32_t W) {
  if (!mask_train_shape_ok(B, H, W)) return 0;
  return magnet::mask_bwd_workspace_bytes(B, H, W);
}

int magnet_mask_train_partials(int32_t B, int32_t H, int32_t W) {
  if (!mask_train_shape_ok(B, H, W)) return MAGNET_ERR_SHAPE;
  return magnet::mask_train_partials(B, H, W);
}

int magnet_mask_pack_train_weights_f32(const float* w1, const float* b1, const float* w2, const float* b2,
                                       const float* w3, const float* b3, void* packed, void* stream) {
  if (!w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !packed) return MAGNET_ERR_NULL;
  if (misaligned16(packed)) return MAGNET_ERR_ALIGN;
  cudaError_t e = magnet::launch_mask_pack_train(w1, b1, w2, b2, w3, b3, packed, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 3;
  return MAGNET_OK;
}

int magnet_mask_train_fwd_f32(const magnet_mask_train_args* a, void* stream) {
  const int st = validate_mask_train(a);
  if (st != MAGNET_OK) return st;
  if (!a->pre0 || !a->pred || !a->gt || !a->gt_mask || !a->pred_scale || !a->partial) return MAGNET_ERR_NULL;
  for (int p = 0; p < a->P; ++p)
    if (!a->pred[p]) return MAGNET_ERR_NULL;
  if (misaligned16(a->pre0)) return MAGNET_ERR_ALIGN;
  for (int p = 0; p < a->P; ++p)
    if (misaligned16(a->pred[p])) return MAGNET_ERR_ALIGN;
  int launches = 0;
  cudaError_t e = magnet::launch_mask_train_fwd(a->P, a->B, a->H, a->W, a->pre0, a->packed_weights, a->pred, a->gt,
                                                a->gt_mask, a->pred_scale, a->save_maps != 0, a->pred_grad != 0,
                                                a->partial, a->saved, (cudaStream_t)stream, &launches);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += launches;
  return MAGNET_OK;
}

int magnet_mask_bwd_f32(const magnet_mask_train_args* a, void* stream) {
  const int st = validate_mask_train(a);
  if (st != MAGNET_OK) return st;
  if (!a->grad_scale || !a->workspace) return MAGNET_ERR_NULL;
  if (misaligned16(a->workspace)) return MAGNET_ERR_ALIGN;
  int launches = 0;
  cudaError_t e = magnet::launch_mask_bwd(a->P, a->B, a->H, a->W, a->packed_weights, a->saved, a->grad_scale,
                                          a->workspace, a->grad_pre0, a->grad_w1, a->grad_b1, a->grad_w2, a->grad_b2,
                                          a->grad_w3, a->grad_b3, a->grad_pred, (cudaStream_t)stream, &launches);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += launches;
  return MAGNET_OK;
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
  for (int p = 0; p < a->P; ++p)
    if (!a->pred[p]) return MAGNET_ERR_NULL;
  cudaError_t e = magnet::launch_depth_metrics(a->pred, a->P, a->k > 0 ? a->up_mask : nullptr, a->gt, a->B, a->H, a->W,
                                               a->k, 0, 0, false, a->row0, a->row1, a->col0, a->col1, a->min_depth,
                                               a->max_depth, a->workspace, a->out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 2;
  return MAGNET_OK;
}

int magnet_depth_metrics_var_f32(const magnet_depth_metrics_args* a, void* stream) {
  const int st = validate_depth_metrics_shape(a);
  if (st != MAGNET_OK) return st;
  if (a->k != 0) return MAGNET_ERR_UNSUPPORTED;
  if (!a->pred || !a->gt || !a->workspace || !a->out) return MAGNET_ERR_NULL;
  for (int p = 0; p < a->P; ++p)
    if (!a->pred[p]) return MAGNET_ERR_NULL;
  cudaError_t e = magnet::launch_depth_metrics(a->pred, a->P, nullptr, a->gt, a->B, a->H, a->W, 0, 0, 0, true, a->row0,
                                               a->row1, a->col0, a->col1, a->min_depth, a->max_depth, a->workspace,
                                               a->out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 2;
  return MAGNET_OK;
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
  int launches = 0;
  cudaError_t e = magnet::launch_dnet_pack(d_w1, d_b1, d_w2, d_b2, m_w1, m_b1, m_w3, m_b3, k == 4, packed,
                                           (cudaStream_t)stream, &launches);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += launches;
  return MAGNET_OK;
}

namespace {
bool dnet_shape_ok(int32_t B, int32_t H, int32_t W) {
  return B > 0 && H > 0 && W > 0 && (int64_t)B * H * W < ((int64_t)1 << 31);
}
}  // namespace

int magnet_dnet_depth_f32(const float* pre_d, const void* packed, int32_t B, int32_t H, int32_t W, int32_t sigma,
                          float* out, void* stream) {
  if (!dnet_shape_ok(B, H, W)) return MAGNET_ERR_SHAPE;
  if (!pre_d || !packed || !out) return MAGNET_ERR_NULL;
  if (misaligned16(pre_d) || misaligned16(packed) || misaligned16(out)) return MAGNET_ERR_ALIGN;
  cudaError_t e = magnet::launch_dnet_depth(B, H, W, pre_d, packed, sigma != 0, out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_dnet_upsample_f32(const float* pre_m, const void* packed, const float* raw, int32_t B, int32_t H, int32_t W,
                             int32_t k, float* out, void* stream) {
  if (!dnet_shape_ok(B, H, W)) return MAGNET_ERR_SHAPE;
  if (k != 4) return MAGNET_ERR_UNSUPPORTED;
  if (!pre_m || !packed || !raw || !out) return MAGNET_ERR_NULL;
  if (misaligned16(pre_m) || misaligned16(packed) || misaligned16(raw) || misaligned16(out)) return MAGNET_ERR_ALIGN;
  cudaError_t e = magnet::launch_dnet_upsample_packed(B, H, W, pre_m, packed, raw, out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

int magnet_plane_depth_f32(const float* volume, const float* planes_host, int32_t B, int32_t D, int32_t H, int32_t W,
                           int32_t scores, float* out, void* stream) {
  if (!volume || !planes_host || !out) return MAGNET_ERR_NULL;
  if (B <= 0 || D <= 0 || H <= 0 || W <= 0 || B > 65535) return MAGNET_ERR_SHAPE;
  if ((int64_t)H * W > (1 << 26)) return MAGNET_ERR_SHAPE;
  if (D > MAGNET_MAX_PLANES) return MAGNET_ERR_UNSUPPORTED;
  cudaError_t e = magnet::launch_plane_depth(volume, planes_host, B, D, H * W, scores != 0, out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 1;
  return MAGNET_OK;
}

namespace {
// Shape fields and box only (the sizing call needs no pointers).
int validate_depth_metrics_nearest_shape(const magnet_depth_metrics_nearest_args* a) {
  if (!a) return MAGNET_ERR_NULL;
  if (a->P <= 0 || a->B <= 0 || a->H <= 0 || a->W <= 0 || a->h <= 0 || a->w <= 0) return MAGNET_ERR_SHAPE;
  if (a->P > MAGNET_METRICS_MAX_PRED) return MAGNET_ERR_UNSUPPORTED;
  if ((int64_t)a->P * a->B > 65535 || (int64_t)a->H * a->W > (1 << 28)) return MAGNET_ERR_SHAPE;
  if (a->h > a->H || a->w > a->W) return MAGNET_ERR_SHAPE;
  if (a->row0 < 0 || a->row0 > a->row1 || a->row1 > a->H) return MAGNET_ERR_SHAPE;
  if (a->col0 < 0 || a->col0 > a->col1 || a->col1 > a->W) return MAGNET_ERR_SHAPE;
  return MAGNET_OK;
}
}  // namespace

int64_t magnet_depth_metrics_nearest_workspace(const magnet_depth_metrics_nearest_args* a) {
  const int st = validate_depth_metrics_nearest_shape(a);
  if (st != MAGNET_OK) return st;
  return (int64_t)magnet::depth_metrics_workspace(a->P, a->B, a->row1 - a->row0, a->col1 - a->col0);
}

int magnet_depth_metrics_nearest_f32(const magnet_depth_metrics_nearest_args* a, void* stream) {
  const int st = validate_depth_metrics_nearest_shape(a);
  if (st != MAGNET_OK) return st;
  if (!a->pred || !a->gt || !a->workspace || !a->out) return MAGNET_ERR_NULL;
  for (int p = 0; p < a->P; ++p)
    if (!a->pred[p]) return MAGNET_ERR_NULL;
  cudaError_t e = magnet::launch_depth_metrics(a->pred, a->P, nullptr, a->gt, a->B, a->H, a->W, 0, a->h, a->w, false, a->row0,
                                               a->row1, a->col0, a->col1, a->min_depth, a->max_depth, a->workspace,
                                               a->out, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(e);
  g_launches += 2;
  return MAGNET_OK;
}

}  // extern "C"
