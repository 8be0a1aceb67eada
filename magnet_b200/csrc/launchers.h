// Host functions that one .cu file of the library defines and another calls: the launchers behind the C ABI (api.cu)
// and the host helpers the kernel files share.  Every file that defines or calls one of them includes this header.
#pragma once
#include <cuda.h>   // CUtensorMap and its enums (types only — cuTensorMapEncodeTiled is resolved at run time)
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <atomic>

#include "common.cuh"

namespace magnet {

// ---- shared host helpers (launch_common.cu) ------------------------------------------------------------------------
int sm_count(int dev);   // SMs of device dev, cached

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn();   // the driver's cuTensorMapEncodeTiled, or NULL

// Work slots of a persistent kernel family (WORK_SLOTS per family, common.cuh): the family's pair of tickets, and the
// slot a launch on `st` takes from them.  Eager launches cycle through the lower half; a launch recorded into a CUDA
// graph takes one of the upper half and keeps it for the life of the graph, so a replay never meets an eager launch.
struct SlotTickets {
  std::atomic<unsigned> eager{0}, captured{0};
};
int work_slot(SlotTickets& tickets, cudaStream_t st);

// ---- cost-volume forward: the kernels report the launches they enqueued through `launches` ----------------------------
cudaError_t launch_cost_mma(const CostParams& p, int mode, bool cw, int layout, const int32_t* src_index, int n_src,
                            cudaStream_t st, int* launches);
bool mma_supports(int C, int D, int V, int layout);
void mma_launch_info(int B, int H, int W, int D, int* grid, int* block, int* smem);
#if defined(MAGNET_MMA_DEBUG) || defined(MAGNET_MMA_PROFILE)
void mma_set_debug_buffer(float* p);
#endif
cudaError_t launch_cost_tma(const CostParams& p, int mode, int C, bool cw, const int32_t* src_index, int n_src,
                            cudaStream_t st, int* launches);
bool tma_supports(int C, int D, int V, int layout);
void tma_launch_info(int B, int H, int W, int D, int* grid, int* block, int* smem);
cudaError_t launch_cost_cells(const CostParams& p, int mode, int C, bool cw, bool reuse, const int32_t* src_index,
                              cudaStream_t st, int* launches);
bool cells_supports(int C, int D, int layout);
void cells_launch_info(int B, int H, int W, int D, int* grid, int* block, int* smem);
cudaError_t launch_cost_direct(const CostParams& p, int depth_mode, int src_layout, int C, bool cw,
                               const int32_t* src_index, cudaStream_t st, int* launches);
cudaError_t launch_softmax_planes(float* vol, int B, int D, int HW, cudaStream_t st);
// the frame table's range check (aux_kernels.cu): `idx` int64 when `wide`, else int32
cudaError_t launch_check_src_index(const void* idx, bool wide, int B, int V, int n_src, int32_t* out, int32_t* bad,
                                   cudaStream_t st);

// ---- source layouts ---------------------------------------------------------------------------------------------------
size_t split16_buffer_bytes(int N, int H, int W);
size_t half16_buffer_bytes(int N, int H, int W);
cudaError_t launch_repack_split16(const float* src, const float* gmm, void* dst, int N, int C, int H, int W,
                                  cudaStream_t st, int* launches);
cudaError_t launch_repack_half16(const void* src, int dtype, const float* gmm, void* dst, int N, int C, int H, int W,
                                 cudaStream_t st, int* launches);
cudaError_t launch_absmax_f32(const float* x, size_t n, unsigned* out, cudaStream_t st);
cudaError_t launch_repack_pixc(const float* src, const float* gmm, float* dst, int N, int C, int H, int W,
                               cudaStream_t st);
cudaError_t launch_repack(const float* src, float* dst, int N, int C, int H, int W, cudaStream_t st);

// ---- cost-volume backwards --------------------------------------------------------------------------------------------
cudaError_t launch_score_grad(const BwdParams& p, cudaStream_t st);
cudaError_t launch_cost_f_bwd(const BwdParams& p, cudaStream_t st, int* launches);
cudaError_t launch_cost_f_bwd_mma(const BwdParams& p, int layout, cudaStream_t st, int* launches);
cudaError_t launch_cost_cw_bwd_mma(const CwBwdParams& p, int mode, int layout, cudaStream_t st);
bool f_bwd_mma_supports(int C, int V);
#ifdef MAGNET_MMA_DEBUG
void f_bwd_mma_set_debug_buffer(float* p);
#endif
cudaError_t launch_cost_cw_bwd(const CwBwdParams& p, const CwBwdParams* split, int split_layout, int C, int mode,
                               bool mask_mma, const float* grad_out, cudaStream_t st, int* launches);
bool cw_bwd_supports(int C);
size_t geom_workspace_bytes(int B, int V, int H, int W);
cudaError_t launch_cost_geom_bwd(const CwBwdParams& p, int C, int mode, bool mask_mma, int softmax, const float* prob,
                                 const float* grad_out, float* partials, float* grad_rays, float* grad_cams,
                                 cudaStream_t st, int* launches);

// ---- cameras, sampling, update, upsampling ----------------------------------------------------------------------------
cudaError_t launch_pack_cameras(const float* intM, const float* R, int64_t r_sb, int64_t r_sv, int64_t r_si,
                                int64_t r_sj, const float* t, int64_t t_sb, int64_t t_sv, int64_t t_si,
                                const int32_t* is_valid, int B, int V, magnet_camera* out, cudaStream_t st);
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
// dnet: DnetLoss (var = activation_G of the upsampled raw v) instead of MagnetLoss (var = sigma^2)
cudaError_t launch_upsample_nll_fwd(bool dnet, const float* depth, const float* mask, const float* gt, const uint8_t* gtm,
                                    int B, int H, int W, int k, float* partial, cudaStream_t st);
// scale_dev: a DEVICE float read in place of `scale` when not NULL
cudaError_t launch_upsample_nll_bwd(bool dnet, const float* depth, const float* mask, const float* gt, const uint8_t* gtm,
                                    float scale, const float* scale_dev, int B, int H, int W, int k, float* gdepth,
                                    float* gmask, cudaStream_t st);

// ---- F-Net loss, plane depth, depth metrics ---------------------------------------------------------------------------
int fnet_l1_partials(int B, int HW);
cudaError_t launch_fnet_l1_fwd(const float* scores, const float* planes, const float* gt, const uint8_t* mask, int B,
                               int D, int HW, float* partial, cudaStream_t st);
cudaError_t launch_fnet_l1_bwd(const float* scores, const float* planes, const float* gt, const uint8_t* mask,
                               float scale, const float* grad_scale, int B, int D, int HW, float* grad_scores,
                               cudaStream_t st);
cudaError_t launch_plane_depth(const float* vol, const float* planes, int B, int D, int HW, bool scores, float* out,
                               cudaStream_t st);
size_t depth_metrics_workspace(int P, int B, int rows, int cols);
cudaError_t launch_depth_metrics(const float* const* preds, int P, const float* up_mask, const float* gt, int B, int H,
                                 int W, int k, int h, int w, bool variance, int r0, int r1, int c0, int c1, float min_d,
                                 float max_d, double* partial, double* out, cudaStream_t st);

// ---- fused heads ------------------------------------------------------------------------------------------------------
size_t dnet_weights_bytes(bool with_mask);
cudaError_t launch_dnet_pack(const float* dw1, const float* db1, const float* dw2, const float* db2, const float* mw1,
                             const float* mb1, const float* mw3, const float* mb3, bool with_mask, void* dst,
                             cudaStream_t st);
cudaError_t launch_dnet_depth(int B, int H, int W, const float* pre_d, const void* weights, bool sigma, float* out,
                              cudaStream_t st);
cudaError_t launch_dnet_upsample_packed(int B, int H, int W, const float* pre_m, const void* weights, const float* raw,
                                        float* out, cudaStream_t st);
size_t dnet_mask_weights_bytes();
cudaError_t launch_dnet_upsample(int B, int H, int W, const float* pre_m, const void* weights, const float* raw,
                                 float* out, cudaStream_t st);
size_t gnet_weights_bytes(int D);
cudaError_t launch_gnet_pack(const float* w0, const float* w1, const float* b1, const float* w2, const float* b2,
                             const float* w3, const float* b3, int D, void* dst, cudaStream_t st);
cudaError_t launch_gnet_update(int B, int D, int H, int W, const float* cost, const float* inv, const void* weights,
                               const float* prev, unsigned* scratch, float* out, cudaStream_t st);
size_t gnet_train_weights_bytes(int D);
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
size_t head_wgrad_partial_floats(int B, int H, int W, int Ma, int Nw);
cudaError_t launch_head_wgrad(int B, int H, int W, int Ma, const float* a, int Nw, const float* b, float* part,
                              float* out_w, float* out_b, cudaStream_t st);
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
                                  const float* scale, bool scale_on_device, bool save_maps, bool pred_grad,
                                  float* partial, float* saved, cudaStream_t st, int* launches);
cudaError_t launch_mask_bwd(int P, int B, int H, int W, const void* weights, const float* saved, const float* gscale,
                            void* workspace, float* grad_pre0, float* gw1, float* gb1, float* gw2, float* gb2,
                            float* gw3, float* gb3, float* const* grad_pred, cudaStream_t st, int* launches);

}  // namespace magnet
