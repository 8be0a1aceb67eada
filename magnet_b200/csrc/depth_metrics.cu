// Depth evaluation on the device: the per-image metrics of validate() (test_MaGNet.py:27-81, train_MaGNet.py:132-182)
// and utils.compute_depth_errors (utils/utils.py:106-144), for up to MAGNET_METRICS_MAX_PRED predictions sharing one GT;
// also the F-Net form of train_FNet.py:165-193 (a depth map on a coarser grid, nearest-upsampled, no variance).
//
// Stage 1 (depth_metrics_partial_kernel): one CTA per (128-column x DM_ROWS-row tile of the evaluation box, image,
// prediction).  Every pixel forms the float32 terms of compute_depth_errors in numpy's operation order and adds them to
// float64 per-thread sums; the CTA reduces its 128 threads in a fixed order and writes one row of DM_SUMS doubles.
// Stage 2 (depth_metrics_final_kernel): one CTA per (prediction, image) adds its rows in a fixed order and forms the
// metrics.  No atomics anywhere, so results are bit-identical from run to run.
//
// Build note: this file relies on IEEE float32 division and full-precision logf / log10f; the library is compiled
// without --use_fast_math, and the explicit __f*_rn intrinsics keep nvcc from contracting terms into FMAs.
#include "common.cuh"
#include "upsample_common.cuh"

namespace magnet {

constexpr int DM_THREADS = 128;
constexpr int DM_ROWS = 4;          // rows of the box per CTA
constexpr int DM_SUMS = 13;         // per-pixel sums (see below); also the width of an output row

// Sum slots.  rmse_log and silog share the squared log error: (log gt - log pred)^2 == (log pred - log gt)^2 exactly,
// because IEEE subtraction is sign-symmetric.
enum : int { S_N = 0, S_A1, S_A2, S_A3, S_ABS, S_ABSREL, S_SQREL, S_SQ, S_LOGSQ, S_LOGERR, S_LOG10, S_INV, S_NLL };

struct DmPreds {
  const float* p[MAGNET_METRICS_MAX_PRED];
};

struct DmBox {
  int r0, c0, rows, cols;
};

// Where a pixel's prediction comes from.
//   DM_FULL: full-resolution (B,2,H,W) [mu, sigma].
//   DM_FUSED: quarter-resolution (B,2,H/k,W/k) [mu, sigma] and the upsampling mask (upsample_depth_via_mask fused in).
//   DM_NEAREST: a (B,1,h,w) depth map, F.interpolate(..., size=(H, W), mode='nearest') fused in (train_FNet.py:181).
//     No variance: the NLL slot stays 0 and the final kernel writes nll = 0.0, as compute_depth_errors(var=None).
//   DM_VAR: full-resolution (B,2,H,W) [mu, var], D-Net's output (test_DNet.py:40-71): channel 1 is the variance itself.
enum : int { DM_FULL = 0, DM_FUSED = 1, DM_NEAREST = 2, DM_VAR = 3 };

// The prediction grid of DM_NEAREST and ATen's source-index scales (float)h / H, (float)w / W.
struct DmNearest {
  int h, w;
  float sh, sw;
};

// ATen's nearest source index (UpSample.h nearest_idx with size=..., CPU and CUDA alike): min(floor(dst * scale),
// in - 1) with the product in float32.  Its shortcuts for equal and doubled sizes give the same index.
__device__ __forceinline__ int nearest_src(int dst, float scale, int in) {
  return min((int)floorf(__fmul_rn((float)dst, scale)), in - 1);
}

template <int FORM>
__global__ void __launch_bounds__(DM_THREADS) depth_metrics_partial_kernel(
    const __grid_constant__ DmPreds preds, const float* __restrict__ up_mask, const float* __restrict__ gt, int B,
    int H, int W, int k, DmNearest nn, DmBox box, float min_d, float max_d, double* __restrict__ partial) {
  const int tile = blockIdx.y * gridDim.x + blockIdx.x, tiles = gridDim.x * gridDim.y;
  const int img = blockIdx.z;                       // p * B + b
  const int p = img / B;
  const size_t b = img % B;
  const float* pred = preds.p[p];
  const int c = blockIdx.x * DM_THREADS + threadIdx.x;
  double s[DM_SUMS];
#pragma unroll
  for (int i = 0; i < DM_SUMS; ++i) s[i] = 0.0;
  const double log_2pi = 0x1.d67f1c864beb4p+0;           // np.log(2*np.pi), a float64 scalar, as the host rounds it
  if (c < box.cols) {
    const int X = box.c0 + c;
    const size_t HW = (size_t)H * W;
    const int xs = FORM == DM_NEAREST ? nearest_src(X, nn.sw, nn.w) : 0;
    for (int j = 0; j < DM_ROWS; ++j) {
      const int r = blockIdx.y * DM_ROWS + j;
      if (r >= box.rows) break;
      const int Y = box.r0 + r;
      float g = gt[b * HW + (size_t)Y * W + X];
      if (g > max_d) g = 0.0f;                            // gt_dmap[gt_dmap > max_depth] = 0
      if (!(g > min_d && g < max_d)) continue;            // valid_mask
      float mu, sg = 0.0f;
      if (FORM == DM_FUSED) {
        float w[9];
        upsampled_gaussian(pred, up_mask, b, H / k, W / k, k, X / k, Y / k, X % k, Y % k, w, mu, sg);
      } else if (FORM == DM_FULL || FORM == DM_VAR) {
        mu = pred[(b * 2 + 0) * HW + (size_t)Y * W + X];
        sg = pred[(b * 2 + 1) * HW + (size_t)Y * W + X];
      } else {
        mu = pred[(b * nn.h + nearest_src(Y, nn.sh, nn.h)) * (size_t)nn.w + xs];
      }
      // masking, in the reference's order
      if (mu < min_d) mu = min_d;
      if (mu > max_d) mu = max_d;
      if (isinf(mu)) mu = max_d;
      if (isnan(mu)) mu = min_d;
      float var = FORM == DM_VAR ? sg : __fmul_rn(sg, sg);   // the variance, or np.square of the unclamped sigma
      if (var < 1e-6f) var = 1e-6f;
      const float r1 = __fdiv_rn(g, mu), r2 = __fdiv_rn(mu, g);
      const float th = (isnan(r1) || isnan(r2)) ? r1 + r2 : fmaxf(r1, r2);   // np.maximum propagates NaN
      const float d = __fsub_rn(g, mu), ad = fabsf(d), d2 = __fmul_rn(d, d);
      const float lg = logf(g), lp = logf(mu);
      const float le = __fsub_rn(lg, lp), err = __fsub_rn(lp, lg);
      const float l10 = fabsf(__fsub_rn(log10f(g), log10f(mu)));
      const float iv = __fsub_rn(__fdiv_rn(1.0f, g), __fdiv_rn(1.0f, mu));
      s[S_N] += 1.0;
      s[S_A1] += th < 1.25f ? 1.0 : 0.0;
      s[S_A2] += th < 1.5625f ? 1.0 : 0.0;
      s[S_A3] += th < 1.953125f ? 1.0 : 0.0;
      s[S_ABS] += (double)ad;
      s[S_ABSREL] += (double)__fdiv_rn(ad, g);
      s[S_SQREL] += (double)__fdiv_rn(d2, g);
      s[S_SQ] += (double)d2;
      s[S_LOGSQ] += (double)__fmul_rn(le, le);
      s[S_LOGERR] += (double)err;
      s[S_LOG10] += (double)l10;
      s[S_INV] += (double)__fmul_rn(iv, iv);
      // 0.5 * (log(var) + log(2 pi) + square(gt - pred) / var): float32 terms, float64 sum (numpy 2 promotion)
      if (FORM != DM_NEAREST)
        s[S_NLL] += 0.5 * __dadd_rn(__dadd_rn((double)logf(var), log_2pi), (double)__fdiv_rn(d2, var));
    }
  }
  // fixed-order CTA reduction: butterfly inside each warp, then the four warps in index order
  __shared__ double red[DM_THREADS / 32][DM_SUMS];
#pragma unroll
  for (int i = 0; i < DM_SUMS; ++i) {
    double v = s[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    s[i] = v;
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int i = 0; i < DM_SUMS; ++i) red[threadIdx.x >> 5][i] = s[i];
  }
  __syncthreads();
  if (threadIdx.x < DM_SUMS) {
    const int i = threadIdx.x;
    partial[((size_t)img * tiles + tile) * DM_SUMS + i] = (red[0][i] + red[1][i]) + (red[2][i] + red[3][i]);
  }
}

// One CTA per (prediction, image): thread t adds rows t, t + 256, ... in order, then a fixed tree over the threads.
// has_var == 0 (DM_NEAREST): nll = 0.0 whatever n, as compute_depth_errors(..., var=None) returns it.
constexpr int DM_FINAL_THREADS = 256;

__global__ void __launch_bounds__(DM_FINAL_THREADS) depth_metrics_final_kernel(const double* __restrict__ partial,
                                                                              int tiles, int has_var,
                                                                              double* __restrict__ out) {
  const int img = blockIdx.x;
  const double* rows = partial + (size_t)img * tiles * DM_SUMS;
  double s[DM_SUMS];
#pragma unroll
  for (int i = 0; i < DM_SUMS; ++i) s[i] = 0.0;
  for (int t = threadIdx.x; t < tiles; t += DM_FINAL_THREADS) {
#pragma unroll
    for (int i = 0; i < DM_SUMS; ++i) s[i] += rows[(size_t)t * DM_SUMS + i];
  }
  __shared__ double red[DM_FINAL_THREADS][DM_SUMS + 1];
#pragma unroll
  for (int i = 0; i < DM_SUMS; ++i) red[threadIdx.x][i] = s[i];
  __syncthreads();
  for (int h = DM_FINAL_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
#pragma unroll
      for (int i = 0; i < DM_SUMS; ++i) red[threadIdx.x][i] += red[threadIdx.x + h][i];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double* S = red[0];
    const double n = S[S_N];          // n == 0: every metric is 0/0 = NaN, as numpy's mean of an empty array
    const double mean_err = S[S_LOGERR] / n;
    double* o = out + (size_t)img * DM_SUMS;
    o[0] = n;
    o[1] = S[S_A1] / n;                                           // a1
    o[2] = S[S_A2] / n;                                           // a2
    o[3] = S[S_A3] / n;                                           // a3
    o[4] = S[S_ABS] / n;                                          // abs_diff
    o[5] = S[S_ABSREL] / n;                                       // abs_rel
    o[6] = S[S_SQREL] / n;                                        // sq_rel
    o[7] = sqrt(S[S_SQ] / n);                                     // rmse
    o[8] = S[S_LOG10] / n;                                        // log_10
    o[9] = sqrt(S[S_INV] / n);                                    // irmse
    o[10] = sqrt(S[S_LOGSQ] / n);                                 // rmse_log
    o[11] = sqrt(__dsub_rn(S[S_LOGSQ] / n, __dmul_rn(mean_err, mean_err))) * 100.0;   // silog (no FMA contraction)
    o[12] = has_var ? S[S_NLL] / n : 0.0;                         // nll
  }
}

// CTA grid over the evaluation box; an empty box still gets one (idle) tile, so every image has a row (n = 0).
static dim3 dm_grid(int rows, int cols) {
  return dim3(cols > 0 ? (cols + DM_THREADS - 1) / DM_THREADS : 1, rows > 0 ? (rows + DM_ROWS - 1) / DM_ROWS : 1);
}

// float64 elements of the partial-row workspace
size_t depth_metrics_workspace(int P, int B, int rows, int cols) {
  const dim3 g = dm_grid(rows, cols);
  return (size_t)P * B * g.x * g.y * DM_SUMS;
}

// k > 0: the fused-upsampling form; else h > 0: the nearest form with a (B,1,h,w) prediction; else full resolution,
// [mu, var] with `variance`, else [mu, sigma].
cudaError_t launch_depth_metrics(const float* const* preds, int P, const float* up_mask, const float* gt, int B, int H,
                                 int W, int k, int h, int w, bool variance, int r0, int r1, int c0, int c1, float min_d,
                                 float max_d, double* partial, double* out, cudaStream_t st) {
  DmPreds pp;
  for (int i = 0; i < MAGNET_METRICS_MAX_PRED; ++i) pp.p[i] = i < P ? preds[i] : nullptr;
  const DmBox box{r0, c0, r1 - r0, c1 - c0};
  // ATen's compute_scales_value without a scale factor: (float)input_size / output_size, rounded to float32
  const DmNearest nn{h, w, h > 0 ? (float)h / (float)H : 0.0f, w > 0 ? (float)w / (float)W : 0.0f};
  dim3 grid = dm_grid(box.rows, box.cols);
  const int gx = grid.x, gy = grid.y;
  grid.z = P * B;
  if (k > 0)
    depth_metrics_partial_kernel<DM_FUSED><<<grid, DM_THREADS, 0, st>>>(pp, up_mask, gt, B, H, W, k, nn, box, min_d,
                                                                        max_d, partial);
  else if (h > 0)
    depth_metrics_partial_kernel<DM_NEAREST><<<grid, DM_THREADS, 0, st>>>(pp, up_mask, gt, B, H, W, k, nn, box, min_d,
                                                                          max_d, partial);
  else if (variance)
    depth_metrics_partial_kernel<DM_VAR><<<grid, DM_THREADS, 0, st>>>(pp, up_mask, gt, B, H, W, k, nn, box, min_d,
                                                                      max_d, partial);
  else
    depth_metrics_partial_kernel<DM_FULL><<<grid, DM_THREADS, 0, st>>>(pp, up_mask, gt, B, H, W, k, nn, box, min_d,
                                                                       max_d, partial);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  depth_metrics_final_kernel<<<P * B, DM_FINAL_THREADS, 0, st>>>(partial, gx * gy, k > 0 || h <= 0, out);
  return cudaGetLastError();
}

}  // namespace magnet
