// Deterministic backward of RoIAlign_v2, the fused FPN RoIAlign and ROIPooling_v1 for sm_90a.
//
// The atomic backward kernels (roi_align.cu, roi_pool.cu) add contributions in whatever order the hardware
// resolves them, so overlapping rois give a gradient whose last bits change from run to run.  These kernels
// return, bit for bit, the serial loop of the reference's backward (oracle/roi_ops.c): for every gradient plane the
// contributions are added with round-to-nearest fadd in ascending flat index ((n*C + c)*PH + ph)*PW + pw, each
// RoIAlign index adding its corners in the order TL, TR, BL, BR.
//
//   plane ownership  a CTA owns a band of rows of one gradient plane (image b, channel c, level l).  It holds the
//                    band in shared memory (value + ticket per pixel), loaded from the gradient for kAddTo and set to
//                    +0.0 for kWriteTo, and writes it back at the end: no other CTA touches those pixels, so there are
//                    no global atomics and no zero fill.
//   index order      the CTA walks its image's entries in index order, one entry per thread per batch.  Each entry
//                    becomes up to four records (pixel, value) with the key 4*thread + corner; records outside the
//                    band are dropped.
//   order in a batch rounds: every pending record does atomicMin(ticket[pixel], key); after a barrier the record
//                    holding its pixel's ticket adds its value and retires; after another barrier the winners reset
//                    their tickets.  atomicMin's result does not depend on arrival order, so each pixel receives its
//                    adds in ascending key order within a batch and in index order across batches: the serial sum.
//                    The number of rounds is the largest number of records that hit one pixel within one batch.
#include <climits>

#include "common.cuh"

namespace {

constexpr int kOrdThreads = 512;
constexpr int kOrdSmemBudget = 96 * 1024;           // bytes per CTA: two CTAs per SM
constexpr int kOrdMaxW = kOrdSmemBudget / 8;        // widest plane row one band can hold (8 bytes per pixel)

struct OrdArgs {
  float* grad;              // this level's gradient (B, C, H, W)
  const float* ograd;       // (total rois, C, PH, PW)
  const float* argx;        // RoIAlign: argmax_x; ROIPooling: max_idx
  const float* argy;        // RoIAlign: argmax_y; ROIPooling: unused
  const float* rois;        // ROIPooling: (R, 5), image index in column 0
  const int32_t* levels;    // fused RoIAlign: level of each roi; nullptr otherwise
  int level;                // level index this launch owns (fused RoIAlign)
  int B, N, C, PP, H, W;    // N: rois per image (RoIAlign), all rois (ROIPooling)
  int rows, bands;          // band height and bands per plane
  int accumulate;
};

template <bool kPool>
__global__ void __launch_bounds__(kOrdThreads, 2)
roi_bwd_ordered_kernel(const __grid_constant__ OrdArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const int tid = threadIdx.x;
  const int band = (int)(blockIdx.x % (unsigned)a.bands);
  const int plane = (int)(blockIdx.x / (unsigned)a.bands);  // b * C + c
  const int b = plane / a.C, c = plane - b * a.C;
  const int r0 = band * a.rows, r1 = min(a.H, r0 + a.rows);
  const int W = a.W;
  const int npx = (r1 - r0) * W;
  float* s_val = reinterpret_cast<float*>(s_raw);
  int* s_tk = reinterpret_cast<int*>(s_raw) + a.rows * W;
  float* g = a.grad + (size_t)plane * a.H * W + (size_t)r0 * W;
  for (int i = tid; i < npx; i += kOrdThreads) {
    s_val[i] = a.accumulate ? g[i] : 0.f;
    s_tk[i] = INT_MAX;
  }
  // RoIAlign: image b owns rois [b*N, (b+1)*N); ROIPooling: every roi, filtered by its image index
  const int n0 = kPool ? 0 : b * a.N;
  const long long count = (long long)a.N * a.PP;
  for (long long base = 0; base < count; base += kOrdThreads) {
    int px[4];
    float v[4];
    unsigned pend = 0;
    const long long j = base + tid;
    if (j < count) {
      const int n = n0 + (int)(j / a.PP), p = (int)(j % a.PP);
      const size_t idx = ((size_t)n * a.C + c) * a.PP + p;
      if (kPool) {
        if ((int)__ldg(a.rois + (size_t)n * 5) == b) {
          const int m = (int)__ldg(a.argx + idx);  // -1: empty bin
          if (m >= 0 && m < a.H * W) {
            const int y = m / W;
            if (y >= r0 && y < r1) {
              px[0] = m - r0 * W;
              v[0] = __ldg(a.ograd + idx);
              pend = 1;
            }
          }
        }
      } else if (a.levels == nullptr || __ldg(a.levels + n) == a.level) {
        const float ax = __ldg(a.argx + idx), ay = __ldg(a.argy + idx);
        if (ax != -1.f && ay != -1.f) {
          // the corner rule and products of roi_align_v2_bwd_kernel (roi_align.cu)
          const int H = a.H;
          const int hl = min(max((int)floorf(ay), 0), H - 1), hh = min(max((int)ceilf(ay), 0), H - 1);
          const int wl = min(max((int)floorf(ax), 0), W - 1), wr = min(max((int)ceilf(ax), 0), W - 1);
          const float al = (hl == hh) ? 0.5f : __fdiv_rn(__fsub_rn(ay, (float)hl), (float)(hh - hl));
          const float be = (wl == wr) ? 0.5f : __fdiv_rn(__fsub_rn(ax, (float)wl), (float)(wr - wl));
          const float d = __ldg(a.ograd + idx);
          const float a0 = __fsub_rn(1.f, al), b0 = __fsub_rn(1.f, be);
          const float dt = __fmul_rn(d, a0), db = __fmul_rn(d, al);
          v[0] = __fmul_rn(dt, b0); v[1] = __fmul_rn(dt, be);
          v[2] = __fmul_rn(db, b0); v[3] = __fmul_rn(db, be);
          if (hl >= r0 && hl < r1) {
            px[0] = (hl - r0) * W + wl; px[1] = (hl - r0) * W + wr;
            pend |= 3u;
          }
          if (hh >= r0 && hh < r1) {
            px[2] = (hh - r0) * W + wl; px[3] = (hh - r0) * W + wr;
            pend |= 12u;
          }
        }
      }
    }
    // the first pass of this barrier also orders the band's initialisation before the first ticket
    while (__syncthreads_or(pend != 0)) {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (pend & (1u << k)) atomicMin(s_tk + px[k], 4 * tid + k);
      __syncthreads();
      unsigned won = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if ((pend & (1u << k)) && s_tk[px[k]] == 4 * tid + k) {
          s_val[px[k]] = __fadd_rn(s_val[px[k]], v[k]);
          won |= 1u << k;
        }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (won & (1u << k)) s_tk[px[k]] = INT_MAX;
      pend &= ~won;
    }
  }
  // the last __syncthreads_or above ordered every add before these reads
  for (int i = tid; i < npx; i += kOrdThreads) g[i] = s_val[i];
}

// Band geometry of one plane: the fewest bands that fit the budget, rows balanced across them.
int band_plan(int H, int W, int& rows, int& bands) {
  if (W > kOrdMaxW)
    return sdet::fail(SDET_ERR_UNSUPPORTED, "plane row of %d pixels does not fit one band (at most %d)", W, kOrdMaxW);
  const int max_rows = kOrdMaxW / W;
  bands = (H + max_rows - 1) / max_rows;
  rows = (H + bands - 1) / bands;
  return SDET_OK;
}

template <bool kPool>
int launch_level(OrdArgs a, cudaStream_t st) {
  const size_t smem = (size_t)a.rows * a.W * 8;
  const unsigned long long ctas = (unsigned long long)a.B * a.C * a.bands;
  auto k = roi_bwd_ordered_kernel<kPool>;
  SDET_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k<<<(unsigned)ctas, kOrdThreads, smem, st>>>(a);
  SDET_LAUNCH_CHECK("roi_bwd_ordered_kernel");
  return SDET_OK;
}

int check_shape(int B, int N, int C, int pooled_h, int pooled_w) {
  if (B <= 0 || N <= 0 || C <= 0) return sdet::fail(SDET_ERR_INVALID_ARG, "B, N, C must be > 0");
  if (pooled_h <= 0 || pooled_w <= 0)
    return sdet::fail(SDET_ERR_INVALID_ARG, "pooled_size must be non-zero (enforce_nonzero)");
  if (pooled_h > SDET_MAX_POOLED || pooled_w > SDET_MAX_POOLED)
    return sdet::fail(SDET_ERR_UNSUPPORTED, "pooled_size > %d per axis is not supported", SDET_MAX_POOLED);
  return SDET_OK;
}

// Every check (including the band geometry of each level) happens before the first memset or launch.
int roi_align_ordered(const float* ograd, const float* argmax_x, const float* argmax_y, const int32_t* levels,
                      float* const* grads, const int* H, const int* W, int num_levels, float* grad_rois, int B,
                      int N, int C, int pooled_h, int pooled_w, int accumulate, cudaStream_t st) {
  int rows[SDET_MAX_LEVELS], bands[SDET_MAX_LEVELS];
  for (int l = 0; l < num_levels; ++l) {
    SDET_REQUIRE(grads[l] && H[l] > 0 && W[l] > 0, "level %d: bad grad pointer / shape", l);
    if (int rc = band_plan(H[l], W[l], rows[l], bands[l])) return rc;
    SDET_REQUIRE((long long)B * C * bands[l] < (1ll << 31), "too many gradient planes");
  }
  if (grad_rois)  // roi_align_v2.cu:139-141
    SDET_CUDA(cudaMemsetAsync(grad_rois, 0, sizeof(float) * (size_t)B * N * 4, st));
  for (int l = 0; l < num_levels; ++l) {
    OrdArgs a{};
    a.grad = grads[l]; a.ograd = ograd; a.argx = argmax_x; a.argy = argmax_y; a.rois = nullptr;
    a.levels = levels; a.level = l;
    a.B = B; a.N = N; a.C = C; a.PP = pooled_h * pooled_w; a.H = H[l]; a.W = W[l];
    a.rows = rows[l]; a.bands = bands[l]; a.accumulate = accumulate ? 1 : 0;
    if (int rc = launch_level<false>(a, st)) return rc;
  }
  return SDET_OK;
}

}  // namespace

extern "C" int sdet_roi_align_v2_backward_ordered(const float* ograd, const float* argmax_x,
                                                  const float* argmax_y, float* grad_data, float* grad_rois,
                                                  int B, int N, int C, int H, int W, int pooled_h,
                                                  int pooled_w, int accumulate, void* stream) {
  if (int rc = check_shape(B, N, C, pooled_h, pooled_w)) return rc;
  SDET_REQUIRE(ograd && argmax_x && argmax_y && grad_data, "NULL argument");
  float* g[1] = {grad_data};
  return roi_align_ordered(ograd, argmax_x, argmax_y, nullptr, g, &H, &W, 1, grad_rois, B, N, C, pooled_h,
                           pooled_w, accumulate, (cudaStream_t)stream);
}

extern "C" int sdet_fpn_roi_align_v2_backward_ordered(const float* ograd, const float* argmax_x,
                                                      const float* argmax_y, const int32_t* levels,
                                                      float* const* grad_feats, const int* H, const int* W,
                                                      int num_levels, int B, int N, int C, int pooled_h,
                                                      int pooled_w, int accumulate, void* stream) {
  if (int rc = check_shape(B, N, C, pooled_h, pooled_w)) return rc;
  SDET_REQUIRE(ograd && argmax_x && argmax_y && levels && grad_feats && H && W, "NULL argument");
  SDET_REQUIRE(num_levels >= 1 && num_levels <= SDET_MAX_LEVELS, "num_levels must be in [1, %d]", SDET_MAX_LEVELS);
  return roi_align_ordered(ograd, argmax_x, argmax_y, levels, grad_feats, H, W, num_levels, nullptr, B, N, C,
                           pooled_h, pooled_w, accumulate, (cudaStream_t)stream);
}

extern "C" int sdet_roi_pooling_v1_backward_ordered(const float* ograd, const float* max_idx, const float* rois,
                                                    float* grad_data, float* grad_rois, int B, int R, int C,
                                                    int H, int W, int pooled_h, int pooled_w, float spatial_scale,
                                                    int accumulate, void* stream) {
  (void)spatial_scale;  // the stored max_idx names the pixel; the bins need not be re-derived
  SDET_REQUIRE(ograd && max_idx && rois && grad_data, "NULL argument");
  SDET_REQUIRE(B > 0 && R > 0 && C > 0 && H > 0 && W > 0 && pooled_h > 0 && pooled_w > 0,
               "shape must be positive");
  if (pooled_h > SDET_MAX_POOLED || pooled_w > SDET_MAX_POOLED)
    return sdet::fail(SDET_ERR_UNSUPPORTED, "pooled_size > %d per axis is not supported", SDET_MAX_POOLED);
  OrdArgs a{};
  if (int rc = band_plan(H, W, a.rows, a.bands)) return rc;
  SDET_REQUIRE((long long)B * C * a.bands < (1ll << 31), "too many gradient planes");
  cudaStream_t st = (cudaStream_t)stream;
  if (grad_rois) SDET_CUDA(cudaMemsetAsync(grad_rois, 0, sizeof(float) * (size_t)R * 5, st));
  a.grad = grad_data; a.ograd = ograd; a.argx = max_idx; a.argy = nullptr; a.rois = rois;
  a.levels = nullptr; a.level = 0;
  a.B = B; a.N = R; a.C = C; a.PP = pooled_h * pooled_w; a.H = H; a.W = W;
  a.accumulate = accumulate ? 1 : 0;
  return launch_level<true>(a, st);
}
