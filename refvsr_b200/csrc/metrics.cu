// rv_region_metrics: squared-error and SSIM-map sums of two (1, 3, H, W) fp32 images over up to 8 axis-aligned boxes, the
// quantities behind every number evaluation/eval_quan_FOV.py prints (metrics.py:18-31 psnr / psnr_masked / ssim /
// ssim_masked with masks that are unions / differences of centred boxes).
//
// One CTA per TH x TW tile of the frame.  Per channel the CTA stages both planes of the tile plus a 3-pixel halo (scipy
// `reflect` borders: -1 -> 0, H -> H-1) in shared memory, takes the horizontal 7-sums of the five moments (a, b, a*a, b*b, a*b) in
// fp64, then the vertical 7-sums per output pixel, and forms skimage's SSIM map value
//   S = ((2 ux uy + C1)(2 vxy + C2)) / ((ux^2 + uy^2 + C1)(vx + vy + C2)),  v = 49/48 (E[..] - E[.]E[.]),  C1 = 1e-4, C2 = 9e-4
// next to the float32 squared error (a - b)^2.  A pixel's two channel sums go to the per-thread sums of every box holding it; the CTA's
// sums go to `work` ([2 * nbox][CTAs]) and a second launch reduces them in a fixed order, so two calls are bit-identical.
#include "common.cuh"

namespace {

constexpr int TW = 32, TH = 16, HALO = 3, NT = 256;
constexpr int SW = TW + 2 * HALO, SH = TH + 2 * HALO;
constexpr int MAXBOX = 8;
constexpr int RED_NT = 256;

static_assert(RV_REGION_METRICS_WORK(TH, TW, 1) == 2, "one CTA per TH x TW tile");
static_assert(TH * TW % NT == 0, "every thread owns the same number of output pixels");

struct Boxes {
  int n;
  int y0[MAXBOX], y1[MAXBOX], x0[MAXBOX], x1[MAXBOX];
};

// scipy.ndimage `reflect` (half-sample symmetric) for i in [-3, n + 2]; tile positions past that (beyond the frame's last
// tile) are clamped so the load stays inside the plane - their outputs are never counted.
__device__ __forceinline__ int reflect_index(int i, int n) {
  i = i < 0 ? -i - 1 : (i >= n ? 2 * n - i - 1 : i);
  return rv::clampi(i, 0, n - 1);
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(NT) region_metrics_kernel(const float* __restrict__ a, const float* __restrict__ b, int H,
                                                            int W, const Boxes bx, double* __restrict__ work) {
  __shared__ float sa[SH][SW], sb[SH][SW];
  __shared__ double hs[5][SH][TW];
  __shared__ double red[NT / 32][2 * MAXBOX];

  const int tid = threadIdx.x;
  const int ty0 = blockIdx.y * TH, tx0 = blockIdx.x * TW;
  const size_t plane = (size_t)H * W;
  constexpr int PPT = TH * TW / NT;                    // output pixels per thread
  double pix_q[PPT], pix_s[PPT];                      // their channel sums
#pragma unroll
  for (int j = 0; j < PPT; ++j) pix_q[j] = pix_s[j] = 0.0;

  for (int c = 0; c < 3; ++c) {
    const float* pa = a + c * plane;
    const float* pb = b + c * plane;
    __syncthreads();                                    // the previous channel's readers are done with sa / sb / hs
    for (int i = tid; i < SH * SW; i += NT) {
      const int r = i / SW, q = i % SW;
      const size_t off = (size_t)reflect_index(ty0 + r - HALO, H) * W + reflect_index(tx0 + q - HALO, W);
      sa[r][q] = pa[off];
      sb[r][q] = pb[off];
    }
    __syncthreads();
    for (int i = tid; i < SH * TW; i += NT) {           // horizontal 7-sums
      const int r = i / TW, x = i % TW;
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0, s4 = 0.0;
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        const double va = sa[r][x + k], vb = sb[r][x + k];
        s0 += va;
        s1 += vb;
        s2 += va * va;
        s3 += vb * vb;
        s4 += va * vb;
      }
      hs[0][r][x] = s0;
      hs[1][r][x] = s1;
      hs[2][r][x] = s2;
      hs[3][r][x] = s3;
      hs[4][r][x] = s4;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < PPT; ++j) {                     // vertical 7-sums, S and the squared error of one output pixel
      const int y = (tid + j * NT) / TW, x = (tid + j * NT) % TW;
      double m[5];
#pragma unroll
      for (int v = 0; v < 5; ++v) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 7; ++k) s += hs[v][y + k][x];
        m[v] = s * (1.0 / 49.0);
      }
      const double cov_norm = 49.0 / 48.0, C1 = 1e-4, C2 = 9e-4;
      const double ux = m[0], uy = m[1];
      const double vx = cov_norm * (m[2] - ux * ux), vy = cov_norm * (m[3] - uy * uy), vxy = cov_norm * (m[4] - ux * uy);
      pix_s[j] += ((2.0 * ux * uy + C1) * (2.0 * vxy + C2)) / ((ux * ux + uy * uy + C1) * (vx + vy + C2));
      const float d = __fsub_rn(sa[y + HALO][x + HALO], sb[y + HALO][x + HALO]);
      pix_q[j] += (double)__fmul_rn(d, d);              // numpy's float32 (img1 - img2) ** 2
    }
  }

  double acc_q[MAXBOX], acc_s[MAXBOX];                  // per box; pixels outside the frame are in no box
#pragma unroll
  for (int k = 0; k < MAXBOX; ++k) acc_q[k] = acc_s[k] = 0.0;
#pragma unroll
  for (int j = 0; j < PPT; ++j) {
    const int gy = ty0 + (tid + j * NT) / TW, gx = tx0 + (tid + j * NT) % TW;
#pragma unroll
    for (int k = 0; k < MAXBOX; ++k) {
      const bool in = k < bx.n && gy >= bx.y0[k] && gy < bx.y1[k] && gx >= bx.x0[k] && gx < bx.x1[k];
      acc_q[k] += in ? pix_q[j] : 0.0;
      acc_s[k] += in ? pix_s[j] : 0.0;
    }
  }

  const int warp = tid >> 5, lane = tid & 31;
#pragma unroll
  for (int k = 0; k < MAXBOX; ++k) {
    const double q = warp_sum(acc_q[k]), s = warp_sum(acc_s[k]);
    if (lane == 0) {
      red[warp][k] = q;
      red[warp][MAXBOX + k] = s;
    }
  }
  __syncthreads();
  const int n = bx.n;
  if (tid < 2 * n) {
    const int col = tid < n ? tid : MAXBOX + tid - n;   // work rows: the n squared-error sums, then the n SSIM sums
    double v = 0.0;
    for (int w = 0; w < NT / 32; ++w) v += red[w][col];
    work[(size_t)tid * gridDim.x * gridDim.y + blockIdx.y * gridDim.x + blockIdx.x] = v;
  }
}

// sums[j] = sum over the CTAs of work[j][.], one CTA per j, in a fixed order
__global__ void __launch_bounds__(RED_NT) region_sums_kernel(const double* __restrict__ work, int nblk, double* __restrict__ sums) {
  __shared__ double part[RED_NT];
  const double* row = work + (size_t)blockIdx.x * nblk;
  double v = 0.0;
  for (int i = threadIdx.x; i < nblk; i += RED_NT) v += row[i];
  part[threadIdx.x] = v;
  __syncthreads();
  for (int s = RED_NT / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) part[threadIdx.x] += part[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) sums[blockIdx.x] = part[0];
}

}  // namespace

extern "C" int rv_region_metrics(const float* a, const float* b, int H, int W, const int32_t* boxes_host, int nbox,
                                 double* work, double* sums, void* stream) {
  RV_REQUIRE(a && b && boxes_host && work && sums, "rv_region_metrics: null pointer");
  RV_REQUIRE(H >= 7 && W >= 7, "rv_region_metrics: the SSIM window needs H, W >= 7 (got %d x %d)", H, W);
  RV_REQUIRE(nbox >= 1 && nbox <= MAXBOX, "rv_region_metrics: 1..%d boxes (got %d)", MAXBOX, nbox);
  Boxes bx{};
  bx.n = nbox;
  for (int k = 0; k < nbox; ++k) {
    const int32_t* q = boxes_host + 4 * k;
    RV_REQUIRE(0 <= q[0] && q[0] <= q[1] && q[1] <= H && 0 <= q[2] && q[2] <= q[3] && q[3] <= W,
               "rv_region_metrics: box %d (y %d..%d, x %d..%d) is not inside the %d x %d frame", k, q[0], q[1], q[2], q[3], H, W);
    bx.y0[k] = q[0];
    bx.y1[k] = q[1];
    bx.x0[k] = q[2];
    bx.x1[k] = q[3];
  }
  const dim3 grid(rv::cdiv(W, TW), rv::cdiv(H, TH));
  region_metrics_kernel<<<grid, NT, 0, (cudaStream_t)stream>>>(a, b, H, W, bx, work);
  RV_LAUNCH_CHECK("region_metrics");
  region_sums_kernel<<<2 * nbox, RED_NT, 0, (cudaStream_t)stream>>>(work, (int)(grid.x * grid.y), sums);
  RV_LAUNCH_CHECK("region_sums");
  return RV_OK;
}
