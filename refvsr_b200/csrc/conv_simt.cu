// CUDA-core implicit-GEMM convolution with the same fused prologue/epilogue contract as the
// wgmma path (conv_tc.cu).  It is the geometry-complete implementation (any kernel size, stride,
// channel count, dtype incl. fp32) and the numerical yardstick the tensor-core kernel is tested
// against on the GPU.  fp32 accumulation in the reference's k-order (ky, kx, c).
//
// GEMM view: M = Ho*Wo output pixels, N = cout, K = kh*kw*(c0+c1).
// CTA tile BM x BN, K step 16, 256 threads, TM x TN register tile per thread.
#include "common.cuh"

namespace rv {

struct ConvP {
  const void* src0;
  const void* src1;
  int c0, c1, H, W, Ho, Wo;
  const float* w;  // [K][ldw]
  int ldw;
  const float* bias;
  int cout, kh, kw, stride, pad, act_pre, act_post;
  const void* gate;
  int gate_cs;
  const void* res;
  int res_cs;
  void* out;
  int out_cs, pixel_shuffle, K;
};

template <typename TO>
__device__ __forceinline__ void store_out(void* out, size_t off, float v) {
  reinterpret_cast<TO*>(out)[off] = from_f<TO>(v);
}

template <typename TI, typename TR, typename TO, int BM, int BN>
__global__ void __launch_bounds__(256) conv_simt_kernel(ConvP p) {
  constexpr int BK = 16;
  constexpr int TN = (BN >= 64) ? 4 : 1;        // columns per thread
  constexpr int TCOLS = BN / TN;                // threads along N
  constexpr int TROWS = 256 / TCOLS;            // threads along M
  constexpr int TM = BM / TROWS;                // rows per thread
  static_assert(TM >= 1 && TROWS * TM == BM, "tile mismatch");
  __shared__ float As[BK][BM + 1];
  __shared__ float Bs[BK][BN];

  const int tid = threadIdx.x;
  const int tn = tid % TCOLS, tm = tid / TCOLS;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int M = p.Ho * p.Wo;
  const int ct = p.c0 + p.c1;
  const TI* s0 = reinterpret_cast<const TI*>(p.src0);
  const TI* s1 = reinterpret_cast<const TI*>(p.src1);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < p.K; k0 += BK) {
    // A tile: BM pixels x BK k-values; consecutive threads walk k fastest so that NHWC channel
    // runs are read contiguously
    for (int e = tid; e < BM * BK; e += 256) {
      int kk = e % BK, mm = e / BK;
      int k = k0 + kk, m = m0 + mm;
      float v = 0.f;
      if (k < p.K && m < M) {
        int tap = k / ct, c = k - tap * ct;
        int ky = tap / p.kw, kx = tap - ky * p.kw;
        int oy = m / p.Wo, ox = m - oy * p.Wo;
        int iy = oy * p.stride + ky - p.pad, ix = ox * p.stride + kx - p.pad;
        if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
          size_t pix = (size_t)iy * p.W + ix;
          v = (c < p.c0) ? to_f(s0[pix * p.c0 + c]) : to_f(s1[pix * p.c1 + (c - p.c0)]);
        }
      }
      As[kk][mm] = v;
    }
    for (int e = tid; e < BK * BN; e += 256) {
      int nn = e % BN, kk = e / BN;
      int k = k0 + kk, n = n0 + nn;
      Bs[kk][nn] = (k < p.K && n < p.ldw) ? p.w[(size_t)k * p.ldw + n] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[kk][tm * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tn * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  const TI* gate = reinterpret_cast<const TI*>(p.gate);
  const TR* res = reinterpret_cast<const TR*>(p.res);
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + tm * TM + i;
    if (m >= M) continue;
    int oy = m / p.Wo, ox = m - oy * p.Wo;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n = n0 + tn * TN + j;
      if (n >= p.cout) continue;
      float v = acc[i][j] + p.bias[n];
      v = apply_act(v, p.act_pre);
      if (gate) v *= to_f(gate[(size_t)m * p.gate_cs + n]);
      if (res) v += to_f(res[(size_t)m * p.res_cs + n]);
      v = apply_act(v, p.act_post);
      size_t off;
      if (p.pixel_shuffle) {
        int c = n >> 2, a = (n >> 1) & 1, b = n & 1;
        off = ((size_t)(2 * oy + a) * (2 * p.Wo) + (2 * ox + b)) * p.out_cs + c;
      } else {
        off = (size_t)m * p.out_cs + n;
      }
      store_out<TO>(p.out, off, v);
    }
  }
}

template <typename TI, typename TR, typename TO>
static int launch_simt(const ConvP& p, cudaStream_t st) {
  const int M = p.Ho * p.Wo;
  if (p.cout > 16) {
    dim3 grid(cdiv(M, 64), cdiv(p.cout, 64));
    conv_simt_kernel<TI, TR, TO, 64, 64><<<grid, 256, 0, st>>>(p);
  } else {
    dim3 grid(cdiv(M, 128), 1);
    conv_simt_kernel<TI, TR, TO, 128, 16><<<grid, 256, 0, st>>>(p);
  }
  RV_LAUNCH_CHECK("conv_simt");
  return RV_OK;
}

int conv2d_simt(const rv_conv_desc* d, cudaStream_t st) {
  ConvP p;
  p.src0 = d->src0; p.src1 = d->src1; p.c0 = d->c0; p.c1 = d->src1 ? d->c1 : 0;
  p.H = d->H; p.W = d->W;
  p.Ho = (d->H + 2 * d->pad - d->kh) / d->stride + 1;
  p.Wo = (d->W + 2 * d->pad - d->kw) / d->stride + 1;
  p.w = (const float*)d->wpack;
  p.ldw = (d->cout + 3) / 4 * 4;
  p.bias = d->bias; p.cout = d->cout; p.kh = d->kh; p.kw = d->kw; p.stride = d->stride; p.pad = d->pad;
  p.act_pre = d->act_pre; p.act_post = d->act_post;
  p.gate = d->gate; p.gate_cs = d->gate_cs; p.res = d->res; p.res_cs = d->res_cs;
  p.out = d->out; p.out_cs = d->out_cs; p.pixel_shuffle = d->pixel_shuffle;
  p.K = d->kh * d->kw * (p.c0 + p.c1);
  RV_REQUIRE(d->k_real == p.K, "rv_conv2d(simt): k_real %d != kh*kw*(c0+c1) = %d", d->k_real, p.K);
  RV_REQUIRE(p.Ho > 0 && p.Wo > 0, "rv_conv2d: empty output");
  RV_REQUIRE(!d->pixel_shuffle || d->cout % 4 == 0, "rv_conv2d: pixel_shuffle needs cout %% 4 == 0");
  const int rdt = d->res ? d->res_dtype : d->out_dtype;
  // instantiate the combinations the engine uses: (in, res, out) in {all same} U {in16, f32, f32}
  if (d->in_dtype == RV_F32 && rdt == RV_F32 && d->out_dtype == RV_F32) return launch_simt<float, float, float>(p, st);
  if (d->in_dtype == RV_F16 && rdt == RV_F16 && d->out_dtype == RV_F16) return launch_simt<__half, __half, __half>(p, st);
  if (d->in_dtype == RV_F16 && rdt == RV_F32 && d->out_dtype == RV_F32) return launch_simt<__half, float, float>(p, st);
  if (d->in_dtype == RV_BF16 && rdt == RV_BF16 && d->out_dtype == RV_BF16) return launch_simt<__nv_bfloat16, __nv_bfloat16, __nv_bfloat16>(p, st);
  if (d->in_dtype == RV_BF16 && rdt == RV_F32 && d->out_dtype == RV_F32) return launch_simt<__nv_bfloat16, float, float>(p, st);
  return fail(RV_E_UNSUPPORTED, "rv_conv2d(simt): unsupported dtype combination in=%d res=%d out=%d",
              d->in_dtype, rdt, d->out_dtype);
}

}  // namespace rv
