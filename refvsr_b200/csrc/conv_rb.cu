// Fused residual block on wgmma:   out = post( x + conv2( act( conv1(x) ) ) )      (3x3, C -> C -> C, C <= 64)
//
// Replaces two rv_conv2d launches per ResidualBlockNoBN / ResBlock
// (mmedit/models/common/sr_backbone_utils.py:85-97, models/archs/RefVSR_/common.py:33-39): the intermediate
// activation never leaves the SM and the skip connection is read from the input box that is already in
// shared memory.
//
// Per output tile of 16 rows x 8 columns (M = 128):
//   * ONE TMA box of the input: 20 rows x 12 columns x 64 channels (2-pixel halo, pitch 12 pixel rows of 128 B,
//     SWIZZLE_128B, out-of-bounds zero fill = conv1's zero padding).
//   * conv1 is evaluated on the 18 x 10 halo region, indexed with the same pitch: m1 = yy*12 + xx, so that
//     input pixel (yy+ky, xx+kx) is simply smem row m1 + ky*12 + kx -> every tap is a row-shifted descriptor view of
//     the box.  216 rows, computed as four m64 blocks (two per consumer warpgroup; rows >= 216 are never read).
//   * epilogue 1 (from the accumulator registers): bias + activation -> 0 outside the image (conv2's zero padding) ->
//     16-bit -> written to shared memory in exactly the swizzled K-major operand layout (pitch 12), fence.proxy.async.
//   * conv2: M = 128 = 16 x 8, row m2 = ty*8 + tx reads intermediate row (ty+ky)*12 + tx + kx: 8-row groups are
//     contiguous, consecutive groups 12 rows apart -> SBO = 1536 bytes; warpgroup g computes tile rows 8g .. 8g + 7.
//   * epilogue 2: + bias + residual (input box pixel (ty+2, tx+2), de-swizzled from smem) -> optional
//     post-activation -> NHWC store.
// Both weight sets stay resident ([9 taps][NB][64] each, host-swizzled).  256 threads = two consumer warpgroups;
// thread 0 also issues the TMA loads.  Persistent CTAs walk the tile list.
#include <algorithm>

#include "common.cuh"
#include "tc_common.cuh"

namespace rv {

static constexpr int RB_TH = 16, RB_TW = 8;      // output tile
static constexpr int RB_P = 12;                  // pixel-row pitch of the input box and of the intermediate
static constexpr int RB_IN_ROWS = RB_TH + 4;     // 20 box rows
static constexpr uint32_t RB_IN_BYTES = RB_IN_ROWS * RB_P * 128;  // 30720
// intermediate: 256 rows; conv1's garbage rows (216..255) read the input up to 26 rows past the box, which lands here
static constexpr uint32_t RB_MID_BYTES = 256 * 128;
static constexpr int RB_MID_VALID = (RB_TH + 2) * RB_P;           // 216

struct RbP {
  int H, W, C, cout, NB, tiles_x, tiles_y, ksteps;
  uint32_t w_bytes;  // one conv: 9 * NB * 128
  const uint8_t* w1;
  const uint8_t* w2;
  const float* b1;
  const float* b2;
  float mid_slope, post_slope;
  void* out;
  int out_cs, pair_ok;
};

// byte offset of channel n of row r in a 128B-swizzled K-major tile whose base is 1024-byte aligned
__device__ __forceinline__ uint32_t sw128_off(int r, int n) {
  return (uint32_t)r * 128u + ((uint32_t)(((n >> 3) ^ (r & 7)) << 4)) + (uint32_t)((n & 7) * 2);
}

template <typename T, int NB>   // NB: output channels (= p.NB)
__global__ void __launch_bounds__(256, 1) conv_rb_kernel(const __grid_constant__ CUtensorMap tmx, const RbP p) {
  constexpr bool BF = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t bar_w, bar_in;
  __shared__ float b1_s[64], b2_s[64];
  const uint32_t raw = tc::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* smW1 = smem;
  uint8_t* smW2 = smW1 + p.w_bytes;
  uint8_t* smIn = smW2 + p.w_bytes;
  uint8_t* smMid = smIn + RB_IN_BYTES;
  const int g = threadIdx.x >> 7, t = threadIdx.x & 127, wq = t >> 5, lane = t & 31;

  if (threadIdx.x == 0) {
    tc::mbar_init(&bar_w, 1);
    tc::mbar_init(&bar_in, 1);
    tc::fence_barrier_init();
    tc::prefetch_tmap(&tmx);
  }
  if (threadIdx.x < 64) {
    b1_s[threadIdx.x] = (int)threadIdx.x < p.cout ? p.b1[threadIdx.x] : 0.f;
    b2_s[threadIdx.x] = (int)threadIdx.x < p.cout ? p.b2[threadIdx.x] : 0.f;
  }
  // intermediate channels the epilogue never writes (NB .. 63) are read by conv2's K slices only with zero weights, but
  // must not hold NaN patterns
  for (int i = threadIdx.x; i < (int)(RB_MID_BYTES / 16); i += blockDim.x) reinterpret_cast<uint4*>(smMid)[i] = make_uint4(0, 0, 0, 0);
  tc::fence_proxy_async();
  __syncthreads();
  if (threadIdx.x == 0) {
    tc::mbar_expect_tx(&bar_w, 2 * p.w_bytes);
    tc::bulk_load(p.w1, &bar_w, smW1, p.w_bytes);
    tc::bulk_load(p.w2, &bar_w, smW2, p.w_bytes);
  }
  tc::mbar_wait(&bar_w, 0);

  const uint32_t in_a = tc::smem_u32(smIn), mid_a = tc::smem_u32(smMid);
  const uint32_t w1_a = tc::smem_u32(smW1), w2_a = tc::smem_u32(smW2);
  T* out = reinterpret_cast<T*>(p.out);
  const int ntiles = p.tiles_x * p.tiles_y;
  uint32_t ph = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ph ^= 1u) {
    const int ty0 = tile / p.tiles_x, tx0 = tile - ty0 * p.tiles_x;
    if (threadIdx.x == 0) {
      tc::mbar_expect_tx(&bar_in, RB_IN_BYTES);
      tc::tma_load_3d(&tmx, &bar_in, smIn, 0, tx0 * RB_TW - 2, ty0 * RB_TH - 2);
    }
    tc::mbar_wait(&bar_in, ph);

    // ---- conv1 over the 18 x 10 halo region: m64 blocks 2g and 2g + 1 ----
    float acc1[2][NB / 2];
    tc::wgmma_fence();
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) {
        const uint64_t bd = tc::desc_sw128(w1_a + (uint32_t)((ky * 3 + kx) * NB * 128));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t ad = tc::desc_sw128(in_a + (uint32_t)((64 * (2 * g + h) + ky * RB_P + kx) * 128));
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < p.ksteps) tc::wgmma<NB, BF>(acc1[h], ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (ky | kx | k) ? 1u : 0u);
        }
      }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    // ---- epilogue 1 -> swizzled 16-bit intermediate ----
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2) {
        const int m1 = 64 * (2 * g + h) + 16 * wq + (lane >> 2) + 8 * r2;
        if (m1 >= RB_MID_VALID) continue;
        const int yy = m1 / RB_P, xx = m1 - yy * RB_P;
        const int iy = ty0 * RB_TH - 1 + yy, ix = tx0 * RB_TW - 1 + xx;
        const bool inside = xx < RB_TW + 2 && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
#pragma unroll
        for (int j = 0; j < NB / 8; ++j) {
          const int n = 8 * j + 2 * (lane & 3);
          float v[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float x = acc1[h][4 * j + 2 * r2 + e] + b1_s[n + e];
            v[e] = inside ? fmaxf(x, x * p.mid_slope) : 0.f;
          }
          T pr[2] = {from_f<T>(v[0]), from_f<T>(v[1])};
          *reinterpret_cast<uint32_t*>(smMid + sw128_off(m1, n)) = *reinterpret_cast<uint32_t*>(pr);
        }
      }
    tc::fence_proxy_async();                           // generic smem writes -> visible to the wgmma operand reads
    asm volatile("bar.sync 1, 256;" ::: "memory");

    // ---- conv2: tile rows 8g .. 8g + 7 ----
    float acc2[NB / 2];
    tc::wgmma_fence();
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) {
        const uint64_t bd = tc::desc_sw128(w2_a + (uint32_t)((ky * 3 + kx) * NB * 128));
        const uint64_t ad = tc::desc_sw128(mid_a + (uint32_t)(((8 * g + ky) * RB_P + kx) * 128), RB_P * 128);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (k < p.ksteps) tc::wgmma<NB, BF>(acc2, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (ky | kx | k) ? 1u : 0u);
      }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    // ---- epilogue 2: + bias + residual from the input box -> NHWC ----
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
      const int m2 = 64 * g + 16 * wq + (lane >> 2) + 8 * r2;
      const int ty = m2 >> 3, tx = m2 & 7;
      const int oy = ty0 * RB_TH + ty, ox = tx0 * RB_TW + tx;
      if (oy >= p.H || ox >= p.W) continue;
      const int rrow = (ty + 2) * RB_P + tx + 2;
#pragma unroll
      for (int j = 0; j < NB / 8; ++j) {
        const int n = 8 * j + 2 * (lane & 3);
        if (n >= p.cout) break;
        const T* rs = reinterpret_cast<const T*>(smIn + sw128_off(rrow, n));
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = acc2[4 * j + 2 * r2 + e] + b2_s[n + e] + to_f(rs[e]);
          v[e] = fmaxf(x, x * p.post_slope);
        }
        T* o = out + ((size_t)oy * p.W + ox) * p.out_cs + n;
        if (p.pair_ok && n + 1 < p.cout) {
          T pr[2] = {from_f<T>(v[0]), from_f<T>(v[1])};
          *reinterpret_cast<uint32_t*>(o) = *reinterpret_cast<uint32_t*>(pr);
        } else {
          o[0] = from_f<T>(v[0]);
          if (n + 1 < p.cout) o[1] = from_f<T>(v[1]);
        }
      }
    }
    __syncthreads();                                   // input box and intermediate are free for the next tile
  }
}

}  // namespace rv

using namespace rv;

extern "C" int rv_resblock(const rv_resblock_desc* d, void* stream) {
  RV_REQUIRE(d && d->src && d->out && d->w1 && d->w2 && d->b1 && d->b2, "rv_resblock: null argument");
  RV_REQUIRE(d->dtype == RV_F16 || d->dtype == RV_BF16, "rv_resblock: activations must be f16/bf16");
  RV_REQUIRE(d->c % 8 == 0 && d->c <= 64 && d->cout <= d->c && d->cout > 0, "rv_resblock: need cout <= c <= 64, c %% 8 == 0 (c=%d cout=%d)", d->c, d->cout);
  RV_REQUIRE(d->nb % 16 == 0 && d->nb >= 16 && d->nb <= 64 && d->nb >= d->cout, "rv_resblock: nb=%d", d->nb);
  RV_REQUIRE(d->H > 0 && d->W > 0, "rv_resblock: bad geometry");
  RV_REQUIRE(((uintptr_t)d->src % 16 == 0) && ((uintptr_t)d->w1 % 16 == 0) && ((uintptr_t)d->w2 % 16 == 0), "rv_resblock: 16-byte alignment");
  RV_REQUIRE(d->act_mid != RV_ACT_CLAMP3 && d->act_post != RV_ACT_CLAMP3, "rv_resblock: clamp3 not supported");
  static int num_sms = 0, max_smem = 0;
  if (num_sms == 0) {
    int dev = 0;
    RV_CUDA_OK(cudaGetDevice(&dev));
    RV_CUDA_OK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    RV_CUDA_OK(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  }
  RbP p;
  p.H = d->H; p.W = d->W; p.C = d->c; p.cout = d->cout; p.NB = d->nb;
  p.tiles_x = (d->W + RB_TW - 1) / RB_TW; p.tiles_y = (d->H + RB_TH - 1) / RB_TH;
  p.ksteps = (d->c + 15) / 16;      // K slices of the input (conv1) and of the intermediate (conv2; zero weights beyond cout)
  p.w_bytes = 9u * (uint32_t)p.NB * 128u;
  p.w1 = (const uint8_t*)d->w1; p.w2 = (const uint8_t*)d->w2; p.b1 = d->b1; p.b2 = d->b2;
  auto slope = [](int act) { return act == RV_ACT_RELU ? 0.f : act == RV_ACT_LRELU01 ? 0.1f : act == RV_ACT_LRELU02 ? 0.2f : 1.f; };
  p.mid_slope = slope(d->act_mid); p.post_slope = slope(d->act_post);
  p.out = d->out; p.out_cs = d->out_cs;
  p.pair_ok = ((uintptr_t)d->out % 4 == 0) && (d->out_cs % 2 == 0);
  const size_t smem = 1024 + 2 * (size_t)p.w_bytes + RB_IN_BYTES + RB_MID_BYTES;
  RV_REQUIRE(smem <= (size_t)max_smem, "rv_resblock: %zu bytes of shared memory do not fit", smem);
  PFN_tmapEncodeTiled enc = get_tmap_encoder();
  if (!enc) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  CUtensorMap tm;
  cuuint64_t gdim[3] = {(cuuint64_t)d->c, (cuuint64_t)d->W, (cuuint64_t)d->H};
  cuuint64_t gstr[2] = {(cuuint64_t)d->c * 2, (cuuint64_t)d->W * d->c * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)RB_P, (cuuint32_t)RB_IN_ROWS};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(&tm, d->dtype == RV_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3,
                   const_cast<void*>(d->src), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled(resblock) failed (%d)", (int)r);
  const int grid = std::min(p.tiles_x * p.tiles_y, num_sms);
  cudaStream_t st = (cudaStream_t)stream;
  static size_t configured[2][4] = {};
  const int ki = d->dtype == RV_BF16 ? 1 : 0, ni = p.NB / 16 - 1;
  void (*const kerns[2][4])(CUtensorMap, RbP) = {
      {conv_rb_kernel<__half, 16>, conv_rb_kernel<__half, 32>, conv_rb_kernel<__half, 48>, conv_rb_kernel<__half, 64>},
      {conv_rb_kernel<__nv_bfloat16, 16>, conv_rb_kernel<__nv_bfloat16, 32>, conv_rb_kernel<__nv_bfloat16, 48>,
       conv_rb_kernel<__nv_bfloat16, 64>}};
  void (*kern)(CUtensorMap, RbP) = kerns[ki][ni];
  if (smem > configured[ki][ni]) {
    RV_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured[ki][ni] = smem;
  }
  kern<<<grid, 256, smem, st>>>(tm, p);
  RV_LAUNCH_CHECK("conv_rb");
  return RV_OK;
}
