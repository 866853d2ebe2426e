// rv_conv_chain: a whole CHAIN of 3x3 C->C convolutions (the trunk of ResidualBlocksWithInputConv, the ResList decoders) in
// ONE persistent wgmma launch, with tile-level instead of grid-level dependencies between layers.
//
//   * tile t of layer l+1 may start as soon as the <= 9 tiles around t have finished layer l.  Every tile has ONE monotone
//     counter in global memory, flags[t] = number of layers completed.  Tiles keep their CTA across layers
//     (t = cta + k * grid), and each CTA walks (layer, k) in lexicographic order, so the wait graph is acyclic (a CTA
//     blocked on layer l+1 never holds back a layer-l tile) as long as all CTAs are co-resident: grid <= #SMs, 1 CTA / SM.
//   * the same condition covers every hazard of ANY layer list over a small set of ping-pong buffers: a layer's source was
//     last written at some layer <= l-1 (RAW: neighbours' flags >= l), and its destination was last read WITH A HALO by the
//     neighbours' tiles of some layer <= l-1 (WAR: same flags).  Residual reads have no halo and belong to the tile itself,
//     i.e. to this CTA.
//   * publication: every thread's stores, __threadfence, CTA barrier, then one release store of flags[t] = l + 1.  The
//     waiting side polls with acquire loads and issues fence.proxy.async before its TMA load reads the data.
// Geometry = conv_tc.cu MODE 1: tile 16 rows x 8 columns, ONE 18 x 10 pixel box per tile (64-channel rows, SWIZZLE_128B,
// out-of-bounds zero fill = conv padding), the 9 taps are row-shifted wgmma descriptor views of it; one warpgroup per CTA.
// The MMA sequence (tap order, K slices, N = NB) and the fp32 epilogue (bias, act, + residual, act, round) are those of
// conv_tc.cu, so a chain is BIT-IDENTICAL to the same layers launched one by one (tests/test_gpu_kernels.py::test_conv_chain_*).
#include <algorithm>

#include "common.cuh"
#include "tc_common.cuh"

namespace rv {
namespace {

constexpr int CH_MAXL = RV_CHAIN_MAX_LAYERS, CH_MAXB = RV_CHAIN_MAX_BUFFERS;
constexpr int CH_TH = 16, CH_TW = 8, CH_BW = CH_TW + 2, CH_BH = CH_TH + 2;
constexpr uint32_t CH_A_TX = CH_BH * CH_BW * 128;              // bytes one activation box delivers (23 040)
constexpr uint32_t CH_A_BYTES = (CH_A_TX + 1023u) & ~1023u;    // 1024-byte swizzle atoms

struct ChLayer {
  const uint8_t* wpack;   // layout-1 weight image [9 taps][NB][64], SWIZZLE_128B byte image (packing.pack_tc)
  const float* bias;
  float pre_slope, post_slope;   // act(v) = max(v, v * slope): 1 none, 0 ReLU, 0.1 / 0.2 LeakyReLU
  int src, res, dst;             // buffer indices; res < 0: no residual
};

struct ChP {
  int H, W, C, NB, tiles_x, tiles_y, nlayers, ksteps;
  uint32_t w_bytes;
  int* flags;
  void* buf[CH_MAXB];
  ChLayer layer[CH_MAXL];
};

struct ChMaps {
  CUtensorMap ld[CH_MAXB];   // box 64 ch x 10 x 18 (tile + halo)
};

__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

template <typename T, int NB>   // NB: rows of the weight image (= p.NB)
__global__ void __launch_bounds__(128, 1) conv_chain_kernel(const __grid_constant__ ChMaps maps, const __grid_constant__ ChP p) {
  constexpr bool BF = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t bar_w, bar_in;
  __shared__ float bias_s[48];
  const uint32_t raw = tc::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* smIn = smem;
  uint8_t* smW = smem + CH_A_BYTES;
  const int t = threadIdx.x, wq = t >> 5, lane = t & 31;
  const uint32_t in_a = tc::smem_u32(smIn), w_a = tc::smem_u32(smW);
  const int ntiles = p.tiles_x * p.tiles_y;

  if (t == 0) {
    tc::mbar_init(&bar_w, 1);
    tc::mbar_init(&bar_in, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  uint32_t ph_in = 0;
  for (int l = 0; l < p.nlayers; ++l) {
    const ChLayer& L = p.layer[l];
    // weights and bias of layer l replace those of layer l - 1 (whose MMAs have all retired: wait<0> + barrier below)
    if (t == 0) {
      tc::mbar_expect_tx(&bar_w, p.w_bytes);
      tc::bulk_load(L.wpack, &bar_w, smW, p.w_bytes);
    }
    if (t < p.NB) bias_s[t] = L.bias[t];
    __syncthreads();
    tc::mbar_wait(&bar_w, (uint32_t)l & 1u);
    const T* res = L.res >= 0 ? reinterpret_cast<const T*>(p.buf[L.res]) : nullptr;
    T* dst = reinterpret_cast<T*>(p.buf[L.dst]);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ph_in ^= 1u) {
      const int ty0 = tile / p.tiles_x, tx0 = tile - ty0 * p.tiles_x;
      if (t == 0) {
        // RAW on the source and WAR on the destination: the <= 9 tiles around this one have completed layer l - 1
        for (int dy = -1; dy <= 1; ++dy)
          for (int dx = -1; dx <= 1; ++dx) {
            const int y = ty0 + dy, x = tx0 + dx;
            if (y < 0 || y >= p.tiles_y || x < 0 || x >= p.tiles_x) continue;
            const int* f = p.flags + y * p.tiles_x + x;
            while (ld_acquire(f) < l) __nanosleep(64);
          }
        asm volatile("fence.proxy.async.global;" ::: "memory");   // generic stores of other CTAs -> this TMA read
        tc::mbar_expect_tx(&bar_in, CH_A_TX);
        tc::tma_load_3d(&maps.ld[L.src], &bar_in, smIn, 0, tx0 * CH_TW - 1, ty0 * CH_TH - 1);
      }
      tc::mbar_wait(&bar_in, ph_in);
      float acc[2][NB / 2];
      tc::wgmma_fence();
      for (int ky = 0; ky < 3; ++ky)
        for (int kx = 0; kx < 3; ++kx) {
          const uint64_t bd = tc::desc_sw128(w_a + (uint32_t)((ky * 3 + kx) * NB * 128));
          const uint32_t at = in_a + (uint32_t)((ky * CH_BW + kx) * 128);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint64_t ad = tc::desc_sw128(at + (uint32_t)h * 8 * CH_BW * 128, CH_BW * 128);
#pragma unroll
            for (int k = 0; k < 3; ++k)
              if (k < p.ksteps) tc::wgmma<NB, BF>(acc[h], ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (ky | kx | k) ? 1u : 0u);
          }
        }
      tc::wgmma_commit();
      tc::wgmma_wait<0>();
      // ---- epilogue (the arithmetic of conv_tc.cu) ----
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r2 = 0; r2 < 2; ++r2) {
          const int m = 64 * h + 16 * wq + (lane >> 2) + 8 * r2;
          const int oy = ty0 * CH_TH + (m >> 3), ox = tx0 * CH_TW + (m & 7);
          if (oy >= p.H || ox >= p.W) continue;
          const size_t pix = (size_t)oy * p.W + ox;
#pragma unroll
          for (int j = 0; j < NB / 8; ++j) {
            const int n = 8 * j + 2 * (lane & 3);
            if (n >= p.C) break;
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float x = acc[h][4 * j + 2 * r2 + e] + bias_s[n + e];
              v[e] = fmaxf(x, x * L.pre_slope);
            }
            if (res != nullptr) {       // written earlier in this launch by this CTA: coherent (non-.nc) loads
              uint32_t rw = *reinterpret_cast<const volatile uint32_t*>(res + pix * p.C + n);
              const T* r = reinterpret_cast<const T*>(&rw);
              v[0] += to_f(r[0]); v[1] += to_f(r[1]);
            }
            T pr[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) pr[e] = from_f<T>(fmaxf(v[e], v[e] * L.post_slope));
            *reinterpret_cast<uint32_t*>(dst + pix * p.C + n) = *reinterpret_cast<uint32_t*>(pr);
          }
        }
      __threadfence();
      __syncthreads();                 // all stores of the tile done; the input box is free again
      if (t == 0) asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p.flags + tile), "r"(l + 1) : "memory");
    }
  }
}

int make_map(CUtensorMap* m, const void* ptr, int C, int W, int H, int fmt) {
  PFN_tmapEncodeTiled enc = get_tmap_encoder();
  if (!enc) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[3] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H};
  cuuint64_t gstr[2] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2};
  cuuint32_t box[3] = {64u, (cuuint32_t)CH_BW, (cuuint32_t)CH_BH};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, fmt ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(ptr), gdim, gstr,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled failed (%d) C=%d W=%d H=%d", (int)r, C, W, H);
  return RV_OK;
}

float slope_of(int act) { return act == RV_ACT_RELU ? 0.f : act == RV_ACT_LRELU01 ? 0.1f : act == RV_ACT_LRELU02 ? 0.2f : 1.f; }

}  // namespace
}  // namespace rv

using namespace rv;

extern "C" int rv_conv_chain(const rv_conv_chain_desc* d, void* stream) {
  RV_REQUIRE(d != nullptr && d->layers != nullptr && d->flags != nullptr, "rv_conv_chain: null descriptor / layers / flags");
  RV_REQUIRE(d->nbuf >= 2 && d->nbuf <= CH_MAXB, "rv_conv_chain: 2..%d buffers (got %d)", CH_MAXB, d->nbuf);
  RV_REQUIRE(d->nlayers >= 1 && d->nlayers <= CH_MAXL, "rv_conv_chain: 1..%d layers per launch (got %d)", CH_MAXL, d->nlayers);
  RV_REQUIRE(d->dtype == RV_F16 || d->dtype == RV_BF16, "rv_conv_chain: activations must be f16 / bf16");
  RV_REQUIRE(d->H > 0 && d->W > 0 && d->C > 0 && d->C % 8 == 0 && d->C <= 48, "rv_conv_chain: C=%d must be a multiple of 8, <= 48", d->C);
  RV_REQUIRE(d->nb >= 16 && d->nb <= 48 && d->nb % 16 == 0 && d->nb >= d->C, "rv_conv_chain: nb=%d must be 16/32/48 and >= C=%d", d->nb, d->C);
  for (int b = 0; b < d->nbuf; ++b)
    RV_REQUIRE(d->buf[b] != nullptr && (uintptr_t)d->buf[b] % 16 == 0, "rv_conv_chain: buffer %d null or not 16-byte aligned", b);
  static int num_sms = 0;
  if (num_sms == 0) {
    int dev = 0;
    RV_CUDA_OK(cudaGetDevice(&dev));
    RV_CUDA_OK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  static ChP p;            // (host-side scratch; the launch copies it by value)
  static ChMaps maps;
  p.H = d->H; p.W = d->W; p.C = d->C; p.NB = d->nb;
  p.tiles_x = (d->W + CH_TW - 1) / CH_TW;
  p.tiles_y = (d->H + CH_TH - 1) / CH_TH;
  p.nlayers = d->nlayers;
  p.ksteps = (d->C + 15) / 16;
  p.w_bytes = 9u * (uint32_t)d->nb * 128u;
  p.flags = d->flags;
  for (int b = 0; b < CH_MAXB; ++b) p.buf[b] = b < d->nbuf ? d->buf[b] : nullptr;
  for (int l = 0; l < d->nlayers; ++l) {
    const rv_chain_layer& s = d->layers[l];
    RV_REQUIRE(s.wpack && s.bias && (uintptr_t)s.wpack % 16 == 0 && (uintptr_t)s.bias % 16 == 0, "rv_conv_chain: layer %d: null / unaligned weights", l);
    RV_REQUIRE(s.src >= 0 && s.src < d->nbuf && s.dst >= 0 && s.dst < d->nbuf && s.res < d->nbuf, "rv_conv_chain: layer %d: bad buffer index", l);
    RV_REQUIRE(s.dst != s.src, "rv_conv_chain: layer %d writes its own source (3x3 conv cannot run in place)", l);
    RV_REQUIRE(s.act_pre != RV_ACT_CLAMP3 && s.act_post != RV_ACT_CLAMP3, "rv_conv_chain: clamp3 is not supported");
    ChLayer& L = p.layer[l];
    L.wpack = (const uint8_t*)s.wpack; L.bias = s.bias;
    L.pre_slope = slope_of(s.act_pre); L.post_slope = slope_of(s.act_post);
    L.src = s.src; L.res = s.res < 0 ? -1 : s.res; L.dst = s.dst;
  }
  const int fmt = d->dtype == RV_BF16 ? 1 : 0;
  for (int b = 0; b < d->nbuf; ++b) {
    const int rc = make_map(&maps.ld[b], d->buf[b], d->C, d->W, d->H, fmt);
    if (rc) return rc;
  }
  for (int b = d->nbuf; b < CH_MAXB; ++b) maps.ld[b] = maps.ld[0];
  const int ntiles = p.tiles_x * p.tiles_y;
  int grid = std::min(num_sms, ntiles);
  if (d->max_ctas > 0) grid = std::min(grid, (int)d->max_ctas);
  const size_t smem = 1024 + CH_A_BYTES + p.w_bytes;
  cudaStream_t st = (cudaStream_t)stream;
  RV_CUDA_OK(cudaMemsetAsync(d->flags, 0, (size_t)ntiles * sizeof(int), st));
  static size_t configured[2][3] = {};
  const int ni = p.NB / 16 - 1;
  void (*const kerns[2][3])(ChMaps, ChP) = {
      {conv_chain_kernel<__half, 16>, conv_chain_kernel<__half, 32>, conv_chain_kernel<__half, 48>},
      {conv_chain_kernel<__nv_bfloat16, 16>, conv_chain_kernel<__nv_bfloat16, 32>, conv_chain_kernel<__nv_bfloat16, 48>}};
  void (*kern)(ChMaps, ChP) = kerns[fmt][ni];
  if (smem > configured[fmt][ni]) {
    RV_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured[fmt][ni] = smem;
  }
  kern<<<grid, 128, smem, st>>>(maps, p);
  RV_LAUNCH_CHECK("conv_chain");
  return RV_OK;
}
