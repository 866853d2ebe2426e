// LR <-> Ref patch matching: conf[l] = max_r <A[l], B[r]>, idx[l] = argmax_r  (attention.py:83-91)
// The reference materialises the (R x P) similarity matrix (16.8 GB fp32 at 270x480) and then
// reduces it; here the GEMM tiles never leave the SM: accumulators live in the registers of the
// consumer warpgroups and the max/argmax over reference patches is a running reduction over the N
// dimension, four threads per LR pixel - no atomics.
//
// Operands are fp16 rows produced by rv_patch_pack (pre-scaled by 2^6).  In "split" mode each row is
// [hi|lo|hi] x [hi|hi|lo], which makes the fp16 tensor-core product equal to the fp32 product up to
// the dropped lo*lo term (~2^-22 relative) - needed because the hard argmax is discontinuous.
#include "common.cuh"
#include "tc_common.cuh"

namespace rv {

// ------------------------------------------------------------------------------------------------
// CUDA-core yardstick (fp32 math on the same fp16 operands)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) match_simt_kernel(const __half* __restrict__ A, int P,
                                                         const __half* __restrict__ B, int R, int kpad,
                                                         float out_scale, float* __restrict__ conf,
                                                         int32_t* __restrict__ idx) {
  constexpr int BM = 64, BN = 64, BK = 32;
  __shared__ float As[BK][BM + 1];
  __shared__ float Bs[BK][BN + 1];
  __shared__ float red_v[BM][16];
  __shared__ int red_i[BM][16];
  const int tid = threadIdx.x, tn = tid % 16, tm = tid / 16;
  const int m0 = blockIdx.x * BM;
  float best[4];
  int bidx[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { best[i] = -INFINITY; bidx[i] = 0; }
  for (int n0 = 0; n0 < R; n0 += BN) {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < kpad; k0 += BK) {
      for (int e = tid; e < BM * BK; e += 256) {
        int kk = e % BK, mm = e / BK;
        int m = m0 + mm, k = k0 + kk;
        As[kk][mm] = (m < P && k < kpad) ? __half2float(A[(size_t)m * kpad + k]) : 0.f;
        int n = n0 + mm;
        Bs[kk][mm] = (n < R && k < kpad) ? __half2float(B[(size_t)n * kpad + k]) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { a[i] = As[kk][tm * 4 + i]; b[i] = Bs[kk][tn * 4 + i]; }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int n = n0 + tn * 4 + j;
        if (n < R && acc[i][j] > best[i]) { best[i] = acc[i][j]; bidx[i] = n; }
      }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) { red_v[tm * 4 + i][tn] = best[i]; red_i[tm * 4 + i][tn] = bidx[i]; }
  __syncthreads();
  if (tid < BM) {
    float bv = red_v[tid][0];
    int bi = red_i[tid][0];
    for (int t = 1; t < 16; ++t) {
      float v = red_v[tid][t];
      int i2 = red_i[tid][t];
      if (v > bv || (v == bv && i2 < bi)) { bv = v; bi = i2; }
    }
    int m = m0 + tid;
    if (m < P) { conf[m] = bv * out_scale; idx[m] = bi; }
  }
}

// ------------------------------------------------------------------------------------------------
// wgmma streaming argmax GEMM
// ------------------------------------------------------------------------------------------------
// 384 threads: warp 0 = TMA producer, warpgroups 1 and 2 = consumers, consumer c multiplies LR rows 64 c .. 64 c + 63 of
// the CTA's 128-row A block (resident in shared memory) by every 128-row B tile streamed through the ring.  Thread t
// of a consumer holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) and the column pairs 8 j + 2 (t % 4) of the tile: a running
// max / argmax per row and thread over the N dimension, then the four threads of a row combine theirs (shuffles).
static constexpr int MT_BM = 128, MT_BN = 128, MT_MAXCH = 7, MT_SLOTS_MAX = 6;

struct MtP {
  int P, R, nk, slots, ntiles_n;
  float out_scale;
  float* conf;
  int32_t* idx;
};

__global__ void __launch_bounds__(384, 1)
match_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const MtP p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t bar_full[MT_SLOTS_MAX], bar_empty[MT_SLOTS_MAX], bar_a;
  const uint32_t raw = tc::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  constexpr uint32_t A_CH = MT_BM * 128, B_ST = MT_BN * 128;
  uint8_t* smemA = smem;
  uint8_t* smemB = smem + (size_t)p.nk * A_CH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int warp_u = __shfl_sync(0xffffffffu, warp, 0);   // provably warp-uniform copy for the role dispatch
  const int m0 = blockIdx.x * MT_BM;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.slots; ++i) { tc::mbar_init(&bar_full[i], 1); tc::mbar_init(&bar_empty[i], 8); }
    tc::mbar_init(&bar_a, 1);
    tc::fence_barrier_init();
    tc::prefetch_tmap(&tmA);
    tc::prefetch_tmap(&tmB);
  }
  __syncthreads();

  if (warp_u == 0) {
    if (tc::elect_one()) {
      tc::mbar_expect_tx(&bar_a, (uint32_t)p.nk * A_CH);
      for (int c = 0; c < p.nk; ++c) tc::tma_load_2d(&tmA, &bar_a, smemA + (size_t)c * A_CH, c * 64, m0);
    }
    __syncwarp();
    int slot = 0;
    uint32_t ph = 0;
    for (int nt = 0; nt < p.ntiles_n; ++nt)
      for (int c = 0; c < p.nk; ++c) {
        tc::mbar_wait(&bar_empty[slot], ph ^ 1u);
        if (tc::elect_one()) {
          tc::mbar_expect_tx(&bar_full[slot], B_ST);
          tc::tma_load_2d(&tmB, &bar_full[slot], smemB + (size_t)slot * B_ST, c * 64, nt * MT_BN);
        }
        __syncwarp();
        if (++slot == p.slots) { slot = 0; ph ^= 1u; }
      }
  } else if (warp_u >= 4) {
    const int cons = (warp_u >> 2) - 1, wq = warp_u & 3;
    const uint32_t a0 = tc::smem_u32(smemA) + (uint32_t)cons * 64 * 128, b0 = tc::smem_u32(smemB);
    float best[2] = {-INFINITY, -INFINITY};
    int bidx[2] = {0, 0};
    float acc[MT_BN / 2];
    tc::mbar_wait(&bar_a, 0);
    int slot = 0, prev = -1;
    uint32_t ph = 0;
    for (int nt = 0; nt < p.ntiles_n; ++nt) {
      for (int c = 0; c < p.nk; ++c) {
        tc::mbar_wait(&bar_full[slot], ph);
        const uint64_t ad = tc::desc_sw128(a0 + (uint32_t)c * A_CH), bd = tc::desc_sw128(b0 + (uint32_t)slot * B_ST);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) tc::wgmma<MT_BN, false>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (c | k) ? 1u : 0u);
        tc::wgmma_commit();
        tc::wgmma_wait<1>();
        if (prev >= 0 && lane == 0) tc::mbar_arrive(&bar_empty[prev]);
        prev = slot;
        if (++slot == p.slots) { slot = 0; ph ^= 1u; }
      }
      tc::wgmma_wait<0>();
      if (lane == 0) tc::mbar_arrive(&bar_empty[prev]);
      prev = -1;
      // columns in increasing order with a strict > keep the earliest maximum of this thread
      const int rbase = nt * MT_BN + 2 * (lane & 3);
      const int nvalid = p.R - rbase;
#pragma unroll
      for (int j = 0; j < MT_BN / 8; ++j)
#pragma unroll
        for (int r2 = 0; r2 < 2; ++r2)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float v = acc[4 * j + 2 * r2 + e];
            if (8 * j + e < nvalid && v > best[r2]) { best[r2] = v; bidx[r2] = rbase + 8 * j + e; }
          }
    }
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) {
#pragma unroll
      for (int off = 1; off < 4; off <<= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best[r2], off);
        const int oi = __shfl_xor_sync(0xffffffffu, bidx[r2], off);
        if (ov > best[r2] || (ov == best[r2] && oi < bidx[r2])) { best[r2] = ov; bidx[r2] = oi; }
      }
      const int m = m0 + cons * 64 + 16 * wq + (lane >> 2) + 8 * r2;
      if ((lane & 3) == 0 && m < p.P) {
        p.conf[m] = best[r2] * p.out_scale;
        p.idx[m] = bidx[r2];
      }
    }
  }
}

static int make_rows_tmap(CUtensorMap* m, const void* ptr, int kpad, int rows, int box_rows) {
  PFN_tmapEncodeTiled enc = get_tmap_encoder();
  if (!enc) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[2] = {(cuuint64_t)kpad, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)kpad * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled(rows) failed (%d)", (int)r);
  return RV_OK;
}

static int match_tc(const void* A, int P, const void* B, int R, int kpad, float out_scale, float* conf,
                    int32_t* idx, cudaStream_t st) {
  RV_REQUIRE(kpad % 64 == 0 && kpad / 64 <= MT_MAXCH, "rv_match_argmax(tc): kpad=%d must be a multiple of 64, <= %d", kpad, 64 * MT_MAXCH);
  RV_REQUIRE(((uintptr_t)A % 16 == 0) && ((uintptr_t)B % 16 == 0), "rv_match_argmax(tc): operands must be 16-byte aligned");
  int dev = 0, max_smem = 0;
  RV_CUDA_OK(cudaGetDevice(&dev));
  RV_CUDA_OK(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  MtP p;
  p.P = P; p.R = R; p.nk = kpad / 64; p.ntiles_n = (R + MT_BN - 1) / MT_BN;
  p.out_scale = out_scale; p.conf = conf; p.idx = idx;
  const size_t a_bytes = (size_t)p.nk * MT_BM * 128;
  const size_t budget = (size_t)max_smem - 1024 - 2048;
  p.slots = (int)std::min<size_t>(MT_SLOTS_MAX, (budget - a_bytes) / ((size_t)MT_BN * 128));
  RV_REQUIRE(p.slots >= 2, "rv_match_argmax(tc): not enough shared memory");
  const size_t smem = 1024 + a_bytes + (size_t)p.slots * MT_BN * 128;
  CUtensorMap tmA, tmB;
  int rc = make_rows_tmap(&tmA, A, kpad, P, MT_BM);
  if (rc) return rc;
  rc = make_rows_tmap(&tmB, B, kpad, R, MT_BN);
  if (rc) return rc;
  static size_t configured = 0;
  if (smem > configured) {
    RV_CUDA_OK(cudaFuncSetAttribute(match_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  match_tc_kernel<<<cdiv(P, MT_BM), 384, smem, st>>>(tmA, tmB, p);
  RV_LAUNCH_CHECK("match_tc");
  return RV_OK;
}

}  // namespace rv

using namespace rv;

extern "C" int rv_match_argmax(const void* A, int P, const void* B, int R, int kpad, float out_scale,
                               float* conf, int32_t* idx, int impl, void* stream) {
  RV_REQUIRE(A && B && conf && idx && P > 0 && R > 0 && kpad > 0, "rv_match_argmax: bad arguments");
  if (impl == 1) return match_tc(A, P, B, R, kpad, out_scale, conf, idx, (cudaStream_t)stream);
  match_simt_kernel<<<cdiv(P, 64), 256, 0, (cudaStream_t)stream>>>((const __half*)A, P, (const __half*)B, R,
                                                                 kpad, out_scale, conf, idx);
  RV_LAUNCH_CHECK("match_simt");
  return RV_OK;
}
