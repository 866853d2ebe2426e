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
// 384 threads: warp 0 = TMA producer, warpgroups 1 and 2 = consumers.  A CTA owns MB x 128 LR rows (its A block, resident in
// shared memory); consumer c multiplies rows 64 MB c .. 64 MB (c + 1) - 1, as MB m64 accumulator blocks, by every 128-row B
// tile streamed through the ring.  In block h, thread t of a consumer holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) and the
// column pairs 8 j + 2 (t % 4) of the tile: a running max / argmax per row and thread over the N dimension, then the four
// threads of a row combine theirs (shuffles).  MB = 2 halves the B traffic from L2 per LR row; it is taken when the 256-row
// A block leaves room for two tiles' chunks in the ring (single mode), otherwise MB = 1 (split mode).
//
// K is streamed in chunks: kpad / 64 chunks of 64 columns (SWIZZLE_128B), then, if kpad % 64 != 0, one tail chunk of up to
// three 16-column slices (SWIZZLE_32B, one TMA box each).  Only real K is multiplied, and each accumulator sees the same
// 16-column k-steps in the same order as with kpad rounded up to a multiple of 64 and zero-filled: the dropped k-steps only
// added exact zeros, so conf / idx do not depend on the padding.
//
// MB = 2: the consumers take turns on the tensor cores.  A consumer issues a tile's MMAs, all chunks as one commit group,
// only after the other consumer has issued its own for the previous tile (consumer 0 starts), and frees the tile's slots once
// they have retired.  The batches then queue back to back, and each consumer's argmax scan runs under the other's MMAs; left
// alone, both issue at once, share the tensor cores and then both scan with them idle.  This needs two tiles' chunks in the
// ring: one consumer's next tile while the other still multiplies the current one.
// MB = 1: the ring may hold a single tile, so both consumers stream it chunk by chunk, each freeing a slot as soon as its
// MMAs on it have retired.
static constexpr int MT_BN = 128, MT_MAXK = 448, MT_SLOTS_MAX = 8;
static constexpr uint32_t MT_SLOT = MT_BN * 128;   // one B chunk: 128 rows x 64 columns (a tail chunk uses part of it)

struct MtP {
  int P, R, nfull, ntail, slots, ntiles_n;
  float out_scale;
  float* conf;
  int32_t* idx;
};

// Running max / argmax over one tile: columns in increasing order with a strict > keep the earliest maximum of this thread.
// Only the last tile can reach past R, so only it tests the column (RAGGED).
template <int MB, bool RAGGED>
__device__ __forceinline__ void mt_scan(const float (&acc)[MB][MT_BN / 2], float (&best)[MB][2], int (&bidx)[MB][2],
                                        int rbase, int nvalid) {
#pragma unroll
  for (int h = 0; h < MB; ++h)
#pragma unroll
    for (int j = 0; j < MT_BN / 8; ++j)
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float v = acc[h][4 * j + 2 * r2 + e];
          if ((!RAGGED || 8 * j + e < nvalid) && v > best[h][r2]) { best[h][r2] = v; bidx[h][r2] = rbase + 8 * j + e; }
        }
}

template <int MB>
__global__ void __launch_bounds__(384, 1)
match_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA16,
                const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmB16, const MtP p) {
  constexpr int BM = 128 * MB;
  constexpr uint32_t A_CH = BM * 128, A_SL = BM * 32, B_SL = MT_BN * 32;   // A chunk; A / B 16-column slice
  extern __shared__ uint8_t smem_raw[];
  constexpr bool TURNS = MB == 2;
  __shared__ uint64_t bar_full[MT_SLOTS_MAX], bar_empty[MT_SLOTS_MAX], bar_a, bar_turn[2];
  const uint32_t raw = tc::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  const int nch = p.nfull + (p.ntail > 0);
  uint8_t* smemA = smem;                                                   // nfull chunks, then ntail slices
  uint8_t* smemB = smem + (size_t)p.nfull * A_CH + (size_t)p.ntail * A_SL;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int warp_u = __shfl_sync(0xffffffffu, warp, 0);   // provably warp-uniform copy for the role dispatch
  const int m0 = blockIdx.x * BM;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.slots; ++i) { tc::mbar_init(&bar_full[i], 1); tc::mbar_init(&bar_empty[i], 8); }
    tc::mbar_init(&bar_a, 1);
    for (int c = 0; c < 2; ++c) tc::mbar_init(&bar_turn[c], 4);   // one arrival per warp of the other consumer
    tc::fence_barrier_init();
    if (p.nfull) {
      tc::prefetch_tmap(&tmA);
      tc::prefetch_tmap(&tmB);
    }
    if (p.ntail) {
      tc::prefetch_tmap(&tmA16);
      tc::prefetch_tmap(&tmB16);
    }
  }
  __syncthreads();

  if (warp_u == 0) {
    if (tc::elect_one()) {
      tc::mbar_expect_tx(&bar_a, (uint32_t)p.nfull * A_CH + (uint32_t)p.ntail * A_SL);
      for (int c = 0; c < p.nfull; ++c) tc::tma_load_2d(&tmA, &bar_a, smemA + (size_t)c * A_CH, c * 64, m0);
      for (int s = 0; s < p.ntail; ++s)
        tc::tma_load_2d(&tmA16, &bar_a, smemA + (size_t)p.nfull * A_CH + (size_t)s * A_SL, p.nfull * 64 + s * 16, m0);
    }
    __syncwarp();
    int slot = 0;
    uint32_t ph = 0;
    for (int nt = 0; nt < p.ntiles_n; ++nt)
      for (int c = 0; c < nch; ++c) {
        tc::mbar_wait(&bar_empty[slot], ph ^ 1u);
        if (tc::elect_one()) {
          uint8_t* dst = smemB + (size_t)slot * MT_SLOT;
          if (c < p.nfull) {
            tc::mbar_expect_tx(&bar_full[slot], MT_SLOT);
            tc::tma_load_2d(&tmB, &bar_full[slot], dst, c * 64, nt * MT_BN);
          } else {
            tc::mbar_expect_tx(&bar_full[slot], (uint32_t)p.ntail * B_SL);
            for (int s = 0; s < p.ntail; ++s)
              tc::tma_load_2d(&tmB16, &bar_full[slot], dst + (size_t)s * B_SL, p.nfull * 64 + s * 16, nt * MT_BN);
          }
        }
        __syncwarp();
        if (++slot == p.slots) { slot = 0; ph ^= 1u; }
      }
  } else if (warp_u >= 4) {
    const int cons = (warp_u >> 2) - 1, wq = warp_u & 3;
    const uint32_t a0 = tc::smem_u32(smemA) + (uint32_t)(cons * MB * 64 * 128);
    const uint32_t a16 = tc::smem_u32(smemA) + (uint32_t)p.nfull * A_CH + (uint32_t)(cons * MB * 64 * 32);
    const uint32_t b0 = tc::smem_u32(smemB);
    float best[MB][2];
    int bidx[MB][2];
#pragma unroll
    for (int h = 0; h < MB; ++h)
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2) { best[h][r2] = -INFINITY; bidx[h][r2] = 0; }
    float acc[MB][MT_BN / 2];
    tc::mbar_wait(&bar_a, 0);
    int slot = 0, prev = -1;
    uint32_t ph = 0, tph = 0;
    for (int nt = 0; nt < p.ntiles_n; ++nt) {
      const int slot0 = slot;
      for (int c = 0; c < nch; ++c) {
        tc::mbar_wait(&bar_full[slot], ph);
        if (TURNS && c == 0 && (cons | nt) != 0) {
          tc::mbar_wait(&bar_turn[cons], tph);
          tph ^= 1u;
        }
        const uint32_t bs = b0 + (uint32_t)slot * MT_SLOT;
        tc::wgmma_fence();
        if (c < p.nfull) {
          const uint64_t bd = tc::desc_sw128(bs);
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int h = 0; h < MB; ++h)
              tc::wgmma<MT_BN, false>(acc[h], tc::desc_sw128(a0 + (uint32_t)c * A_CH + (uint32_t)h * 64 * 128) + (uint64_t)(2 * k),
                                      bd + (uint64_t)(2 * k), (c | k) ? 1u : 0u);
        } else {
#pragma unroll
          for (int k = 0; k < 3; ++k)
            if (k < p.ntail) {
              const uint64_t bd = tc::desc_sw32(bs + (uint32_t)k * B_SL);
#pragma unroll
              for (int h = 0; h < MB; ++h)
                tc::wgmma<MT_BN, false>(acc[h], tc::desc_sw32(a16 + (uint32_t)k * A_SL + (uint32_t)h * 64 * 32), bd,
                                        (c | k) ? 1u : 0u);
            }
        }
        if (!TURNS) {
          // the previous chunk's MMAs have retired once at most this chunk's group is in flight: free its slot
          tc::wgmma_commit();
          tc::wgmma_wait<1>();
          if (prev >= 0 && lane == 0) tc::mbar_arrive(&bar_empty[prev]);
          prev = slot;
        }
        if (++slot == p.slots) { slot = 0; ph ^= 1u; }
      }
      if (TURNS) {
        tc::wgmma_commit();
        if (lane == 0) tc::mbar_arrive(&bar_turn[cons ^ 1]);   // the other consumer's turn
        tc::wgmma_wait<0>();
        if (lane == 0)
          for (int c = 0, s = slot0; c < nch; ++c, s = (s + 1 == p.slots) ? 0 : s + 1) tc::mbar_arrive(&bar_empty[s]);
      } else {
        tc::wgmma_wait<0>();
        if (lane == 0) tc::mbar_arrive(&bar_empty[prev]);
        prev = -1;
      }
      const int rbase = nt * MT_BN + 2 * (lane & 3);
      if (nt == p.ntiles_n - 1) mt_scan<MB, true>(acc, best, bidx, rbase, p.R - rbase);
      else mt_scan<MB, false>(acc, best, bidx, rbase, 0);
    }
#pragma unroll
    for (int h = 0; h < MB; ++h)
#pragma unroll
      for (int r2 = 0; r2 < 2; ++r2) {
        float bv = best[h][r2];
        int bi = bidx[h][r2];
#pragma unroll
        for (int off = 1; off < 4; off <<= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
          if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        const int m = m0 + (cons * MB + h) * 64 + 16 * wq + (lane >> 2) + 8 * r2;
        if ((lane & 3) == 0 && m < p.P) {
          p.conf[m] = bv * p.out_scale;
          p.idx[m] = bi;
        }
      }
  }
}

// rows of kpad fp16 values; a box of box_k columns (64: SWIZZLE_128B, 16: SWIZZLE_32B) by box_rows rows
static int make_rows_tmap(CUtensorMap* m, const void* ptr, int kpad, int rows, int box_k, int box_rows) {
  PFN_tmapEncodeTiled enc = get_tmap_encoder();
  if (!enc) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[2] = {(cuuint64_t)kpad, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)kpad * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_k, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, box_k == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_32B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled(rows) failed (%d)", (int)r);
  return RV_OK;
}

template <int MB>
static int launch_match_tc(const void* A, int P, const void* B, int R, int kpad, MtP& p, size_t smem, cudaStream_t st) {
  CUtensorMap tmA, tmA16, tmB, tmB16;
  memset(&tmA16, 0, sizeof(tmA16));
  memset(&tmB16, 0, sizeof(tmB16));
  memset(&tmA, 0, sizeof(tmA));
  memset(&tmB, 0, sizeof(tmB));
  int rc = RV_OK;
  if (p.nfull) rc = make_rows_tmap(&tmA, A, kpad, P, 64, 128 * MB);
  if (!rc && p.nfull) rc = make_rows_tmap(&tmB, B, kpad, R, 64, MT_BN);
  if (!rc && p.ntail) rc = make_rows_tmap(&tmA16, A, kpad, P, 16, 128 * MB);
  if (!rc && p.ntail) rc = make_rows_tmap(&tmB16, B, kpad, R, 16, MT_BN);
  if (rc) return rc;
  static size_t configured = 0;
  if (smem > configured) {
    RV_CUDA_OK(cudaFuncSetAttribute(match_tc_kernel<MB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  match_tc_kernel<MB><<<cdiv(P, 128 * MB), 384, smem, st>>>(tmA, tmA16, tmB, tmB16, p);
  RV_LAUNCH_CHECK("match_tc");
  return RV_OK;
}

static int match_tc(const void* A, int P, const void* B, int R, int kpad, float out_scale, float* conf,
                    int32_t* idx, cudaStream_t st) {
  RV_REQUIRE(kpad % 16 == 0 && kpad <= MT_MAXK, "rv_match_argmax(tc): kpad=%d must be a multiple of 16, <= %d", kpad, MT_MAXK);
  RV_REQUIRE(((uintptr_t)A % 16 == 0) && ((uintptr_t)B % 16 == 0), "rv_match_argmax(tc): operands must be 16-byte aligned");
  int dev = 0, max_smem = 0;
  RV_CUDA_OK(cudaGetDevice(&dev));
  RV_CUDA_OK(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  MtP p;
  p.P = P; p.R = R; p.nfull = kpad / 64; p.ntail = (kpad % 64) / 16; p.ntiles_n = (R + MT_BN - 1) / MT_BN;
  p.out_scale = out_scale; p.conf = conf; p.idx = idx;
  // a 256-row A block (and turns) when the ring can then hold two tiles' chunks, see match_tc_kernel
  const int nch = p.nfull + (p.ntail > 0);
  const size_t budget = (size_t)max_smem - 1024 - 2048;
  const size_t a2 = (size_t)256 * kpad * 2, a1 = (size_t)128 * kpad * 2;
  const int mb = budget >= a2 + (size_t)(2 * nch) * MT_SLOT ? 2 : 1;
  const size_t a_bytes = mb == 2 ? a2 : a1;
  p.slots = (int)std::min<size_t>(MT_SLOTS_MAX, (budget - a_bytes) / MT_SLOT);
  RV_REQUIRE(p.slots >= nch, "rv_match_argmax(tc): not enough shared memory for kpad=%d", kpad);
  const size_t smem = 1024 + a_bytes + (size_t)p.slots * MT_SLOT;
  return mb == 2 ? launch_match_tc<2>(A, P, B, R, kpad, p, smem, st) : launch_match_tc<1>(A, P, B, R, kpad, p, smem, st);
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
