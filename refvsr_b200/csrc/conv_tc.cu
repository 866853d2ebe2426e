// wgmma implicit-GEMM convolution for NHWC f16/bf16 activations (stride 1, "same"-style zero padding), the
// tensor-core implementation of rv_conv2d (sm_90a).
//
// GEMM view per CTA tile: M = 128 output pixels, N = NB output channels, K = taps x 64-channel chunks of src0|src1 in
// K = 16 steps.  There is no im2col buffer:
//   * A operand: TMA box loads of the tile + halo, 64 channels wide.  TMA's out-of-bounds zero fill implements the
//     convolution's zero padding and the channel padding to 64.  The box lands in shared memory as 128-byte pixel rows
//     with the 128B swizzle, i.e. directly in the canonical K-major wgmma layout, and the taps are row-shifted
//     descriptor views of it.
//     MODE 0: one box per (kx, chunk), tile 8 x 16 (y-halo only; tap views start on 1024-byte swizzle atoms);
//     MODE 1: ONE box per (tile, chunk), tile 16 x 8, all kh x kw taps are views (layouts 1 and 3 of the weights);
//     MODE 2: 32B-swizzled 16-channel quads per kx, one K = 16 slice per row (layout 2).
//   * B operand: weights pre-packed on the host in exactly the swizzled shared-memory image, fetched with plain bulk
//     copies; resident for the whole CTA lifetime when they fit, otherwise streamed through the ring with A.
//   * D: fp32 accumulators in the registers of the consumer warpgroup (two m64nNk16 halves of the 128-pixel tile).
// MODE 1 3 x 3 convolutions whose every channel chunk takes 3 K-steps (48 channels: the trunk, fusions, pixel shuffles and
// the HR tail) at NB 16 / 48 / 96 run a kernel whose tap and K-step loops are unrolled at compile time (p.fixed): a stage
// is then one fence, 54 wgmmas with no branch between them and one commit, where the runtime loop makes ptxas fence and
// wait on every wgmma.  Other shapes (8 + 48 channels, 7 x 7) keep the runtime loop; both issue the same MMAs in the same order.
// Warp roles (128 (1 + NCONS) threads): warpgroup 0 = TMA producers, warpgroups 1 .. NCONS = consumers.  Consumer c owns the
// CTA's local tiles c, c + NCONS, ... and its own ring of shared-memory slots, so one consumer's MMAs overlap the others'
// epilogues (bias / act / gate / residual / act / NHWC or pixel-shuffled store straight from the accumulator registers).
// Producer warp c fills consumer c's ring only, each with its own slot and phase state, so a consumer that is slow to free a
// slot never holds back another consumer's fills.  The gate / residual buffers are filled by warp 2 + c for consumer c
// with two consumers, and by warp 3 for all three, in tile order, with three.  In the compile-time kernels the A warps
// still issue their first ring fills round-robin (a start-up hand-off through bar_fill), as the single producer before them
// did, so that consumer 1's first box does not queue behind all of consumer 0's.
// NCONS is 2 everywhere but in the single-source 48 -> 48 3 x 3 kernel (conv_tc3_kernel: the trunk convs and conv_hr,
// plain or with a residual), whose epilogue (about 2 000 - 2 600 cycles, latency-bound) is longer than its 54-wgmma batch
// (about 1 750): with two consumers taking turns a tile costs about MMA + epilogue, with three each batch covers the other
// two consumers' epilogues.  Its 512 threads get 128 registers each, so its epilogue reads the gate / residual values from
// their TMA buffer where they are used instead of copying them to registers first.
// Up to NB = 48 the epilogue never waits on a global load of the gate / residual: with 16-bit, 16-byte aligned operands
// they arrive as TMA boxes in a ring of epi_depth per-consumer shared-memory buffers (plan_tc counts them, shrinking the
// A ring), issued by warp 2 + c as soon as a buffer is free; otherwise each thread loads them into registers before
// issuing the tile's MMAs.
// NB >= 64 loads each channel pair where it is used.  The kernels up to NB = 48 with a plain 16-bit output (compile-time
// and runtime tap loops alike) write the tile into a per-consumer shared-memory buffer and store it with one TMA box
// store (p.out_tma): a tile's channel-pair stores per thread, each behind its own bounds branches, made the epilogue the
// longest phase of a tile.
// In every compile-time kernel the two consumers also take turns issuing their MMA batches, so that each epilogue
// overlaps the other consumer's MMAs.  Other epilogues store from registers.  The upsampling
// convs (3 x 3, 48 -> 192 = 2 NB, pixel shuffle into a 16-bit map, no gate / residual; p.ps_vec) are packed in the
// HR-row column order (ps_order 1, see below TcP): column block a is HR sub-row a of both sub-pixels and all 48 channels, so
// a CTA writes whole 96-byte HR pixels and every L2 sector of the map gets one full write (in the conv's own order, each
// block wrote half of every pixel, and the other half came from the other block at some other time).  They run a twin of
// the compile-time kernel (PSV) in which each lane's accumulators form 16-byte vectors of one HR pixel with no lane
// exchange.  Each 8-row half of a tile goes into a per-consumer [8 rows][16 HR pixels][48] shared-memory buffer and out
// by one TMA box store; when those buffers do not fit, the vectors are 16-byte global stores.
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "tc_common.cuh"

namespace rv {

static constexpr int TH = 8, TW = 16;
static constexpr int MAX_SLOTS = 6;  // ring slots per consumer
static constexpr int MAX_EPI = 2;    // gate / residual buffers per consumer
static constexpr int MAX_NB = 96;

struct TcP {
  int Ho, Wo, kh, kw, pad;
  int nch0, nch1, c0, c1;
  int S, NB, cout, tiles_x, tiles_y, slots, resident;
  uint32_t a_bytes, w_bytes, a_tx, slot_bytes;   // a_tx = bytes one A-stage TMA load delivers (<= a_bytes)
  int th, tw, tw_shift, bw;                      // tile rows / columns, box width in pixels
  int mode;                                      // 0, 1, 2 (see the file comment)
  int nq0, nq1;                                  // MODE 2: 16-channel quads of src0 / src1
  uint32_t q_bytes;                              // MODE 2: bytes of one quad sub-buffer of an A stage
  const uint8_t* wpack;
  const float* bias;
  float pre_slope, post_slope;   // act(v) = max(v, v * slope)  (none: 1, relu: 0, lrelu: 0.1 / 0.2)
  int post_clamp3;               // clamp(-3, 3) after everything (AlignedConv2d affine map)
  const void* gate;
  int gate_cs;
  const void* res;
  int res_cs;
  void* out;
  int out_cs, pixel_shuffle, pair_ok, fmt;
  int epi_tma;                   // gate / residual tiles arrive by TMA in per-consumer shared-memory buffers
  int epi_depth;                 // tiles of those buffers per consumer (1 or 2)
  uint32_t epi_bytes, epi_tx;    // bytes of one such buffer ([128 pixels][NB] 16-bit) / of all buffers of one tile
  int fixed;                     // MODE 1 with FIX_KS x FIX_KS taps and FIX_KST K-steps in every chunk (compile-time loop)
  int ps_order;                  // pixel shuffle, HR-row column order (rv_conv_desc::ps_order, see below)
  int ps_vec;                    // pixel shuffle in that order: HR rows as 16-byte vectors or TMA boxes (PSV kernel)
  int out_tma;                   // the output tile is staged in a per-consumer shared-memory buffer and written by TMA
  uint32_t out_off, out_bytes;   // byte offset of those buffers from the ring / bytes of one
  int ncons;                     // consumer warpgroups (3: conv_tc3_kernel, see plan_tc)
  // Batch (rv_conv_desc::n): the persistent loop runs over nimg x tiles_x x tiles_y tiles, image-major.  With nimg > 1 every
  // tensor map has the image as its last dimension, so a box never reaches into a neighbouring image (TMA's out-of-bounds fill
  // is each image's own zero padding); per-thread loads and stores step by these element strides.  nimg = 1 keeps the 3-D maps.
  int nimg;
  long long bs_gate, bs_res, bs_out;
};

// HR-row column order of the pixel-shuffle convs (ps_order 1, cout = 2 NB, packing.ps_rows_order): column nl of block
// nblk is HR sub-row a = nblk.  Lane q of a wgmma accumulator holds the column pairs nl = 8 j + 2 q, + 1; its pairs
// j = 4 g .. 4 g + 3 are the 8 consecutive channels 8 c8 .. 8 c8 + 7 of sub-pixel b, (b, c8) = divmod(4 g + q, NB / 16), so
// each is one 16-byte vector with no lane exchange.  Only the PSV kernel knows this order: the plan refuses it elsewhere.

// MODE 1 shapes whose tap / K-step loops are unrolled at compile time: KS x KS taps and KST K = 16 steps in every channel
// chunk (3 x 3 over 48-channel chunks: the trunk, fusions, pixel shuffles and the HR tail), at the NB the window uses.
static constexpr int FIX_KS = 3, FIX_KST = 3;
__host__ __device__ constexpr bool fixed_nb(int nb) { return nb == 16 || nb == 48 || nb == 96; }

// Timeline instrumentation, compiled only with -DRV_CONV_TIMELINE into a separate library (tools/conv_timeline.py); the
// product library has none of it.  Lane 0 of each role writes clock64 stamps of consumer c's i-th local tile:
// tl[cta][role][i][event], cta = blockIdx.y * gridDim.x + blockIdx.x, role c = the producer warps of consumer c (A warp
// events 0-2, gate / residual warp events 3-5), role TL_MAX_CONS + c = consumer c (a two-consumer kernel leaves roles 2 and 5
// empty).
//   producer: 0 empty-slot wait start, 1 wait end, 2 A box (all stages of the tile) issued,
//             3 empty epilogue-buffer wait start, 4 wait end, 5 gate / residual boxes issued
//   consumer: 0 full-slot wait start, 1 full-slot wait end, 2 turn wait end, 3 first wgmma issued,
//             4 wgmma.wait_group 0 returned, 5 epilogue-buffer wait end, 6 store-drain wait start, 7 store-drain wait end,
//             8 epilogue end
// tl_diag splits the cost (S = 1 convs only): 1 = MMA-only (every tile re-issues its batch on the consumer's first,
// resident slot: no full-slot waits after the first, no slot release, no epilogue), 2 = the same with every A view on a
// 1024-byte swizzle atom (wrong values, same wgmma count), 3 = epilogue-only (no A loads, no MMAs), 4 = the full pipeline
// with an epilogue that touches no shared memory (TMA-store epilogue only: the gate / residual buffers are waited for and
// released but not read, the values are folded into a register instead of the staging buffer, no TMA store).
#ifdef RV_CONV_TIMELINE
static constexpr int TL_TILES = 128, TL_EV = 10, TL_MAX_CONS = 3, TL_ROLES = 2 * TL_MAX_CONS;
__device__ long long* g_tl;
__device__ int g_tl_diag;
static int g_tl_max_slots = 0;   // host: ring slots per consumer at most (0: the plan's)
__device__ __forceinline__ void tl_stamp(long long* tl, int role, int it, int ev) {
  if (tl != nullptr && it < TL_TILES) {
    long long c;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(c) :: "memory");
    tl[(((size_t)(blockIdx.y * gridDim.x + blockIdx.x) * TL_ROLES + role) * TL_TILES + it) * TL_EV + ev] = c;
  }
}
// the buffer pointer and the variant are read once per thread (RV_TL_INIT), so that a stamp costs a clock read and a
// store, and a variant test no global load
#define RV_TL_INIT long long* const tl_buf = g_tl; const int tl_diag = g_tl_diag
#define RV_TL(on, role, it, ev) do { if (on) tl_stamp(tl_buf, role, it, ev); } while (0)
#define RV_TL_DIAG tl_diag
#define RV_TL_MMA_ONLY (tl_diag == 1 || tl_diag == 2)
#else
#define RV_TL_INIT do { } while (0)
#define RV_TL(on, role, it, ev) do { } while (0)
#define RV_TL_DIAG 0
#define RV_TL_MMA_ONLY false
#endif

// All MMAs of one pipeline stage into both 64-row halves.  Descriptor start addresses are in 16-byte units: +2 per
// K = 16 slice of a 128-byte row, whole rows per tap.  KS > 0 (MODE 1 only): kh = kw = KS and KST K-steps per chunk known
// at compile time, so the stage is one unbranched run of wgmmas that ptxas issues behind a single warpgroup.arrive; the
// MMA order per accumulator half (ky, kx, k) is the runtime loop's, so the results are the same bits.
// ALIGNED (timeline diagnostic only): every A view at the slot's first swizzle atom, 8-row groups 1024 bytes apart.
template <int MODE, bool BF, int NB, int KS = 0, int KST = 0, bool ALIGNED = false>
__device__ __forceinline__ void issue_stage(const TcP& p, float (&acc)[2][NB / 2], uint32_t a_addr, uint32_t b_addr,
                                            int s, int ksteps) {
  if constexpr (MODE == 1 && KS > 0) {
    constexpr uint32_t sbo = ALIGNED ? 1024u : (uint32_t)(8 + KS - 1) * 128;   // box width bw = tw + KS - 1 pixels of 128 bytes
#pragma unroll
    for (int ky = 0; ky < KS; ++ky)
#pragma unroll
      for (int kx = 0; kx < KS; ++kx) {
        const uint64_t bd = tc::desc_sw128(b_addr + (uint32_t)((ky * KS + kx) * NB * 128));
        const uint32_t at = a_addr + (ALIGNED ? 0u : (uint32_t)((ky * (8 + KS - 1) + kx) * 128));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t ad = tc::desc_sw128(at + (uint32_t)h * 8 * sbo, sbo);
#pragma unroll
          for (int k = 0; k < KST; ++k)
            tc::wgmma<NB, BF>(acc[h], ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (s | ky | kx | k) ? 1u : 0u);
        }
      }
  } else if constexpr (MODE == 2) {
    const int nq = p.nq0 + p.nq1;
    for (int ky = 0; ky < p.kh; ++ky)
      for (int qd = 0; qd < nq; ++qd) {
        const uint64_t bd = tc::desc_sw32(b_addr + (uint32_t)((ky * nq + qd) * NB * 32));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t ad = tc::desc_sw32(a_addr + (uint32_t)(qd * p.q_bytes + (h * 4 + ky) * TW * 32));
          tc::wgmma<NB, BF>(acc[h], ad, bd, (s | ky | qd) ? 1u : 0u);
        }
      }
  } else if constexpr (MODE == 1) {
    const uint32_t sbo = (uint32_t)p.bw * 128;        // 8-row groups of M = consecutive tile rows of the box
    for (int ky = 0; ky < p.kh; ++ky)
      for (int kx = 0; kx < p.kw; ++kx) {
        const uint64_t bd = tc::desc_sw128(b_addr + (uint32_t)((ky * p.kw + kx) * NB * 128));
        const uint32_t at = a_addr + (uint32_t)((ky * p.bw + kx) * 128);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t ad = tc::desc_sw128(at + (uint32_t)h * 8 * sbo, sbo);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < ksteps) tc::wgmma<NB, BF>(acc[h], ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (s | ky | kx | k) ? 1u : 0u);
        }
      }
  } else {
    for (int ky = 0; ky < p.kh; ++ky) {
      const uint64_t bd = tc::desc_sw128(b_addr + (uint32_t)(ky * NB * 128));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint64_t ad = tc::desc_sw128(a_addr + (uint32_t)((h * 4 + ky) * TW * 128));
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (k < ksteps) tc::wgmma<NB, BF>(acc[h], ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (s | ky | k) ? 1u : 0u);
      }
    }
  }
}

// Gate / residual values of the channel pair (n, n + 1) as loaded, before conversion: 16-bit types packed into one
// register (half the registers of a float2 while the loads are in flight), fp32 as float2.  `second`: n + 1 < cout.
template <typename T> struct RawPair { using type = uint32_t; };
template <> struct RawPair<float> { using type = float2; };

template <typename T>
__device__ __forceinline__ typename RawPair<T>::type ld_raw2(const T* q, bool pair, bool second) {
  if constexpr (sizeof(T) == 2) {
    const uint16_t* u = reinterpret_cast<const uint16_t*>(q);
    if (pair) return *reinterpret_cast<const uint32_t*>(q);
    return (uint32_t)u[0] | (second ? (uint32_t)u[1] << 16 : 0u);
  } else {
    if (pair) return *reinterpret_cast<const float2*>(q);
    return make_float2(q[0], second ? q[1] : 0.f);
  }
}

template <typename T>
__device__ __forceinline__ float2 raw2_to_f2(typename RawPair<T>::type r) {
  if constexpr (std::is_same<T, __half>::value) return __half22float2(*reinterpret_cast<const __half2*>(&r));
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&r));
  else return r;
}

template <typename T>
__device__ __forceinline__ void st2(T* q, float a, float b, bool pair) {
  if constexpr (sizeof(T) == 2) {
    if (pair) {
      if constexpr (std::is_same<T, __half>::value) *reinterpret_cast<__half2*>(q) = __floats2half2_rn(a, b);
      else *reinterpret_cast<__nv_bfloat162*>(q) = __floats2bfloat162_rn(a, b);
      return;
    }
  } else {
    if (pair) { *reinterpret_cast<float2*>(q) = make_float2(a, b); return; }
  }
  q[0] = from_f<T>(a);
}

// two 16-bit values, a in the low half (the lower address of a little-endian store)
template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  const T lo = from_f<T>(a), hi = from_f<T>(b);
  return (uint32_t)*reinterpret_cast<const uint16_t*>(&lo) | (uint32_t)*reinterpret_cast<const uint16_t*>(&hi) << 16;
}

// NB: output channels per CTA (= p.NB); KS, KST: compile-time taps and K-steps of MODE 1 (0: the runtime loop, p.fixed = 0);
// PSV: the 16-byte pixel-shuffle epilogue (p.ps_vec), which has no gate / residual
// BATCH: p.nimg > 1 (a separate instantiation, so that one image keeps its single-image tile loop and addressing)
// NCONS: consumer warpgroups (2, or 3 in conv_tc3_kernel)
template <int NCONS, typename TI, typename TR, typename TO, bool BATCH, int MODE, int NB, int KS, int KST, bool PSV>
__device__ __forceinline__ void conv_tc_body(const CUtensorMap& tm0, const CUtensorMap& tm1, const CUtensorMap& tmg,
                                             const CUtensorMap& tmr, const CUtensorMap& tmo, const TcP& p) {
  static_assert(NCONS == 2 || (NCONS == 3 && MODE == 1 && NB == 48 && KS > 0 && !PSV && sizeof(TR) == 2 && sizeof(TO) == 2),
                "three consumers: the compile-time 48-channel kernel with 16-bit operands only");
  constexpr bool BF = std::is_same<TI, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t bar_full[NCONS][MAX_SLOTS], bar_empty[NCONS][MAX_SLOTS], bar_w, bar_turn[NCONS];
  __shared__ uint64_t bar_efull[NCONS][MAX_EPI], bar_eempty[NCONS][MAX_EPI], bar_fill[NCONS];
  __shared__ __align__(16) float bias_s[MAX_NB];

  const uint32_t raw = tc::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* smemW = smem;                                            // resident weights (S stages)
  uint8_t* ring = smem + (p.resident ? (size_t)p.S * p.w_bytes : 0);  // consumer c: slots x slot_bytes
  const int warp = threadIdx.x >> 5;
  const int warp_u = __shfl_sync(0xffffffffu, warp, 0);
  const int nblk = blockIdx.y;
  const int tiles_img = p.tiles_x * p.tiles_y;
  const int ntiles = BATCH ? tiles_img * p.nimg : tiles_img;
  constexpr bool batched = BATCH;
  const int nchunks = p.nch0 + p.nch1;
  RV_TL_INIT;

  // Programmatic dependent launch: the next kernel of the stream may start its prologue now; activations are read and
  // written only after griddepcontrol.wait, while barrier init, bias and the (constant) weight fetch overlap the tail
  // of the previous kernel.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (threadIdx.x == 0) {
    for (int c = 0; c < NCONS; ++c)
      for (int i = 0; i < p.slots; ++i) {
        tc::mbar_init(&bar_full[c][i], 1);
        tc::mbar_init(&bar_empty[c][i], 4);   // one arrival per consumer warp
      }
    tc::mbar_init(&bar_w, 1);
    for (int c = 0; c < NCONS; ++c)
      for (int i = 0; i < p.epi_depth; ++i) {
        tc::mbar_init(&bar_efull[c][i], 1);
        tc::mbar_init(&bar_eempty[c][i], 1);   // released by one consumer thread after a named barrier
      }
    for (int c = 0; c < NCONS; ++c) tc::mbar_init(&bar_turn[c], 4);   // one arrival per warp of the previous consumer
    for (int c = 0; c < NCONS; ++c) tc::mbar_init(&bar_fill[c], 1);   // the previous A producer warp's start-up hand-off
    tc::fence_barrier_init();
    tc::prefetch_tmap(&tm0);
    if (p.nch1 || p.nq1) tc::prefetch_tmap(&tm1);
  }
  for (int i = threadIdx.x; i < p.NB; i += blockDim.x) {
    const int n = nblk * p.NB + i;
    bias_s[i] = (n < p.cout) ? p.bias[n] : 0.f;
  }
  __syncthreads();

  // Up to NB = 48 the epilogue takes a tile's gate and residual values from registers filled before it starts (loaded
  // where they are used, each pair's load would cost the epilogue a full global-memory latency):
  //  * p.epi_tma (16-bit, 16-byte aligned operands): producer warp 2 + c loads consumer c's [128 pixels][NB] gate /
  //    residual boxes by TMA into a ring of p.epi_depth buffers, up to p.epi_depth tiles ahead of the epilogue, which
  //    copies a buffer to registers and releases it;
  //  * otherwise each thread loads its values from global memory before issuing the tile's MMAs.
  // Wider tiles keep per-pair loads: their accumulators leave no room for the whole tile's operands in 168 registers.
  constexpr int NJ = NB / 8;
  constexpr bool EARLY = NB <= 48;
  constexpr bool TMA_OK = EARLY && sizeof(TR) == 2;
  const bool epi_tma = TMA_OK && p.epi_tma;
  const void* const gate_p = p.gate;
  // consumer c's gate / residual buffer b: the gate box, then the residual box
  auto epi_buf = [&](int c, int b) {
    return ring + (size_t)NCONS * p.slots * p.slot_bytes + (size_t)(c * p.epi_depth + b) * p.epi_tx;
  };
  auto epi_res = [&](uint8_t* g) { return g + (gate_p != nullptr ? p.epi_bytes : 0u); };

  if (warp_u < 4) {
    // ============================ TMA producers ============================
    // warp c < NCONS: consumer c's A boxes (and streamed weights); the other warps: the gate / residual boxes, warp 2 + c
    // those of consumer c with two consumers, warp 3 those of all three with three
    const int pc = warp_u % NCONS;
    const uint8_t* wsrc = p.wpack + (size_t)nblk * p.S * p.w_bytes;
    if (warp_u == 0 && p.resident && tc::elect_one()) {
      tc::mbar_expect_tx(&bar_w, (uint32_t)p.S * p.w_bytes);
      for (int s = 0; s < p.S; ++s) tc::bulk_load(wsrc + (size_t)s * p.w_bytes, &bar_w, smemW + (size_t)s * p.w_bytes, p.w_bytes);
    }
    __syncwarp();
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const bool tl0 = (threadIdx.x & 31) == 0;
    (void)tl0;
    if (warp_u >= NCONS) {
      // MMA-only diagnostics run no epilogue, so nothing would free the buffers
      if (!epi_tma || RV_TL_MMA_ONLY) return;
      if (tc::elect_one()) {
        tc::prefetch_tmap(&tmg);
        tc::prefetch_tmap(&tmr);
      }
      // local tile l is consumer l % NCONS's (l / NCONS)-th; with three consumers the turns make them consume in local
      // tile order, so one in-order issuer never waits on a buffer behind a later tile's
      constexpr int LSTEP = NCONS == 2 ? 2 : 1;
      for (int l = NCONS == 2 ? pc : 0, tile = blockIdx.x + l * gridDim.x; tile < ntiles; l += LSTEP, tile += LSTEP * gridDim.x) {
        const int c = l % NCONS, it = l / NCONS;
        const int buf = it & (p.epi_depth - 1);                           // epi_depth 1 or 2
        const uint32_t eph = (uint32_t)(it >> (p.epi_depth - 1)) & 1u;
        const int img = BATCH ? tile / tiles_img : 0, ti = BATCH ? tile - img * tiles_img : tile;
        const int ty = ti / p.tiles_x, tx = ti - ty * p.tiles_x;
        RV_TL(tl0, c, it, 3);
        tc::mbar_wait(&bar_eempty[c][buf], eph ^ 1u);
        RV_TL(tl0, c, it, 4);
        if (tc::elect_one()) {
          uint64_t* bar = &bar_efull[c][buf];
          uint8_t* g = epi_buf(c, buf);
          tc::mbar_expect_tx(bar, p.epi_tx);
          if (batched) {
            if (gate_p != nullptr) tc::tma_load_4d(&tmg, bar, g, nblk * NB, tx * p.tw, ty * p.th, img);
            if (p.res != nullptr) tc::tma_load_4d(&tmr, bar, epi_res(g), nblk * NB, tx * p.tw, ty * p.th, img);
          } else {
            if (gate_p != nullptr) tc::tma_load_3d(&tmg, bar, g, nblk * NB, tx * p.tw, ty * p.th);
            if (p.res != nullptr) tc::tma_load_3d(&tmr, bar, epi_res(g), nblk * NB, tx * p.tw, ty * p.th);
          }
        }
        __syncwarp();
        RV_TL(tl0, c, it, 5);
      }
      return;
    }
    const uint32_t tx_bytes = p.a_tx + (p.resident ? 0u : p.w_bytes);
    // Start-up hand-off (compile-time kernels): the A warps issue the tiles of their first ring fill round-robin
    // (consumer 0's tile 0, consumer 1's tile 0, ..., consumer 0's tile 1, ...), so that consumer 1's first box does not
    // queue behind consumer 0's whole fill.  Tile it of warp c > 0 follows tile it of warp c - 1, tile it of warp 0 follows
    // tile it - 1 of the last warp; after the first `lead` tiles (at most two) each waits on its own consumer's slots only.
    // The runtime-loop kernels (7 x 7, 1 x 1, 64-channel chunks) measured slower with it and keep independent fills.
    const int lead = KS > 0 ? min(2, (p.slots + p.S - 1) / p.S) : 0;
    const int pprev = pc == 0 ? NCONS - 1 : pc - 1, pnext = pc == NCONS - 1 ? 0 : pc + 1;
    auto tiles_of = [&](int w) {                                    // local tiles of A warp w
      const int rest = ntiles - (int)blockIdx.x - w * (int)gridDim.x;
      return rest > 0 ? (int)((rest + NCONS * gridDim.x - 1) / (NCONS * gridDim.x)) : 0;
    };
    const int n_prev = tiles_of(pprev), n_next = tiles_of(pnext);
    uint32_t fph = 0;
    int slot = 0, it = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x + pc * gridDim.x; tile < ntiles; tile += NCONS * gridDim.x, ++it) {
      if (RV_TL_DIAG == 3 || (RV_TL_MMA_ONLY && it >= 1)) break;   // diagnostics: only the resident slot / nothing
      const int after = it - (pc == 0 ? 1 : 0);                     // the previous warp's tile this one follows
      if (it < lead && after >= 0 && after < n_prev) {
        tc::mbar_wait(&bar_fill[pc], fph);
        fph ^= 1u;
      }
      const int img = BATCH ? tile / tiles_img : 0, ti = BATCH ? tile - img * tiles_img : tile;
      const int ty0 = ti / p.tiles_x, tx0 = ti - ty0 * p.tiles_x;
      const int yc = ty0 * p.th - p.pad, xc = tx0 * p.tw - p.pad;
      int kx = 0, ch = 0;
      for (int s = 0; s < p.S; ++s) {
        RV_TL(tl0 && s == 0, pc, it, 0);
        tc::mbar_wait(&bar_empty[pc][slot], ph ^ 1u);
        RV_TL(tl0 && s == 0, pc, it, 1);
        if (tc::elect_one()) {
          uint64_t* bar = &bar_full[pc][slot];
          uint8_t* dst = ring + ((size_t)pc * p.slots + slot) * p.slot_bytes;
          tc::mbar_expect_tx(bar, tx_bytes);
          auto load = [&](const CUtensorMap* m, uint8_t* d, int c) {
            if (batched) tc::tma_load_4d(m, bar, d, c, xc + kx, yc, img);
            else tc::tma_load_3d(m, bar, d, c, xc + kx, yc);
          };
          if constexpr (MODE == 2) {
            for (int qd = 0; qd < p.nq0 + p.nq1; ++qd) {
              if (qd < p.nq0) load(&tm0, dst + (size_t)qd * p.q_bytes, qd * 16);
              else load(&tm1, dst + (size_t)qd * p.q_bytes, (qd - p.nq0) * 16);
            }
          } else {
            if (ch < p.nch0) load(&tm0, dst, ch * 64);
            else load(&tm1, dst, (ch - p.nch0) * 64);
          }
          if (!p.resident) tc::bulk_load(wsrc + (size_t)s * p.w_bytes, bar, dst + p.a_bytes, p.w_bytes);
        }
        __syncwarp();
        RV_TL(tl0 && s == p.S - 1, pc, it, 2);
        // stage order: mode 0 = (kx, chunk), mode 1 = (chunk), mode 2 = (kx)
        if (MODE == 2) ++kx;
        else if (++ch == nchunks) { ch = 0; kx += (MODE == 1) ? 0 : 1; }
        if (++slot == p.slots) { slot = 0; ph ^= 1u; }
      }
      const int next = it + (pc == NCONS - 1 ? 1 : 0);              // the next warp's tile that follows this one
      if (next < lead && next < n_next && tl0) tc::mbar_arrive(&bar_fill[pnext]);
    }
  } else {
    // ============================ consumers ================================
    const int cons = (warp_u >> 2) - 1;
    const int t = threadIdx.x & 127, wq = t >> 5, lane = t & 31;
    const TI* const gate0 = reinterpret_cast<const TI*>(p.gate);
    const TR* const res0 = reinterpret_cast<const TR*>(p.res);
    TO* const out0 = reinterpret_cast<TO*>(p.out);
    const uint32_t ring_addr = tc::smem_u32(ring + (size_t)cons * p.slots * p.slot_bytes);
    const uint32_t w_addr = tc::smem_u32(smemW);
    if (p.resident) tc::mbar_wait(&bar_w, 0);
    asm volatile("griddepcontrol.wait;" ::: "memory");     // gate / residual reads and all stores come after this
    int slot = 0;
    uint32_t ph = 0;
    // Compile-time kernels: the consumers take turns on the tensor cores, in a ring.  Consumer c issues a tile's MMAs only
    // after consumer c - 1 (the last one for consumer 0) has issued its MMAs of the tile before (consumer 0 starts), so
    // the batches queue back to back and the epilogues run under the other consumers' MMAs; left alone, the consumers tend
    // to issue at once, share the tensor cores, and then run their epilogues with the tensor cores idle.
    constexpr bool TURNS = KS > 0;
    uint32_t tph = 0;
    // two consumers copy a tile's gate / residual values to registers before the epilogue and release the buffer at once;
    // three read them from the buffer where they are used and release it after the values pass (128 registers a thread)
    constexpr bool EPI_REGS = NCONS == 2;
    const uint8_t* epi_g = nullptr;
    const uint8_t* epi_r = nullptr;
    float acc[2][NB / 2];
    int ebuf = 0;
    uint32_t eph = 0;
    // p.out_tma (kernels up to NB = 48 with a 16-bit output TMA can address, and the PSV kernel): the epilogue writes the
    // tile's values into this consumer's buffer with no bounds branches, and one thread stores the buffer with TMA, which
    // clips edge tiles and channels >= cout.  Otherwise each thread stores its values itself.
    constexpr bool OUT_TMA_OK = (EARLY || PSV) && sizeof(TO) == 2;
    const bool out_tma = OUT_TMA_OK && p.out_tma;
    uint8_t* out_s = ring + p.out_off + (size_t)cons * p.out_bytes;
    if (out_tma && t == 0) tc::prefetch_tmap(&tmo);
    int it = 0;
    const bool tl0 = t == 0;
    (void)tl0;
    // three consumers: the gate / residual word of tile pixel m, channels nl, nl + 1 in buffer b (tl_diag 4: not read), and
    // the buffer's release once every thread of the consumer has passed its reads and a proxy fence
    auto epi_word = [&](const uint8_t* b, int m, int nl) {
      const uint32_t off = (uint32_t)(m * NB + nl) * 2u;
      return RV_TL_DIAG == 4 ? 0x3c003c00u ^ off : *reinterpret_cast<const uint32_t*>(b + off);
    };
    auto release_epi = [&]() {
      if (t == 0) tc::mbar_arrive(&bar_eempty[cons][ebuf]);
      if (++ebuf == p.epi_depth) { ebuf = 0; eph ^= 1u; }
    };
    (void)epi_word; (void)release_epi;
    for (int tile = blockIdx.x + cons * gridDim.x; tile < ntiles; tile += NCONS * gridDim.x, ++it) {
      const int img = BATCH ? tile / tiles_img : 0, ti = BATCH ? tile - img * tiles_img : tile;
      const int ty0 = ti / p.tiles_x, tx0 = ti - ty0 * p.tiles_x;
      const TI* const gate = BATCH && gate0 != nullptr ? gate0 + img * p.bs_gate : gate0;
      const TR* const res = BATCH && res0 != nullptr ? res0 + img * p.bs_res : res0;
      TO* const out = BATCH ? out0 + img * p.bs_out : out0;
      if (RV_TL_DIAG == 3) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < NB / 2; ++i) acc[h][i] = 0.f;
      }
      typename RawPair<TI>::type gv[2][2][NJ];   // [h][r2][j], as the epilogue below indexes the accumulators
      typename RawPair<TR>::type rv[2][2][NJ];
      // skipped whole when there is nothing to load: its unrolled, branchy code is several KB of instructions that every
      // tile of a plain conv would otherwise fetch and step through between its epilogue and its next MMA batch
      if (EARLY && EPI_REGS && !epi_tma && (gate != nullptr || res != nullptr)) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int r2 = 0; r2 < 2; ++r2) {
            const int m = 64 * h + 16 * wq + (lane >> 2) + 8 * r2;
            const int oy = ty0 * p.th + (m >> p.tw_shift), ox = tx0 * p.tw + (m & (p.tw - 1));
            if (oy >= p.Ho || ox >= p.Wo) continue;
            const size_t pix = (size_t)oy * p.Wo + ox;
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
              const int n = nblk * NB + 8 * j + 2 * (lane & 3);
              if (n >= p.cout) continue;
              const bool second = n + 1 < p.cout, pair = p.pair_ok && second;
              if (gate != nullptr) gv[h][r2][j] = ld_raw2<TI>(gate + pix * p.gate_cs + n, pair, second);
              if (res != nullptr) rv[h][r2][j] = ld_raw2<TR>(res + pix * p.res_cs + n, pair, second);
            }
          }
      }
      int ch = 0, prev = -1;
      for (int s = 0; s < p.S; ++s) {
        int ksteps = 4;
        if (MODE != 2) {
          const int crem = (ch < p.nch0) ? (p.c0 - ch * 64) : (p.c1 - (ch - p.nch0) * 64);
          ksteps = (min(crem, 64) + 15) >> 4;
          if (++ch == nchunks) ch = 0;
        }
        if (RV_TL_DIAG == 3) break;
        RV_TL(tl0 && s == 0, TL_MAX_CONS + cons, it, 0);
        if (!RV_TL_MMA_ONLY || it == 0) tc::mbar_wait(&bar_full[cons][slot], ph);
        RV_TL(tl0 && s == 0, TL_MAX_CONS + cons, it, 1);
        if (TURNS && s == 0 && (cons != 0 || it != 0)) {
          tc::mbar_wait(&bar_turn[cons], tph);
          tph ^= 1u;
        }
        RV_TL(tl0 && s == 0, TL_MAX_CONS + cons, it, 2);
        const uint32_t a_addr = ring_addr + (uint32_t)slot * p.slot_bytes;
        const uint32_t b_addr = p.resident ? w_addr + (uint32_t)s * p.w_bytes : a_addr + p.a_bytes;
        tc::wgmma_fence();
        RV_TL(tl0 && s == 0, TL_MAX_CONS + cons, it, 3);
        if (RV_TL_DIAG == 2) issue_stage<MODE, BF, NB, KS, KST, true>(p, acc, a_addr, b_addr, s, ksteps);
        else issue_stage<MODE, BF, NB, KS, KST>(p, acc, a_addr, b_addr, s, ksteps);
        tc::wgmma_commit();
        if (TURNS && s == p.S - 1 && lane == 0) tc::mbar_arrive(&bar_turn[cons == NCONS - 1 ? 0 : cons + 1]);   // the next turn
        if (RV_TL_MMA_ONLY) continue;    // MMA-only: the slot stays resident (S = 1)
        if (p.slots == 1) {
          // a single slot is refilled only after these MMAs have read it
          tc::wgmma_wait<0>();
          if (lane == 0) tc::mbar_arrive(&bar_empty[cons][slot]);
        } else {
          // the previous stage's MMAs have retired once at most this stage's group is in flight: free its slot
          tc::wgmma_wait<1>();
          if (prev >= 0 && lane == 0) tc::mbar_arrive(&bar_empty[cons][prev]);
          prev = slot;
        }
        if (++slot == p.slots) { slot = 0; ph ^= 1u; }
      }
      tc::wgmma_wait<0>();
      RV_TL(tl0, TL_MAX_CONS + cons, it, 4);
      if (RV_TL_MMA_ONLY) continue;
      if (prev >= 0 && lane == 0) tc::mbar_arrive(&bar_empty[cons][prev]);
      if constexpr (TMA_OK) {
        if (epi_tma) {
          tc::mbar_wait(&bar_efull[cons][ebuf], eph);
          RV_TL(tl0, TL_MAX_CONS + cons, it, 5);
          epi_g = epi_buf(cons, ebuf);
          epi_r = epi_res(epi_buf(cons, ebuf));
        }
        if (epi_tma && EPI_REGS) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int r2 = 0; r2 < 2; ++r2)
#pragma unroll
              for (int j = 0; j < NJ; ++j) {
                const int m = 64 * h + 16 * wq + (lane >> 2) + 8 * r2;
                const uint32_t off = (uint32_t)(m * NB + 8 * j + 2 * (lane & 3)) * 2u;
                if (RV_TL_DIAG == 4) {
                  gv[h][r2][j] = rv[h][r2][j] = 0x3c003c00u ^ off;
                  continue;
                }
                if (gate != nullptr) gv[h][r2][j] = *reinterpret_cast<const uint32_t*>(epi_g + off);
                if (res != nullptr) rv[h][r2][j] = *reinterpret_cast<const uint32_t*>(epi_r + off);
              }
          // all 128 threads have read the buffer: order those reads before the async proxy's writes of a later tile, then
          // hand the buffer back to its producer warp
          asm volatile("bar.sync %0, 128;" ::"r"(1 + cons) : "memory");
          if (t == 0) {
            tc::fence_proxy_async();
            tc::mbar_arrive(&bar_eempty[cons][ebuf]);
          }
          if (++ebuf == p.epi_depth) { ebuf = 0; eph ^= 1u; }
        }
      }
      RV_TL(tl0 && !epi_tma, TL_MAX_CONS + cons, it, 5);

      // ---- epilogue: thread t holds rows 64 h + 16 wq + lane / 4 (+ 8) and column pairs 8 j + 2 (lane % 4) ----
      if constexpr (PSV) {
        // Pixel shuffle into a 16-bit map without gate / residual, columns in the HR-row order (after TcP): block nblk is
        // HR sub-row a = nblk, and lane q's column pairs j = 4 g .. 4 g + 3 are 8 consecutive channels of sub-pixel b, one
        // 16-byte vector.  The CTA writes whole HR pixels: tile row r gives the 2 tw pixels x NB / 2 channels of HR row
        // 2 (ty0 th + r) + a from 2 tx0 tw on, contiguous in memory.  With p.out_tma each 8-row half of the tile goes
        // into this consumer's [8 rows][2 tw pixels][NB / 2] buffer and out by one TMA box store (4-D map over
        // (channel, HR x, a, LR y)); otherwise each vector is a 16-byte global store.  The general epilogue below is not
        // compiled into this kernel.
        static_assert(sizeof(TO) == 2 && NB % 32 == 0, "16-byte pixel-shuffle rows need 16-bit outputs, NB % 32 == 0");
        constexpr int CV = NB / 16;                     // 16-byte vectors per HR pixel
        const int q = lane & 3;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (out_tma) {
            RV_TL(tl0 && h == 0, TL_MAX_CONS + cons, it, 6);
            if (t == 0) tc::bulk_wait_read<0>();      // this consumer's previous store has read the buffer
            asm volatile("bar.sync %0, 128;" ::"r"(1 + cons) : "memory");
            RV_TL(tl0 && h == 0, TL_MAX_CONS + cons, it, 7);
          }
#pragma unroll
          for (int r2 = 0; r2 < 2; ++r2) {
            const int m = 64 * h + 16 * wq + (lane >> 2) + 8 * r2;
            const int r = m >> p.tw_shift, x = m & (p.tw - 1);
            const int oy = ty0 * p.th + r, ox = tx0 * p.tw + x;
            const bool in = oy < p.Ho && ox < p.Wo;
#pragma unroll
            for (int g = 0; g < NB / 32; ++g) {
              const int J = 4 * g + q, b = J >= CV ? 1 : 0, c8 = J - b * CV;
              uint32_t pk[4];
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const int j = 4 * g + jj;
                float v[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const float xv = acc[h][4 * j + 2 * r2 + e] + bias_s[8 * j + 2 * q + e];
                  v[e] = fmaxf(xv, xv * p.pre_slope);
                  v[e] = fmaxf(v[e], v[e] * p.post_slope);
                  if (p.post_clamp3) v[e] = fminf(fmaxf(v[e], -3.f), 3.f);
                }
                pk[jj] = pack2<TO>(v[0], v[1]);
              }
              const uint4 vec = make_uint4(pk[0], pk[1], pk[2], pk[3]);
              if (out_tma) {
                const uint32_t pix = (uint32_t)(r - 8 * h) * 2 * p.tw + 2 * x + b;
                *reinterpret_cast<uint4*>(out_s + (pix * (NB / 2) + 8 * c8) * 2u) = vec;
              } else if (in) {
                if constexpr (BATCH) {
                  // in 16-byte units from the image's base (out_cs and the image stride are multiples of 8), so that the
                  // store stays one 16-byte access
                  uint4* o = reinterpret_cast<uint4*>(out0) + (size_t)img * (p.bs_out >> 3) +
                             ((size_t)(2 * oy + nblk) * (2 * p.Wo) + 2 * ox + b) * (p.out_cs >> 3) + c8;
                  *o = vec;
                } else {
                  TO* o = out + ((size_t)(2 * oy + nblk) * (2 * p.Wo) + 2 * ox + b) * p.out_cs + 8 * c8;
                  *reinterpret_cast<uint4*>(o) = vec;
                }
              }
            }
          }
          if (out_tma) {
            tc::fence_proxy_async();                  // the buffer's writes, before the async proxy reads them
            asm volatile("bar.sync %0, 128;" ::"r"(1 + cons) : "memory");
            if (t == 0) {
              if (batched) tc::tma_store_5d(&tmo, out_s, 0, 2 * tx0 * p.tw, nblk, ty0 * p.th + 8 * h, img);
              else tc::tma_store_4d(&tmo, out_s, 0, 2 * tx0 * p.tw, nblk, ty0 * p.th + 8 * h);
              tc::bulk_commit();
            }
          }
        }
        RV_TL(tl0, TL_MAX_CONS + cons, it, 8);
        continue;
      }
      if constexpr (OUT_TMA_OK && !PSV) {
        if (out_tma) {
          RV_TL(tl0, TL_MAX_CONS + cons, it, 6);
          if (RV_TL_DIAG != 4) {
            if (t == 0) tc::bulk_wait_read<0>();      // this consumer's previous store has read the buffer
            asm volatile("bar.sync %0, 128;" ::"r"(1 + cons) : "memory");
          }
          RV_TL(tl0, TL_MAX_CONS + cons, it, 7);
          uint32_t fold = 0;    // tl_diag 4: the epilogue's values, kept live without a shared-memory store
          (void)fold;
          // HG / HR / HP: the conv may have a gate / a residual / a post-activation or clamp.  The compile-time kernels run
          // the variant of exactly what the conv applies: with runtime tests only, every value of a plain conv also issued
          // the predicated-off gate and residual conversions and the identity post-activation and clamp, more than half
          // of the pass's instructions, on the consumer's critical path.  The runtime-loop kernels keep the general one.
          auto values = [&](auto hg, auto hr, auto hp) {
            constexpr bool HG = decltype(hg)::value, HR = decltype(hr)::value, HP = decltype(hp)::value;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int r2 = 0; r2 < 2; ++r2) {
                const int m = 64 * h + 16 * wq + (lane >> 2) + 8 * r2;
#pragma unroll
                for (int j = 0; j < NJ; ++j) {
                  const int nl = 8 * j + 2 * (lane & 3);
                  float v[2];
#pragma unroll
                  for (int e = 0; e < 2; ++e) {
                    const float x = acc[h][4 * j + 2 * r2 + e] + bias_s[nl + e];
                    v[e] = fmaxf(x, x * p.pre_slope);
                  }
                  if (HG && gate != nullptr) {
                    // __fmul_rn: never contracted with the residual add into one FMA, whose single rounding would change
                    // the bits of gate + residual convs (with runtime tests the two were separate predicated instructions)
                    const float2 g = raw2_to_f2<TI>(EPI_REGS ? gv[h][r2][j] : epi_word(epi_g, m, nl));
                    v[0] = __fmul_rn(v[0], g.x); v[1] = __fmul_rn(v[1], g.y);
                  }
                  if (HR && res != nullptr) {
                    typename RawPair<TR>::type rw;
                    if constexpr (EPI_REGS) rw = rv[h][r2][j];
                    else rw = epi_word(epi_r, m, nl);
                    const float2 r = raw2_to_f2<TR>(rw);
                    v[0] += r.x; v[1] += r.y;
                  }
                  if (HP) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                      v[e] = fmaxf(v[e], v[e] * p.post_slope);
                      if (p.post_clamp3) v[e] = fminf(fmaxf(v[e], -3.f), 3.f);
                    }
                  }
                  if (RV_TL_DIAG == 4) fold ^= pack2<TO>(v[0], v[1]);
                  else *reinterpret_cast<uint32_t*>(out_s + (uint32_t)(m * NB + nl) * 2u) = pack2<TO>(v[0], v[1]);
                }
              }
          };
          using Y = std::true_type;
          using N = std::false_type;
          if constexpr (KS > 0) {
            // post slope 1 without clamp is the identity: skipping it leaves every finite value's bits unchanged
            const bool hp = p.post_slope != 1.f || p.post_clamp3;
            if (gate != nullptr) {
              if (res != nullptr) { if (hp) values(Y{}, Y{}, Y{}); else values(Y{}, Y{}, N{}); }
              else { if (hp) values(Y{}, N{}, Y{}); else values(Y{}, N{}, N{}); }
            } else {
              if (res != nullptr) { if (hp) values(N{}, Y{}, Y{}); else values(N{}, Y{}, N{}); }
              else { if (hp) values(N{}, N{}, Y{}); else values(N{}, N{}, N{}); }
            }
          } else {
            values(Y{}, Y{}, Y{});
          }
          if (RV_TL_DIAG == 4) {
            if (fold == 0x7fc00001u) out[0] = from_f<TO>(0.f);   // practically never taken: keeps the values live
            if (!EPI_REGS && epi_tma) release_epi();             // (not read)
            RV_TL(tl0, TL_MAX_CONS + cons, it, 8);
            continue;
          }
          // the buffer's writes (and, with three consumers, this thread's gate / residual reads), before the async proxy
          // reads the one / overwrites the other
          tc::fence_proxy_async();
          asm volatile("bar.sync %0, 128;" ::"r"(1 + cons) : "memory");
          if (!EPI_REGS && epi_tma) release_epi();
          if (t == 0) {
            if (batched) tc::tma_store_4d(&tmo, out_s, nblk * NB, tx0 * p.tw, ty0 * p.th, img);
            else tc::tma_store_3d(&tmo, out_s, nblk * NB, tx0 * p.tw, ty0 * p.th);
            tc::bulk_commit();
          }
          RV_TL(tl0, TL_MAX_CONS + cons, it, 8);
          continue;
        }
      }
      // three consumers: the plan gives them the TMA-store epilogue only
      if constexpr (EPI_REGS) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int r2 = 0; r2 < 2; ++r2) {
          const int m = 64 * h + 16 * wq + (lane >> 2) + 8 * r2;
          const int oy = ty0 * p.th + (m >> p.tw_shift), ox = tx0 * p.tw + (m & (p.tw - 1));
          if (oy >= p.Ho || ox >= p.Wo) continue;
          const size_t pix = (size_t)oy * p.Wo + ox;
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            const int nl = 8 * j + 2 * (lane & 3);
            const int n = nblk * NB + nl;
            if (n >= p.cout) continue;
            const bool pair = p.pair_ok && (n + 1 < p.cout);
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float x = acc[h][4 * j + 2 * r2 + e] + bias_s[nl + e];
              v[e] = fmaxf(x, x * p.pre_slope);     // slope in [0,1]: identity / ReLU / LeakyReLU without a select
            }
            if (gate != nullptr) {
              const float2 g = raw2_to_f2<TI>(EARLY ? gv[h][r2][j] : ld_raw2<TI>(gate + pix * p.gate_cs + n, pair, n + 1 < p.cout));
              v[0] *= g.x; v[1] *= g.y;
            }
            if (res != nullptr) {
              const float2 r = raw2_to_f2<TR>(EARLY ? rv[h][r2][j] : ld_raw2<TR>(res + pix * p.res_cs + n, pair, n + 1 < p.cout));
              v[0] += r.x; v[1] += r.y;
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              v[e] = fmaxf(v[e], v[e] * p.post_slope);
              if (p.post_clamp3) v[e] = fminf(fmaxf(v[e], -3.f), 3.f);
            }
            if (p.pixel_shuffle) {
              // n = 4c + 2a + b  ->  out[(2oy+a, 2ox+b)][c]; the pair (n, n+1) is b = 0, 1 of one (c, a)
              const int cc = n >> 2, a = (n >> 1) & 1;
              TO* o = out + ((size_t)(2 * oy + a) * (2 * p.Wo) + 2 * ox) * p.out_cs + cc;
              o[0] = from_f<TO>(v[0]);
              if (n + 1 < p.cout) o[p.out_cs] = from_f<TO>(v[1]);
            } else {
              TO* o = out + pix * p.out_cs + n;
              st2<TO>(o, v[0], v[1], pair);
              if (!pair && n + 1 < p.cout) o[1] = from_f<TO>(v[1]);
            }
          }
        }
      }
      }
      RV_TL(tl0, TL_MAX_CONS + cons, it, 8);
    }
    if (out_tma && t == 0) tc::bulk_wait<0>();     // the last stores are complete before the CTA exits
  }
}

template <typename TI, typename TR, typename TO, bool BATCH, int MODE, int NB, int KS, int KST, bool PSV>
__global__ void __launch_bounds__(128 * (1 + 2), 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1,
               const __grid_constant__ CUtensorMap tmg, const __grid_constant__ CUtensorMap tmr,
               const __grid_constant__ CUtensorMap tmo, const TcP p) {
  conv_tc_body<2, TI, TR, TO, BATCH, MODE, NB, KS, KST, PSV>(tm0, tm1, tmg, tmr, tmo, p);
}

// the single-source 48 -> 48 3 x 3 conv with three consumers (p.ncons == 3): one 16-bit type T for every operand
template <typename T, bool BATCH>
__global__ void __launch_bounds__(128 * (1 + 3), 1)
conv_tc3_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1,
                const __grid_constant__ CUtensorMap tmg, const __grid_constant__ CUtensorMap tmr,
                const __grid_constant__ CUtensorMap tmo, const TcP p) {
  conv_tc_body<3, T, T, T, BATCH, 1, 48, FIX_KS, FIX_KST, false>(tm0, tm1, tmg, tmr, tmo, p);
}

PFN_tmapEncodeTiled get_tmap_encoder() {
  static PFN_tmapEncodeTiled fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_tmapEncodeTiled)f;
  }
  return fn;
}

// 16-bit NHWC map [H][W][C] with `cs` (default C) channels between pixels, boxes of box_c x box_w x box_rows;
// out-of-bounds elements read as zero and are not written.  n > 1: [n][H][W][C] with `bs` elements between images, a 4th
// dimension of box size 1, so that a box stops at its own image's border.
static int make_tmap_3d(CUtensorMap* m, const void* ptr, int C, int W, int H, int box_c, int box_w, int box_rows, int fmt,
                        CUtensorMapSwizzle swz, int cs = 0, int n = 1, long long bs = 0) {
  PFN_tmapEncodeTiled enc = get_tmap_encoder();
  if (!enc) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if (cs == 0) cs = C;
  cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)n};
  cuuint64_t gstr[3] = {(cuuint64_t)cs * 2, (cuuint64_t)W * cs * 2, (cuuint64_t)bs * 2};
  cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(m, fmt ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, n > 1 ? 4 : 3,
                   const_cast<void*>(ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled failed (%d) C=%d W=%d H=%d", (int)r, C, W, H);
  return RV_OK;
}

// the 16-bit pixel-shuffled output [2 Ho][2 Wo][cs] of an LR Ho x Wo map as (channel, HR x, sub-row a, LR y), so that one
// box of C x 2 tw x 1 x rows is HR rows 2 y + a of `rows` LR rows; out-of-bounds elements are not written.  n > 1: the image
// is a 5th dimension, `bs` elements apart.
static int make_ps_rows_tmap(CUtensorMap* m, const void* ptr, int C, int cs, int Wo, int Ho, int tw, int rows, int fmt,
                             int n = 1, long long bs = 0) {
  PFN_tmapEncodeTiled enc = get_tmap_encoder();
  if (!enc) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const cuuint64_t px = (cuuint64_t)cs * 2;
  cuuint64_t gdim[5] = {(cuuint64_t)C, (cuuint64_t)2 * Wo, 2, (cuuint64_t)Ho, (cuuint64_t)n};
  cuuint64_t gstr[4] = {px, 2 * Wo * px, 4 * Wo * px, (cuuint64_t)bs * 2};
  cuuint32_t box[5] = {(cuuint32_t)C, (cuuint32_t)2 * tw, 1, (cuuint32_t)rows, 1};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(m, fmt ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, n > 1 ? 5 : 4, const_cast<void*>(ptr), gdim,
                   gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(RV_E_CUDA, "cuTensorMapEncodeTiled (HR rows) failed (%d) C=%d W=%d H=%d", (int)r, C, Wo, Ho);
  return RV_OK;
}

static int make_act_tmap(CUtensorMap* m, const void* ptr, int C, int W, int H, int box_w, int box_rows, int fmt, int sw32,
                         int n, long long bs) {
  return make_tmap_3d(m, ptr, C, W, H, sw32 ? 16 : 64, box_w, box_rows, fmt, sw32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_128B,
                      0, n, bs);
}

static int g_num_sms = 0;
static int g_max_smem = 0;
static int g_cta_cap = 0;          // rv_set_conv_cta_cap: upper bound of the persistent grid (0 = one CTA per SM)
int set_conv_cta_cap(int cap) { const int old = g_cta_cap; g_cta_cap = cap > 0 ? cap : 0; return old; }
static int g_smem_cap = 0;         // rv_set_conv_smem_cap: upper bound of a launch's shared memory (0 = the device's opt-in limit)
int set_conv_smem_cap(int bytes) { const int old = g_smem_cap; g_smem_cap = bytes > 0 ? bytes : 0; return old; }
static int g_conv_consumers = 0;   // rv_set_conv_consumers: 2 = the two-consumer kernel for every conv (0 = the plan's choice)
int set_conv_consumers(int n) { const int old = g_conv_consumers; g_conv_consumers = n == 2 ? 2 : 0; return old; }

template <typename TI, typename TR, typename TO, int MODE, int NB, int KS = 0, int KST = 0, bool PSV = false, int NCONS = 2>
static int launch_tc_mode(const CUtensorMap* tm, const TcP& p, dim3 grid, size_t smem, cudaStream_t st) {
  const int batch = p.nimg > 1 ? 1 : 0;
  auto kern = batch ? conv_tc_kernel<TI, TR, TO, true, MODE, NB, KS, KST, PSV> : conv_tc_kernel<TI, TR, TO, false, MODE, NB, KS, KST, PSV>;
  if constexpr (NCONS == 3) kern = batch ? conv_tc3_kernel<TO, true> : conv_tc3_kernel<TO, false>;
  static size_t configured[2] = {0, 0};   // per template instantiation
  if (smem > configured[batch]) {
    RV_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured[batch] = smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(128 * (1 + NCONS));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  static const bool use_pdl = getenv("REFVSR_NO_PDL") == nullptr;
  cfg.attrs = attr;
  cfg.numAttrs = use_pdl ? 1 : 0;
  RV_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, tm[0], tm[1], tm[2], tm[3], tm[4], p));
  RV_LAUNCH_CHECK("conv_tc");
  return RV_OK;
}

template <typename TI, typename TR, typename TO, int NB>
static int launch_tc_nb(const CUtensorMap* tm, const TcP& p, dim3 grid, size_t smem, cudaStream_t st) {
  switch (p.mode) {
    case 2: return launch_tc_mode<TI, TR, TO, 2, NB>(tm, p, grid, smem, st);
    case 1:
      if constexpr (fixed_nb(NB)) {
        if constexpr (NB == 96 && sizeof(TO) == 2)
          if (p.ps_vec) return launch_tc_mode<TI, TR, TO, 1, NB, FIX_KS, FIX_KST, true>(tm, p, grid, smem, st);
        if constexpr (NB == 48 && sizeof(TO) == 2 && std::is_same<TI, TO>::value && std::is_same<TR, TO>::value)
          if (p.ncons == 3) return launch_tc_mode<TI, TR, TO, 1, NB, FIX_KS, FIX_KST, false, 3>(tm, p, grid, smem, st);
        if (p.fixed) return launch_tc_mode<TI, TR, TO, 1, NB, FIX_KS, FIX_KST>(tm, p, grid, smem, st);
      }
      return launch_tc_mode<TI, TR, TO, 1, NB>(tm, p, grid, smem, st);
    default: return launch_tc_mode<TI, TR, TO, 0, NB>(tm, p, grid, smem, st);
  }
}

template <typename TI, typename TR, typename TO>
static int launch_tc(const CUtensorMap* tm, const TcP& p, dim3 grid, size_t smem, cudaStream_t st) {
  switch (p.NB) {
    case 16: return launch_tc_nb<TI, TR, TO, 16>(tm, p, grid, smem, st);
    case 32: return launch_tc_nb<TI, TR, TO, 32>(tm, p, grid, smem, st);
    case 48: return launch_tc_nb<TI, TR, TO, 48>(tm, p, grid, smem, st);
    case 64: return launch_tc_nb<TI, TR, TO, 64>(tm, p, grid, smem, st);
    case 80: return launch_tc_nb<TI, TR, TO, 80>(tm, p, grid, smem, st);
    default: return launch_tc_nb<TI, TR, TO, 96>(tm, p, grid, smem, st);
  }
}

// Everything about a launch that does not need a device: geometry, layout mode and the shared-memory rings.
// (rv_conv2d_tc_plan exposes it so that the ring invariants are checked on a machine without a GPU.)
static int plan_tc(const rv_conv_desc* d, TcP& p, size_t& smem_out, int& nblk_out) {
  RV_REQUIRE(d->stride == 1, "rv_conv2d(tc): stride must be 1 (got %d)", d->stride);
  RV_REQUIRE(d->in_dtype == RV_F16 || d->in_dtype == RV_BF16, "rv_conv2d(tc): activations must be f16/bf16");
  RV_REQUIRE(d->c0 % 8 == 0 && (!d->src1 || d->c1 % 8 == 0), "rv_conv2d(tc): channel counts must be multiples of 8");
  RV_REQUIRE(((uintptr_t)d->src0 % 16 == 0) && ((uintptr_t)d->src1 % 16 == 0) && ((uintptr_t)d->wpack % 16 == 0),
             "rv_conv2d(tc): src/wpack must be 16-byte aligned");
  RV_REQUIRE(d->nb >= 16 && d->nb <= MAX_NB && d->nb % 16 == 0, "rv_conv2d(tc): nb=%d must be a multiple of 16 in [16,96]", d->nb);
  RV_REQUIRE(d->kh >= 1 && d->kh <= 7 && d->kw >= 1 && d->kw <= 7, "rv_conv2d(tc): kernel size up to 7x7");
  RV_REQUIRE(!d->pixel_shuffle || d->cout % 4 == 0, "rv_conv2d: pixel_shuffle needs cout %% 4 == 0");
  RV_REQUIRE(d->layout >= 0 && d->layout <= 3, "rv_conv2d(tc): unknown layout %d", d->layout);
  RV_REQUIRE(g_num_sms > 0 && g_max_smem > 0, "rv_conv2d(tc): device limits not set");
  RV_REQUIRE(d->ps_order == 0 || (d->ps_order == 1 && d->pixel_shuffle && d->cout == 2 * d->nb && d->nb % 32 == 0),
             "rv_conv2d(tc): ps_order=%d needs a pixel shuffle with cout == 2 * nb and nb %% 32 == 0 (cout=%d nb=%d ps=%d)",
             d->ps_order, d->cout, d->nb, d->pixel_shuffle);
  p.Ho = d->H + 2 * d->pad - d->kh + 1;
  p.Wo = d->W + 2 * d->pad - d->kw + 1;
  RV_REQUIRE(p.Ho > 0 && p.Wo > 0, "rv_conv2d: empty output");
  p.nimg = d->n > 1 ? d->n : 1;
  const bool batched = p.nimg > 1;
  // the activation maps' image strides must keep every image's base 16-byte aligned (TMA global strides)
  RV_REQUIRE(!batched || (d->bs_src0 % 8 == 0 && (!d->src1 || d->bs_src1 % 8 == 0)),
             "rv_conv2d(tc): n=%d needs image strides of src0 / src1 that are multiples of 8 elements", d->n);
  p.bs_gate = batched && d->gate ? d->bs_gate : 0;
  p.bs_res = batched && d->res ? d->bs_res : 0;
  p.bs_out = batched ? d->bs_out : 0;
  p.kh = d->kh; p.kw = d->kw; p.pad = d->pad;
  p.c0 = d->c0; p.c1 = d->src1 ? d->c1 : 0;
  p.nch0 = (p.c0 + 63) / 64; p.nch1 = (p.c1 + 63) / 64;
  p.nq0 = p.nq1 = 0; p.q_bytes = 0;
  p.NB = d->nb; p.cout = d->cout;
  const int nblk = (d->cout + p.NB - 1) / p.NB;
  const int smem_lim = g_smem_cap > 0 ? std::min(g_smem_cap, g_max_smem) : g_max_smem;
  RV_REQUIRE(smem_lim > 3072, "rv_conv2d(tc): shared-memory limit %d too small", smem_lim);
  const size_t budget = (size_t)smem_lim - 1024 /*alignment*/ - 2048 /*static: barriers, bias*/;
  p.mode = (d->layout == 1 || d->layout == 3) ? 1 : d->layout;
  if (p.mode == 1) {
    RV_REQUIRE(d->kh == d->kw && (d->kh == 1 || d->kh == 3 || d->kh == 5 || d->kh == 7), "rv_conv2d(tc): layout 1 needs a square 1/3/5/7 kernel");
    p.th = 16; p.tw = 8; p.tw_shift = 3;
    p.bw = p.tw + d->kw - 1;            // box = tile + halo; rows of the box are bw pixels (bw * 128 B) apart
    p.S = p.nch0 + p.nch1;
    p.a_tx = (uint32_t)(p.th + d->kh - 1) * p.bw * 128;
    p.a_bytes = (p.a_tx + 1023u) & ~1023u;   // slots stay 1024-byte aligned (swizzle atom)
    p.w_bytes = (uint32_t)d->kh * d->kw * p.NB * 128;
  } else if (p.mode == 2) {
    p.th = TH; p.tw = TW; p.tw_shift = 4; p.bw = TW;
    p.nq0 = (p.c0 + 15) / 16; p.nq1 = (p.c1 + 15) / 16;
    p.S = d->kw;
    p.q_bytes = (uint32_t)(TH + d->kh - 1) * TW * 32;
    p.a_bytes = (uint32_t)(p.nq0 + p.nq1) * p.q_bytes;
    p.a_tx = p.a_bytes;
    p.w_bytes = (uint32_t)d->kh * (p.nq0 + p.nq1) * p.NB * 32;
  } else {
    p.th = TH; p.tw = TW; p.tw_shift = 4; p.bw = TW;
    p.S = d->kw * (p.nch0 + p.nch1);
    p.a_bytes = (uint32_t)(TH + d->kh - 1) * TW * 128;
    p.a_tx = p.a_bytes;
    p.w_bytes = (uint32_t)d->kh * p.NB * 128;
  }
  p.tiles_x = (p.Wo + p.tw - 1) / p.tw; p.tiles_y = (p.Ho + p.th - 1) / p.th;
  // the compile-time tap loop: a square FIX_KS kernel whose every channel chunk takes FIX_KST K-steps (e.g. 48 + 48
  // channels, not 8 + 48); other shapes keep the runtime loop
  p.fixed = p.mode == 1 && d->kh == FIX_KS && d->kw == FIX_KS && fixed_nb(p.NB);
  for (int ch = 0; ch < p.nch0 + p.nch1 && p.fixed; ++ch) {
    const int crem = (ch < p.nch0) ? (p.c0 - ch * 64) : (p.c1 - (ch - p.nch0) * 64);
    p.fixed = (std::min(crem, 64) + 15) / 16 == FIX_KST;
  }
  // the upsampling convs (compile-time 3 x 3 loop, NB = 96, pixel shuffle in the HR-row column order into a 16-bit map, no
  // gate / residual) run the PSV kernel when the HR pixel rows stay 16-byte aligned; other pixel shuffles keep the 2-byte
  // stores of the general epilogue
  p.ps_order = d->ps_order;
  p.ps_vec = p.fixed && d->pixel_shuffle && d->ps_order && p.NB == 96 && dtype_size(d->out_dtype) == 2 && !d->gate &&
             !d->res && d->out != nullptr && (uintptr_t)d->out % 16 == 0 && (d->out_cs * 2) % 16 == 0 && (!batched || d->bs_out % 8 == 0);
  RV_REQUIRE(!d->ps_order || p.ps_vec, "rv_conv2d(tc): ps_order=1 needs the 3x3 48-channel nb=96 kernel with a 16-bit output "
             "whose HR pixel rows are 16-byte aligned (out_cs=%d), no gate / residual", d->out_cs);
  // shared-memory plan for nc consumers (buffers below): weights resident when they leave room for two slots per consumer
  // (layout 1: one), else streamed with A; a consumer with a single slot still overlaps with the other consumers' rings
  const size_t w_all = (size_t)p.S * p.w_bytes;
  // TMA epilogue: 16-bit gate / residual whose boxes TMA can address (16-byte aligned base and pixel stride), tiles the
  // register epilogue keeps whole (NB <= 48), and room for the buffers next to resident weights and the minimal ring
  const int rdt0 = d->res ? d->res_dtype : d->in_dtype;
  auto tma_ok = [batched](const void* q, int cs, long long bs) {
    return q == nullptr || ((uintptr_t)q % 16 == 0 && cs > 0 && cs % 8 == 0 && (!batched || bs % 8 == 0));
  };
  p.epi_bytes = (uint32_t)p.th * p.tw * p.NB * 2;
  p.epi_tx = (uint32_t)((d->gate ? 1 : 0) + (d->res ? 1 : 0)) * p.epi_bytes;
  // TMA-store epilogue, when its buffer per consumer fits next to the resident weights, the gate / residual buffers and the
  // minimal ring: kernels up to NB = 48 writing a plain (not pixel-shuffled) map of the input's 16-bit type whose base
  // and pixel stride TMA can address ([128 pixels][NB] buffer, th x tw of the layout mode), and the PSV kernel (half a tile of HR rows,
  // [8 rows][16 pixels][NB / 2]: a whole tile's buffers would leave one A slot per consumer next to the 108 KB of weights)
  const bool out_plain = p.NB <= 48 && !d->pixel_shuffle && d->out_dtype == d->in_dtype && d->out != nullptr &&
                         tma_ok(d->out, d->out_cs, d->bs_out);
  p.out_bytes = p.ps_vec ? p.epi_bytes / 2 : p.epi_bytes;
  size_t epi_all = 0, out_all = 0;
  // the epilogue buffers of nc consumers; true when they, the resident weights and the minimal ring fit
  auto buffers = [&](int nc) {
    const size_t ring_min = (size_t)nc * (p.mode == 1 ? 1 : 2) * p.a_bytes;
    p.epi_tma = (d->gate || d->res) && p.NB <= 48 && rdt0 == d->in_dtype && tma_ok(d->gate, d->gate_cs, d->bs_gate) &&
                tma_ok(d->res, d->res_cs, d->bs_res) && w_all + ring_min + (size_t)nc * p.epi_tx <= budget;
    // a second buffer lets the boxes arrive up to two tiles ahead of the epilogue; it is taken only while two A slots and
    // the output buffer per consumer still fit (gate + residual at NB = 48 keeps two A slots and one buffer)
    p.epi_depth = p.epi_tma && w_all + (size_t)nc * (2 * p.a_bytes + MAX_EPI * p.epi_tx + p.epi_bytes) <= budget ? MAX_EPI : 1;
    epi_all = p.epi_tma ? (size_t)nc * p.epi_depth * p.epi_tx : 0;
    p.out_tma = (out_plain || p.ps_vec) && w_all + ring_min + epi_all + (size_t)nc * p.out_bytes <= budget;
    out_all = p.out_tma ? (size_t)nc * p.out_bytes : 0;
    return w_all + ring_min + epi_all + out_all <= budget;
  };
  // Three consumers (conv_tc3_kernel) for the single-source 48 -> 48 3 x 3 convs with a 16-bit output, plain or with a
  // residual, when the weights, one A slot, the output buffer and (residual) one residual buffer per consumer fit (199 680
  // bytes with a residual).  Measured on an H100 at 700 W against two consumers (README "Three consumers"): 14.9 -> 13.7 us
  // plain and 18.4 -> 17.4 us with a residual at 270 x 480, 44.7 -> 42.3 / 57.0 -> 55.1 us at 540 x 960, conv_hr 163 -> 159
  // us.  Gate + residual needs 236 544 bytes and keeps two consumers (a gate alone, not in the window, too).
  const bool three = g_conv_consumers != 2 && p.fixed && p.NB == 48 && p.S == 1 && !d->gate && out_plain && rdt0 == d->in_dtype;
  p.ncons = three && buffers(3) && p.out_tma && (p.epi_tma || !d->res) ? 3 : 2;
  const size_t nc = (size_t)p.ncons;
  if (buffers(p.ncons)) {
    p.resident = 1;
    p.slot_bytes = p.a_bytes;
    p.slots = (int)std::min<size_t>(MAX_SLOTS, (budget - w_all - epi_all - out_all) / (nc * p.a_bytes));
#ifdef RV_CONV_TIMELINE
    if (g_tl_max_slots > 0) p.slots = std::min(p.slots, g_tl_max_slots);
#endif
  } else {
    RV_REQUIRE(p.mode != 1, "rv_conv2d(tc): layout 1 weights do not fit in shared memory");
    p.resident = 0;
    p.slot_bytes = p.a_bytes + p.w_bytes;
    p.slots = (int)std::min<size_t>(MAX_SLOTS, budget / (nc * p.slot_bytes));
    RV_REQUIRE(p.slots >= 1, "rv_conv2d(tc): stage of %u bytes does not fit once per consumer in shared memory", p.slot_bytes);
  }
  p.out_off = (uint32_t)(nc * p.slots * p.slot_bytes + epi_all);
  const size_t smem = 1024 + (p.resident ? w_all : 0) + nc * p.slots * p.slot_bytes + epi_all + out_all;
  p.wpack = (const uint8_t*)d->wpack; p.bias = d->bias;
  auto slope = [](int act) { return act == RV_ACT_RELU ? 0.f : act == RV_ACT_LRELU01 ? 0.1f : act == RV_ACT_LRELU02 ? 0.2f : 1.f; };
  RV_REQUIRE(d->act_pre != RV_ACT_CLAMP3, "rv_conv2d(tc): clamp3 is only supported as act_post");
  p.pre_slope = slope(d->act_pre); p.post_slope = slope(d->act_post);
  p.post_clamp3 = d->act_post == RV_ACT_CLAMP3;
  p.gate = d->gate; p.gate_cs = d->gate_cs; p.res = d->res; p.res_cs = d->res_cs;
  p.out = d->out; p.out_cs = d->out_cs; p.pixel_shuffle = d->pixel_shuffle;
  // channel pairs (n, n + 1), n even, are one 4- / 8-byte access when every row stride keeps them aligned
  const int rdt = d->res ? d->res_dtype : d->out_dtype;
  auto al = [](const void* q, int cs, int dt) { return q == nullptr || (((uintptr_t)q % (2 * dtype_size(dt)) == 0) && cs % 2 == 0); };
  p.pair_ok = al(d->out, d->out_cs, d->out_dtype) && al(d->gate, d->gate_cs, d->in_dtype) && al(d->res, d->res_cs, rdt);
  p.fmt = d->in_dtype == RV_BF16 ? 1 : 0;
  smem_out = smem;
  nblk_out = nblk;
  return RV_OK;
}

int conv2d_tc(const rv_conv_desc* d, cudaStream_t st) {
  if (g_num_sms == 0) {
    int dev = 0;
    RV_CUDA_OK(cudaGetDevice(&dev));
    RV_CUDA_OK(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
    RV_CUDA_OK(cudaDeviceGetAttribute(&g_max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  }
  TcP p;
  size_t smem = 0;
  int nblk = 1;
  {
    const int rc0 = plan_tc(d, p, smem, nblk);
    if (rc0) return rc0;
  }
  const int rdt = d->res ? d->res_dtype : d->out_dtype;
  const int sw32 = p.mode == 2;
  CUtensorMap tm[5];    // src0, src1, gate, res, out (unused ones: copies of src0)
  const int n = p.nimg;
  int rc = make_act_tmap(&tm[0], d->src0, p.c0, d->W, d->H, p.mode == 1 ? p.tw + d->kw - 1 : p.tw, p.th + d->kh - 1, p.fmt, sw32,
                         n, d->bs_src0);
  if (rc) return rc;
  tm[1] = tm[2] = tm[3] = tm[4] = tm[0];
  if (p.c1) {
    rc = make_act_tmap(&tm[1], d->src1, p.c1, d->W, d->H, p.mode == 1 ? p.tw + d->kw - 1 : p.tw, p.th + d->kh - 1, p.fmt, sw32,
                       n, d->bs_src1);
    if (rc) return rc;
  }
  // gate / residual boxes for the TMA epilogue: [th][tw][NB], unswizzled, so box pixel m sits at m * NB channels
  if (p.epi_tma && d->gate &&
      (rc = make_tmap_3d(&tm[2], d->gate, d->gate_cs, p.Wo, p.Ho, p.NB, p.tw, p.th, p.fmt, CU_TENSOR_MAP_SWIZZLE_NONE, 0, n, d->bs_gate)))
    return rc;
  if (p.epi_tma && d->res &&
      (rc = make_tmap_3d(&tm[3], d->res, d->res_cs, p.Wo, p.Ho, p.NB, p.tw, p.th, p.fmt, CU_TENSOR_MAP_SWIZZLE_NONE, 0, n, d->bs_res)))
    return rc;
  // output tiles [th][tw][NB] of the TMA-store epilogue; channels >= cout (and pixels outside the map) are not written
  if (p.out_tma && !p.ps_vec &&
      (rc = make_tmap_3d(&tm[4], d->out, d->cout, p.Wo, p.Ho, p.NB, p.tw, p.th, p.fmt, CU_TENSOR_MAP_SWIZZLE_NONE, d->out_cs,
                         n, d->bs_out)))
    return rc;
  if (p.out_tma && p.ps_vec &&
      (rc = make_ps_rows_tmap(&tm[4], d->out, d->cout / 4, d->out_cs, p.Wo, p.Ho, p.tw, p.th / 2, p.fmt, n, d->bs_out)))
    return rc;
  const int ntiles = p.tiles_x * p.tiles_y * n;
  int gx = std::min(ntiles, std::max(1, g_num_sms / nblk));
  if (g_cta_cap > 0) gx = std::min(gx, std::max(1, g_cta_cap / nblk));     // two capped launches on different streams share the SMs
  dim3 grid(gx, nblk);
  if (d->in_dtype == RV_F16 && rdt == RV_F16 && d->out_dtype == RV_F16) return launch_tc<__half, __half, __half>(tm, p, grid, smem, st);
  if (d->in_dtype == RV_F16 && rdt == RV_F32 && d->out_dtype == RV_F32) return launch_tc<__half, float, float>(tm, p, grid, smem, st);
  if (d->in_dtype == RV_BF16 && rdt == RV_BF16 && d->out_dtype == RV_BF16) return launch_tc<__nv_bfloat16, __nv_bfloat16, __nv_bfloat16>(tm, p, grid, smem, st);
  if (d->in_dtype == RV_BF16 && rdt == RV_F32 && d->out_dtype == RV_F32) return launch_tc<__nv_bfloat16, float, float>(tm, p, grid, smem, st);
  return fail(RV_E_UNSUPPORTED, "rv_conv2d(tc): unsupported dtype combination in=%d res=%d out=%d", d->in_dtype, rdt, d->out_dtype);
}

// host-only: the launch plan of rv_conv2d (tensor-core path) for given device limits.  `consumers` 2 plans the two-consumer
// kernel whatever rv_set_conv_consumers holds, 0 takes that setting (and so the kernel a launch would run).
static int plan_for(const rv_conv_desc* d, int max_smem, int num_sms, int consumers, TcP& p, size_t& smem) {
  const int s0 = g_num_sms, s1 = g_max_smem, s2 = g_smem_cap, s3 = g_conv_consumers;
  g_num_sms = num_sms; g_max_smem = max_smem; g_smem_cap = 0;
  if (consumers == 2) g_conv_consumers = 2;
  int nblk = 1;
  const int rc = plan_tc(d, p, smem, nblk);
  g_num_sms = s0; g_max_smem = s1; g_smem_cap = s2; g_conv_consumers = s3;
  return rc;
}

// host-only, the two-consumer plan -> out[8] = {mode, slots per consumer, weights resident, S, consumer warpgroups,
// accumulator sets, nb, smem bytes}.  mode: 0 boxes per (kx, chunk), 1 single box, 2 32B-swizzled quads.
int conv2d_tc_plan(const rv_conv_desc* d, int max_smem, int num_sms, int* out) {
  TcP p;
  size_t smem = 0;
  const int rc = plan_for(d, max_smem, num_sms, 2, p, smem);
  if (rc) return rc;
  out[0] = p.mode;
  out[1] = p.slots; out[2] = p.resident; out[3] = p.S; out[4] = p.ncons; out[5] = p.ncons; out[6] = p.NB; out[7] = (int)smem;
  return RV_OK;
}

// host-only: gate / residual buffers per consumer of that plan (0: the epilogue loads them itself)
int conv2d_tc_epi_depth(const rv_conv_desc* d, int max_smem, int num_sms, int* depth) {
  TcP p;
  size_t smem = 0;
  const int rc = plan_for(d, max_smem, num_sms, 2, p, smem);
  if (rc) return rc;
  *depth = p.epi_tma ? p.epi_depth : 0;
  return RV_OK;
}

// host-only: how that plan stores the output -> *kind = 0 per-thread stores from registers, 1 TMA boxes of [th][tw][NB]
// NHWC tiles, 2 TMA boxes of pixel-shuffled HR rows (PSV), 3 pixel-shuffled HR rows as 16-byte stores from registers (PSV)
int conv2d_tc_out_store(const rv_conv_desc* d, int max_smem, int num_sms, int* kind) {
  TcP p;
  size_t smem = 0;
  const int rc = plan_for(d, max_smem, num_sms, 2, p, smem);
  if (rc) return rc;
  *kind = p.ps_vec ? (p.out_tma ? 2 : 3) : (p.out_tma ? 1 : 0);
  return RV_OK;
}

// host-only: the plan a launch takes under the current rv_set_conv_consumers -> out[4] = {consumer warpgroups, slots per
// consumer, gate / residual buffers per consumer (0: none by TMA), smem bytes}
int conv2d_tc_consumers(const rv_conv_desc* d, int max_smem, int num_sms, int* out) {
  TcP p;
  size_t smem = 0;
  const int rc = plan_for(d, max_smem, num_sms, 0, p, smem);
  if (rc) return rc;
  out[0] = p.ncons; out[1] = p.slots; out[2] = p.epi_tma ? p.epi_depth : 0; out[3] = (int)smem;
  return RV_OK;
}

}  // namespace rv

#ifdef RV_CONV_TIMELINE
// instrumented library only: stamp buffer (nullptr: off) of TL_ROLES x TL_TILES x TL_EV int64 per CTA, and the diagnostic
// variant (0 = the product kernel) for the following launches
extern "C" int rv_conv_timeline_set(void* buf, int diag) {
  long long* b = static_cast<long long*>(buf);
  if (cudaMemcpyToSymbol(rv::g_tl, &b, sizeof(b)) != cudaSuccess) return 1;
  if (cudaMemcpyToSymbol(rv::g_tl_diag, &diag, sizeof(diag)) != cudaSuccess) return 1;
  return 0;
}
extern "C" int rv_conv_timeline_max_slots(int n) {
  const int old = rv::g_tl_max_slots;
  rv::g_tl_max_slots = n;
  return old;
}
extern "C" int rv_conv_timeline_dims(int* out3) {
  out3[0] = rv::TL_ROLES; out3[1] = rv::TL_TILES; out3[2] = rv::TL_EV;
  return 0;
}
#endif
