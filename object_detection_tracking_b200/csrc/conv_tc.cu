// Implicit-GEMM convolution on the Hopper tensor cores (wgmma), operands staged by TMA.
//
//   D[M = B*Ho*Wo pixels, N = Cout] = A[M, K = R*S*Cin] * W[N, K]^T   (+bias, +residual, ReLU / swish)
//
// * A is never materialised: each K-block (one filter tap x 64 input channels) of a 128-pixel tile
//   is fetched straight from the NHWC activation tensor by ONE TMA im2col load
//   (cp.async.bulk.tensor.4d...im2col): padding, stride, dilation and the wrap of a pixel run across
//   image rows / batch images are all resolved by the tensor map (zero fill outside the image).
// * W is pre-packed [Cout][R][S][Cin] (K-major); a 2D tiled TMA load brings block_n x 64 per K-block.
// * Both land in shared memory in the 128-byte-swizzled K-major layout wgmma reads directly.
// * Warpgroup roles (384 threads): warpgroup 0 = TMA producer (warp 0 issues the operand loads, warp 1 is the output
//   warp of the staged epilogue, the others retire at once and hand their registers to the consumers), warpgroups 1 and
//   2 = consumers: each issues wgmma.m64n{64,128}k16 for its 64 rows of the 128-row tile, keeps the accumulators in
//   registers and runs the epilogue of those rows (bias / residual / activation).  The two consumers interleave their
//   MMAs on the tensor cores; they own halves of the same tile and reach its epilogue together.
// * Epilogue, two paths chosen by the plan (p.epi_slots):
//   - staged (fp16-plane outputs that are dense [M][Cout_pad] matrices, with no residual or an unshifted one of the
//     same size): results go through 64 x 64 shared-memory slots, one ring per consumer warpgroup, and leave by TMA
//     store.  The output warp loads the residual into the slots by TMA, running up to kResSlots chunks ahead of the
//     consumers across tile boundaries, so the consumers never wait on a DRAM round trip; they add the residual in place,
//     write the result into the slot and move on.
//   - direct (fp32 outputs, outputs at a placement offset, 2x-upsampled residuals): loads and stores straight from and to
//     global memory.
// * Persistent: grid = min(#tiles, #SMs), static round-robin tile schedule; the producer runs ahead into the next
//   tile while the consumers are in the epilogue of the current one.
// * SPLIT precision: every operand is an fp16 pair (hi, lo') with x = hi + lo'/2048.  Three MMAs per
//   K-step -- acc0 += Ahi*Bhi ; acc1 += Ahi*Blo' + Alo'*Bhi -- and D = acc0 + acc1/2048 recover
//   ~fp32 products on the fp16 tensor pipe (needed for the 1e-3 box parity of the north star).
//
// Reference ops replaced: nn.conv2d (nn.py:337-381) + BatchNorm inference (nn.py:1771-1774, folded into
// weights/bias) + ReLU (nn.py:606-613) + residual add (nn.py:519-521) + FPN upsample-add
// (nn.py:989-996) + dense (nn.py:730-774).
#include <stdlib.h>

#include <type_traits>
#include <vector>

#include "common.h"
#include "planes.cuh"
#include "ptx.cuh"

namespace b2 {

namespace {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;                 // fp16 elements = one 128-byte swizzle row
constexpr int kABytes = kBlockM * kBlockK * 2;   // 16 KB
constexpr int kWgRows = 64;                 // tile rows per consumer warpgroup (the M of wgmma)
constexpr int kWgmmaK = 16;
constexpr int kThreads = 384;               // producer warpgroup + two consumer warpgroups
constexpr int kMaxStages = 8;
constexpr int kSmemBudget = 224 * 1024;     // stages + epilogue slots (alignment slack and barriers on top, 227 KB in all)
constexpr int kSmemLimit = 227 * 1024;
// staged epilogue: a slot holds one consumer warpgroup's 64 rows x 64 columns (one 128-byte swizzle row), per plane
constexpr int kChunkN = 64;
constexpr uint32_t kSlotPlaneBytes = kWgRows * kChunkN * 2;   // 8 KB
constexpr int kMaxSlots = 4;                // per consumer warpgroup
constexpr int kResSlots = 3;                // slots per warpgroup with a residual (the ring the residual is loaded ahead in)
constexpr int kRes3x3Slots = 1;             // the same for a layer with R x S > 1
constexpr int kOutSlots = 1;                // slots per warpgroup without one

struct ConvTcParams {
  int M, Ho, Wo, HoWo;
  int stride, dil, lower_h, lower_w;
  int S, cin_blocks, num_kb;
  int n_cols;        // Cout_pad: columns at or past it (the ragged last n-block) are not stored
  int num_n_blocks, num_tiles;
  int a_mode;        // 0 = A is a plain [M][Cin] matrix (2D tiled TMA), 1 = im2col TMA
  int a_window;      // grouped conv (64-column tiles, one 64-channel block per tap): A reads input channels [n0, n0 + 64)
  uint32_t b_slot_bytes;   // one B plane of a stage in shared memory (block_n rows)
  uint32_t stage_bytes;    // shared-memory footprint of a stage
  uint32_t tx_bytes;       // bytes the TMA loads of a stage deliver (B boxes are clipped to Cout_pad rows)
  int num_stages;
  __half* out_hi;
  __half* out_lo;
  float* out_f32;
  int ldc, out_H, out_W, off_h, off_w;
  const float* bias;
  const __half* res_hi;
  const __half* res_lo;
  int ldr, res_H, res_W, res_shift;
  int relu;
  int acc_kb;        // ACC: K-blocks per tensor-core accumulation chunk
  float acc_delta;   // SPLIT: relative compensation of the tensor-core accumulator's truncation (kAccDelta)
  unsigned int* range_flag;   // ORed with 1 when a plane output exceeds the fp16 range (nullptr = not monitored)
  int epi_slots;     // 0 = direct epilogue (registers -> global); > 0 = staged epilogue with this many slots per warpgroup
  uint32_t slot_bytes;     // one slot: kSlotPlaneBytes per plane (hi, and lo' in split precision)
};

template <bool SWISH>
__device__ __forceinline__ void activate(int relu, float& v0, float& v1) {
  if (relu == 1) {
    v0 = fmaxf(v0, 0.0f);
    v1 = fmaxf(v1, 0.0f);
  } else if (SWISH && relu == 2) {   // swish: x * sigmoid(x) -- only in the SWISH instantiations (EfficientDet)
    v0 = __fmul_rn(v0, 1.f / (1.f + expf(-v0)));   // x * sigmoid(x) as the other kernels compute it
    v1 = __fmul_rn(v1, 1.f / (1.f + expf(-v1)));
  }
}

// The arithmetic of every epilogue path, for two adjacent output channels (n, n + 1) of one pixel: bias, residual (hi,
// then lo'), activation.  load_res(plane) returns the residual's hi (0) or lo' (1) pair.  The full-tile paths pass the
// flags as constants, the general paths as run-time values; either way the expressions and their order are these.
template <bool SWISH, class LoadRes>
__device__ __forceinline__ void pair_math(float& v0, float& v1, float2 b, bool res, bool res_lo, int relu,
                                          LoadRes&& load_res) {
  v0 += b.x;
  v1 += b.y;
  if (res) {
    const float2 r = __half22float2(load_res(0));
    v0 += r.x;
    v1 += r.y;
    if (res_lo) {
      const float2 s = join2(make_float2(v0, v1), load_res(1));
      v0 = s.x;
      v1 = s.y;
    }
  }
  activate<SWISH>(relu, v0, v1);
}

// fp16 (hi, lo') planes of two adjacent outputs, and the range monitor's running maximum
__device__ __forceinline__ void to_planes(float v0, float v1, __half2& hi, __half2& lo, float& amax) {
  amax = fmaxf(amax, fmaxf(fabsf(v0), fabsf(v1)));
  split2(v0, v1, hi, lo);
}

__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<const uint32_t*>(&h); }
__device__ __forceinline__ __half2 bits_h2(uint32_t u) { return *reinterpret_cast<const __half2*>(&u); }

// fp16 (hi, lo') planes of two adjacent outputs; lo == nullptr stores the hi plane only
template <bool SPLIT>
__device__ __forceinline__ void store_planes(float v0, float v1, __half2* hi_dst, __half2* lo_dst, float& amax) {
  __half2 hi, lo;
  to_planes(v0, v1, hi, lo, amax);
  *hi_dst = hi;
  if (SPLIT && lo_dst != nullptr) *lo_dst = lo;
}

// Two adjacent output channels (n, n + 1) of one pixel: bias, residual, activation, store (fp16 hi/lo planes or fp32)
// straight to global memory.
template <bool SPLIT, bool SWISH>
__device__ __forceinline__ void epilogue_pair(const ConvTcParams& p, float v0, float v1, size_t opix, size_t rpix, int n,
                                              float& amax) {
  const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
  pair_math<SWISH>(v0, v1, b, p.res_hi != nullptr, SPLIT && p.res_lo != nullptr, p.relu, [&](int plane) {
    return __ldg(reinterpret_cast<const __half2*>((plane == 0 ? p.res_hi : p.res_lo) + rpix * p.ldr + n));
  });
  if (p.out_f32 != nullptr) {
    *reinterpret_cast<float2*>(p.out_f32 + opix * p.ldc + n) = make_float2(v0, v1);
    return;
  }
  store_planes<SPLIT>(v0, v1, reinterpret_cast<__half2*>(p.out_hi + opix * p.ldc + n),
                      p.out_lo != nullptr ? reinterpret_cast<__half2*>(p.out_lo + opix * p.ldc + n) : nullptr, amax);
}

// The same arithmetic in a staged-epilogue slot: the residual (when there is one) was loaded into the slot by TMA, and
// the result overwrites it in place (hi at s_hi, lo' at s_lo), to leave by TMA store.
template <bool SPLIT, bool SWISH>
__device__ __forceinline__ void epilogue_pair_slot(const ConvTcParams& p, float v0, float v1, int n, __half2* s_hi,
                                                   __half2* s_lo, float& amax) {
  const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
  pair_math<SWISH>(v0, v1, b, p.res_hi != nullptr, SPLIT && p.res_lo != nullptr, p.relu,
                   [&](int plane) { return plane == 0 ? *s_hi : *s_lo; });
  store_planes<SPLIT>(v0, v1, s_hi, p.out_lo != nullptr ? s_lo : nullptr, amax);
}

// Runs f(RES, ACT) with the layer's residual flag and activation as compile-time constants (std::bool_constant,
// std::integral_constant).  A SWISH instantiation only runs swish layers (plan_build), and without SWISH, activate()
// applies nothing but ReLU.
template <bool SWISH, class F>
__device__ __forceinline__ void with_layer_flags(bool res, int relu, F&& f) {
  using Res = std::true_type;
  using NoRes = std::false_type;
  if constexpr (SWISH) {
    if (res) f(Res{}, std::integral_constant<int, 2>{});
    else f(NoRes{}, std::integral_constant<int, 2>{});
  } else if (relu == 1) {
    if (res) f(Res{}, std::integral_constant<int, 1>{});
    else f(NoRes{}, std::integral_constant<int, 1>{});
  } else {
    if (res) f(Res{}, std::integral_constant<int, 0>{});
    else f(NoRes{}, std::integral_constant<int, 0>{});
  }
}

// ACC (split precision only): the tensor core adds into its fp32 accumulator with truncation (round
// toward zero), a bias that grows with the number of accumulation steps (K/16) and compounds through 100+
// layers.  With ACC the hi*hi accumulator is restarted every kAccChunkKb K-blocks and the consumer warpgroup sums the
// chunk results in registers with round-to-nearest fp32 adds, which brings the result to CUDA-core fp32 accuracy.
constexpr int kAccChunkKb = 1;   // default: restart every K-block (64 K-elements = 4 truncating accumulations)
// The truncating adds that remain inside a chunk of four wgmma.k16 shrink every chunk sum toward zero by a small
// relative amount, i.e. the whole conv output by the same factor (sum_q t_q (1 - eta) = (1 - eta) sum_q t_q).
// fmaf(v, kAccDelta, v) (one FFMA per output) gives the loss back: for delta in [2^-24, 1.5 * 2^-24) = [5.96e-8, 8.94e-8)
// the product is between half an ulp and one and a half ulps of v for every mantissa, so the result is v moved away from
// zero by exactly one ulp (0.72 * 2^-23 = 8.6e-8 relative on average); smaller values act on part of the mantissa range,
// values below 2.98e-8 are no-ops.  B2_ACC_DELTA / B2_ACC_DELTA2 override the two constants for calibration sweeps.
constexpr float kAccDelta = 6.8e-8f;
constexpr float kAccDelta2 = 1.7e-7f;   // chunks of two or more K-blocks (seven or more truncating adds)

template <int BN, bool SPLIT, bool ACC, bool SWISH>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
               const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
               const __grid_constant__ CUtensorMap tmO_hi, const __grid_constant__ CUtensorMap tmO_lo,
               const __grid_constant__ CUtensorMap tmR_hi, const __grid_constant__ CUtensorMap tmR_lo,
               const __grid_constant__ ConvTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle atoms need 1024-byte aligned tiles (an offset from smem_raw, so that the compiler knows the pointers
  // below are shared memory and accesses through them are LDS / STS)
  uint8_t* tiles = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  // staged epilogue: slot s of consumer warpgroup w at slots + (w * epi_slots + s) * slot_bytes
  uint8_t* slots = tiles + static_cast<size_t>(p.num_stages) * p.stage_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(slots + static_cast<size_t>(2 * p.epi_slots) * p.slot_bytes);
  uint64_t* empty_bar = full_bar + kMaxStages;
  uint64_t* slot_full = empty_bar + kMaxStages;        // [w * kMaxSlots + s]: residual landed / slot free to write
  uint64_t* slot_written = slot_full + 2 * kMaxSlots;  // [w * kMaxSlots + s]: the warpgroup's result is in the slot

  // broadcast from lane 0 so that the compiler treats the warp index (and everything derived from it) as warp-uniform
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA_hi);
    tma_prefetch_desc(&tmB_hi);
    if (SPLIT) {
      tma_prefetch_desc(&tmA_lo);
      tma_prefetch_desc(&tmB_lo);
    }
    for (int i = 0; i < p.num_stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // one arrive per consumer warp
    }
    if (p.epi_slots > 0) {
      tma_prefetch_desc(&tmO_hi);
      if (SPLIT && p.out_lo != nullptr) tma_prefetch_desc(&tmO_lo);
      if (p.res_hi != nullptr) tma_prefetch_desc(&tmR_hi);
      if (SPLIT && p.res_lo != nullptr) tma_prefetch_desc(&tmR_lo);
      for (int i = 0; i < 2 * kMaxSlots; ++i) {
        mbar_init(&slot_full[i], 1);
        mbar_init(&slot_written[i], 4);   // one arrive per warp of the consumer warpgroup
      }
    }
    fence_mbar_init();
  }
  __syncthreads();

  const uint32_t a_lo_off = kABytes;
  const uint32_t b_hi_off = SPLIT ? 2 * kABytes : kABytes;
  const uint32_t b_lo_off = b_hi_off + p.b_slot_bytes;

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (warp == 1 && p.epi_slots > 0) {
      // ===================== output warp (staged epilogue), one lane =====================
      // Walks this CTA's (tile, 64-column chunk) sequence twice: arming slots (residual TMA load, or a plain arrive)
      // epi_slots chunks ahead of the consumers, across tile boundaries, and storing each chunk once both
      // warpgroups have written it.  A slot is re-armed when the store has finished reading it.
      if (lane != 0) return;
      constexpr int kChunks = BN / kChunkN;
      const bool res = p.res_hi != nullptr;
      const bool res_lo = SPLIT && p.res_lo != nullptr;
      const bool out_lo = SPLIT && p.out_lo != nullptr;
      const uint32_t res_tx = kSlotPlaneBytes * (res_lo ? 2 : 1);
      int arm_tile = blockIdx.x, arm_chunk = 0;
      auto arm = [&](int s) {   // slot s of both warpgroups <- chunk (arm_tile, arm_chunk)
        const int m_blk = arm_tile / p.num_n_blocks;
        const int n = (arm_tile - m_blk * p.num_n_blocks) * BN + arm_chunk * kChunkN;
#pragma unroll
        for (int w = 0; w < 2; ++w) {
          uint64_t* bar = &slot_full[w * kMaxSlots + s];
          const int m = m_blk * kBlockM + w * kWgRows;
          if (res && m < p.M) {
            uint8_t* dst = slots + static_cast<size_t>(w * p.epi_slots + s) * p.slot_bytes;
            mbar_expect_tx(bar, res_tx);
            tma_load_2d(dst, &tmR_hi, bar, n, m);
            if (res_lo) tma_load_2d(dst + kSlotPlaneBytes, &tmR_lo, bar, n, m);
          } else {
            mbar_arrive(bar);
          }
        }
        if (++arm_chunk == kChunks) {
          arm_chunk = 0;
          arm_tile += gridDim.x;
        }
      };
      for (int s = 0; s < p.epi_slots && arm_tile < p.num_tiles; ++s) arm(s);
      int slot = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int m_blk = tile / p.num_n_blocks;
        const int n0 = (tile - m_blk * p.num_n_blocks) * BN;
        for (int c = 0; c < kChunks; ++c) {
#pragma unroll
          for (int w = 0; w < 2; ++w) {
            mbar_wait(&slot_written[w * kMaxSlots + slot], phase);
            const int m = m_blk * kBlockM + w * kWgRows;
            if (m < p.M) {
              const uint8_t* src = slots + static_cast<size_t>(w * p.epi_slots + slot) * p.slot_bytes;
              tma_store_2d(&tmO_hi, src, n0 + c * kChunkN, m);
              if (out_lo) tma_store_2d(&tmO_lo, src + kSlotPlaneBytes, n0 + c * kChunkN, m);
            }
          }
          bulk_commit();
          if (arm_tile < p.num_tiles) {
            bulk_wait_read<0>();
            arm(slot);
          }
          if (++slot == p.epi_slots) {
            slot = 0;
            phase ^= 1;
          }
        }
      }
      bulk_wait<0>();   // the shared-memory sources must outlive the stores
      return;
    }
    if (warp != 0) return;
    // converged warp, one elected lane issues
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int m_blk = tile / p.num_n_blocks;
      const int n0 = (tile - m_blk * p.num_n_blocks) * BN;
      const int m0 = m_blk * kBlockM;
      int img = 0, ch = 0, cw = 0;
      if (p.a_mode == 1) {
        img = m0 / p.HoWo;
        const int rem = m0 - img * p.HoWo;
        const int pp = rem / p.Wo;
        const int qq = rem - pp * p.Wo;
        ch = p.lower_h + pp * p.stride;
        cw = p.lower_w + qq * p.stride;
      }
      int tap = 0, cb = 0;   // K-block = (filter tap, 64-channel block)
      const int c0 = p.a_window ? n0 : 0;   // first input channel of the K-blocks
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* st = tiles + static_cast<size_t>(stage) * p.stage_bytes;
        if (elect_one()) {
          mbar_expect_tx(&full_bar[stage], p.tx_bytes);
          if (p.a_mode == 1) {
            const int r = tap / p.S;
            const int s = tap - r * p.S;
            const uint16_t ow = static_cast<uint16_t>(s * p.dil);
            const uint16_t oh = static_cast<uint16_t>(r * p.dil);
            tma_load_im2col_4d(st, &tmA_hi, &full_bar[stage], c0 + cb * kBlockK, cw, ch, img, ow, oh);
            if (SPLIT) tma_load_im2col_4d(st + a_lo_off, &tmA_lo, &full_bar[stage], c0 + cb * kBlockK, cw, ch, img, ow, oh);
          } else {
            tma_load_2d(st, &tmA_hi, &full_bar[stage], c0 + cb * kBlockK, m0);
            if (SPLIT) tma_load_2d(st + a_lo_off, &tmA_lo, &full_bar[stage], c0 + cb * kBlockK, m0);
          }
          tma_load_2d(st + b_hi_off, &tmB_hi, &full_bar[stage], kb * kBlockK, n0);
          if (SPLIT) tma_load_2d(st + b_lo_off, &tmB_lo, &full_bar[stage], kb * kBlockK, n0);
        }
        __syncwarp();
        if (++cb == p.cin_blocks) {
          cb = 0;
          ++tap;
        }
        if (++stage == p.num_stages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  // 128 x 40 + 256 x 232 registers = what the CTA was launched with (384 x 168): the increase must fit in what the
  // producer warpgroup gave back, or setmaxnreg.inc never returns.
  setmaxnreg_inc<232>();
  constexpr int kAcc = BN / 2;   // fp32 accumulator registers per thread for a 64 x BN block
  const int cwg = wg - 1;        // rows cwg * 64 .. of the tile
  // wgmma accumulator layout: warp q of the warpgroup holds rows 16q..16q+15; lane l holds rows l/4 and l/4 + 8 of
  // those, columns 8j + 2(l%4) + {0, 1} of every 8-column block j in registers 4j + {0, 1} (first row) / 4j + {2, 3}
  const int wg_row = (warp & 3) * 16 + (lane >> 2);   // first row inside the warpgroup's 64 (the other is + 8)
  const int row0 = cwg * kWgRows + wg_row;
  const int col0 = 2 * (lane & 3);
  int eslot = 0;         // staged epilogue: slot of this warpgroup's next chunk
  uint32_t ephase = 0;
  const uint32_t tiles_u32 = smem_u32(tiles);
  float acc0[kAcc];
  float acc1[SPLIT ? kAcc : 1];
  float sums[ACC ? kAcc : 1];
  int stage = 0;
  uint32_t phase = 0;
  auto release = [&](int s) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  };
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int m_blk = tile / p.num_n_blocks;
    const int n0 = (tile - m_blk * p.num_n_blocks) * BN;
    if (ACC) {
#pragma unroll
      for (int i = 0; i < kAcc; ++i) sums[i] = 0.0f;
    }
    // The wait structure is the same on every K-block: no wgmma_wait sits on a run-time branch.  A wait whose count
    // depends on a divergent path makes ptxas serialise every wgmma of the loop (C7518) or insert waits of its own
    // (C7517); tests/test_conv_ptxas_cpu.py keeps both out.
    int kq = 0;       // ACC: K-block inside the current chunk
    int held = -1;    // stage the newest commit group may still be reading (released after the next wait)
    for (int kb = 0; kb < p.num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t st = tiles_u32 + static_cast<uint32_t>(stage) * p.stage_bytes;
      const uint32_t a_hi = st + cwg * (kWgRows * kBlockK * 2);
      const uint32_t b_hi = st + b_hi_off;
      const uint32_t first = kb > 0 ? 1u : 0u;
      wgmma_fence();
      if constexpr (ACC) {
        // two commit groups: the four hi*hi MMAs of the chunk accumulator, then the eight cross terms.
#pragma unroll
        for (int k = 0; k < kBlockK / kWgmmaK; ++k) {
          const uint32_t ko = k * kWgmmaK * 2;   // 32 bytes along K inside the 128-byte swizzle row
          wgmma_f16<BN>(acc0, make_smem_desc_sw128(a_hi + ko), make_smem_desc_sw128(b_hi + ko),
                        (kq > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        // all but the newest group done: the previous K-block's cross terms have finished with their stage, which
        // goes back to the producer while this K-block's hi*hi MMAs run
        wgmma_wait<1>();
        if (held >= 0) release(held);
#pragma unroll
        for (int k = 0; k < kBlockK / kWgmmaK; ++k) {
          const uint32_t ko = k * kWgmmaK * 2;
          const uint64_t da_hi = make_smem_desc_sw128(a_hi + ko);
          const uint64_t db_hi = make_smem_desc_sw128(b_hi + ko);
          wgmma_f16<BN>(acc1, da_hi, make_smem_desc_sw128(st + b_lo_off + ko), (first | k) ? 1u : 0u);
          wgmma_f16<BN>(acc1, make_smem_desc_sw128(a_hi + a_lo_off + ko), db_hi, 1u);
        }
        wgmma_commit();
        // acc0 is final: at the end of a chunk it is folded into the running sums with round-to-nearest adds (a
        // select, not a branch) while the cross terms -- two thirds of the K-block's MMAs -- are still on the tensor
        // cores
        wgmma_wait<1>();
        fence_regs(acc0);
        const bool fold = kq + 1 == p.acc_kb || kb == p.num_kb - 1;
#pragma unroll
        for (int i = 0; i < kAcc; ++i) sums[i] = fold ? __fadd_rn(sums[i], acc0[i]) : sums[i];
        kq = fold ? 0 : kq + 1;
      } else {
#pragma unroll
        for (int k = 0; k < kBlockK / kWgmmaK; ++k) {
          const uint32_t ko = k * kWgmmaK * 2;
          const uint64_t da_hi = make_smem_desc_sw128(a_hi + ko);
          const uint64_t db_hi = make_smem_desc_sw128(b_hi + ko);
          const uint32_t acc = (first | k) ? 1u : 0u;
          wgmma_f16<BN>(acc0, da_hi, db_hi, acc);
          if constexpr (SPLIT) {
            const uint64_t da_lo = make_smem_desc_sw128(a_hi + a_lo_off + ko);
            const uint64_t db_lo = make_smem_desc_sw128(st + b_lo_off + ko);
            wgmma_f16<BN>(acc1, da_hi, db_lo, acc);
            wgmma_f16<BN>(acc1, da_lo, db_hi, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous K-block's MMAs are done with their stage
        if (held >= 0) release(held);
      }
      held = stage;
      if (++stage == p.num_stages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();   // num_kb >= 1: held is a stage here
    release(held);
    fence_regs(acc0);
    if constexpr (SPLIT) fence_regs(acc1);

    // ---- epilogue: this thread's two rows
    auto out_value = [&](int i) -> float {   // accumulator register i -> conv output before bias
      if constexpr (!SPLIT) {
        return acc0[i];
      } else if constexpr (ACC) {
        const float s = fmaf(acc1[i], kLoInv, sums[i]);
        return fmaf(s, p.acc_delta, s);
      } else {   // single-chunk (K <= 64) split layers: the same compensation
        const float v = fmaf(acc0[i], p.acc_delta, acc0[i]);
        return fmaf(acc1[i], kLoInv, v);
      }
    };
    bool valid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) valid[h] = m_blk * kBlockM + row0 + 8 * h < p.M;
    float amax = 0.f;   // largest |output| this thread writes in this tile (range monitor)
    // A full tile (every row below M, every column below Cout_pad) of a layer whose planes are the precision's (lo'
    // planes in split precision) takes an epilogue with the layer's flags as compile-time constants: no per-pair row or
    // column checks and no flag reloads.  Other tiles take the general path, which clips and reads the flags per pair.
    const bool res = p.res_hi != nullptr;
    const bool full = m_blk * kBlockM + kBlockM <= p.M && n0 + BN <= p.n_cols && (!SWISH || p.relu == 2) &&
                      (!SPLIT || ((!res || p.res_lo != nullptr) && (p.out_f32 != nullptr || p.out_lo != nullptr)));
    if (p.epi_slots == 0) {
      // output and residual pixel of this thread's two rows (rows past M: 0, never stored).  Each branch below computes
      // them itself: computed once ahead of the branch, they spill in the 128-column split + ACC kernel's ragged path.
      size_t opix[2] = {0, 0}, rpix[2] = {0, 0};
      auto row_pixels = [&] {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = m_blk * kBlockM + row0 + 8 * h;
          if (valid[h]) {
            const int img = m / p.HoWo;
            const int rem = m - img * p.HoWo;
            const int pp = rem / p.Wo + p.off_h;
            const int qq = rem - (rem / p.Wo) * p.Wo + p.off_w;
            opix[h] = (static_cast<size_t>(img) * p.out_H + pp) * p.out_W + qq;
            rpix[h] = (static_cast<size_t>(img) * p.res_H + (pp >> p.res_shift)) * p.res_W + (qq >> p.res_shift);
          }
        }
      };
      if (full) {
        row_pixels();
        auto direct_full = [&](auto F32, auto RES, auto ACT) {
          constexpr bool kF32 = decltype(F32)::value;
          constexpr bool kRes = decltype(RES)::value;
          const float2* bias = reinterpret_cast<const float2*>(p.bias + n0 + col0);
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {   // 8-column block j: pair 4 * j of the row's float2 / __half2 view
            const float2 b = __ldg(bias + 4 * j);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int i = 4 * j + 2 * h;
              const size_t o = opix[h] * p.ldc + n0 + col0;
              const size_t r = rpix[h] * p.ldr + n0 + col0;
              float v0 = out_value(i), v1 = out_value(i + 1);
              pair_math<SWISH>(v0, v1, b, kRes, SPLIT && kRes, ACT, [&](int plane) {
                return __ldg(reinterpret_cast<const __half2*>((plane == 0 ? p.res_hi : p.res_lo) + r) + 4 * j);
              });
              if constexpr (kF32) {
                reinterpret_cast<float2*>(p.out_f32 + o)[4 * j] = make_float2(v0, v1);
              } else {
                __half2 hi, lo;
                to_planes(v0, v1, hi, lo, amax);
                reinterpret_cast<__half2*>(p.out_hi + o)[4 * j] = hi;
                if (SPLIT) reinterpret_cast<__half2*>(p.out_lo + o)[4 * j] = lo;
              }
            }
          }
        };
        if (p.out_f32 != nullptr)
          with_layer_flags<SWISH>(res, p.relu, [&](auto RES, auto ACT) { direct_full(std::true_type{}, RES, ACT); });
        else
          with_layer_flags<SWISH>(res, p.relu, [&](auto RES, auto ACT) { direct_full(std::false_type{}, RES, ACT); });
      } else {
        row_pixels();
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int n = n0 + 8 * j + col0;
          if (n >= p.n_cols) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (!valid[h]) continue;
            const int i = 4 * j + 2 * h;
            epilogue_pair<SPLIT, SWISH>(p, out_value(i), out_value(i + 1), opix[h], rpix[h], n, amax);
          }
        }
      }
    } else {
      // staged: one 64-column chunk at a time through this warpgroup's slot ring.  Slot layout = the TMA box with
      // 128-byte swizzle: row r at r * 128, 16-byte unit u at (u ^ (r % 8)) * 16.  The 8 rows a warp's lanes hold
      // have distinct r % 8, so every 4-byte access of the warp hits 32 distinct banks.
      auto run_chunks = [&](auto&& chunk) {   // chunk(c, byte offset of the slot from `slots`)
#pragma unroll
        for (int c = 0; c < BN / kChunkN; ++c) {
          mbar_wait(&slot_full[cwg * kMaxSlots + eslot], ephase);
          chunk(c, static_cast<uint32_t>(cwg * p.epi_slots + eslot) * p.slot_bytes);
          fence_proxy_async_smem();   // the TMA store reads what this thread wrote
          __syncwarp();
          if (lane == 0) mbar_arrive(&slot_written[cwg * kMaxSlots + eslot]);
          if (++eslot == p.epi_slots) {
            eslot = 0;
            ephase ^= 1;
          }
        }
      };
      if (full) {
        with_layer_flags<SWISH>(res, p.relu, [&](auto RES, auto ACT) {
          constexpr bool kRes = decltype(RES)::value;
          run_chunks([&](int c, uint32_t slot_off) {
            // The slot is 1024-byte aligned and r % 8 = lane / 4, so the swizzle phase sits alone in address bits 4-6:
            // unit u of this thread's first row is at row ^ (u << 4), and its second row (r + 8) 1024 bytes on.
            const uint32_t row = smem_u32(slots) + slot_off + wg_row * 128 + ((lane >> 2) << 4) + col0 * 2;
            const float2* bias = reinterpret_cast<const float2*>(p.bias + n0 + col0);
#pragma unroll
            for (int u = 0; u < kChunkN / 8; ++u) {
              const int j = c * (kChunkN / 8) + u;
              const float2 b = __ldg(bias + 4 * j);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int i = 4 * j + 2 * h;
                const uint32_t a = (row ^ (u << 4)) + h * 1024;
                float v0 = out_value(i), v1 = out_value(i + 1);
                pair_math<SWISH>(v0, v1, b, kRes, SPLIT && kRes, ACT,
                                 [&](int plane) { return bits_h2(ld_shared_b32(a + plane * kSlotPlaneBytes)); });
                __half2 hi, lo;
                to_planes(v0, v1, hi, lo, amax);
                st_shared_b32(a, h2_bits(hi));
                if (SPLIT) st_shared_b32(a + kSlotPlaneBytes, h2_bits(lo));
              }
            }
          });
        });
      } else {
        run_chunks([&](int c, uint32_t slot_off) {
          uint8_t* s_hi = slots + slot_off;
#pragma unroll
          for (int u = 0; u < kChunkN / 8; ++u) {
            const int j = c * (kChunkN / 8) + u;
            const int n = n0 + 8 * j + col0;
            if (n >= p.n_cols) continue;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              if (!valid[h]) continue;
              const int i = 4 * j + 2 * h;
              const uint32_t off = (wg_row + 8 * h) * 128 + ((u ^ (lane >> 2)) << 4) + col0 * 2;
              epilogue_pair_slot<SPLIT, SWISH>(p, out_value(i), out_value(i + 1), n,
                                               reinterpret_cast<__half2*>(s_hi + off),
                                               reinterpret_cast<__half2*>(s_hi + kSlotPlaneBytes + off), amax);
            }
          }
        });
      }
    }
    // inf included; a NaN can only follow an inf, which an earlier launch has flagged
    if (p.range_flag != nullptr && amax > 65504.f) atomicOr(p.range_flag, 1u);
  }
}

// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode_tiled = nullptr;
EncodeIm2colFn g_encode_im2col = nullptr;
int g_driver_version = 0;

void small_tensor_fixup(CUtensorMap* m, size_t bytes) {
  // Driver <= 13.1 mis-encodes maps of tensors smaller than 128 KiB (bit 21 of the 2nd qword); the
  // vendored CuTe applies the same fix-up (cute/atom/copy_traits_sm90_tma.hpp).
  if (g_driver_version <= 13010 && bytes < 131072) reinterpret_cast<uint64_t*>(m)[1] &= ~(1ull << 21);
}

int encode_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
              uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed: " + std::to_string(static_cast<int>(r)));
    return -1;
  }
  small_tensor_fixup(m, static_cast<size_t>(outer) * row_stride_bytes);
  return 0;
}


typedef void (*ConvKernel)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap,
                           CUtensorMap, ConvTcParams);

template <int BN>
ConvKernel kernel_for(bool split, bool acc, bool swish) {
  if (split && acc) return swish ? conv_tc_kernel<BN, true, true, true> : conv_tc_kernel<BN, true, true, false>;
  if (split) return swish ? conv_tc_kernel<BN, true, false, true> : conv_tc_kernel<BN, true, false, false>;
  return swish ? conv_tc_kernel<BN, false, false, true> : conv_tc_kernel<BN, false, false, false>;
}

ConvKernel kernel_for(int block_n, bool split, bool acc, bool swish) {
  return block_n == 64 ? kernel_for<64>(split, acc, swish) : kernel_for<128>(split, acc, swish);
}

}  // namespace

struct ConvPlan {
  CUtensorMap tmA_hi, tmA_lo, tmB_hi, tmB_lo;
  CUtensorMap tmO_hi, tmO_lo, tmR_hi, tmR_lo;   // staged epilogue: output / residual planes as [M][Cout_pad]
  ConvTcParams p;
  ConvKernel kernel;
  int grid;
  size_t smem_bytes;
};

int conv_tc_init() {
  if (g_encode_tiled && g_encode_im2col) return 0;
  B2_CUDA(cudaDriverGetVersion(&g_driver_version));
  cudaDriverEntryPointQueryResult q;
  void* fn = nullptr;
  B2_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  B2_CHECK(fn != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
  g_encode_tiled = reinterpret_cast<EncodeTiledFn>(fn);
  fn = nullptr;
  B2_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &q));
  B2_CHECK(fn != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeIm2col not available");
  g_encode_im2col = reinterpret_cast<EncodeIm2colFn>(fn);
  for (int bn : {64, 128})
    for (int mode = 0; mode < 3; ++mode)   // fp16, split, split + ACC
      for (int swish = 0; swish < 2; ++swish)
        B2_CUDA(cudaFuncSetAttribute(kernel_for(bn, mode >= 1, mode == 2, swish != 0),
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit));
  return 0;
}

// 128-column tiles unless 64-column tiles pad Cout_pad less (Cout_pad <= 64, or 64 past a multiple of 128)
static int pick_block_n(int cout_pad) {
  const int pad128 = (cout_pad + 127) / 128 * 128;
  const int pad64 = (cout_pad + 63) / 64 * 64;
  return pad64 < pad128 ? 64 : 128;
}

static int plan_build(ConvPlan* pl, const ConvDesc& d, const ConvWeights& w, const ConvIO& io, bool split,
                      int num_sms, int force_a_mode) {
  B2_CHECK(conv_tc_init() == 0, "conv_tc_init failed");
  B2_CHECK(d.Cin % kBlockK == 0, "conv_tc: Cin must be a multiple of 64");
  B2_CHECK(w.Cout_pad % 16 == 0, "conv_tc: Cout_pad must be a multiple of 16");
  // grouped conv as block-diagonal 64-channel windows: a 64-column tile's outputs read only the same 64 input channels
  const bool grouped = d.groups > 1;
  B2_CHECK(!grouped || (d.Cin % d.groups == 0 && d.Cout == d.Cin && kGroupWindow % (d.Cin / d.groups) == 0),
           "conv_tc: a grouped conv needs Cout == Cin and groups whose channel count divides 64");
  B2_CHECK(w.K == d.R * d.S * (grouped ? kGroupWindow : d.Cin), "conv_tc: packed weight K mismatch");
  B2_CHECK(!split || (io.in_lo && w.w_lo), "conv_tc: split precision needs lo planes");
  ConvTcParams& p = pl->p;
  const int Ho = d.Ho(), Wo = d.Wo();
  B2_CHECK(Ho > 0 && Wo > 0, "conv_tc: empty output");
  p.M = d.B * Ho * Wo;
  p.Ho = Ho;
  p.Wo = Wo;
  p.HoWo = Ho * Wo;
  p.stride = d.stride;
  p.dil = d.dil;
  p.lower_h = -d.pad_t;
  p.lower_w = -d.pad_l;
  p.S = d.S;
  p.cin_blocks = grouped ? 1 : d.Cin / kBlockK;
  p.num_kb = d.R * d.S * p.cin_blocks;
  p.a_window = grouped ? 1 : 0;
  const int block_n = grouped ? kGroupWindow : pick_block_n(w.Cout_pad);
  const int b_rows = w.Cout_pad < block_n ? w.Cout_pad : block_n;   // rows of the B box (<= the tensor's)
  p.n_cols = w.Cout_pad;
  p.num_n_blocks = (w.Cout_pad + block_n - 1) / block_n;
  const int num_m_blocks = (p.M + kBlockM - 1) / kBlockM;
  p.num_tiles = num_m_blocks * p.num_n_blocks;
  p.b_slot_bytes = static_cast<uint32_t>(block_n) * kBlockK * 2;
  p.stage_bytes = (kABytes + p.b_slot_bytes) * (split ? 2 : 1);
  p.tx_bytes = (kABytes + static_cast<uint32_t>(b_rows) * kBlockK * 2) * (split ? 2 : 1);
  // Staged epilogue (results leave by TMA store, the residual arrives by TMA load) when output and residual are dense
  // [M][Cout_pad] row-major matrices the tensor maps can describe: fp16 planes written without a placement offset, an
  // unshifted residual of the same size, 16-byte aligned bases and row strides.
  auto aligned16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  const char* not_staged = nullptr;   // why the staged epilogue cannot take this layer (nullptr: it can)
  if (io.out_f32 != nullptr)
    not_staged = "the output is fp32";
  else if (d.off_h != 0 || d.off_w != 0 || d.out_H != Ho || d.out_W != Wo)
    not_staged = "the output is placed inside a larger buffer";
  else if (!aligned16(io.out_hi) || (split && !aligned16(io.out_lo)))
    not_staged = "the output planes are not 16-byte aligned";
  else if (io.res_hi != nullptr && (d.res_shift != 0 || d.res_H != Ho || d.res_W != Wo))
    not_staged = "the residual is upsampled or not the output's size";
  else if (io.res_hi != nullptr && (d.ldr % 8 != 0 || !aligned16(io.res_hi) || (split && !aligned16(io.res_lo))))
    not_staged = "the residual rows or planes are not 16-byte aligned";
  B2_CHECK(d.force_epi != 1 || not_staged == nullptr,
           std::string("conv_tc: force_epi = 1 asks for the staged epilogue, but ") + (not_staged ? not_staged : ""));
  const bool staged = not_staged == nullptr && d.force_epi != 0;
  // a 1x1 residual layer (1-4 K-blocks) loads its residual kResSlots chunks ahead; an R x S > 1 one (9-72 K-blocks) is
  // mainloop-bound and gets one slot, so that its operand ring keeps a stage more (DESIGN 4, Basic block)
  int res_slots = d.R * d.S > 1 ? kRes3x3Slots : kResSlots;
  if (const char* e = getenv("B2_RES_SLOTS"))   // experiment hook: slots of the staged R x S > 1 residual layers
    if (d.R * d.S > 1 && atoi(e) >= 1 && atoi(e) <= kMaxSlots) res_slots = atoi(e);
  p.epi_slots = !staged ? 0 : io.res_hi != nullptr ? res_slots : kOutSlots;
  p.slot_bytes = kSlotPlaneBytes * (split ? 2 : 1);
  const int slot_total = 2 * p.epi_slots * static_cast<int>(p.slot_bytes);
  p.num_stages = (kSmemBudget - slot_total) / static_cast<int>(p.stage_bytes);
  if (p.num_stages > kMaxStages) p.num_stages = kMaxStages;
  B2_CHECK(p.num_stages >= 2, "conv_tc: tile too large for shared memory");
  p.out_hi = io.out_hi;
  p.out_lo = io.out_lo;
  p.out_f32 = io.out_f32;
  p.ldc = d.ldc;
  p.out_H = d.out_H;
  p.out_W = d.out_W;
  p.off_h = d.off_h;
  p.off_w = d.off_w;
  B2_CHECK(d.ldc >= w.Cout_pad && d.ldc % 8 == 0, "conv_tc: ldc must cover Cout_pad");
  B2_CHECK(Ho + d.off_h <= d.out_H && Wo + d.off_w <= d.out_W, "conv_tc: output does not fit buffer");
  p.bias = w.bias;
  p.res_hi = io.res_hi;
  p.res_lo = io.res_lo;
  p.ldr = d.ldr;
  // both epilogues read residual columns [0, Cout_pad) of every row
  B2_CHECK(io.res_hi == nullptr || (d.ldr % 2 == 0 && d.ldr >= w.Cout_pad), "conv_tc: ldr must be even and cover Cout_pad");
  p.res_H = d.res_H;
  p.res_W = d.res_W;
  p.res_shift = d.res_shift;
  p.relu = d.relu;
  p.range_flag = io.range_flag;
  // accurate accumulation: on by default in split precision when K spans more than one chunk
  p.acc_kb = d.acc_kb > 0 ? d.acc_kb : kAccChunkKb;
  if (const char* e = getenv("B2_ACC_KB")) p.acc_kb = atoi(e) > 0 ? atoi(e) : kAccChunkKb;
  const bool acc = split && d.acc_kb >= 0 && p.num_kb > p.acc_kb && getenv("B2_NO_ACC") == nullptr;
  p.acc_delta = getenv("B2_ACC_DELTA") ? static_cast<float>(atof(getenv("B2_ACC_DELTA"))) : kAccDelta;
  if (p.acc_kb >= 2) p.acc_delta = getenv("B2_ACC_DELTA2") ? static_cast<float>(atof(getenv("B2_ACC_DELTA2"))) : kAccDelta2;
  pl->kernel = kernel_for(block_n, split, acc, d.relu == 2);
  pl->grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
  pl->smem_bytes = static_cast<size_t>(p.num_stages) * p.stage_bytes + slot_total + 1024 /*align*/ +
                   (2 * kMaxStages + 4 * kMaxSlots) * 8 /*barriers*/;
  const int in_ld = d.in_ld > 0 ? d.in_ld : d.Cin;
  const bool plain = (d.R == 1 && d.S == 1 && d.stride == 1 && d.pad_t == 0 && d.pad_b == 0 && d.pad_l == 0 &&
                      d.pad_r == 0 && d.in_H == d.in_pitch_H && d.in_W == d.in_pitch_W);
  p.a_mode = plain ? 0 : 1;
  if (force_a_mode >= 0) {
    B2_CHECK(force_a_mode == 1 || plain, "conv_tc: tiled A mode needs a plain 1x1 conv");
    p.a_mode = force_a_mode;
  }
  const size_t in_bytes = static_cast<size_t>(d.B) * d.in_pitch_H * d.in_pitch_W * in_ld * 2;
  for (int plane = 0; plane < (split ? 2 : 1); ++plane) {
    CUtensorMap* mA = plane == 0 ? &pl->tmA_hi : &pl->tmA_lo;
    CUtensorMap* mB = plane == 0 ? &pl->tmB_hi : &pl->tmB_lo;
    const __half* a = plane == 0 ? io.in_hi : io.in_lo;
    const __half* b = plane == 0 ? w.w_hi : w.w_lo;
    if (p.a_mode == 0) {
      if (encode_2d(mA, a, d.Cin, static_cast<uint64_t>(d.B) * d.in_H * d.in_W, static_cast<uint64_t>(in_ld) * 2,
                    kBlockK, kBlockM))
        return -1;
    } else {
      cuuint64_t dims[4] = {static_cast<cuuint64_t>(d.Cin), static_cast<cuuint64_t>(d.in_W),
                            static_cast<cuuint64_t>(d.in_H), static_cast<cuuint64_t>(d.B)};
      cuuint64_t strides[3] = {static_cast<cuuint64_t>(in_ld) * 2,
                               static_cast<cuuint64_t>(d.in_pitch_W) * in_ld * 2,
                               static_cast<cuuint64_t>(d.in_pitch_H) * d.in_pitch_W * in_ld * 2};
      // bounding box of filter base positions: lower = -pad, upper = pad_after - (k-1)*dilation  {W, H}
      int lower[2] = {-d.pad_l, -d.pad_t};
      int upper[2] = {d.pad_r - (d.S - 1) * d.dil, d.pad_b - (d.R - 1) * d.dil};
      cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(d.stride), static_cast<cuuint32_t>(d.stride), 1};
      CUresult r = g_encode_im2col(mA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(a), dims, strides,
                                   lower, upper, kBlockK, kBlockM, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeIm2col failed: " + std::to_string(static_cast<int>(r)) + " (Cin=" +
                  std::to_string(d.Cin) + " W=" + std::to_string(d.in_W) + " H=" + std::to_string(d.in_H) + ")");
        return -1;
      }
      small_tensor_fixup(mA, in_bytes);
    }
    if (encode_2d(mB, b, w.K, w.Cout_pad, static_cast<uint64_t>(w.K) * 2, kBlockK, b_rows)) return -1;
  }
  if (!split) {
    pl->tmA_lo = pl->tmA_hi;
    pl->tmB_lo = pl->tmB_hi;
  }
  // staged epilogue: 64 x 64 boxes of [M][Cout_pad]; stores clip the ragged last m- and n-blocks, loads zero-fill them
  pl->tmO_hi = pl->tmO_lo = pl->tmR_hi = pl->tmR_lo = pl->tmB_hi;   // unused maps: any valid map
  if (p.epi_slots > 0) {
    const int planes = split ? 2 : 1;
    for (int plane = 0; plane < planes; ++plane) {
      const __half* o = plane == 0 ? io.out_hi : io.out_lo;
      if (o && encode_2d(plane == 0 ? &pl->tmO_hi : &pl->tmO_lo, o, w.Cout_pad, p.M, static_cast<uint64_t>(d.ldc) * 2,
                         kChunkN, kWgRows))
        return -1;
      const __half* r = plane == 0 ? io.res_hi : io.res_lo;
      if (r && encode_2d(plane == 0 ? &pl->tmR_hi : &pl->tmR_lo, r, w.Cout_pad, p.M, static_cast<uint64_t>(d.ldr) * 2,
                         kChunkN, kWgRows))
        return -1;
    }
  }
  return 0;
}

ConvPlan* conv_tc_plan_create(const ConvDesc& d, const ConvWeights& w, const ConvIO& io, bool split, int num_sms) {
  ConvPlan* pl = new ConvPlan();
  if (plan_build(pl, d, w, io, split, num_sms, d.force_a_mode) != 0) {
    delete pl;
    return nullptr;
  }
  return pl;
}

void conv_tc_plan_destroy(ConvPlan* p) { delete p; }

int conv_tc_launch(const ConvPlan* pl, cudaStream_t stream) {
  pl->kernel<<<pl->grid, kThreads, pl->smem_bytes, stream>>>(pl->tmA_hi, pl->tmA_lo, pl->tmB_hi, pl->tmB_lo, pl->tmO_hi,
                                                             pl->tmO_lo, pl->tmR_hi, pl->tmR_lo, pl->p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
