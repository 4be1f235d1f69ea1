// tapgemm_tc.cu -- wgmma / TMA implementation of the shifted-tap GEMM (see tapgemm.h) for Hopper (sm_90a).
//
// A persistent CTA (one per SM) computes 128 (pixels) x BN (output channels) tiles of the output phases:
//   warp 8     : TMA producer.  Per K step (one tap x 64 input channels) two bulk-tensor loads:
//                a 5-D box {64 ch, Wt, Ht, Nt, 2 planes} of the activation view the tap reads -- the
//                tap shift is just a coordinate offset and the zero padding of the convolution is
//                TMA's out-of-bounds fill -- and a 3-D box {64 ch, BN, 2 planes} of the tap's weights.
//                Both land in the 128B-swizzled K-major layout wgmma consumes; no im2col buffer
//                ever exists in HBM or shared memory.
//   warps 0..7 : two consumer warpgroups, one per 64-row half of the tile.  fp32 fidelity from bf16 tensor
//                cores: per K=16 slice   main  += A_hi * B_hi
//                                         cross += A_lo * B_hi ;  cross += A_hi * B_lo
//                in two separate register accumulators (the 2^-9-smaller cross terms get their own
//                accumulator so their rounding does not ride on the main sum's exponent).  After the last K
//                step cross is added into main and the sums go through a float32 staging tile in shared memory
//                (in float32 mode 32 columns at a time, in four rounds), and the same eight warps run the epilogue
//                one pixel row per thread: BatchNorm scale/shift + activation (or backward scale * ReLU-mask),
//                re-split to bf16 hi/lo planes and store NHWC at the phase's output stride; or store raw sums to
//                this K split's workspace slab.  Plain whole tiles in float32 mode (g.epi_tma) skip the float32
//                staging: the epilogue runs on the accumulator fragments and each round leaves through TMA stores
//                that drain while the next tile's MMAs run.
// Pipeline: STAGES-deep smem ring with full/empty mbarriers (TMA -> wgmma -> release after wgmma.wait_group); the
// producer runs ahead across work items, so the next tile's operands load while the epilogue of this one runs.
#include <cuda.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "tapgemm.h"
#include "tc_ptx.cuh"

namespace ian {

struct TcMaps {
  CUtensorMap a[4];     // activation views, box = {64 ch, Wt, Ht, Nt, 2 planes}   (3-pass float32-split mode)
  CUtensorMap b;        // weights, box = {64 ch, BN, 2 planes}
  CUtensorMap a1[4];    // same tensors, hi plane only (single-pass bf16 mode)
  CUtensorMap b1;
  // the output's hi and lo planes as 5-D views {C, pw, Wq, ph, N*Hq} (the TMA-store epilogue), box {32 ch, 1, Wt, 1, Ht*Nt};
  // built for o_out / o_plane only, so a launch whose `out` differs keeps the thread-store epilogue
  CUtensorMap o[2];
  const __nv_bfloat16* o_out;
  long long o_plane;
  int Wt, Ht, Nt, BN;
  mutable int sk_choice;   // cached stream-K decision of launch_tapgemm_tc: -1 unknown, 0 whole tiles, 1 stream-K
};

namespace {

using namespace tc;

constexpr int BM = 128;
constexpr int BK = 64;

constexpr int kEpiWarps = 8;                 // the two consumer warpgroups
constexpr int kThreadsCta = 32 * kEpiWarps + 32;

// PASSES = 3: float32 fidelity, operands are bf16 hi|lo planes, 3 MMAs per K slice, main|cross accumulators.
// PASSES = 1: plain bf16 (BASELINE configs[2]): hi planes only, 1 MMA per K slice, one accumulator.
// BN <= 128: a warpgroup holds 64 x BN float32 accumulators (BN / 2 registers per thread, twice that in float32 mode).
template <int BN, int PASSES> struct TcCfg {
  static constexpr int kPlanes = PASSES == 3 ? 2 : 1;
  static constexpr int kATileBytes = BM * BK * 2 * kPlanes;
  static constexpr int kBTileBytes = BN * BK * 2 * kPlanes;
  static constexpr int kStageBytes = kATileBytes + kBTileBytes;
  // accumulator columns staged per epilogue round.  Float32 mode stages 32 at a time (a 20 KB tile instead of 68 KB) so
  // that a third 64 KB operand stage fits; bf16 mode's 32 KB stages fit four deep next to a whole-tile round, and its
  // short K loops would feel the extra barriers of more rounds.
  static constexpr int kRound = (PASSES == 3 && BN > 32) ? 32 : BN;
  static constexpr int kRounds = BN / kRound;
  static constexpr int kLd = kRound + 8;                       // staging row pitch in floats (conflict-free fragment stores)
  // float32 mode at BN = 128 may write plain tiles with TMA stores straight from the accumulators (g.epi_tma): one
  // round's 32 columns as bf16 hi|lo tiles of BM rows x 64 B (64B-swizzled), double-buffered so that a round's
  // stores drain while the next round (or the next tile's K loop) runs.  The float32 staging tile of the other
  // epilogues aliases the two buffers.
  static constexpr bool kTmaEpi = PASSES == 3 && BN == 128;
  static constexpr int kOutPlaneBytes = BM * kRound * 2;
  static constexpr int kOutRoundBytes = 2 * kOutPlaneBytes;
  static constexpr int kStagingBytes = kTmaEpi && 2 * kOutRoundBytes > BM * kLd * 4 ? 2 * kOutRoundBytes : BM * kLd * 4;
  // scale|shift of the tile's columns: one copy per CTA where the TMA-store buffers need the room, else one per warp
  static constexpr int kStageSmem = kTmaEpi ? 1024 : kEpiWarps * 1024;
  static constexpr int kStagesFit = (232448 - 1024 - 256 - kStagingBytes - kStageSmem) / kStageBytes;
  static constexpr int kStages = kStagesFit > 6 ? 6 : kStagesFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/ + kStageSmem + kStagingBytes;
  static_assert(kStages >= 2 && kSmemBytes <= 232448, "tapgemm_tc: shared memory budget");
};
// float32 mode at BN = 128 runs the heavy layers: one K step's 64 KB load must not be the only one in flight, and the
// TMA-store buffers take their own 32 KB next to the three stages: 3 * 65536 + 32768 + 1024 + 1024 + 256
static_assert(TcCfg<128, 3>::kStages == 3 && TcCfg<128, 3>::kSmemBytes == 231680, "tapgemm_tc: three float32-mode stages");
static_assert(TcCfg<128, 3>::kRound == 32 && TcCfg<128, 3>::kOutRoundBytes == 16384, "tapgemm_tc: 32-column TMA-store rounds");

// ---------------------------------------------------------------- kernel
// Persistent, warp-specialised.  Work items w = blockIdx.x + i*gridDim.x over
// (phase | k-split | m-tile | n-tile), longest phases first.  The n-tiles of one m-tile are neighbouring work items, so
// they run at the same time on neighbouring CTAs and read the same activation boxes: HBM delivers each box once and L2
// serves the rest.  (With m-tiles innermost, a layer whose input outgrows L2 -- enc_conv2 reads 134 MB at batch 256 --
// fetches its activations from HBM once per n-tile.)  The order does not change any sum.  The smem ring runs ACROSS
// work items: the producer prefetches the next tile's operands while the consumers run the epilogue of the current one.
struct WorkItem {
  int phase, ks, co0, it0, it1;
  int n0, p0, q0, mtile;
  // stream-K (SK): 0 = the segment is a whole tile; 1 = contributor (a later part of a tile: raw sums go to this
  // CTA's workspace slot); 2 = finisher (the first part of a tile cut by a CTA boundary: adds the partial sums of
  // CTAs blockIdx.x+1 .. sk_last, then runs the epilogue)
  int sk_role, sk_last;
};

// CH float32 values -> bf16 hi|lo planes (hi only in single-pass mode), packed bf16x2 conversions, 32-byte sector stores
template <int CH, int PASSES>
__device__ __forceinline__ void store_split(__nv_bfloat16* dst, long long plane, const float (&v)[CH]) {
  __align__(16) __nv_bfloat162 hi[CH / 2], lo[CH / 2];
#pragma unroll
  for (int j = 0; j < CH / 2; ++j) {
    hi[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
    if (PASSES == 3) {
      const float2 hf = __bfloat1622float2(hi[j]);
      lo[j] = __floats2bfloat162_rn(v[2 * j] - hf.x, v[2 * j + 1] - hf.y);
    }
  }
  static_assert(CH % 16 == 0, "an epilogue chunk is a whole number of 32-byte sectors per plane");
  const uint4* h4 = reinterpret_cast<const uint4*>(hi);
  const uint4* l4 = reinterpret_cast<const uint4*>(lo);
#pragma unroll
  for (int j = 0; j < CH / 16; ++j) {                    // dst is 32-byte aligned: channel offsets are multiples of CH >= 16
    tc::st_global_256(dst + 16 * j, h4[2 * j], h4[2 * j + 1]);
    if (PASSES == 3) tc::st_global_256(dst + plane + 16 * j, l4[2 * j], l4[2 * j + 1]);
  }
}

template <int BN>
__device__ __forceinline__ WorkItem decode_work(const TapGemm& g, const TcMaps& maps, int w) {
  WorkItem wi;
  const int tiles_q = g.Wg / maps.Wt, tiles_p = g.Hg / maps.Ht;
  const int tiles_m = tiles_q * tiles_p * ((g.n_img + maps.Nt - 1) / maps.Nt);
  const int tiles_n = g.Cout / BN;
  const int per_phase = tiles_m * tiles_n * g.ksplit;
  wi.phase = w / per_phase;
  int r = w % per_phase;
  const int nt = r % tiles_n; r /= tiles_n;
  int mt = r % tiles_m; r /= tiles_m;
  wi.ks = r;
  wi.mtile = mt;
  const int qb = mt % tiles_q; mt /= tiles_q;
  const int pb = mt % tiles_p; mt /= tiles_p;
  wi.n0 = mt * maps.Nt; wi.p0 = pb * maps.Ht; wi.q0 = qb * maps.Wt;
  wi.co0 = nt * BN;
  const int total_it = g.phase[wi.phase].ntaps * (g.Cin / BK);
  wi.it0 = (int)((long long)total_it * wi.ks / g.ksplit);
  wi.it1 = (int)((long long)total_it * (wi.ks + 1) / g.ksplit);
  return wi;
}

// Work iteration of one CTA.  SK = false: whole tiles, w = blockIdx.x + i*gridDim.x (longest phases first).
// SK = true (stream-K): the launch is ONE linear space of T K-steps over (phase | n-tile | m-tile | K step) and CTA c
// owns steps [T*c/G, T*(c+1)/G): every SM gets the same tensor work however the tile count divides by the SM count and
// however unequal the phases are.  A tile cut by a CTA boundary is finished by the CTA holding its FIRST K steps
// (which it reaches at the END of its range), after the CTAs holding the later steps (which they run FIRST) have
// published their raw partial sums -- an ordered, atomic-free, deterministic fix-up.
template <int BN, bool SK>
struct WorkIter {
  int w, total, stride;                 // !SK
  int T, G, cur, end, iters[kMaxPhases], tiles_per_phase, tiles_m, tiles_q, tiles_p;   // SK
  __device__ __forceinline__ int boundary(int c) const { return (int)((long long)T * c / G); }
  __device__ __forceinline__ int owner(int gi) const {
    int c = (int)((long long)gi * G / T);
    while (c + 1 < G && boundary(c + 1) <= gi) ++c;
    while (c > 0 && boundary(c) > gi) --c;
    return c;
  }
  __device__ __forceinline__ void init(const TapGemm& g, const TcMaps& maps, int total_work) {
    if (!SK) { w = blockIdx.x; total = total_work; stride = gridDim.x; return; }
    T = total_work; G = gridDim.x;
    tiles_q = g.Wg / maps.Wt; tiles_p = g.Hg / maps.Ht;
    tiles_m = tiles_q * tiles_p * ((g.n_img + maps.Nt - 1) / maps.Nt);
    tiles_per_phase = tiles_m * (g.Cout / BN);
    for (int p = 0; p < kMaxPhases; ++p) iters[p] = p < g.nphase ? g.phase[p].ntaps * (g.Cin / BK) : 0;
    cur = boundary(blockIdx.x); end = boundary(blockIdx.x + 1);
  }
  __device__ __forceinline__ bool next(const TapGemm& g, const TcMaps& maps, WorkItem& wi) {
    if (!SK) {
      if (w >= total) return false;
      wi = decode_work<BN>(g, maps, w);
      wi.sk_role = 0; wi.sk_last = 0;
      w += stride;
      return true;
    }
    if (cur >= end) return false;
    int gi = cur, ph = 0, phase_start = 0;
    while (ph + 1 < g.nphase && gi >= phase_start + tiles_per_phase * iters[ph]) { phase_start += tiles_per_phase * iters[ph]; ++ph; }
    const int ip = iters[ph];
    const int tile = (gi - phase_start) / ip, it = (gi - phase_start) % ip;
    int len = ip - it;
    if (len > end - gi) len = end - gi;
    wi.phase = ph; wi.ks = 0; wi.it0 = it; wi.it1 = it + len;
    int mt = tile % tiles_m;
    const int nt = tile / tiles_m;
    wi.mtile = mt;
    const int qb = mt % tiles_q; mt /= tiles_q;
    const int pb = mt % tiles_p; mt /= tiles_p;
    wi.n0 = mt * maps.Nt; wi.p0 = pb * maps.Ht; wi.q0 = qb * maps.Wt; wi.co0 = nt * BN;
    wi.sk_role = it > 0 ? 1 : (len < ip ? 2 : 0);
    wi.sk_last = wi.sk_role == 2 ? owner(phase_start + tile * ip + ip - 1) : 0;
    cur = gi + len;
    return true;
  }
};

template <int BN, int PASSES, bool SK>
__global__ void __launch_bounds__(kThreadsCta, 1)
tapgemm_tc_kernel(const __grid_constant__ TapGemm g, const __grid_constant__ TcMaps maps, const int total_work) {
  using Cfg = TcCfg<BN, PASSES>;
  constexpr int kATileBytes = Cfg::kATileBytes;
  constexpr int S = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t stg_base = smem_base + S * Cfg::kStageBytes;   // epilogue staging, 1024-aligned (swizzled TMA-store tiles)
  const uint32_t bar_base = stg_base + Cfg::kStagingBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };
  const uint32_t stage_smem = bar_base + 256u;       // scale|shift of the tile's columns: (1 or 8) x (128 + 128) floats
  uint8_t* smem_al = smem_raw + (smem_base - smem_u32(smem_raw));
  float* stage_ptr = reinterpret_cast<float*>(smem_al + (stage_smem - smem_base));
  float* acc_tile = reinterpret_cast<float*>(smem_al + (stg_base - smem_base));   // [BM][kLd] float32 round staging

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    pdl_trigger();                                      // the next kernel of the chain may move in as this grid's CTAs retire
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);                       // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                                           // prologue done; everything below reads / writes activations (tapgemm.h: PDL)

  if (warp == kEpiWarps) {
    // ===================== TMA producer (whole warp in uniform control flow, one elected lane issues) =====================
    uint32_t i = 0;                                     // running K-step counter across work items
    WorkIter<BN, SK> iter;
    iter.init(g, maps, total_work);
    WorkItem wi;
    while (iter.next(g, maps, wi)) {
      const Phase ph = g.phase[wi.phase];
      // K order is chunk-major: step it = channel chunk it / ntaps of tap it % ntaps, so consecutive steps read the same
      // 64 channels of (almost) the same pixels, which stay hot in L2 across the taps of a chunk
      int t = wi.it0 % ph.ntaps, c0 = wi.it0 / ph.ntaps * BK;
      for (int it = wi.it0; it < wi.it1; ++it, ++i) {
        const int s = i % S;
        const uint32_t par = (i / S) & 1u;
        const Tap tap = g.taps[ph.tap_begin + t];
        mbar_wait(empty_bar(s), par ^ 1u);
        const uint32_t sa = smem_base + s * Cfg::kStageBytes;
        if (elect_one_sync()) {
          mbar_expect_tx(full_bar(s), Cfg::kStageBytes);
          tma_load_5d(PASSES == 3 ? &maps.a[tap.view] : &maps.a1[tap.view], full_bar(s), sa, c0, wi.q0 + tap.dw,
                      wi.p0 + tap.dh, wi.n0, 0);
          tma_load_3d(PASSES == 3 ? &maps.b : &maps.b1, full_bar(s), sa + kATileBytes, c0, tap.wtile * g.Cout + wi.co0, 0);
        }
        __syncwarp();
        if (++t == ph.ntaps) { t = 0; c0 += BK; }
      }
    }
    return;
  }

  // ===================== consumers (warps 0..7): wgmma main loop, then the epilogue =====================
  constexpr int R = BN / 2;                             // accumulator registers per thread and accumulator
  constexpr int RW = Cfg::kRound;                     // tile columns per staging round
  constexpr int TC = RW >= 32 ? RW / 2 : RW;          // columns per thread and round (BN = 16: all 16, on warps 0-3 only)
  constexpr int CH = TC >= 32 ? 32 : 16;              // columns per epilogue chunk: whole 32-byte sectors per plane
  constexpr int kThreadCols = Cfg::kRounds * TC;      // columns per thread and tile (its stream-K slot)
  const int wg = warp >> 2, wtid = threadIdx.x & 127;
  const int ew = warp;
  const int lg = warp & 3;                              // 32-row group of the tile this warp's epilogue handles
  const int half = ew >> 2;                           // which half of a round's columns
  const bool has_cols = RW >= 32 || half == 0;
  float* my_stage = stage_ptr + (Cfg::kTmaEpi ? 0 : ew * 256);   // [0,128): scale, [128,256): shift of the tile's columns
  // activation as a branch-free a*t + b*|t| (none / LeakyRectify(0.2) / rectify; lasagne forms, SURVEY C.5)
  const float act_a = g.act == ACT_LRELU ? 0.6f : g.act == ACT_RELU ? 0.5f : 1.f;
  const float act_b = g.act == ACT_LRELU ? 0.4f : g.act == ACT_RELU ? 0.5f : 0.f;
  const int ml = lg * 32 + lane;                        // tile row of this thread's epilogue
  const int wl0 = ml % maps.Wt;
  const int hl0 = (ml / maps.Wt) % maps.Ht;
  const int nl0 = ml / (maps.Wt * maps.Ht);
  uint32_t i = 0;
  WorkIter<BN, SK> iter;
  iter.init(g, maps, total_work);
  WorkItem wi;
  while (iter.next(g, maps, wi)) {
    const Phase ph = g.phase[wi.phase];
    if (wi.it1 <= wi.it0) continue;                     // (uniform over the CTA)
    if (g.scale_pix_stride == 0) {                      // stage this tile's per-channel scale/shift while the MMAs run
      if constexpr (Cfg::kTmaEpi) {
        // one copy per CTA: every consumer warp has finished the previous tile's epilogue, which reads it; the first
        // barrier of this tile's epilogue publishes the new values
        asm volatile("bar.sync 1, 256;" ::: "memory");
        for (int c = threadIdx.x; c < BN; c += 32 * kEpiWarps) {
          my_stage[c] = g.scale ? __ldg(g.scale + wi.co0 + c) : 1.f;
          my_stage[128 + c] = g.shift ? __ldg(g.shift + wi.co0 + c) : 0.f;
        }
      } else if (has_cols) {
        __syncwarp();
        for (int c = lane; c < BN; c += 32) {
          my_stage[c] = g.scale ? __ldg(g.scale + wi.co0 + c) : 1.f;
          my_stage[128 + c] = g.shift ? __ldg(g.shift + wi.co0 + c) : 0.f;
        }
        __syncwarp();
      }
    }
    // ---- main loop: this warpgroup's 64 rows x BN columns (declared per tile: dead during the epilogue)
    float acc_m[R], acc_c[PASSES == 3 ? R : 1];
#pragma unroll
    for (int j = 0; j < R; ++j) acc_m[j] = 0.f;
#pragma unroll
    for (int j = 0; j < (PASSES == 3 ? R : 1); ++j) acc_c[j] = 0.f;
    wgmma_fence_regs(acc_m);
    if (PASSES == 3) wgmma_fence_regs(acc_c);
    for (int it = wi.it0; it < wi.it1; ++it, ++i) {
      const int s = i % S;
      mbar_wait(full_bar(s), (i / S) & 1u);
      const uint32_t sa = smem_base + s * Cfg::kStageBytes;
      const uint64_t a_hi = make_sw128_desc(sa + wg * 64 * 128), a_lo = make_sw128_desc(sa + BM * BK * 2 + wg * 64 * 128);
      const uint64_t b_hi = make_sw128_desc(sa + kATileBytes), b_lo = make_sw128_desc(sa + kATileBytes + BN * BK * 2);
      const uint32_t first = (it == wi.it0) ? 0u : 1u;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t ko = (uint64_t)(k * 2);         // 32 bytes per K=16 slice, in 16-byte units
        const uint32_t acc = k > 0 ? 1u : first;
        wgmma_bf16<BN>(acc_m, a_hi + ko, b_hi + ko, acc);
        if constexpr (PASSES == 3) {
          wgmma_bf16<BN>(acc_c, a_lo + ko, b_hi + ko, acc);
          wgmma_bf16<BN>(acc_c, a_hi + ko, b_lo + ko, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                                  // the previous K step's MMAs have retired: free its stage
      if (it > wi.it0 && wtid == 0) mbar_arrive(empty_bar((i - 1) % S));
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc_m);
    if (PASSES == 3) wgmma_fence_regs(acc_c);
    if (wtid == 0) mbar_arrive(empty_bar((i - 1) % S));
    if constexpr (PASSES == 3) {
#pragma unroll
      for (int j = 0; j < R; ++j) acc_m[j] += acc_c[j];   // main + cross: the one float32 add of every output
    }
    // ===================== TMA-store epilogue (plain whole tiles, float32 mode) =====================
    // The same float operations per element as the thread-store epilogue below, run on the accumulator fragments; each
    // 32-column round is written as bf16 hi|lo into a swizzled staging buffer and leaves through two TMA stores issued by
    // thread 0.  Nothing waits for those stores here: the warps go on to the next tile and its K loop hides them.
    // Hazards: (1) a buffer is rewritten only after thread 0's cp.async.bulk.wait_group.read has seen the stores that
    // read it (round r-2, possibly of the previous tile) and a barrier has passed that on; (2) the generic epilogue's
    // float32 staging aliases the buffers and waits for every outstanding store first; (3) thread 0 waits for all its
    // stores to complete before the CTA exits (shared memory must outlive them, and the next kernel's
    // griddepcontrol.wait relies on this grid's writes being done); (4) the choice is uniform over the CTA.
    if constexpr (Cfg::kTmaEpi) {
      if (g.epi_tma && wi.sk_role == 0) {
#pragma unroll
        for (int r = 0; r < Cfg::kRounds; ++r) {
          const uint32_t buf = stg_base + (uint32_t)(r & 1) * Cfg::kOutRoundBytes;
          if (threadIdx.x == 0) bulk_wait_group_read1();   // (1): every group but the newest (round r-1) has been read
          asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
          for (int j = 0; j < RW / 2; j += 2) {         // registers [r*RW/2, (r+1)*RW/2) hold this round's columns
            const float2 a = make_float2(acc_m[r * RW / 2 + j], acc_m[r * RW / 2 + j + 1]);
            const int row = wg * 64 + frag_row(wtid, j);
            const int c = frag_col(wtid, j);            // column inside the round (even)
            const float2 sc = *reinterpret_cast<const float2*>(my_stage + r * RW + c);
            const float2 sf = *reinterpret_cast<const float2*>(my_stage + 128 + r * RW + c);
            float v0 = fmaf(a.x, sc.x, sf.x), v1 = fmaf(a.y, sc.y, sf.y);
            if (g.act == ACT_ELU) {
              v0 = v0 > 0.f ? v0 : expm1f(v0);
              v1 = v1 > 0.f ? v1 : expm1f(v1);
            } else if (g.act != ACT_NONE) {
              v0 = fmaf(act_b, fabsf(v0), act_a * v0);
              v1 = fmaf(act_b, fabsf(v1), act_a * v1);
            }
            const __nv_bfloat162 hi = __floats2bfloat162_rn(v0, v1);
            const float2 hf = __bfloat1622float2(hi);
            const __nv_bfloat162 lo = __floats2bfloat162_rn(v0 - hf.x, v1 - hf.y);
            // 64-byte rows, 64B swizzle: 16-byte unit c/8 of row `row` sits at unit (c/8) ^ ((row/2) % 4)
            const uint32_t off = (uint32_t)row * 64u + ((((uint32_t)c >> 3) ^ (((uint32_t)row >> 1) & 3u)) << 4) + ((uint32_t)c & 7u) * 2u;
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(buf + off), "r"(*reinterpret_cast<const uint32_t*>(&hi)) : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(buf + Cfg::kOutPlaneBytes + off), "r"(*reinterpret_cast<const uint32_t*>(&lo))
                         : "memory");
          }
          fence_proxy_async_smem();                     // generic-proxy writes -> visible to the TMA store
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (threadIdx.x == 0) {
            // rows of an image n >= n_img fall outside the map's N*Hq extent and are not written
            const int c4 = wi.n0 * g.Hg + wi.p0;
            tma_store_5d(&maps.o[0], buf, wi.co0 + r * RW, ph.ow0, wi.q0, ph.oh0, c4);
            tma_store_5d(&maps.o[1], buf + Cfg::kOutPlaneBytes, wi.co0 + r * RW, ph.ow0, wi.q0, ph.oh0, c4);
            bulk_commit_group();
          }
        }
        continue;
      }
      if (threadIdx.x == 0) bulk_wait_group_read0();   // (2): the float32 staging below overwrites the store buffers
    }
    // ===================== epilogue =====================
    if (SK && wi.sk_role == 2 && has_cols) {          // finisher: the later parts were computed first; wait for them
      for (int k = (int)blockIdx.x + 1 + lane; k <= wi.sk_last; k += 32) {
        if (iter.boundary(k) == iter.boundary(k + 1)) continue;   // a CTA without K steps (T < G) publishes nothing
        const int* fl = g.sk_flags + k * kEpiWarps + ew;
        const long long t0 = clock64();
        int fv;
        do {
          asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(fv) : "l"(fl) : "memory");
          if (clock64() - t0 > 4000000000LL) __trap();
        } while (fv != g.sk_epoch);
      }
      __syncwarp();
    }
    // the row's (n, p, q) offsets in the tile; the stream-K float32 form derives them here from a fresh %tid.x rather
    // than keeping them live across the main loop, whose 128 accumulator registers leave no room for them there
    int nl = nl0, hl = hl0, wl = wl0;
    if constexpr (SK && Cfg::kTmaEpi) {
      uint32_t tid;
      asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tid));
      const int row = (int)((tid >> 5) & 3u) * 32 + (int)(tid & 31u);
      wl = row % maps.Wt;
      hl = (row / maps.Wt) % maps.Ht;
      nl = row / (maps.Wt * maps.Ht);
    }
    const int n = wi.n0 + nl, p = wi.p0 + hl, q = wi.q0 + wl;
    const bool valid = n < g.n_img;
    const int oh = p * g.osh + ph.oh0, ow = q * g.osw + ph.ow0;
    const long long pix = (long long)(n * g.Hout + oh) * g.Wout + ow;
    // the sums leave through a BM x RW staging tile, RW columns per round (row-per-thread access for the epilogue)
#pragma unroll 1
    for (int r = 0; r < Cfg::kRounds; ++r) {
      asm volatile("bar.sync 1, 256;" ::: "memory");  // every warp has read the staging tile of the previous round
#pragma unroll
      for (int j = 0; j < RW / 2; j += 2) {           // registers [r*RW/2, (r+1)*RW/2) hold this round's columns
        float2 v = make_float2(acc_m[j], acc_m[j + 1]);
#pragma unroll
        for (int rr = 1; rr < Cfg::kRounds; ++rr)
          if (rr == r) v = make_float2(acc_m[rr * RW / 2 + j], acc_m[rr * RW / 2 + j + 1]);
        *reinterpret_cast<float2*>(acc_tile + (wg * 64 + frag_row(wtid, j)) * Cfg::kLd + frag_col(wtid, j)) = v;
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (!has_cols) continue;
#pragma unroll 1
      for (int cc = 0; cc < TC; cc += CH) {
        const int cb = r * RW + half * TC + cc;         // tile column of this chunk's first channel
        const int co = wi.co0 + cb;
        const int cs = r * TC + cc;                     // offset in this thread's stream-K slot
        float v[CH];
        const float* srow = acc_tile + ml * Cfg::kLd + half * TC + cc;
#pragma unroll
        for (int j = 0; j < CH / 4; ++j) {
          const float4 t4 = *reinterpret_cast<const float4*>(srow + 4 * j);
          v[4 * j] = t4.x; v[4 * j + 1] = t4.y; v[4 * j + 2] = t4.z; v[4 * j + 3] = t4.w;
        }
        if (SK && wi.sk_role == 1) {                   // contributor: raw partial sums -> this CTA's workspace slot
          float4* wp = reinterpret_cast<float4*>(g.sk_ws + (((long long)blockIdx.x * kEpiWarps + ew) * 32 + lane) * kThreadCols + cs);
#pragma unroll
          for (int j = 0; j < CH / 4; ++j) __stcg(wp + j, make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]));
          continue;
        }
        if (SK && wi.sk_role == 2) {                   // finisher: add the later parts, in CTA order
          for (int k = (int)blockIdx.x + 1; k <= wi.sk_last; ++k) {
            if (iter.boundary(k) == iter.boundary(k + 1)) continue;
            const float4* rp = reinterpret_cast<const float4*>(g.sk_ws + (((long long)k * kEpiWarps + ew) * 32 + lane) * kThreadCols + cs);
#pragma unroll
            for (int j = 0; j < CH / 4; ++j) {
              const float4 a = __ldcg(rp + j);
              v[4 * j] += a.x; v[4 * j + 1] += a.y; v[4 * j + 2] += a.z; v[4 * j + 3] += a.w;
            }
          }
        }
        if (g.ksplit > 1) {
          if (valid) {                                  // this K split's slab; the finalize kernel adds them in order
            float4* wsp = reinterpret_cast<float4*>(g.ws + (long long)wi.ks * g.ws_slab + pix * g.Cout + co);
#pragma unroll
            for (int j = 0; j < CH / 4; ++j) __stcg(wsp + j, make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]));
          }
          continue;
        }
        if (valid) {
          const long long off = pix * g.Cout + co;
          if (g.out_raw) store_split<CH, PASSES>(g.out_raw + off, g.out_raw_plane, v);   // pre-BN value (MDBLOCK residual input)
          if (g.res && !g.res_after) {                                   // residual add before BatchNorm (MDBLOCK, layers.py:411-416)
            const uint4* rh = reinterpret_cast<const uint4*>(g.res + off);
            const uint4* rl = reinterpret_cast<const uint4*>(g.res + g.res_plane + off);
#pragma unroll
            for (int j8 = 0; j8 < CH / 8; ++j8) {
              const uint4 h4 = __ldg(rh + j8);
              const __nv_bfloat16* hb = reinterpret_cast<const __nv_bfloat16*>(&h4);
              if (PASSES == 3) {
                const uint4 l4 = __ldg(rl + j8);
                const __nv_bfloat16* lb = reinterpret_cast<const __nv_bfloat16*>(&l4);
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j8 * 8 + j] += __bfloat162float(hb[j]) + __bfloat162float(lb[j]);
              } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j8 * 8 + j] += __bfloat162float(hb[j]);
              }
            }
          }
          if (g.act == ACT_MASK) {
            const int si = co + (oh * g.Wout + ow) * g.scale_pix_stride;
            const uint4* mk = reinterpret_cast<const uint4*>(g.mask + off);
#pragma unroll
            for (int j8 = 0; j8 < CH / 8; ++j8) {
              const uint4 m4 = __ldg(mk + j8);
              const __nv_bfloat16* mb = reinterpret_cast<const __nv_bfloat16*>(&m4);
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float sc = g.scale_pix_stride ? __ldg(g.scale + si + j8 * 8 + j) : my_stage[cb + j8 * 8 + j];
                v[j8 * 8 + j] = v[j8 * 8 + j] * sc * (__bfloat162float(mb[j]) > 0.f ? 1.f : g.mask_slope);
              }
            }
            if (g.res && g.res_after) {                  // gradient of the block's residual branch joins after the mask/scale
              const uint4* rh = reinterpret_cast<const uint4*>(g.res + off);
              const uint4* rl = reinterpret_cast<const uint4*>(g.res + g.res_plane + off);
#pragma unroll
              for (int j8 = 0; j8 < CH / 8; ++j8) {
                const uint4 h4 = __ldg(rh + j8);
                const __nv_bfloat16* hb = reinterpret_cast<const __nv_bfloat16*>(&h4);
                if (PASSES == 3) {
                  const uint4 l4 = __ldg(rl + j8);
                  const __nv_bfloat16* lb = reinterpret_cast<const __nv_bfloat16*>(&l4);
#pragma unroll
                  for (int j = 0; j < 8; ++j) v[j8 * 8 + j] += __bfloat162float(hb[j]) + __bfloat162float(lb[j]);
                } else {
#pragma unroll
                  for (int j = 0; j < 8; ++j) v[j8 * 8 + j] += __bfloat162float(hb[j]);
                }
              }
            }
          } else {
#pragma unroll
            for (int j4 = 0; j4 < CH / 4; ++j4) {
              const float4 sc = *reinterpret_cast<const float4*>(my_stage + cb + 4 * j4);
              const float4 sf = *reinterpret_cast<const float4*>(my_stage + 128 + cb + 4 * j4);
              v[4 * j4 + 0] = fmaf(v[4 * j4 + 0], sc.x, sf.x);
              v[4 * j4 + 1] = fmaf(v[4 * j4 + 1], sc.y, sf.y);
              v[4 * j4 + 2] = fmaf(v[4 * j4 + 2], sc.z, sf.z);
              v[4 * j4 + 3] = fmaf(v[4 * j4 + 3], sc.w, sf.w);
            }
            if (g.act == ACT_ELU) {
#pragma unroll
              for (int j = 0; j < CH; ++j) v[j] = v[j] > 0.f ? v[j] : expm1f(v[j]);
            } else if (g.act != ACT_NONE) {
#pragma unroll
              for (int j = 0; j < CH; ++j) v[j] = fmaf(act_b, fabsf(v[j]), act_a * v[j]);
            }
          }
          if (g.out) store_split<CH, PASSES>(g.out + off, g.out_plane, v);
          if (g.out_f32_t) {                         // tile-blocked channel-major table: [m-tile][co][128 rows]
            const long long tbase = ((long long)wi.mtile * g.cout_real + co) * BM + ml;
            if (g.out_t_bf16) {
              __nv_bfloat16* ot = reinterpret_cast<__nv_bfloat16*>(g.out_f32_t) + tbase;
#pragma unroll
              for (int j = 0; j < CH; ++j)
                if (co + j < g.cout_real) ot[j * BM] = __float2bfloat16_rn(v[j]);   // a warp writes 64 contiguous bytes per column
            } else {
              float* ot = g.out_f32_t + tbase;
#pragma unroll
              for (int j = 0; j < CH; ++j)
                if (co + j < g.cout_real) ot[j * BM] = v[j];   // a warp writes 128 contiguous bytes per column
            }
          }
          if (g.out_f32) {
            float4* of = reinterpret_cast<float4*>(g.out_f32 + off);
#pragma unroll
            for (int j = 0; j < CH / 4; ++j) of[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
          }
        }
      }
    }
    if (SK && wi.sk_role == 1 && has_cols) {          // publish this warp's sub-block of partial sums
      __threadfence();
      __syncwarp();
      if (lane == 0) {
        int* fl = g.sk_flags + (int)blockIdx.x * kEpiWarps + ew;
        asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(fl), "r"(g.sk_epoch) : "memory");
      }
    }
  }
  if constexpr (Cfg::kTmaEpi) {
    if (threadIdx.x == 0) bulk_wait_group0();          // (3): every TMA-stored byte has landed before the CTA retires
  }
}

}  // namespace

TcMaps* tc_build_maps(const TapGemm& g, char* err, int errlen) {
  tc::EncodeTiledFn enc = tc::get_encode_fn();
  if (!enc) { snprintf(err, errlen, "cuTensorMapEncodeTiled entry point not available"); return nullptr; }
  if (g.Cin % 64 || (g.Cout % 128 && g.Cout != 16)) { snprintf(err, errlen, "tc path needs Cin%%64==0 and Cout%%128==0 or Cout==16 (got %d,%d)", g.Cin, g.Cout); return nullptr; }
  TcMaps* m = new TcMaps();
  memset(m, 0, sizeof(*m));
  tile_shape(g.Hg, g.Wg, m->Wt, m->Ht, m->Nt);
  m->sk_choice = -1;
  m->BN = (g.Cout % 128 == 0) ? 128 : 16;   // 128: the widest tile whose float32-mode accumulators fit a warpgroup's registers
  if (g.Wg % m->Wt || g.Hg % m->Ht || m->Wt * m->Ht * m->Nt != BM) {
    snprintf(err, errlen, "M grid %dx%d does not tile into 128-row boxes", g.Hg, g.Wg);
    delete m; return nullptr;
  }
  // which views are used
  bool used[4] = {false, false, false, false};
  int max_tile = 0;
  for (int p = 0; p < g.nphase; ++p)
    for (int t = 0; t < g.phase[p].ntaps; ++t) {
      const Tap& tp = g.taps[g.phase[p].tap_begin + t];
      used[tp.view] = true;
      if (tp.wtile > max_tile) max_tile = tp.wtile;
    }
  for (int v = 0; v < 4; ++v) {
    if (!used[v]) continue;
    const int vh = v >> 1, vw = v & 1;
    const cuuint64_t Hv = (g.Hin - vh + g.sh - 1) / g.sh, Wv = (g.Win - vw + g.sw - 1) / g.sw;
    cuuint64_t dims[5] = {(cuuint64_t)g.Cin, Wv, Hv, (cuuint64_t)g.n_img, 2};
    cuuint64_t strides[4] = {(cuuint64_t)g.sw * g.Cin * 2, (cuuint64_t)g.sh * g.Win * g.Cin * 2,
                             (cuuint64_t)g.Hin * g.Win * g.Cin * 2, (cuuint64_t)g.a_plane * 2};
    cuuint32_t box[5] = {BK, (cuuint32_t)m->Wt, (cuuint32_t)m->Ht, (cuuint32_t)m->Nt, 2};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    void* base = (void*)(g.a + ((long long)vh * g.Win + vw) * g.Cin);
    CUresult r = enc(&m->a[v], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(A view %d) failed: %d", v, (int)r); delete m; return nullptr; }
    box[4] = 1;
    r = enc(&m->a1[v], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(A1 view %d) failed: %d", v, (int)r); delete m; return nullptr; }
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)g.Cin, (cuuint64_t)(max_tile + 1) * g.Cout, 2};
    cuuint64_t strides[2] = {(cuuint64_t)g.Cin * 2, (cuuint64_t)g.b_plane * 2};
    cuuint32_t box[3] = {BK, (cuuint32_t)m->BN, 2};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&m->b, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)g.b, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(B) failed: %d", (int)r); delete m; return nullptr; }
    box[2] = 1;
    r = enc(&m->b1, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)g.b, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(B1) failed: %d", (int)r); delete m; return nullptr; }
  }
  // Output planes for the TMA-store epilogue, where a map can describe the output: output pixel
  // (n, p*os_h + oh0, q*os_w + ow0) of NHWC [n][Hout][Wout][C] is element (c, ow0, q, oh0, n*Hg + p) of the view
  // {C, os_w, Wg, os_h, N*Hg}.  H and N merge because stride(N) = Hg * stride(Hg); a tile's box {32, 1, Wt, 1, Ht*Nt} then
  // covers its rows in tile order, since Nt > 1 only when Ht = Hg.  One map per plane, so the rows n >= n_img of a
  // partial last m-tile are clipped at the N*Hg extent instead of landing in the other plane.
  if (g.out && m->BN == 128 && g.Hout == g.osh * g.Hg && g.Wout == g.osw * g.Wg && (g.out_plane * 2) % 16 == 0 &&
      (uintptr_t)g.out % 16 == 0) {
    const cuuint64_t C = (cuuint64_t)g.Cout;
    cuuint64_t dims[5] = {C, (cuuint64_t)g.osw, (cuuint64_t)g.Wg, (cuuint64_t)g.osh, (cuuint64_t)g.n_img * g.Hg};
    cuuint64_t strides[4] = {C * 2, C * 2 * g.osw, C * 2 * g.Wout, C * 2 * g.Wout * g.osh};
    cuuint32_t box[5] = {32, 1, (cuuint32_t)m->Wt, 1, (cuuint32_t)(m->Ht * m->Nt)};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    bool ok = true;
    for (int pl = 0; pl < 2 && ok; ++pl)
      ok = enc(&m->o[pl], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, (void*)(g.out + pl * g.out_plane), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    if (ok) { m->o_out = g.out; m->o_plane = g.out_plane; }   // otherwise this layer keeps the thread-store epilogue
  }
  return m;
}

void tc_free_maps(TcMaps* m) { delete m; }

int tc_tile_width(const TcMaps* maps) { return maps->BN; }

int tc_num_sms() {
  static std::atomic<int> num_sms[kMaxDevices];
  const int dev = cur_device();
  int n = num_sms[dev].load(std::memory_order_relaxed);
  if (!n) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    num_sms[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}
size_t tc_sk_workspace_floats() { return (size_t)tc_num_sms() * kEpiWarps * 32 * 128; }
size_t tc_sk_flag_ints() { return (size_t)tc_num_sms() * kEpiWarps; }

template <int BN, int PASSES, bool SK>
static int launch_one(const TapGemm& g, const TcMaps* maps, int tiles_m, int num_sms, cudaStream_t st) {
  using Cfg = TcCfg<BN, PASSES>;
  static DeviceOnce attr_set;
  const int dev = cur_device();
  if (!attr_set.is_done(dev)) {
    if (cudaFuncSetAttribute(tapgemm_tc_kernel<BN, PASSES, SK>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes) != cudaSuccess)
      return -1;
    attr_set.set_done(dev);
  }
  int total_work, grid;
  if (SK) {                                              // T K-steps, one CTA per SM, every CTA gets T/G of them
    long long T = 0;
    for (int p = 0; p < g.nphase; ++p) T += (long long)tiles_m * (g.Cout / maps->BN) * g.phase[p].ntaps * (g.Cin / BK);
    total_work = (int)T;
    grid = num_sms;
  } else {
    total_work = tiles_m * (g.Cout / maps->BN) * g.nphase * g.ksplit;
    grid = total_work < num_sms ? total_work : num_sms;
  }
  if (launch_pdl(tapgemm_tc_kernel<BN, PASSES, SK>, dim3(grid), dim3(kThreadsCta), Cfg::kSmemBytes, st, g, *maps, total_work) != cudaSuccess)
    return -1;
  return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_tapgemm_tc(const TapGemm& g_in, const TcMaps* maps, cudaStream_t st) {
  // TMA-store epilogue only for plain outputs: float32 mode, whole K, scale/shift + none/LReLU/ReLU/ELU into `out` and
  // nothing else, into the planes the output maps were built for.  Stream-K tiles cut by a CTA boundary, split-K slabs,
  // MDBLOCK, the backward mask and the head's tables keep the thread-store epilogue.
  TapGemm g = g_in;
  g.epi_tma = g_in.epi_tma && g.passes == 3 && maps->BN == 128 && g.ksplit == 1 && g.out && g.out == maps->o_out &&
              g.out_plane == maps->o_plane && g.scale_pix_stride == 0 &&
              (g.act == ACT_NONE || g.act == ACT_LRELU || g.act == ACT_RELU || g.act == ACT_ELU) && !g.out_raw && !g.res &&
              !g.mask && !g.out_f32 && !g.out_f32_t;
  const int num_sms = tc_num_sms();
  const int tiles_m = (g.Wg / maps->Wt) * (g.Hg / maps->Ht) * ((g.n_img + maps->Nt - 1) / maps->Nt);
  const long long tiles = (long long)tiles_m * (g.Cout / maps->BN) * g.nphase;
  // stream-K pays for one extra partial-sum round trip per cut tile, so it is used only where whole-tile scheduling
  // leaves >= 20 % of the SM-time idle (e.g. dec_conv1 of IAN_simple, whose 9/6/6/4-tap phases map badly onto the SMs).
  bool sk = false;
  if (g.sk_force) {
    sk = g.sk_ws && g.ksplit == 1 && maps->BN == 128 && !g.out_f32_t;
  } else if (maps->sk_choice >= 0) {
    sk = maps->sk_choice == 1 && g.sk_ws != nullptr;
  } else if (g.sk_ws && g.ksplit == 1 && maps->BN == 128 && tiles >= num_sms / 2 && !g.out_f32_t) {
    const int per_phase = tiles_m * (g.Cout / maps->BN);
    std::vector<long long> load(num_sms, 0);
    long long T = 0;
    for (long long w = 0; w < tiles; ++w) {              // the static schedule: tile w -> CTA w % G, phases in order
      const int it = g.phase[w / per_phase].ntaps * (g.Cin / BK);
      load[w % num_sms] += it;
      T += it;
    }
    long long makespan = 0;
    for (long long v : load) makespan = v > makespan ? v : makespan;
    sk = makespan * num_sms >= (T * 6) / 5;
    maps->sk_choice = sk ? 1 : 0;
  } else if (g.sk_ws) {
    maps->sk_choice = 0;
  }
  if (g.passes == 1) {
    if (maps->BN == 128) return sk ? launch_one<128, 1, true>(g, maps, tiles_m, num_sms, st) : launch_one<128, 1, false>(g, maps, tiles_m, num_sms, st);
    return launch_one<16, 1, false>(g, maps, tiles_m, num_sms, st);
  }
  if (maps->BN == 128) return sk ? launch_one<128, 3, true>(g, maps, tiles_m, num_sms, st) : launch_one<128, 3, false>(g, maps, tiles_m, num_sms, st);
  return launch_one<16, 3, false>(g, maps, tiles_m, num_sms, st);
}

}  // namespace ian
