// linear_tc_dw.cu — dW of the Linear op on wgmma (sm_90a), fed by TMA (3xTF32).
//
// Replaces cublasSgemm(OP_N, OP_T) of Linear::backward_task (linear_kernel.cu:220-224):
//     dW[o][i] += sum_v dY[v][o] * X[v][i]
//   M = i (X columns, tiles of 128), N = o (<= 256), K = v (vertices).  A CTA owns one M-tile and a
//   vertex range (split-K), so X streams through HBM once; the accumulator [128 x N] sits in the
//   registers of two consumer warpgroups.  Partials go to a workspace [splits][out][in]; a reduce
//   kernel adds them into dW in split order (deterministic).
//
// wgmma takes tf32 operands from shared memory only K-major, and both X and dY are vertex-major
// (MN-major for this product), so:
//   A = X^T comes from registers: each consumer thread reads its fragment straight from the TMA tile
//       (32-column boxes, 128-byte swizzle), applies the fused dropout mask and splits it hi / lo;
//   B = dY^T is transposed and split once per 32-vertex block by the consumers into two K-major tiles
//       [N][KS] (hi, lo; 128-byte swizzle) that the MMAs of every consumer warpgroup read.
//
// Both kernels below do that arithmetic with the same per-element MMA order (blocks in vertex order, k8 steps 0..3,
// then lo_x*hi_y, hi_x*lo_y, hi_x*hi_y), so every bit of dW is the same in both.  They share the per-block steps
// (DwLane, dw_transpose, dw_fragments, dw_store) and differ in their pipelines and in how they issue the MMAs.
//
// k_tc_linear_dw_ws (N <= 128, the default there): one TMA producer warp and 1 or 2 consumer warpgroups.
//   The producer fills a ring of stages (X boxes, the dY box and the [KS][4]-word box of the packed dropout
//   mask) on full / empty mbarriers.  Each consumer warpgroup waits for its stage, transposes its share of dY
//   into one of two or three dY^T buffers, reads its A fragments and mask words, releases the stage, waits for
//   the other warpgroup's share of the buffer (bfull) and issues the block's MMAs; `wgmma.wait_group 1` then
//   retires the previous block's, whose buffer is released (bempty).  No CTA-wide barrier, and the MMA queue
//   never drains inside the loop.  Each operand pair is one m64n(32 NC)k8 MMA over all N columns rather than NC
//   of n32 (an element's sums and their order are those of its n32 chunk).  With inDim <= 64 the tile is 64
//   columns and one warpgroup, so no MMA multiplies the zero fill past inDim.
// k_tc_linear_dw (N > 128, or ROC_B200_DW=sync): two consumer warpgroups of 64 X columns each and nothing
//   else: with the accumulator of up to 256 columns in registers a third (producer) warp would cap them at
//   168 registers.  Thread 0 refills a stage with TMA (X boxes + dY box) once both warpgroups are past it.
//   The dY^T tiles are double-buffered and the step is software-pipelined: while the MMAs of vertex block k
//   run, the consumers transpose block k + 1 into the other buffer and then read block k + 1's A fragments
//   into a second register set.  One CTA-wide barrier per block publishes the next dY^T buffer and certifies
//   that both warpgroups' MMAs of the previous block have retired (which frees that buffer and the ring
//   stage).
// A bf16 X (a leaf node tensor) takes the same two kernels with 64-byte X box rows and the 64-byte swizzle; each
// element is widened exactly as its fragment is read, so dW is the fp32 kernel's on X.float(), bit for bit.
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "tc_common.cuh"

namespace roc {

using namespace tc;

constexpr int DW_BM = 128;         // X columns per CTA (k_tc_linear_dw_ws: 64 when inDim <= 64)
constexpr int DW_KS = 32;          // vertices per stage = one 128-byte swizzle row of dY^T
constexpr int DW_XBOX = 32;        // X columns per TMA box = one 128-byte swizzle row
constexpr int DW_THREADS = 256;    // k_tc_linear_dw: two consumer warpgroups
constexpr int DW_MAX_STAGES = 4;
// dY^T buffers of k_tc_linear_dw_ws, chosen by measurement: two ran faster at N = 64, three at N = 128
__host__ __device__ constexpr int dw_ws_bufs(int NC) { return NC <= 2 ? 2 : 3; }
constexpr int DW_MASK_WORDS = 4;   // mask words per vertex in a stage (the 128 columns of a tile; 16-byte TMA rows)

struct TcDwParams {
  float* ws; int64_t rows; int inDim, outDim;
  int64_t vPerSplit;       // multiple of DW_KS
  int stages;
  const uint32_t* mask; int64_t ldm; float mscale;   // fused dropout of X (NULL = none)
};

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// Accumulator row 16 (w % 4) + g + 8 h of warpgroup w / 4, held by lane (g, t) of warp w (0..7), is X column
// dw_col(w, g, h) of the tile.  The permutation (any one gives the same sums: an accumulator row depends only on its
// own A row) puts the 32 lanes' A fragment reads of the swizzled X boxes on 32 distinct banks: within a warp the
// 16-byte chunk (col % 32) / 4 is 4 (g / 4) + 2 (w % 2) + h, so chunk ^ t (the swizzle of vertex row t) is distinct
// over (g / 4, t), and col % 4 = g % 4.  Both columns of a thread sit in one 32-column box, so in one mask word.
__device__ __forceinline__ int dw_col(int w, int g, int h) {
  return (w >> 1) * DW_XBOX + (g >> 2) * 16 + (w & 1) * 8 + h * 4 + (g & 3);
}

// What a consumer thread needs to find its A fragment: the element offsets of (vertex k = t + 4 e, column c) of k8
// step 0 in the swizzled X boxes, and the mask bits of its two columns.  fp32 X (TX = float, 128-byte swizzle):
// box(c) * 32 KS + k * 32 + ((c % 32 / 4) ^ k) * 4 + c % 4.  bf16 X (TX = uint16_t, rows of 64 bytes, 64-byte
// swizzle): box(c) * 32 KS + k * 32 + ((c % 32 / 8) ^ ((k / 2) % 4)) * 8 + c % 8.  Either swizzle term is the same
// for vertex k + 8 kk, so the k8 steps add 8 kk * 32 elements.
template <class TX>
struct DwLane {
  int ca, cb;       // X columns of this thread in the tile
  int xo[2][2];
  int mb0, mb1;
  __device__ __forceinline__ DwLane(int warp, int lane) {
    const int g = lane >> 2, t = lane & 3;
    ca = dw_col(warp, g, 0); cb = dw_col(warp, g, 1);
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int c = h ? cb : ca, k = t + 4 * e;
        if constexpr (sizeof(TX) == 4)
          xo[h][e] = (c / DW_XBOX) * (DW_KS * DW_XBOX) + k * DW_XBOX + ((((c % DW_XBOX) >> 2) ^ k) << 2) + (c & 3);
        else
          xo[h][e] = (c / DW_XBOX) * (DW_KS * DW_XBOX) + k * DW_XBOX + ((((c % DW_XBOX) >> 3) ^ ((k >> 1) & 3)) << 3) +
                     (c & 7);
      }
    mb0 = ca & 31; mb1 = cb & 31;
  }
};

// dY [KS][BN] -> dY^T hi / lo [BN][KS]; 128-byte swizzle: element (o, k) at o*32 + ((k/4 ^ o%8) * 4) + k%4.  Thread
// `tid` of CT takes 4 consecutive k of one o per item: 4 conflict-free loads, one 16-byte store per tile, and the 8
// lanes of a store phase (8 consecutive o) fill the 32 banks.
template <int NC, int CT>
__device__ __forceinline__ void dw_transpose(const float* ys, float* hiT, float* loT, int tid) {
  constexpr int BN = 32 * NC;
#pragma unroll
  for (int j = 0; j < (DW_KS / 4) * BN / CT; j++) {
    const int idx = tid + CT * j;
    const int q = idx / BN, o = idx - q * BN;
    uint32_t h[4], l[4];
#pragma unroll
    for (int r = 0; r < 4; r++) split_tf32(ys[(4 * q + r) * BN + o], h[r], l[r]);
    const int d = o * DW_KS + ((q ^ (o & 7)) << 2);
    *reinterpret_cast<uint4*>(hiT + d) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(loT + d) = make_uint4(l[0], l[1], l[2], l[3]);
  }
  fence_proxy_async_smem();
}

// A fragments (hi, lo) of every k8 step of the block whose X boxes start at xs; mw[2 kk + e] is the mask word of
// vertex 8 kk + 4 e + t (all ones without a mask).  A bf16 X is widened exactly as it is read.
template <class TX>
__device__ __forceinline__ void dw_fragments(const TX* xs, const DwLane<TX>& L, bool masked, float mscale,
                                             const uint32_t (&mw)[8], uint32_t (&fr)[DW_KS / 8][2][4]) {
#pragma unroll
  for (int kk = 0; kk < DW_KS / 8; kk++) {
    const int kb = kk * 8 * DW_XBOX;
    float x[4] = {to_f32(xs[kb + L.xo[0][0]]), to_f32(xs[kb + L.xo[1][0]]), to_f32(xs[kb + L.xo[0][1]]),
                  to_f32(xs[kb + L.xo[1][1]])};
    if (masked) {
      const uint32_t m0 = mw[2 * kk], m1 = mw[2 * kk + 1];
      x[0] = ((m0 >> L.mb0) & 1u) ? x[0] * mscale : 0.f;   // == k_dropout
      x[1] = ((m0 >> L.mb1) & 1u) ? x[1] * mscale : 0.f;
      x[2] = ((m1 >> L.mb0) & 1u) ? x[2] * mscale : 0.f;
      x[3] = ((m1 >> L.mb1) & 1u) ? x[3] * mscale : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 4; i++) split_tf32(x[i], fr[kk][0][i], fr[kk][1][i]);
  }
}

// the block's MMAs on dY^T hi / lo at shared addresses dHi / dLo, committed as one group: per k8 step and operand
// pair one m64n(32 NC)k8 over the NC stacked n32 tiles (k_tc_linear_dw issues NC m64n32k8 instead; each element gets
// the same products in the same order)
template <int NC>
__device__ __forceinline__ void dw_mmas(float (&acc)[NC][16], uint32_t dHi, uint32_t dLo,
                                        const uint32_t (&fr)[DW_KS / 8][2][4]) {
#pragma unroll
  for (int kk = 0; kk < DW_KS / 8; kk++) {
    wgmma_fence();
    const uint32_t off = (uint32_t)kk * 32u;
    const uint64_t bh = make_sdesc_sw128(dHi + off), bl = make_sdesc_sw128(dLo + off);
    wgmma_m64nNk8_tf32<NC>(acc, fr[kk][1], bh);
    wgmma_m64nNk8_tf32<NC>(acc, fr[kk][0], bl);
    wgmma_m64nNk8_tf32<NC>(acc, fr[kk][0], bh);
  }
  wgmma_commit();
}

// acc[c][4j + {0,1}] = (i0 + ca, o, o + 1), [4j + {2,3}] = (i0 + cb, ...), o = 32c + 8j + 2t -> this split's partial
template <int NC, class TX>
__device__ __forceinline__ void dw_store(const TcDwParams& p, const DwLane<TX>& L, int i0, int t,
                                         const float (&acc)[NC][16]) {
  float* ws = p.ws + (size_t)blockIdx.x * ((size_t)p.inDim * p.outDim);
  const int ia = i0 + L.ca, ib = i0 + L.cb;
#pragma unroll
  for (int c = 0; c < NC; c++)
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int o = c * 32 + j * 8 + 2 * t;
#pragma unroll
      for (int h = 0; h < 2; h++) {
        if (o + h >= p.outDim) continue;
        float* col = ws + (size_t)(o + h) * p.inDim;
        if (ia < p.inDim) col[ia] = acc[c][4 * j + h];
        if (ib < p.inDim) col[ib] = acc[c][4 * j + 2 + h];
      }
    }
}

// TX: float, or uint16_t for a bf16 X (boxes of 64-byte rows, 64-byte swizzle), in both kernels below
template <int NC, class TX>
__global__ void __launch_bounds__(DW_THREADS, 1)
k_tc_linear_dw(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapDY,
               const TcDwParams p) {
  constexpr int BN = 32 * NC;
  constexpr uint32_t xBytes = DW_KS * DW_BM * sizeof(TX);      // four [KS][32] boxes of X
  constexpr uint32_t xBoxBytes = DW_KS * DW_XBOX * sizeof(TX);
  constexpr uint32_t yBytes = DW_KS * BN * 4;         // [KS][BN] of dY
  constexpr uint32_t stageBytes = xBytes + yBytes;
  constexpr uint32_t bBytes = BN * DW_KS * 4;         // one dY^T tile; buffer b holds hi at 2b, lo at 2b + 1
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* bT = reinterpret_cast<float*>(smem);
  uint8_t* stages = smem + 4 * bBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(stages + (size_t)p.stages * stageBytes);   // [stages] TMA landed

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i0 = blockIdx.y * DW_BM;
  const int64_t v0 = (int64_t)blockIdx.x * p.vPerSplit;
  const int64_t v1 = min(p.rows, v0 + p.vPerSplit);
  const int numSteps = (v1 > v0) ? (int)((v1 - v0 + DW_KS - 1) / DW_KS) : 0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapX); tma_prefetch_desc(&mapDY);
    for (int s = 0; s < p.stages; s++) mbar_init(&full[s], 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto load = [&](int step) {     // TMA of vertex block `step` into stage step % stages (thread 0)
    uint8_t* st = stages + (size_t)(step % p.stages) * stageBytes;
    uint64_t* bar = &full[step % p.stages];
    const int v = (int)(v0 + (int64_t)step * DW_KS);
    mbar_arrive_expect_tx(bar, stageBytes);
#pragma unroll
    for (int b = 0; b < DW_BM / DW_XBOX; b++) tma_load_2d(st + b * xBoxBytes, &mapX, i0 + b * DW_XBOX, v, bar);
    tma_load_2d(st + xBytes, &mapDY, 0, v, bar);
  };
  if (threadIdx.x == 0)
    for (int step = 0; step < p.stages && step < numSteps; step++) load(step);

  // ================================== consumers ===================================
  const DwLane<TX> L(warp, lane);
  const int t = lane & 3;
  const bool masked = p.mask != nullptr && i0 + L.ca < p.inDim;   // (columns past inDim are zero-filled by TMA)
  const int mcol = (i0 + L.ca) >> 5;
  // dropout fused into the operand load: this thread's mask words of vertices v + 8 kk + t (+ 4); all ones for a
  // column past inDim, as in k_tc_linear_dw_ws
  auto load_mask = [&](int step, uint32_t (&mw)[8]) {
    const int64_t v = v0 + (int64_t)step * DW_KS;
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const int64_t row = v + 4 * q + t;                    // q = 2 kk + h: vertex 8 kk + 4 h + t
      mw[q] = masked ? ((row < p.rows) ? __ldg(p.mask + row * p.ldm + mcol) : 0u) : 0xFFFFFFFFu;
    }
  };
  auto transpose = [&](int s, int b) {   // dY of stage s -> dY^T of buffer b
    float* hiT = bT + (size_t)(2 * b) * (BN * DW_KS);
    dw_transpose<NC, DW_THREADS>(reinterpret_cast<const float*>(stages + (size_t)s * stageBytes + xBytes), hiT,
                                 hiT + BN * DW_KS, threadIdx.x);
  };
  auto fragments = [&](int s, const uint32_t (&mw)[8], uint32_t (&fr)[DW_KS / 8][2][4]) {   // of the block in stage s
    dw_fragments(reinterpret_cast<const TX*>(stages + (size_t)s * stageBytes), L, p.mask != nullptr, p.mscale, mw, fr);
  };
  float acc[NC][16];
#pragma unroll
  for (int c = 0; c < NC; c++)
#pragma unroll
    for (int i = 0; i < 16; i++) acc[c][i] = 0.f;
  auto mmas = [&](int b, const uint32_t (&fr)[DW_KS / 8][2][4]) {
    const uint32_t dHi = smem_u32(bT + (size_t)(2 * b) * (BN * DW_KS)), dLo = dHi + bBytes;
#pragma unroll
    for (int kk = 0; kk < DW_KS / 8; kk++) {
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < NC; c++) {
        const uint32_t off = (uint32_t)c * 32u * 128u + (uint32_t)kk * 32u;
        const uint64_t bh = make_sdesc_sw128(dHi + off), bl = make_sdesc_sw128(dLo + off);
        wgmma_m64n32k8_tf32(acc[c], fr[kk][1], bh);
        wgmma_m64n32k8_tf32(acc[c], fr[kk][0], bl);
        wgmma_m64n32k8_tf32(acc[c], fr[kk][0], bh);
      }
    }
    wgmma_commit();
  };
  // Block `step` sits in stage step % stages, its dY^T in buffer step % 2.  On entry to body(step) that dY^T is written
  // but not yet published, the block's A fragments are in `fr`, and the MMAs of block step - 1 (A fragments in
  // `frPrev`) may still run.  The two register sets alternate, so the loop is unrolled by two.
  int sn = 0; uint32_t phn = 0;  // stage and parity of the next block to wait for
  auto next_stage = [&]() { if (++sn == p.stages) { sn = 0; phn ^= 1; } };
  uint32_t mw[8];
  auto body = [&](int step, uint32_t (&fr)[DW_KS / 8][2][4], uint32_t (&frPrev)[DW_KS / 8][2][4]) {
    wgmma_wait_all();            // this warpgroup's MMAs of block step - 1 have retired
    keep_live(frPrev);
#pragma unroll
    for (int c = 0; c < NC; c++) wgmma_fence_acc(acc[c]);
    consumer_sync();             // dY^T of `step` is published; both warpgroups are past block step - 1 and its stage
    if (threadIdx.x == 0 && step + p.stages < numSteps) load(step + p.stages);   // into the stage of `step`
    mmas(step & 1, fr);
    if (step + 1 < numSteps) {   // block step + 1 while the MMAs run: dY^T, A fragments
      mbar_wait(&full[sn], phn);
      transpose(sn, (step + 1) & 1);
      fragments(sn, mw, frPrev);
      next_stage();
      load_mask(step + 2, mw);   // a whole block ahead of its use: the load latency stays off the step
    }
  };
  uint32_t frA[DW_KS / 8][2][4], frB[DW_KS / 8][2][4] = {};
  if (numSteps > 0) {
    load_mask(0, mw);
    mbar_wait(&full[0], 0);
    transpose(0, 0);
    fragments(0, mw, frA);
    next_stage();
    load_mask(1, mw);
  }
  for (int step = 0; step < numSteps; step += 2) {
    body(step, frA, frB);
    if (step + 1 < numSteps) body(step + 1, frB, frA);
  }
  wgmma_wait_all();
  keep_live(frA);
  keep_live(frB);
#pragma unroll
  for (int c = 0; c < NC; c++) wgmma_fence_acc(acc[c]);
  dw_store<NC>(p, L, i0, t, acc);
}

// WG consumer warpgroups (tile of 64 WG X columns) + one TMA producer warp
template <int NC, int WG, class TX>
__global__ void __launch_bounds__(128 * WG + 32, 1)
k_tc_linear_dw_ws(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapDY,
                  const __grid_constant__ CUtensorMap mapM, const TcDwParams p) {
  constexpr int BN = 32 * NC;
  constexpr int CT = 128 * WG, CW = 4 * WG;            // consumer threads, warps
  constexpr int BM = 64 * WG;                          // X columns of the tile
  constexpr uint32_t xBoxBytes = DW_KS * DW_XBOX * sizeof(TX);
  constexpr uint32_t xBytes = (BM / DW_XBOX) * xBoxBytes;
  constexpr uint32_t yBytes = DW_KS * BN * 4;          // [KS][BN] of dY
  constexpr uint32_t stageBytes = xBytes + yBytes;     // a multiple of 1024: every box stays swizzle-aligned
  constexpr uint32_t mBytes = DW_KS * DW_MASK_WORDS * 4;
  constexpr uint32_t bBytes = BN * DW_KS * 4;          // one dY^T tile; buffer b holds hi at 2b, lo at 2b + 1
  constexpr int BUFS = dw_ws_bufs(NC);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* bT = reinterpret_cast<float*>(smem);
  uint8_t* stages = smem + 2 * BUFS * bBytes;
  const uint32_t* masks = reinterpret_cast<const uint32_t*>(stages + (size_t)p.stages * stageBytes);   // [stages]
  uint64_t* full = reinterpret_cast<uint64_t*>(stages + (size_t)p.stages * (stageBytes + mBytes));  // TMA landed
  uint64_t* empty = full + DW_MAX_STAGES;              // [stages] the consumers have taken the stage
  uint64_t* bfull = empty + DW_MAX_STAGES;             // [BUFS] dY^T buffer written by every consumer warp
  uint64_t* bempty = bfull + BUFS;                     // [BUFS] every warpgroup's MMAs on the buffer have retired

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i0 = blockIdx.y * DW_BM;
  const int64_t v0 = (int64_t)blockIdx.x * p.vPerSplit;
  const int64_t v1 = min(p.rows, v0 + p.vPerSplit);
  const int numSteps = (v1 > v0) ? (int)((v1 - v0 + DW_KS - 1) / DW_KS) : 0;
  const bool masked = p.mask != nullptr;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapX); tma_prefetch_desc(&mapDY);
    if (masked) tma_prefetch_desc(&mapM);
    for (int s = 0; s < p.stages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], CW); }
    for (int b = 0; b < BUFS; b++) { mbar_init(&bfull[b], CW); mbar_init(&bempty[b], CW); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == CW) {
    // ================================ TMA producer ================================
    const uint32_t txBytes = stageBytes + (masked ? mBytes : 0u);
    int s = 0; uint32_t ph = 0;
    for (int step = 0; step < numSteps; step++) {
      mbar_wait(&empty[s], ph ^ 1);
      if (elect_one()) {
        uint8_t* st = stages + (size_t)s * stageBytes;
        const int v = (int)(v0 + (int64_t)step * DW_KS);
        mbar_arrive_expect_tx(&full[s], txBytes);
#pragma unroll
        for (int b = 0; b < BM / DW_XBOX; b++) tma_load_2d(st + b * xBoxBytes, &mapX, i0 + b * DW_XBOX, v, &full[s]);
        tma_load_2d(st + xBytes, &mapDY, 0, v, &full[s]);
        if (masked) tma_load_2d((uint8_t*)masks + (size_t)s * mBytes, &mapM, i0 / 32, v, &full[s]);
      }
      __syncwarp();
      if (++s == p.stages) { s = 0; ph ^= 1; }
    }
    return;
  }

  // ================================== consumers ===================================
  const DwLane<TX> L(warp, lane);
  const int t = lane & 3;
  // Mask word of the thread's two columns for vertex r of the stage: masks[s][r][ca / 32].  A column past inDim is
  // zero-filled by TMA and keeps all bits, as in k_tc_linear_dw; rows past `rows` read the TMA zero fill (dropped).
  const int mcol = L.ca >> 5;
  const uint32_t mpast = (i0 + L.ca < p.inDim) ? 0u : 0xFFFFFFFFu;
  float acc[NC][16];
#pragma unroll
  for (int c = 0; c < NC; c++)
#pragma unroll
    for (int i = 0; i < 16; i++) acc[c][i] = 0.f;
  int s = 0; uint32_t ph = 0;    // ring stage of the block and its parity
  int b = 0; uint32_t bph = 0;   // dY^T buffer of the block and its parity
  int bPrev = 0;
  // Block `step`: its A fragments go to `fr`, whose last MMAs (block step - 2) retired in body(step - 1); the MMAs of
  // block step - 1 (A fragments in `frPrev`) may still run until the wait_group 1 that follows block step's issue.
  // The two register sets alternate, so the loop is unrolled by two.
  auto body = [&](int step, uint32_t (&fr)[DW_KS / 8][2][4], uint32_t (&frPrev)[DW_KS / 8][2][4]) {
    mbar_wait(&full[s], ph);
    mbar_wait(&bempty[b], bph ^ 1);     // the MMAs of block step - BUFS on buffer b have retired in every warpgroup
    const uint8_t* st = stages + (size_t)s * stageBytes;
    float* hiT = bT + (size_t)(2 * b) * (BN * DW_KS);
    dw_transpose<NC, CT>(reinterpret_cast<const float*>(st + xBytes), hiT, hiT + BN * DW_KS, threadIdx.x);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bfull[b]);
    uint32_t mw[8];
    const uint32_t* ms = masks + (size_t)s * (DW_KS * DW_MASK_WORDS);
#pragma unroll
    for (int q = 0; q < 8; q++) mw[q] = masked ? (ms[(4 * q + t) * DW_MASK_WORDS + mcol] | mpast) : 0xFFFFFFFFu;
    dw_fragments(reinterpret_cast<const TX*>(st), L, masked, p.mscale, mw, fr);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
    mbar_wait(&bfull[b], bph);          // every warp's share of block step's dY^T is written
    const uint32_t dHi = smem_u32(hiT);
    dw_mmas<NC>(acc, dHi, dHi + bBytes, fr);
    wgmma_wait_1();                    // this warpgroup's MMAs of block step - 1 have retired
    keep_live(frPrev);
    if (step > 0 && lane == 0) mbar_arrive(&bempty[bPrev]);
    if (++s == p.stages) { s = 0; ph ^= 1; }
    bPrev = b;
    if (++b == BUFS) { b = 0; bph ^= 1; }
  };
  uint32_t frA[DW_KS / 8][2][4], frB[DW_KS / 8][2][4] = {};
  for (int step = 0; step < numSteps; step += 2) {
    body(step, frA, frB);
    if (step + 1 < numSteps) body(step + 1, frB, frA);
  }
  wgmma_wait_all();
  keep_live(frA);
  keep_live(frB);
#pragma unroll
  for (int c = 0; c < NC; c++) wgmma_fence_acc(acc[c]);
  dw_store<NC>(p, L, i0, t, acc);
}

int splitk_reduce(int64_t count, int splits, const float* part, float* dW, cudaStream_t st);   // linear_simt.cu

// ws: k_tc_linear_dw_ws with WG consumer warpgroups; otherwise k_tc_linear_dw
struct DwPlan { int NC, MT, splits, stages; bool ws; int WG; size_t smemBytes; };

// maskOk: no mask, or one whose [KS][4]-word box TMA can load (16-byte aligned base); xElem: bytes per X element (4,
// or 2 for bf16).  The split count does not depend on xElem, so one workspace size serves both.
static int tc_dw_plan(int64_t rows, int inDim, int outDim, bool maskOk, size_t xElem, DwPlan* q) {
  if (outDim > 256 || outDim < 1 || inDim < 4 || rows < 8) return ROC_ERR_UNSUPPORTED;
  const int nc = (outDim + 31) / 32;
  q->NC = nc <= 1 ? 1 : nc <= 2 ? 2 : nc <= 4 ? 4 : 8;
  q->MT = (inDim + DW_BM - 1) / DW_BM;
  // ROC_B200_DW=sync is read on every call, so a test or benchmark can compare the two kernels call by call
  { const char* e = getenv("ROC_B200_DW"); q->ws = q->NC <= 4 && maskOk && !(e && strcmp(e, "sync") == 0); }
  q->WG = (q->ws && inDim <= 64) ? 1 : 2;
  const size_t bn = (size_t)32 * q->NC;
  size_t stageBytes, fixedBytes;
  if (q->ws) {
    stageBytes = (size_t)DW_KS * 64 * q->WG * xElem + (size_t)DW_KS * bn * 4 + (size_t)DW_KS * DW_MASK_WORDS * 4;
    fixedBytes = 1024 /*align*/ + 128 /*barriers*/ + (size_t)2 * dw_ws_bufs(q->NC) * bn * DW_KS * 4 /*dY^T hi / lo*/;
  } else {
    stageBytes = (size_t)DW_KS * DW_BM * xElem + (size_t)DW_KS * bn * 4;
    fixedBytes = 1024 /*align*/ + 64 /*barriers*/ + 4 * bn * DW_KS * 4 /*two dY^T hi / lo buffers*/;
  }
  q->stages = ring_stages(stageBytes, fixedBytes, DW_MAX_STAGES);
  if (!q->stages) return ROC_ERR_UNSUPPORTED;
  q->smemBytes = (size_t)q->stages * stageBytes + fixedBytes;
  int sp = sm_count() / q->MT;
  if (sp < 1) sp = 1;
  int64_t maxSp = (rows + 63) / 64;
  if (sp > maxSp) sp = (int)maxSp;
  q->splits = sp;
  return ROC_OK;
}

size_t tc_dw_workspace_bytes(int64_t rows, int inDim, int outDim) {
  DwPlan q;
  if (tc_dw_plan(rows, inDim, outDim, true, 4, &q) != ROC_OK) return 0;
  return (size_t)q.splits * (size_t)inDim * (size_t)outDim * sizeof(float);
}

template <int NC, class TX>
static int dw_launch(const DwPlan& q, const CUtensorMap& mapX, const CUtensorMap& mapDY, const CUtensorMap& mapM,
                     const TcDwParams& t, cudaStream_t st) {
  const dim3 grid((unsigned)q.splits, (unsigned)q.MT, 1);
  if constexpr (NC <= 4) {
    if (q.ws && q.WG == 1)
      return launch_dyn<k_tc_linear_dw_ws<NC, 1, TX>>(grid, 128 + 32, q.smemBytes, st, mapX, mapDY, mapM, t);
    if (q.ws) return launch_dyn<k_tc_linear_dw_ws<NC, 2, TX>>(grid, 256 + 32, q.smemBytes, st, mapX, mapDY, mapM, t);
  }
  return launch_dyn<k_tc_linear_dw<NC, TX>>(grid, DW_THREADS, q.smemBytes, st, mapX, mapDY, t);
}

template <class TX>
static int dw_launch_nc(const DwPlan& q, const CUtensorMap& mapX, const CUtensorMap& mapDY, const CUtensorMap& mapM,
                        const TcDwParams& t, cudaStream_t st) {
  switch (q.NC) {
    case 1: return dw_launch<1, TX>(q, mapX, mapDY, mapM, t, st);
    case 2: return dw_launch<2, TX>(q, mapX, mapDY, mapM, t, st);
    case 4: return dw_launch<4, TX>(q, mapX, mapDY, mapM, t, st);
    default: return dw_launch<8, TX>(q, mapX, mapDY, mapM, t, st);
  }
}

// X is fp32, or bf16 (raw bits) when xBf16
int tc_linear_dw(int64_t rows, int inDim, int outDim, const void* X, bool xBf16, int64_t ldX, const float* dY,
                 int64_t ldDY, float* dW, float* workspace, size_t wsBytes, const DropMask* dm, cudaStream_t st,
                 roc_gemm_info* info) {
  // the mask box is [KS vertices][4 words]: TMA wants a 16-byte aligned base (the row stride is a multiple of 4 words,
  // which the C ABI requires), so a mask that starts elsewhere goes to k_tc_linear_dw, which loads it word by word
  const bool maskOk = !dm || aligned16(dm->bits);
  DwPlan q;
  if (tc_dw_plan(rows, inDim, outDim, maskOk, xBf16 ? 2 : 4, &q) != ROC_OK) return ROC_ERR_UNSUPPORTED;
  if ((ldX % (xBf16 ? 8 : 4)) || (ldDY % 4) || !aligned16(X) || !aligned16(dY)) return ROC_ERR_UNSUPPORTED;
  if (rows > 0x7FFFFF00ll || !encode_tiled_fn()) return ROC_ERR_UNSUPPORTED;
  const size_t count = (size_t)inDim * outDim;
  if (wsBytes < (size_t)q.splits * count * sizeof(float)) return ROC_ERR_INVALID;
  CUtensorMap mapX, mapDY, mapM;
  memset(&mapM, 0, sizeof(mapM));
  if (xBf16 ? !make_tmap_bf16_2d(&mapX, static_cast<const uint16_t*>(X), (uint64_t)rows, (uint64_t)inDim,
                                 (uint64_t)ldX, DW_KS, DW_XBOX)
            : !make_tmap_f32_2d(&mapX, static_cast<const float*>(X), (uint64_t)rows, (uint64_t)inDim, (uint64_t)ldX,
                                DW_KS, DW_XBOX))
    return ROC_ERR_UNSUPPORTED;
  if (!make_tmap_f32_2d(&mapDY, dY, (uint64_t)rows, (uint64_t)outDim, (uint64_t)ldDY, DW_KS, (uint32_t)(32 * q.NC),
                        CU_TENSOR_MAP_SWIZZLE_NONE))
    return ROC_ERR_UNSUPPORTED;
  if (q.ws && dm &&
      !make_tmap_u32_2d(&mapM, dm->bits, (uint64_t)rows, (uint64_t)dm->ld, (uint64_t)dm->ld, DW_KS, DW_MASK_WORDS))
    return ROC_ERR_UNSUPPORTED;
  TcDwParams t{};
  t.ws = workspace; t.rows = rows; t.inDim = inDim; t.outDim = outDim; t.stages = q.stages;
  t.vPerSplit = ((rows + q.splits - 1) / q.splits + DW_KS - 1) / DW_KS * DW_KS;
  if (dm) { t.mask = dm->bits; t.ldm = dm->ld; t.mscale = dm->scale; }
  if (info) {
    info->nc = q.NC; info->epi = q.ws ? 1 : 0; info->grid_x = q.splits; info->grid_y = q.MT; info->stages = q.stages;
    info->splits = q.splits; info->v_per_split = t.vPerSplit;
  }
  const int rc = xBf16 ? dw_launch_nc<uint16_t>(q, mapX, mapDY, mapM, t, st)
                        : dw_launch_nc<float>(q, mapX, mapDY, mapM, t, st);
  if (rc != ROC_OK) return rc;
  return splitk_reduce((int64_t)count, q.splits, workspace, dW, st);
}

}  // namespace roc
