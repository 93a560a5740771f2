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
//       (four [KS][32] boxes, 128-byte swizzle), applies the fused dropout mask and splits it hi / lo;
//   B = dY^T is transposed and split once per stage by the consumers into two K-major tiles
//       [N][KS] (hi, lo; 128-byte swizzle) that the MMAs of both warpgroups read.
// The dY^T tiles are double-buffered and the step is software-pipelined: while the MMAs of vertex
// block k run, the consumers transpose block k + 1 into the other buffer and then read block k + 1's
// A fragments into a second register set, so the tensor cores and the load / split work overlap.
// One CTA-wide barrier per block publishes the next dY^T buffer and certifies that both warpgroups'
// MMAs of the previous block have retired (which frees that buffer and the ring stage).
// Two warpgroups of 64 X columns each and nothing else: with the accumulator of up to 256 columns in
// registers a third (producer) warp would cap them at 168 registers and serialise the MMAs.  Thread 0
// refills a stage with TMA (X boxes + dY box) once both warpgroups are past it.
#include <cstdlib>
#include "common.cuh"
#include "tc_common.cuh"

namespace roc {

using namespace tc;

constexpr int DW_BM = 128;         // X columns per CTA
constexpr int DW_KS = 32;          // vertices per stage = one 128-byte swizzle row of dY^T
constexpr int DW_XBOX = 32;        // X columns per TMA box = one 128-byte swizzle row
constexpr int DW_THREADS = 256;    // two consumer warpgroups
constexpr int DW_MAX_STAGES = 4;

struct TcDwParams {
  float* ws; int64_t rows; int inDim, outDim;
  int64_t vPerSplit;       // multiple of DW_KS
  int stages;
  const uint32_t* mask; int64_t ldm; float mscale;   // fused dropout of X (NULL = none)
};

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Accumulator row 16 (w % 4) + g + 8 h of warpgroup w / 4, held by lane (g, t) of warp w (0..7), is X column
// dw_col(w, g, h) of the tile.  The permutation (any one gives the same sums: an accumulator row depends only on its
// own A row) puts the 32 lanes' A fragment reads of the swizzled X boxes on 32 distinct banks: within a warp the
// 16-byte chunk (col % 32) / 4 is 4 (g / 4) + 2 (w % 2) + h, so chunk ^ t (the swizzle of vertex row t) is distinct
// over (g / 4, t), and col % 4 = g % 4.  Both columns of a thread sit in one 32-column box, so in one mask word.
__device__ __forceinline__ int dw_col(int w, int g, int h) {
  return (w >> 1) * DW_XBOX + (g >> 2) * 16 + (w & 1) * 8 + h * 4 + (g & 3);
}

template <int NC>
__global__ void __launch_bounds__(DW_THREADS, 1)
k_tc_linear_dw(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapDY,
               const TcDwParams p) {
  constexpr int BN = 32 * NC;
  constexpr uint32_t xBytes = DW_KS * DW_BM * 4;      // four [KS][32] boxes of X
  constexpr uint32_t xBoxBytes = DW_KS * DW_XBOX * 4;
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
  const int g = lane >> 2, t = lane & 3;
  const int ca = dw_col(warp, g, 0), cb = dw_col(warp, g, 1);   // X columns of this thread: i0 + ca and i0 + cb
  // offsets of the fragment (k8 step 0) in the swizzled X boxes: (vertex t + 4 e, column c) at
  // box(c) * 32 KS + (t + 4 e) * 32 + ((c % 32 / 4) ^ (t + 4 e)) * 4 + c % 4
  int xo[2][2];
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const int c = h ? cb : ca, k = t + 4 * e;
      xo[h][e] = (c / DW_XBOX) * (DW_KS * DW_XBOX) + k * DW_XBOX + ((((c % DW_XBOX) >> 2) ^ k) << 2) + (c & 3);
    }
  const bool masked = p.mask != nullptr && i0 + ca < p.inDim;   // (columns past inDim are zero-filled by TMA)
  const int mcol = (i0 + ca) >> 5, mb0 = ca & 31, mb1 = cb & 31;
  // dropout fused into the operand load: this thread's mask words of vertices v + 8 kk + t (+ 4)
  auto load_mask = [&](int step, uint32_t (&mw)[8]) {
    const int64_t v = v0 + (int64_t)step * DW_KS;
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const int64_t row = v + 4 * q + t;                    // q = 2 kk + h: vertex 8 kk + 4 h + t
      mw[q] = masked ? ((row < p.rows) ? __ldg(p.mask + row * p.ldm + mcol) : 0u) : 0xFFFFFFFFu;
    }
  };
  // dY [KS][BN] of stage s -> dY^T hi / lo [BN][KS] of buffer b; 128-byte swizzle: element (o, k) at
  // o*32 + ((k/4 ^ o%8) * 4) + k%4.  A thread takes 4 consecutive k of one o: 4 conflict-free loads, one 16-byte
  // store per tile, and the 8 lanes of a store phase (8 consecutive o) fill the 32 banks.
  auto transpose = [&](int s, int b) {
    const float* ys = reinterpret_cast<const float*>(stages + (size_t)s * stageBytes + xBytes);
    float* hiT = bT + (size_t)(2 * b) * (BN * DW_KS);
    float* loT = hiT + BN * DW_KS;
#pragma unroll
    for (int j = 0; j < NC; j++) {
      const int idx = threadIdx.x + DW_THREADS * j;
      const int q = idx / BN, o = idx - q * BN;
      uint32_t h[4], l[4];
#pragma unroll
      for (int r = 0; r < 4; r++) split_tf32(ys[(4 * q + r) * BN + o], h[r], l[r]);
      const int d = o * DW_KS + ((q ^ (o & 7)) << 2);
      *reinterpret_cast<uint4*>(hiT + d) = make_uint4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<uint4*>(loT + d) = make_uint4(l[0], l[1], l[2], l[3]);
    }
    fence_proxy_async_smem();
  };
  // A fragments (hi, lo) of every k8 step of the block in stage s
  auto fragments = [&](int s, const uint32_t (&mw)[8], uint32_t (&fr)[DW_KS / 8][2][4]) {
    const float* xs = reinterpret_cast<const float*>(stages + (size_t)s * stageBytes);
#pragma unroll
    for (int kk = 0; kk < DW_KS / 8; kk++) {
      const int kb = kk * 8 * DW_XBOX;
      float x[4] = {xs[kb + xo[0][0]], xs[kb + xo[1][0]], xs[kb + xo[0][1]], xs[kb + xo[1][1]]};
      if (p.mask) {
        const uint32_t m0 = mw[2 * kk], m1 = mw[2 * kk + 1];
        x[0] = ((m0 >> mb0) & 1u) ? x[0] * p.mscale : 0.f;   // == k_dropout
        x[1] = ((m0 >> mb1) & 1u) ? x[1] * p.mscale : 0.f;
        x[2] = ((m1 >> mb0) & 1u) ? x[2] * p.mscale : 0.f;
        x[3] = ((m1 >> mb1) & 1u) ? x[3] * p.mscale : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 4; i++) split_tf32(x[i], fr[kk][0][i], fr[kk][1][i]);
    }
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
  // ---- epilogue: acc[c][4j + {0,1}] = (i0 + ca, o, o + 1), [4j + {2,3}] = (i0 + cb, ...), o = 32c + 8j + 2t
  float* ws = p.ws + (size_t)blockIdx.x * ((size_t)p.inDim * p.outDim);
  const int ia = i0 + ca, ib = i0 + cb;
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

__global__ void __launch_bounds__(256)
k_tc_splitk_reduce(int64_t count, int splits, const float* __restrict__ part, float* __restrict__ dW) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int z = 0; z < splits; z++) s += part[(int64_t)z * count + i];
    dW[i] += s;
  }
}

struct DwPlan { int NC, MT, splits, stages; size_t smemBytes; };

static int tc_dw_plan(int64_t rows, int inDim, int outDim, DwPlan* q) {
  if (outDim > 256 || outDim < 1 || inDim < 4 || rows < 8) return ROC_ERR_UNSUPPORTED;
  { const char* e = getenv("ROC_B200_GEMM"); if (e && e[0] == 'n' && e[1] == 'o') return ROC_ERR_UNSUPPORTED; }   // "notc"
  const int nc = (outDim + 31) / 32;
  q->NC = nc <= 1 ? 1 : nc <= 2 ? 2 : nc <= 4 ? 4 : 8;
  q->MT = (inDim + DW_BM - 1) / DW_BM;
  const size_t bn = (size_t)32 * q->NC;
  const size_t stageBytes = (size_t)DW_KS * DW_BM * 4 + (size_t)DW_KS * bn * 4;
  const size_t fixedBytes = 1024 /*align*/ + 64 /*barriers*/ + 4 * bn * DW_KS * 4 /*two dY^T hi / lo buffers*/;
  int st = (int)(((size_t)227 * 1024 - fixedBytes) / stageBytes);
  if (st > DW_MAX_STAGES) st = DW_MAX_STAGES;
  if (st < 2) return ROC_ERR_UNSUPPORTED;
  q->stages = st;
  q->smemBytes = (size_t)st * stageBytes + fixedBytes;
  int sp = sm_count() / q->MT;
  if (sp < 1) sp = 1;
  int64_t maxSp = (rows + 63) / 64;
  if (sp > maxSp) sp = (int)maxSp;
  q->splits = sp;
  return ROC_OK;
}

size_t tc_dw_workspace_bytes(int64_t rows, int inDim, int outDim) {
  DwPlan q;
  if (tc_dw_plan(rows, inDim, outDim, &q) != ROC_OK) return 0;
  return (size_t)q.splits * (size_t)inDim * (size_t)outDim * sizeof(float);
}

template <int NC>
static int dw_launch(const DwPlan& q, const CUtensorMap& mapX, const CUtensorMap& mapDY, const TcDwParams& t,
                     cudaStream_t st) {
  static DynSmemCache configured;
  ROC_CUDA(ensure_dyn_smem(k_tc_linear_dw<NC>, q.smemBytes, configured));
  k_tc_linear_dw<NC><<<dim3((unsigned)q.splits, (unsigned)q.MT, 1), DW_THREADS, q.smemBytes, st>>>(mapX, mapDY, t);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

int tc_linear_dw(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX, const float* dY, int64_t ldDY,
                 float* dW, float* workspace, size_t wsBytes, const DropMask* dm, cudaStream_t st,
                 roc_gemm_info* info) {
  DwPlan q;
  if (tc_dw_plan(rows, inDim, outDim, &q) != ROC_OK) return ROC_ERR_UNSUPPORTED;
  if ((ldX % 4) || (ldDY % 4) || !aligned16(X) || !aligned16(dY)) return ROC_ERR_UNSUPPORTED;
  if (rows > 0x7FFFFF00ll || !encode_tiled_fn()) return ROC_ERR_UNSUPPORTED;
  const size_t count = (size_t)inDim * outDim;
  if (wsBytes < (size_t)q.splits * count * sizeof(float)) return ROC_ERR_INVALID;
  CUtensorMap mapX, mapDY;
  if (!make_tmap_f32_2d(&mapX, X, (uint64_t)rows, (uint64_t)inDim, (uint64_t)ldX, DW_KS, DW_XBOX))
    return ROC_ERR_UNSUPPORTED;
  if (!make_tmap_f32_2d(&mapDY, dY, (uint64_t)rows, (uint64_t)outDim, (uint64_t)ldDY, DW_KS, (uint32_t)(32 * q.NC),
                        CU_TENSOR_MAP_SWIZZLE_NONE))
    return ROC_ERR_UNSUPPORTED;
  TcDwParams t{};
  t.ws = workspace; t.rows = rows; t.inDim = inDim; t.outDim = outDim; t.stages = q.stages;
  t.vPerSplit = ((rows + q.splits - 1) / q.splits + DW_KS - 1) / DW_KS * DW_KS;
  if (dm) { t.mask = dm->bits; t.ldm = dm->ld; t.mscale = dm->scale; }
  if (info) {
    info->nc = q.NC; info->epi = 0; info->grid_x = q.splits; info->grid_y = q.MT; info->stages = q.stages;
    info->splits = q.splits; info->v_per_split = t.vPerSplit;
  }
  int rc;
  switch (q.NC) {
    case 1: rc = dw_launch<1>(q, mapX, mapDY, t, st); break;
    case 2: rc = dw_launch<2>(q, mapX, mapDY, t, st); break;
    case 4: rc = dw_launch<4>(q, mapX, mapDY, t, st); break;
    default: rc = dw_launch<8>(q, mapX, mapDY, t, st); break;
  }
  if (rc != ROC_OK) return rc;
  int64_t blocks = ((int64_t)count + 255) / 256;
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  k_tc_splitk_reduce<<<(unsigned)blocks, 256, 0, st>>>((int64_t)count, q.splits, workspace, dW);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

}  // namespace roc
