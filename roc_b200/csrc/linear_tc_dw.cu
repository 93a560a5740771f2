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
//       [KS][128] (column i = row of A), applies the fused dropout mask and splits it hi / lo;
//   B = dY^T is transposed and split once per stage by the consumers into two K-major tiles
//       [N][KS] (hi, lo; 128-byte swizzle) that the MMAs of both warpgroups read.
// Two warpgroups of 64 X columns each and nothing else: with the accumulator of up to 256 columns in
// registers a third (producer) warp would cap them at 168 registers and serialise the MMAs.  Thread 0
// refills a stage with TMA (X box + dY box) once both warpgroups are past it.
#include <cstdlib>
#include "common.cuh"
#include "tc_common.cuh"

namespace roc {

using namespace tc;

constexpr int DW_BM = 128;         // X columns per CTA
constexpr int DW_KS = 32;          // vertices per stage = one 128-byte swizzle row of dY^T
constexpr int DW_THREADS = 256;    // two consumer warpgroups
constexpr int DW_MAX_STAGES = 4;

struct TcDwParams {
  float* ws; int64_t rows; int inDim, outDim;
  int64_t vPerSplit;       // multiple of DW_KS
  int stages;
  const uint32_t* mask; int64_t ldm; float mscale;   // fused dropout of X (NULL = none)
};

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

template <int NC>
__global__ void __launch_bounds__(DW_THREADS, 1)
k_tc_linear_dw(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapDY,
               const TcDwParams p) {
  constexpr int BN = 32 * NC;
  constexpr uint32_t xBytes = DW_KS * DW_BM * 4;      // [KS][128] of X
  constexpr uint32_t yBytes = DW_KS * BN * 4;         // [KS][BN] of dY
  constexpr uint32_t stageBytes = xBytes + yBytes;
  constexpr uint32_t bBytes = BN * DW_KS * 4;         // dY^T hi; lo beside it
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* bHi = reinterpret_cast<float*>(smem);
  float* bLo = reinterpret_cast<float*>(smem + bBytes);
  uint8_t* stages = smem + 2 * bBytes;
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
    tma_load_2d(st, &mapX, i0, v, bar);
    tma_load_2d(st + xBytes, &mapDY, 0, v, bar);
  };
  if (threadIdx.x == 0)
    for (int step = 0; step < p.stages && step < numSteps; step++) load(step);

  // ================================== consumers ===================================
  const int g = lane >> 2, t = lane & 3;
  const int il = (warp >> 2) * 64 + (warp & 3) * 16 + g;   // X columns of this thread: i0 + il and i0 + il + 8
  const bool masked = p.mask != nullptr && i0 + il < p.inDim;   // (columns past inDim are zero-filled by TMA)
  const int mcol = (i0 + il) >> 5, mb0 = (i0 + il) & 31, mb1 = mb0 + 8;   // both columns sit in one mask word
  float acc[NC][16];
#pragma unroll
  for (int c = 0; c < NC; c++)
#pragma unroll
    for (int i = 0; i < 16; i++) acc[c][i] = 0.f;
  int s = 0; uint32_t ph = 0;
  for (int step = 0; step < numSteps; step++) {
    const int64_t v = v0 + (int64_t)step * DW_KS;
    // dropout fused into the operand load: this thread's mask words of vertices v + 8 kk + t (+ 4)
    uint32_t mw[8];
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const int64_t row = v + 4 * q + t;                    // q = 2 kk + h: vertex 8 kk + 4 h + t
      mw[q] = masked ? ((row < p.rows) ? __ldg(p.mask + row * p.ldm + mcol) : 0u) : 0xFFFFFFFFu;
    }
    mbar_wait(&full[s], ph);
    const float* xs = reinterpret_cast<const float*>(stages + (size_t)s * stageBytes);
    const float* ys = xs + DW_KS * DW_BM;
    consumer_sync();              // both warpgroups are done with the previous stage (and its MMAs have completed)
    if (threadIdx.x == 0 && step > 0 && step - 1 + p.stages < numSteps) load(step - 1 + p.stages);
    // dY [KS][BN] -> dY^T hi / lo [BN][KS]; 128-byte swizzle: element (o, k) at o*32 + ((k/4 ^ o%8) * 4) + k%4
    for (int idx = threadIdx.x; idx < DW_KS * BN; idx += 256) {
      const int k = idx / BN, o = idx - k * BN;
      uint32_t h, l;
      split_tf32(ys[idx], h, l);
      const int d = o * DW_KS + ((((k >> 2) ^ (o & 7))) << 2) + (k & 3);
      bHi[d] = __uint_as_float(h);
      bLo[d] = __uint_as_float(l);
    }
    fence_proxy_async_smem();
    consumer_sync();
    const uint32_t dHi = smem_u32(bHi), dLo = smem_u32(bLo);
    uint32_t fr[DW_KS / 8][2][4];      // A fragments (hi, lo) of every k8 step: live until the MMAs are retired
#pragma unroll
    for (int kk = 0; kk < DW_KS / 8; kk++) {
      const int k0 = 8 * kk + t, k1 = k0 + 4;
      float x[4] = {xs[k0 * DW_BM + il], xs[k0 * DW_BM + il + 8], xs[k1 * DW_BM + il], xs[k1 * DW_BM + il + 8]};
      if (p.mask) {
        const uint32_t m0 = mw[2 * kk], m1 = mw[2 * kk + 1];
        x[0] = ((m0 >> mb0) & 1u) ? x[0] * p.mscale : 0.f;   // == k_dropout
        x[1] = ((m0 >> mb1) & 1u) ? x[1] * p.mscale : 0.f;
        x[2] = ((m1 >> mb0) & 1u) ? x[2] * p.mscale : 0.f;
        x[3] = ((m1 >> mb1) & 1u) ? x[3] * p.mscale : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 4; i++) split_tf32(x[i], fr[kk][0][i], fr[kk][1][i]);
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
    wgmma_wait_all();
    keep_live(fr);
#pragma unroll
    for (int c = 0; c < NC; c++) wgmma_fence_acc(acc[c]);
    if (++s == p.stages) { s = 0; ph ^= 1; }
  }
  // ---- epilogue: acc[c][4j + {0,1}] = (i0 + il, o, o + 1), [4j + {2,3}] = (i0 + il + 8, ...), o = 32c + 8j + 2t
  float* ws = p.ws + (size_t)blockIdx.x * ((size_t)p.inDim * p.outDim);
  const int ia = i0 + il, ib = ia + 8;
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
  const size_t fixedBytes = 1024 /*align*/ + 64 /*barriers*/ + 2 * bn * DW_KS * 4 /*dY^T hi / lo*/;
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
                 float* dW, float* workspace, size_t wsBytes, const DropMask* dm, cudaStream_t st) {
  DwPlan q;
  if (tc_dw_plan(rows, inDim, outDim, &q) != ROC_OK) return ROC_ERR_UNSUPPORTED;
  if ((ldX % 4) || (ldDY % 4) || !aligned16(X) || !aligned16(dY)) return ROC_ERR_UNSUPPORTED;
  if (rows > 0x7FFFFF00ll || !encode_tiled_fn()) return ROC_ERR_UNSUPPORTED;
  const size_t count = (size_t)inDim * outDim;
  if (wsBytes < (size_t)q.splits * count * sizeof(float)) return ROC_ERR_INVALID;
  CUtensorMap mapX, mapDY;
  if (!make_tmap_f32_2d(&mapX, X, (uint64_t)rows, (uint64_t)inDim, (uint64_t)ldX, DW_KS, DW_BM, CU_TENSOR_MAP_SWIZZLE_NONE))
    return ROC_ERR_UNSUPPORTED;
  if (!make_tmap_f32_2d(&mapDY, dY, (uint64_t)rows, (uint64_t)outDim, (uint64_t)ldDY, DW_KS, (uint32_t)(32 * q.NC),
                        CU_TENSOR_MAP_SWIZZLE_NONE))
    return ROC_ERR_UNSUPPORTED;
  TcDwParams t{};
  t.ws = workspace; t.rows = rows; t.inDim = inDim; t.outDim = outDim; t.stages = q.stages;
  t.vPerSplit = ((rows + q.splits - 1) / q.splits + DW_KS - 1) / DW_KS * DW_KS;
  if (dm) { t.mask = dm->bits; t.ldm = dm->ld; t.mscale = dm->scale; }
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
