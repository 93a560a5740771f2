// linear_tc.cu — wgmma tensor-core GEMMs for the Linear op, fed by TMA (sm_90a).
//
// Replaces cublasSgemm of Linear::forward_task (linear_kernel.cu:76-80) and the dX sgemm of
// Linear::backward_task (linear_kernel.cu:227-231):
//     fwd: Y[v][o]  = sum_i X[v][i]  * W[o*in + i]      M = rows, N = outDim, K = inDim
//     dX : dX[v][i] = sum_o dY[v][o] * W[o*in + i]      M = rows, N = inDim,  K = outDim
// fp32 in, fp32 out, within 1e-4 of sgemm: the tensor cores have no fp32 MMA, so
// each operand is split hi + lo (hi = fp32 truncated to TF32's 10-bit mantissa,
// lo = exact remainder) and three tf32 MMAs accumulate lo*hi + hi*lo + hi*hi
// in fp32 registers (3xTF32: error ~2^-20 relative per product).
//
// One kernel serves both: a row-major [rows][K] streaming operand A (X or dY) times a
// small K-major weight operand prepared by k_split_w ([N][K] hi / lo; dX passes W
// transposed).  The streaming operand is split where it is consumed: each consumer thread
// reads its wgmma A fragment from the TMA tile (128-byte swizzle, conflict-free), applies the
// fused dropout mask, splits it hi / lo in registers and issues wgmma with A from registers,
// so the tile crosses shared memory once.  W_hi / W_lo come from shared memory (K-major,
// 128-byte swizzle).  One persistent CTA per SM (x N-tiles of <= 128 columns in grid.y):
//   warps 0-7  two consumer warpgroups, 64 rows of the 128-row tile each: fragment load,
//              [dropout mask ->] hi/lo split, 3 x wgmma m64n32k8 per 32-column chunk and k8
//              step, then the epilogue (relu / dropout-backward mask / relu mask / row norm /
//              accumulate) straight from the accumulator registers
//   warp 8     TMA producer (A tile [128 rows][32 k] + W_hi + W_lo tile per stage)
// HBM-bound on A (rows*K*4 bytes read once); W (tens of KB) stays in L2.
#include <cstdio>
#include <cstdlib>
#include "common.cuh"
#include "tc_common.cuh"

namespace roc {

using namespace tc;

constexpr int TC_BM = 128;        // rows per tile: two consumer warpgroups of 64
constexpr int TC_BK = 32;         // fp32 per k-block = one 128-byte swizzle row
constexpr int TC_THREADS = 288;   // 8 consumer warps + 1 producer warp
constexpr int TC_MAX_STAGES = 8;

// Whi/Wlo[n][k] (n < Npad, k < Kpad, zero padded) = split of B(n, k), where
//   transposed == 0: B(n, k) = W[n * ldW + k]   (fwd: n = output o, k = input i, ldW = inDim)
//   transposed == 1: B(n, k) = W[k * ldW + n]   (dX : n = input i,  k = output o)
__global__ void k_split_w(int N, int K, int Npad, int Kpad, int ldW, int transposed, const float* __restrict__ W,
                          float* __restrict__ Whi, float* __restrict__ Wlo) {
  int total = Npad * Kpad;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int n = i / Kpad, k = i - n * Kpad;
    float w = 0.f;
    if (n < N && k < K) w = transposed ? W[(size_t)k * ldW + n] : W[(size_t)n * ldW + k];
    float hi = __uint_as_float(__float_as_uint(w) & 0xFFFFE000u);
    Whi[i] = hi;
    Wlo[i] = w - hi;
  }
}

struct TcParams {
  float* Y; int64_t ldY;
  int64_t rows; int outDim; int numKb; int stages;
  const uint32_t* mask; int64_t ldm; float mscale;      // dropout of A fused into the operand load (NULL = none)
  // epilogue, applied in this order to acc(row, col):
  int relu;                                             //   relu (Linear's activation, linear_kernel.cu:83-104)
  const uint32_t* omask; int64_t oldm; float oscale;    //   dropout backward: keep ? x * scale : 0
  const float* reluOf; int64_t ldR;                     //   relu backward: reluOf(row, col) > 0 ? x : 0
  const uint64_t* rowEnd; uint64_t colLeft;             //   indegree norm: x / sqrtf(deg(row))
  int accumulate;                                       //   Y += x instead of Y = x
};

// Epilogue stage switches: compile-time when the kernel is instantiated for a fixed combination
// (EPI >= 0, a bit mask), read from the parameters for the generic instantiation (EPI < 0).
enum { EPI_RELU = 1, EPI_OMASK = 2, EPI_RELUOF = 4, EPI_NORM = 8, EPI_ACC = 16 };
#define EPI_FLAGS(EPI, p)                                                        \
  const bool fRelu = (EPI) < 0 ? (p).relu != 0 : ((EPI) & EPI_RELU) != 0;         \
  const bool fOmask = (EPI) < 0 ? (p).omask != nullptr : ((EPI) & EPI_OMASK) != 0; \
  const bool fReluOf = (EPI) < 0 ? (p).reluOf != nullptr : ((EPI) & EPI_RELUOF) != 0; \
  const bool fNorm = (EPI) < 0 ? (p).rowEnd != nullptr : ((EPI) & EPI_NORM) != 0;  \
  const bool fAcc = (EPI) < 0 ? (p).accumulate != 0 : ((EPI) & EPI_ACC) != 0;

__device__ __forceinline__ float row_norm_divisor(const TcParams& p, int64_t row) {
  if (!p.rowEnd || row >= p.rows) return 1.0f;
  const uint64_t st = (row == 0) ? p.colLeft : p.rowEnd[row - 1];
  return sqrtf((float)(uint32_t)(p.rowEnd[row] - st));
}

// Epilogue of two adjacent columns (col even) of one row: the accumulator pair a thread holds.
template <int EPI>
__device__ __forceinline__ void tc_store_pair(const TcParams& p, int64_t row, int col, float x0, float x1,
                                              const RowDiv& rd) {
  EPI_FLAGS(EPI, p)
  if (row >= p.rows || col >= p.outDim) return;
  const bool two = col + 1 < p.outDim;
  float* y = p.Y + row * p.ldY + col;
  uint32_t mw = 3u;                 // col is even: col and col + 1 sit in one mask word
  if (fOmask) mw = __ldg(p.omask + row * p.oldm + (col >> 5)) >> (col & 31);
  float old[2] = {0.f, 0.f}, ro[2] = {1.f, 1.f};
  if (fAcc) {
    if (two) { const float2 o = *reinterpret_cast<const float2*>(y); old[0] = o.x; old[1] = o.y; }
    else old[0] = y[0];
  }
  if (fReluOf) {
    const float* rp = p.reluOf + row * p.ldR + col;
    if (two) { const float2 o = __ldg(reinterpret_cast<const float2*>(rp)); ro[0] = o.x; ro[1] = o.y; }
    else ro[0] = rp[0];
  }
  float v[2] = {x0, x1};
#pragma unroll
  for (int k = 0; k < 2; k++) {
    float x = v[k];
    if (fRelu) x = relu_nanprop(x);
    if (fOmask) x = ((mw >> k) & 1u) ? x * p.oscale : 0.f;
    if (fReluOf) x = (ro[k] > 0.f) ? x : 0.f;
    if (fNorm) x = rowdiv(x, rd);   // == x / d bit for bit (common.cuh)
    if (fAcc) x = old[k] + x;
    v[k] = x;
  }
  if (two) *reinterpret_cast<float2*>(y) = make_float2(v[0], v[1]);
  else y[0] = v[0];
}

template <int NC, int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_tc_linear(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapWhi,
            const __grid_constant__ CUtensorMap mapWlo, const TcParams p) {
  constexpr int BN = 32 * NC;
  constexpr uint32_t aBytes = TC_BM * TC_BK * 4;       // 16 KB of A per stage
  constexpr uint32_t bBytes = BN * TC_BK * 4;
  constexpr uint32_t stageBytes = aBytes + 2 * bBytes;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * stageBytes);   // [stages] TMA landed
  uint64_t* empty = full + TC_MAX_STAGES;                                                // [stages] consumers done

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t numTiles = (p.rows + TC_BM - 1) / TC_BM;
  const int n0 = blockIdx.y * BN;          // this CTA's slice of the N (output column) dimension

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapA); tma_prefetch_desc(&mapWhi); tma_prefetch_desc(&mapWlo);
    for (int s = 0; s < p.stages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ================================ TMA producer ================================
    int s = 0; uint32_t ph = 0;
    for (int64_t tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
      for (int kb = 0; kb < p.numKb; kb++) {
        mbar_wait(&empty[s], ph ^ 1);
        uint8_t* st = smem + (size_t)s * stageBytes;
        if (elect_one()) {
          mbar_arrive_expect_tx(&full[s], stageBytes);
          tma_load_2d(st, &mapA, kb * TC_BK, (int)(tile * TC_BM), &full[s]);
          tma_load_2d(st + aBytes, &mapWhi, kb * TC_BK, n0, &full[s]);
          tma_load_2d(st + aBytes + bBytes, &mapWlo, kb * TC_BK, n0, &full[s]);
        }
        __syncwarp();
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ================================== consumers ===================================
  const bool fNorm = (EPI) < 0 ? p.rowEnd != nullptr : ((EPI) & EPI_NORM) != 0;
  const int g = lane >> 2, t = lane & 3;
  const int rl = (warp >> 2) * 64 + (warp & 3) * 16 + g;    // tile rows of this thread: rl and rl + 8 (both == g mod 8)
  const bool masked = p.mask != nullptr;
  int s = 0; uint32_t ph = 0;
  for (int64_t tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
    const int64_t row0 = tile * TC_BM + rl, row1 = row0 + 8;
    // the rows' norm divisors are fetched before the main loop so their DRAM latency overlaps it
    const float d0 = fNorm ? row_norm_divisor(p, row0) : 1.0f;
    const float d1 = fNorm ? row_norm_divisor(p, row1) : 1.0f;
    float acc[NC][16];
#pragma unroll
    for (int c = 0; c < NC; c++)
#pragma unroll
      for (int i = 0; i < 16; i++) acc[c][i] = 0.f;
    for (int kb = 0; kb < p.numKb; kb++) {
      // dropout fused into the operand load: bit c of mask[row][kb] keeps column 32 kb + c
      uint32_t mw0 = 0xFFFFFFFFu, mw1 = 0xFFFFFFFFu;
      if (masked) {
        mw0 = (row0 < p.rows) ? __ldg(p.mask + row0 * p.ldm + kb) : 0u;
        mw1 = (row1 < p.rows) ? __ldg(p.mask + row1 * p.ldm + kb) : 0u;
      }
      mbar_wait(&full[s], ph);
      const float* as = reinterpret_cast<const float*>(smem + (size_t)s * stageBytes);
      const uint32_t bHi = smem_u32(smem + (size_t)s * stageBytes + aBytes), bLo = bHi + bBytes;
      uint32_t fr[TC_BK / 8][2][4];    // A fragments (hi, lo) of every k8 step: live until the MMAs are retired
#pragma unroll
      for (int kk = 0; kk < TC_BK / 8; kk++) {
        // 128B swizzle: 16-byte chunk j of row r sits at chunk j ^ (r & 7); columns 8 kk + t and 8 kk + t + 4
        const int o0 = (((2 * kk) ^ g) << 2) + t, o1 = (((2 * kk + 1) ^ g) << 2) + t;
        float x[4] = {as[rl * TC_BK + o0], as[(rl + 8) * TC_BK + o0], as[rl * TC_BK + o1], as[(rl + 8) * TC_BK + o1]};
        if (masked) {
          const int b0 = 8 * kk + t, b1 = b0 + 4;
          x[0] = ((mw0 >> b0) & 1u) ? x[0] * p.mscale : 0.f;   // == k_dropout
          x[1] = ((mw1 >> b0) & 1u) ? x[1] * p.mscale : 0.f;
          x[2] = ((mw0 >> b1) & 1u) ? x[2] * p.mscale : 0.f;
          x[3] = ((mw1 >> b1) & 1u) ? x[3] * p.mscale : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 4; i++) split_tf32(x[i], fr[kk][0][i], fr[kk][1][i]);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < NC; c++) {
          const uint32_t off = (uint32_t)c * 32u * 128u + (uint32_t)kk * 32u;
          const uint64_t dBh = make_sdesc_sw128(bHi + off), dBl = make_sdesc_sw128(bLo + off);
          wgmma_m64n32k8_tf32(acc[c], fr[kk][1], dBh);
          wgmma_m64n32k8_tf32(acc[c], fr[kk][0], dBl);
          wgmma_m64n32k8_tf32(acc[c], fr[kk][0], dBh);
        }
      }
      wgmma_commit();
      wgmma_wait_all();
      keep_live(fr);
#pragma unroll
      for (int c = 0; c < NC; c++) wgmma_fence_acc(acc[c]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      if (++s == p.stages) { s = 0; ph ^= 1; }
    }
    // epilogue: acc[c][4j + {0,1}] = (row0, col, col + 1), acc[c][4j + {2,3}] = (row1, ...), col = n0 + 32c + 8j + 2t
    const RowDiv rd0 = rowdiv_make(d0), rd1 = rowdiv_make(d1);
#pragma unroll
    for (int c = 0; c < NC; c++)
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int col = n0 + c * 32 + j * 8 + 2 * t;
        tc_store_pair<EPI>(p, row0, col, acc[c][4 * j], acc[c][4 * j + 1], rd0);
        tc_store_pair<EPI>(p, row1, col, acc[c][4 * j + 2], acc[c][4 * j + 3], rd1);
      }
  }
}

// The split weights (W_hi / W_lo, padded) live in a stream-ordered allocation made for this call
// (cudaMallocAsync / cudaFreeAsync on the caller's stream): no process-wide scratch, so the C ABI can be driven
// from several threads, devices and streams at once (the reference's task bodies run one per GPU in one process).

struct TsEpilogue {
  int relu = 0;
  const DropMask* outMask = nullptr;
  const float* reluOf = nullptr; int64_t ldR = 0;
  const uint64_t* rowEnd = nullptr; uint64_t colLeft = 0;
  int accumulate = 0;
};

// the epilogue instantiation that serves `epi`: the combinations the GCN path produces have their own, anything else
// takes the generic kernel (-1)
static int tc_instance(int epi) {
  return (epi == 0 || epi == EPI_NORM || epi == EPI_OMASK || epi == (EPI_OMASK | EPI_RELUOF | EPI_NORM)) ? epi : -1;
}

template <int NC>
static int tc_launch(dim3 grid, size_t smemBytes, int epi, const CUtensorMap& mapA, const CUtensorMap& mapWhi,
                     const CUtensorMap& mapWlo, const TcParams& q, cudaStream_t st) {
  constexpr int E1 = EPI_NORM, E2 = EPI_OMASK, E3 = EPI_OMASK | EPI_RELUOF | EPI_NORM;
  switch (tc_instance(epi)) {
    case 0: return launch_dyn<k_tc_linear<NC, 0>>(grid, TC_THREADS, smemBytes, st, mapA, mapWhi, mapWlo, q);
    case E1: return launch_dyn<k_tc_linear<NC, E1>>(grid, TC_THREADS, smemBytes, st, mapA, mapWhi, mapWlo, q);
    case E2: return launch_dyn<k_tc_linear<NC, E2>>(grid, TC_THREADS, smemBytes, st, mapA, mapWhi, mapWlo, q);
    case E3: return launch_dyn<k_tc_linear<NC, E3>>(grid, TC_THREADS, smemBytes, st, mapA, mapWhi, mapWlo, q);
    default: return launch_dyn<k_tc_linear<NC, -1>>(grid, TC_THREADS, smemBytes, st, mapA, mapWhi, mapWlo, q);
  }
}

// Y[rows][N] (op)= A[rows][K] * B^T with B(n, k) taken from W as k_split_w describes
static int ts_gemm(int64_t rows, int K, int N, const float* A, int64_t ldA, const float* W, int ldW, int transposed,
                   float* Y, int64_t ldY, const DropMask* inMask, const TsEpilogue& e, cudaStream_t st,
                   roc_gemm_info* info) {
  if (K < 8 || N < 1 || rows < 1) return ROC_ERR_UNSUPPORTED;
  if ((ldA % 4) || (ldY % 4) || !aligned16(A) || !aligned16(Y)) return ROC_ERR_UNSUPPORTED;
  if (e.reluOf && ((e.ldR % 4) || !aligned16(e.reluOf))) return ROC_ERR_UNSUPPORTED;
  if (rows > 0x7FFFFF00ll) return ROC_ERR_UNSUPPORTED;   // TMA coordinates are int32
  if (!encode_tiled_fn()) return ROC_ERR_UNSUPPORTED;
  // N-tile of 32, 64 or 128 columns (wgmma chunks of 32): the widest tile streams A once per 128 output columns
  const int NC = (N <= 32) ? 1 : (N <= 64) ? 2 : 4;
  const int BN = 32 * NC;
  const int nTiles = (N + BN - 1) / BN;
  const int Npad = nTiles * BN;
  const int Kpad = (K + TC_BK - 1) / TC_BK * TC_BK;
  const size_t need = (size_t)2 * Npad * Kpad;
  float* wsplit = nullptr;
  ROC_CUDA(cudaMallocAsync((void**)&wsplit, need * sizeof(float), st));
  struct FreeOnExit {   // returned to the pool in stream order, after the GEMM below (or at once on an early return)
    float* p; cudaStream_t s;
    ~FreeOnExit() { if (p) cudaFreeAsync(p, s); }
  } wsplitGuard{wsplit, st};
  float* Whi = wsplit;
  float* Wlo = wsplit + (size_t)Npad * Kpad;
  k_split_w<<<(Npad * Kpad + 255) / 256, 256, 0, st>>>(N, K, Npad, Kpad, ldW, transposed, W, Whi, Wlo);
  ROC_LAUNCH_CHECK();

  CUtensorMap mapA, mapWhi, mapWlo;
  if (!make_tmap_f32_2d(&mapA, A, (uint64_t)rows, (uint64_t)K, (uint64_t)ldA, TC_BM, TC_BK)) return ROC_ERR_UNSUPPORTED;
  if (!make_tmap_f32_2d(&mapWhi, Whi, (uint64_t)Npad, (uint64_t)Kpad, (uint64_t)Kpad, (uint32_t)BN, TC_BK)) return ROC_ERR_UNSUPPORTED;
  if (!make_tmap_f32_2d(&mapWlo, Wlo, (uint64_t)Npad, (uint64_t)Kpad, (uint64_t)Kpad, (uint32_t)BN, TC_BK)) return ROC_ERR_UNSUPPORTED;

  const size_t stageBytes = (size_t)TC_BM * TC_BK * 4 + (size_t)2 * BN * TC_BK * 4;
  const size_t fixedBytes = 1024 /*align*/ + 256 /*barriers*/;
  const int stages = ring_stages(stageBytes, fixedBytes, TC_MAX_STAGES);
  if (!stages) return ROC_ERR_UNSUPPORTED;
  TcParams q{};
  q.Y = Y; q.ldY = ldY; q.rows = rows; q.outDim = N; q.numKb = Kpad / TC_BK; q.stages = stages;
  q.accumulate = e.accumulate;
  if (inMask) { q.mask = inMask->bits; q.ldm = inMask->ld; q.mscale = inMask->scale; }
  q.relu = e.relu;
  if (e.outMask) { q.omask = e.outMask->bits; q.oldm = e.outMask->ld; q.oscale = e.outMask->scale; }
  q.reluOf = e.reluOf; q.ldR = e.ldR;
  q.rowEnd = e.rowEnd; q.colLeft = e.colLeft;
  const size_t smemBytes = (size_t)stages * stageBytes + fixedBytes;
  const int64_t numTiles = (rows + TC_BM - 1) / TC_BM;
  int gx = sm_count() / nTiles;
  if (gx < 1) gx = 1;
  if (numTiles < gx) gx = (int)numTiles;
  dim3 grid((unsigned)gx, (unsigned)nTiles, 1);
  const int epi = (q.relu ? EPI_RELU : 0) | (q.omask ? EPI_OMASK : 0) | (q.reluOf ? EPI_RELUOF : 0) |
                  (q.rowEnd ? EPI_NORM : 0) | (q.accumulate ? EPI_ACC : 0);
  if (info) {
    info->nc = NC; info->epi = tc_instance(epi); info->grid_x = (int)grid.x; info->grid_y = (int)grid.y;
    info->stages = stages;
  }
  switch (NC) {
    case 1: return tc_launch<1>(grid, smemBytes, epi, mapA, mapWhi, mapWlo, q, st);
    case 2: return tc_launch<2>(grid, smemBytes, epi, mapA, mapWhi, mapWlo, q, st);
    default: return tc_launch<4>(grid, smemBytes, epi, mapA, mapWhi, mapWlo, q, st);
  }
}

int tc_linear_fwd(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX, const float* W, float* Y,
                  int64_t ldY, int relu, const uint64_t* rowEnd, uint64_t colLeft, const DropMask* dm,
                  cudaStream_t st, roc_gemm_info* info) {
  TsEpilogue e;
  e.relu = relu; e.rowEnd = rowEnd; e.colLeft = colLeft;
  return ts_gemm(rows, inDim, outDim, X, ldX, W, inDim, 0, Y, ldY, dm, e, st, info);
}

// dX (+)= dY W, optionally followed in the epilogue by the dropout backward of X's producer
int tc_linear_dx(int64_t rows, int inDim, int outDim, const float* dY, int64_t ldDY, const float* W, float* dX,
                 int64_t ldDX, int accumulate, const DropMask* dm, const float* reluOf, int64_t ldR,
                 const uint64_t* rowEnd, uint64_t colLeft, cudaStream_t st, roc_gemm_info* info) {
  TsEpilogue e;
  e.outMask = dm; e.accumulate = accumulate;
  e.reluOf = reluOf; e.ldR = ldR; e.rowEnd = rowEnd; e.colLeft = colLeft;
  return ts_gemm(rows, outDim, inDim, dY, ldDY, W, inDim, 1, dX, ldDX, nullptr, e, st, info);
}

}  // namespace roc
