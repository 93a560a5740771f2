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
//              [dropout mask ->] hi/lo split, per k8 step one wgmma m64n(32 NC)k8 per operand pair,
//              then the epilogue (relu / dropout-backward mask / relu mask / row norm / accumulate)
//              from the accumulator registers; at NC <= 2 a written (not accumulated) Y leaves through
//              a shared-memory staging tile by TMA stores
//   warp 8     TMA producer: per tile the epilogue operands (reluOf boxes and output-mask words, into
//              one of 1 or 2 buffers), then per k-block the A tile [128 rows][32 k] and its input-mask
//              words, with W_hi + W_lo of the k-block when W does not stay resident
// The mainloop keeps two k-blocks of MMAs in flight: the fragments of k-block kb and kb - 1 live in two
// register sets, `wgmma.wait_group 1` after kb's issue retires kb - 1 and frees its stage, and the queue
// drains only at the end of a tile.  The row ends of the norm divisors are loaded a tile ahead of their use,
// so no global load waits in front of an MMA.
// When the CTA's W_hi / W_lo slice (2 * 32 NC * Kpad floats) fits beside the epilogue buffers and a ring
// of TC_RES_MIN_A_BYTES of A, it is loaded once per CTA and the ring carries A alone; otherwise W streams
// through the ring with A, from L2.  A is read once (rows*K*4 bytes, or rows*K*2 for a bf16 A).
// The forward of a leaf bf16 X runs the same kernel with TA = uint16_t (see k_tc_linear).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "tc_common.cuh"

namespace roc {

using namespace tc;

constexpr int TC_BM = 128;        // rows per tile: two consumer warpgroups of 64
constexpr int TC_BK = 32;         // k per k-block: one 128-byte swizzle row of fp32 A and of W, a 64-byte one of bf16 A
constexpr int TC_THREADS = 288;   // 8 consumer warps + 1 producer warp
constexpr int TC_MAX_STAGES = 8;        // ring depth with fp32 A (16 KB of A per stage)
constexpr int TC_MAX_STAGES_BF16 = 12;  // with bf16 A (8 KB per stage)
constexpr int TC_BAR_STAGES = 12;       // full / empty barrier slots: the deeper of the two rings
constexpr size_t TC_RES_MIN_A_BYTES = 64 * 1024;  // A in flight a resident W must leave room for, per SM

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
  const uint32_t* omask; float oscale;                  //   dropout backward: keep ? x * scale : 0 (words by TMA)
  const float* reluOf;                                  //   relu backward: reluOf(row, col) > 0 ? x : 0 (by TMA)
  const uint64_t* rowEnd; uint64_t colLeft;             //   indegree norm: x / sqrtf(deg(row))
  int accumulate;                                       //   Y += x instead of Y = x
  // shared memory (offsets from the 1024-aligned base): [W_hi | W_lo of every k-block when wres] [ring] [epilogue
  // operand buffers] [Y staging tile] [barriers]
  int wres;                                             // W resident: the ring stages carry only A (and mask words)
  uint32_t stageOff, stageBytes, mOff;                  // stage: A [128][32], W_hi + W_lo unless wres, at mOff the
                                                        // input-mask words [128][4] when mask
  uint32_t eOff, eBytes, eMaskOff; int eb;              // eb buffers of eBytes: [NC][128][32] reluOf, [128][4] mask words
  int ystage; uint32_t yOff; int yCols;                 // Y leaves through [NC][128][32] at yOff, columns < yCols by
                                                        // TMA stores
  uint32_t barOff;
};

// Epilogue stage switches: compile-time when the kernel is instantiated for a fixed combination
// (EPI >= 0, a bit mask), read from the parameters for the generic instantiation (EPI < 0, or EPI_GEN with
// EPI_YBF16).  EPI_YBF16 stores Y in bf16 (ROC_LINEAR_Y_BF16): always compile-time, so the fp32 instantiations do not
// change.
enum { EPI_RELU = 1, EPI_OMASK = 2, EPI_RELUOF = 4, EPI_NORM = 8, EPI_ACC = 16, EPI_YBF16 = 32, EPI_GEN = 64 };
#define EPI_FLAGS(EPI, p)                                                        \
  constexpr bool fGen = (EPI) < 0 || ((EPI) & EPI_GEN) != 0;                     \
  constexpr bool fYb = (EPI) >= 0 && ((EPI) & EPI_YBF16) != 0;                   \
  const bool fRelu = fGen ? (p).relu != 0 : ((EPI) & EPI_RELU) != 0;              \
  const bool fOmask = fGen ? (p).omask != nullptr : ((EPI) & EPI_OMASK) != 0;      \
  const bool fReluOf = fGen ? (p).reluOf != nullptr : ((EPI) & EPI_RELUOF) != 0;   \
  const bool fNorm = fGen ? (p).rowEnd != nullptr : ((EPI) & EPI_NORM) != 0;       \
  const bool fAcc = fGen ? (p).accumulate != 0 : ((EPI) & EPI_ACC) != 0;

// b = the low words of the row's (start, end) offsets, so that end - start is its indegree; (0, 1) past the last row
__device__ __forceinline__ void row_bounds(const TcParams& p, int64_t row, uint32_t (&b)[2]) {
  if (!p.rowEnd || row >= p.rows) { b[0] = 0u; b[1] = 1u; return; }
  b[0] = (uint32_t)((row == 0) ? p.colLeft : p.rowEnd[row - 1]);
  b[1] = (uint32_t)p.rowEnd[row];
}
__device__ __forceinline__ float row_norm_divisor(const uint32_t (&b)[2]) { return sqrtf((float)(b[1] - b[0])); }

// Y[row][col, col + 1] (+)= x0, x1 (col even): the accumulator pair a thread holds, after the rest of the epilogue
__device__ __forceinline__ void tc_store_pair(const TcParams& p, bool fAcc, int64_t row, int col, float x0, float x1) {
  if (row >= p.rows || col >= p.outDim) return;
  float* y = p.Y + row * p.ldY + col;
  if (col + 1 < p.outDim) {
    if (fAcc) { const float2 o = *reinterpret_cast<const float2*>(y); x0 = o.x + x0; x1 = o.y + x1; }
    *reinterpret_cast<float2*>(y) = make_float2(x0, x1);
  } else {
    y[0] = fAcc ? y[0] + x0 : x0;
  }
}

// The same for a bf16 Y (EPI_YBF16, never accumulated): each value narrowed by f32_to_bf16_rne
__device__ __forceinline__ uint32_t pack_bf16x2(float x0, float x1) {
  return (uint32_t)f32_to_bf16_rne(x0) | ((uint32_t)f32_to_bf16_rne(x1) << 16);
}
__device__ __forceinline__ void tc_store_pair_bf16(const TcParams& p, int64_t row, int col, float x0, float x1) {
  if (row >= p.rows || col >= p.outDim) return;
  uint16_t* y = reinterpret_cast<uint16_t*>(p.Y) + row * p.ldY + col;
  if (col + 1 < p.outDim) *reinterpret_cast<uint32_t*>(y) = pack_bf16x2(x0, x1);
  else y[0] = f32_to_bf16_rne(x0);
}

__device__ __forceinline__ void wgmma_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// TA: float, or uint16_t for an A in bf16 (the forward of a leaf bf16 X): its [128][32] box has 64-byte rows with the
// 64-byte swizzle, and each element is widened exactly as the fragment is read, so everything after the load is the
// fp32 kernel's arithmetic on A.float().
template <int NC, int EPI, class TA>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_tc_linear(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapWhi,
            const __grid_constant__ CUtensorMap mapWlo, const __grid_constant__ CUtensorMap mapR,
            const __grid_constant__ CUtensorMap mapM, const __grid_constant__ CUtensorMap mapIM,
            const __grid_constant__ CUtensorMap mapY,
            const TcParams p) {
  constexpr int BN = 32 * NC;
  constexpr uint32_t aBytes = TC_BM * TC_BK * sizeof(TA);   // 16 KB (fp32) or 8 KB (bf16) of A per stage
  constexpr uint32_t bBytes = BN * TC_BK * 4;          // one k-block of W_hi (or W_lo)
  constexpr uint32_t rBytes = TC_BM * 32 * 4;          // one 32-column box of reluOf
  EPI_FLAGS(EPI, p)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.barOff);   // [stages] TMA landed
  uint64_t* empty = full + TC_BAR_STAGES;                          // [stages] consumers done
  uint64_t* efull = empty + TC_BAR_STAGES;                         // [eb] epilogue operands landed
  uint64_t* eempty = efull + 2;                                    // [eb] consumers have read them
  uint64_t* wfull = eempty + 2;                                    // resident W landed

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t numTiles = (p.rows + TC_BM - 1) / TC_BM;
  const int n0 = blockIdx.y * BN;          // this CTA's slice of the N (output column) dimension
  const bool masked = p.mask != nullptr;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapA); tma_prefetch_desc(&mapWhi); tma_prefetch_desc(&mapWlo);
    if (fReluOf) tma_prefetch_desc(&mapR);
    if (fOmask) tma_prefetch_desc(&mapM);
    if (masked) tma_prefetch_desc(&mapIM);
    for (int s = 0; s < p.stages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    for (int e = 0; e < p.eb; e++) { mbar_init(&efull[e], 1); mbar_init(&eempty[e], 8); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ================================ TMA producer ================================
    if (p.wres) {
      if (elect_one()) {
        mbar_arrive_expect_tx(wfull, 2u * p.numKb * bBytes);
        for (int kb = 0; kb < p.numKb; kb++) {
          tma_load_2d(smem + (size_t)kb * bBytes, &mapWhi, kb * TC_BK, n0, wfull);
          tma_load_2d(smem + (size_t)(p.numKb + kb) * bBytes, &mapWlo, kb * TC_BK, n0, wfull);
        }
      }
      __syncwarp();
    }
    int s = 0; uint32_t ph = 0;
    int e = 0; uint32_t eph = 0;
    for (int64_t tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
      const int r0 = (int)(tile * TC_BM);
      if (p.eb) {   // the tile's epilogue operands, ahead of its A stages
        mbar_wait(&eempty[e], eph ^ 1);
        if (elect_one()) {
          uint8_t* eb = smem + p.eOff + (size_t)e * p.eBytes;
          mbar_arrive_expect_tx(&efull[e], p.eBytes);
          if (fReluOf)
            for (int c = 0; c < NC; c++) tma_load_2d(eb + c * rBytes, &mapR, n0 + 32 * c, r0, &efull[e]);
          if (fOmask) tma_load_2d(eb + p.eMaskOff, &mapM, n0 / 32, r0, &efull[e]);
        }
        __syncwarp();
        if (++e == p.eb) { e = 0; eph ^= 1; }
      }
      for (int kb = 0; kb < p.numKb; kb++) {
        mbar_wait(&empty[s], ph ^ 1);
        uint8_t* st = smem + p.stageOff + (size_t)s * p.stageBytes;
        if (elect_one()) {
          mbar_arrive_expect_tx(&full[s], p.stageBytes);
          tma_load_2d(st, &mapA, kb * TC_BK, r0, &full[s]);
          // the box starts 16-byte aligned in global memory: words (kb & ~3) .. + 3, of which word kb is used
          if (masked) tma_load_2d(st + p.mOff, &mapIM, kb & ~3, r0, &full[s]);
          if (!p.wres) {
            tma_load_2d(st + aBytes, &mapWhi, kb * TC_BK, n0, &full[s]);
            tma_load_2d(st + aBytes + bBytes, &mapWlo, kb * TC_BK, n0, &full[s]);
          }
        }
        __syncwarp();
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ================================== consumers ===================================
  const int g = lane >> 2, t = lane & 3;
  const int rl = (warp >> 2) * 64 + (warp & 3) * 16 + g;    // tile rows of this thread: rl and rl + 8 (both == g mod 8)
  if (p.wres) mbar_wait(wfull, 0);
  int s = 0; uint32_t ph = 0;
  int e = 0; uint32_t eph = 0;
  // The row ends of the norm divisors are loaded a whole tile ahead of their use, into registers.
  uint32_t nb0[2] = {0u, 1u}, nb1[2] = {0u, 1u};
  if (fNorm) {
    row_bounds(p, (int64_t)blockIdx.x * TC_BM + rl, nb0);
    row_bounds(p, (int64_t)blockIdx.x * TC_BM + rl + 8, nb1);
  }
  uint32_t frA[TC_BK / 8][2][4], frB[TC_BK / 8][2][4] = {};   // A fragments (hi, lo) of two k-blocks in flight
  for (int64_t tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
    const int64_t row0 = tile * TC_BM + rl, row1 = row0 + 8;
    const uint32_t rb0[2] = {nb0[0], nb0[1]}, rb1[2] = {nb1[0], nb1[1]};   // this tile's
    if (fNorm) {
      row_bounds(p, row0 + (int64_t)gridDim.x * TC_BM, nb0);
      row_bounds(p, row1 + (int64_t)gridDim.x * TC_BM, nb1);
    }
    float acc[NC][16];
#pragma unroll
    for (int c = 0; c < NC; c++)
#pragma unroll
      for (int i = 0; i < 16; i++) acc[c][i] = 0.f;
    int sPrev = 0;
    // k-block kb: its A fragments go to `fr`, whose MMAs (k-block kb - 2) retired in the previous step; the MMAs of
    // kb - 1 (fragments in `frPrev`) may run until the wait_group 1 that follows kb's issue, which then frees kb - 1's
    // stage.  The MMA queue drains only at the end of the tile.
    auto body = [&](int kb, uint32_t (&fr)[TC_BK / 8][2][4], uint32_t (&frPrev)[TC_BK / 8][2][4]) {
      mbar_wait(&full[s], ph);
      const uint8_t* st = smem + p.stageOff + (size_t)s * p.stageBytes;
      const TA* as = reinterpret_cast<const TA*>(st);
      const uint32_t bHi = p.wres ? smem_u32(smem + (size_t)kb * bBytes) : smem_u32(st + aBytes);
      const uint32_t bLo = p.wres ? bHi + (uint32_t)p.numKb * bBytes : bHi + bBytes;
      // dropout fused into the operand load: bit c of mask[row][kb] keeps column 32 kb + c ([128][4] words by TMA,
      // with the stage)
      uint32_t mw0 = 0u, mw1 = 0u;
      if (masked) {
        const uint32_t* mw = reinterpret_cast<const uint32_t*>(st + p.mOff);
        mw0 = mw[rl * 4 + (kb & 3)];
        mw1 = mw[(rl + 8) * 4 + (kb & 3)];
      }
#pragma unroll
      for (int kk = 0; kk < TC_BK / 8; kk++) {
        // columns 8 kk + t and 8 kk + t + 4 of rows rl and rl + 8.  fp32, 128B swizzle: 16-byte chunk j of row r sits
        // at chunk j ^ (r & 7).  bf16, 64B swizzle: chunk j (8 elements) of row r at j ^ ((r >> 1) & 3), the same for
        // rl and rl + 8; the 8 rows of a warp then read 8 distinct 4-bank groups
        int o0, o1;
        if constexpr (sizeof(TA) == 4) {
          o0 = (((2 * kk) ^ g) << 2) + t; o1 = (((2 * kk + 1) ^ g) << 2) + t;
        } else {
          o0 = ((kk ^ ((rl >> 1) & 3)) << 3) + t; o1 = o0 + 4;
        }
        float x[4] = {to_f32(as[rl * TC_BK + o0]), to_f32(as[(rl + 8) * TC_BK + o0]), to_f32(as[rl * TC_BK + o1]),
                      to_f32(as[(rl + 8) * TC_BK + o1])};
        if (masked) {
          const int b0 = 8 * kk + t, b1 = b0 + 4;
          x[0] = ((mw0 >> b0) & 1u) ? x[0] * p.mscale : 0.f;   // == k_dropout
          x[1] = ((mw1 >> b0) & 1u) ? x[1] * p.mscale : 0.f;
          x[2] = ((mw0 >> b1) & 1u) ? x[2] * p.mscale : 0.f;
          x[3] = ((mw1 >> b1) & 1u) ? x[3] * p.mscale : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 4; i++) split_tf32(x[i], fr[kk][0][i], fr[kk][1][i]);
      }
      // per k8 step one m64n(32 NC)k8 per operand pair, lo*hi, hi*lo, hi*hi: each element gets the products of its
      // n32 chunk in the same order
#pragma unroll
      for (int kk = 0; kk < TC_BK / 8; kk++) {
        wgmma_fence();
        const uint64_t dBh = make_sdesc_sw128(bHi + kk * 32u), dBl = make_sdesc_sw128(bLo + kk * 32u);
        wgmma_m64nNk8_tf32<NC>(acc, fr[kk][1], dBh);
        wgmma_m64nNk8_tf32<NC>(acc, fr[kk][0], dBl);
        wgmma_m64nNk8_tf32<NC>(acc, fr[kk][0], dBh);
      }
      wgmma_commit();
      wgmma_wait_1();
      keep_live(frPrev);
      if (kb > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[sPrev]);
      }
      sPrev = s;
      if (++s == p.stages) { s = 0; ph ^= 1; }
    };
    for (int kb = 0; kb < p.numKb; kb += 2) {
      body(kb, frA, frB);
      if (kb + 1 < p.numKb) body(kb + 1, frB, frA);
    }
    wgmma_wait_all();
    keep_live(frA);
    keep_live(frB);
#pragma unroll
    for (int c = 0; c < NC; c++) wgmma_fence_acc(acc[c]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[sPrev]);

    // epilogue: acc[c][4j + {0,1}] = (row0, col, col + 1), acc[c][4j + {2,3}] = (row1, ...), col = n0 + 32c + 8j + 2t.
    // The reluOf boxes ([128][32], 128-byte swizzle) and mask words ([128][4]) of the tile are in shared memory.
    const RowDiv rd[2] = {rowdiv_make(row_norm_divisor(rb0)), rowdiv_make(row_norm_divisor(rb1))};
    const float* eo = nullptr;
    const uint32_t* em = nullptr;
    if (p.eb) {
      mbar_wait(&efull[e], eph);
      const uint8_t* eb = smem + p.eOff + (size_t)e * p.eBytes;
      eo = reinterpret_cast<const float*>(eb);
      em = reinterpret_cast<const uint32_t*>(eb + p.eMaskOff);
    }
#pragma unroll
    for (int c = 0; c < NC; c++)
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int r = rl + 8 * h, cc = 8 * j + 2 * t;   // tile row, column in chunk c
          const uint32_t mw = fOmask ? em[r * 4 + c] >> cc : 3u;
          float2 ro = make_float2(1.f, 1.f);
          if (fReluOf) ro = *reinterpret_cast<const float2*>(eo + c * (rBytes / 4) + r * 32 + (((cc >> 2) ^ g) << 2) + (cc & 3));
          float v[2] = {acc[c][4 * j + 2 * h], acc[c][4 * j + 2 * h + 1]};
          const float rov[2] = {ro.x, ro.y};
#pragma unroll
          for (int k = 0; k < 2; k++) {
            float x = v[k];
            if (fRelu) x = relu_nanprop(x);
            if (fOmask) x = ((mw >> k) & 1u) ? x * p.oscale : 0.f;
            if (fReluOf) x = (rov[k] > 0.f) ? x : 0.f;
            if (fNorm) x = rowdiv(x, rd[h]);   // == x / d bit for bit (common.cuh)
            v[k] = x;
          }
          acc[c][4 * j + 2 * h] = v[0];
          acc[c][4 * j + 2 * h + 1] = v[1];
        }
    if (p.eb) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&eempty[e]);
      if (++e == p.eb) { e = 0; eph ^= 1; }
    }
    if (NC <= 2 && p.ystage) {
      // The tile leaves through shared memory: each warpgroup writes its 64 rows of every chunk ([64][32], 128-byte
      // swizzle) and one of its threads stores them by TMA, which skips the rows past Y's last.  The stores run on
      // while the next tile is computed; the buffer is refilled once they have read it.
      const int wg = warp >> 2;
      const bool leader = (threadIdx.x & 127) == 0;
      float* yb = reinterpret_cast<float*>(smem + p.yOff) + wg * 64 * 32;   // chunk c at + c * TC_BM * 32
      uint16_t* ybh = reinterpret_cast<uint16_t*>(smem + p.yOff) + wg * 64 * 32;   // the same for a bf16 Y
      if (leader) bulk_wait_read();
      named_barrier(1 + wg, 128);
#pragma unroll
      for (int c = 0; c < NC; c++)
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const int r = (rl & 63) + 8 * h, cc = 8 * j + 2 * t;
            if constexpr (fYb) {
              // [64][32] bf16, 64-byte rows with the 64-byte swizzle: 16-byte unit j of row r at j ^ ((r >> 1) & 3)
              *reinterpret_cast<uint32_t*>(ybh + c * TC_BM * 32 + r * 32 + ((j ^ ((r >> 1) & 3)) << 3) + 2 * t) =
                  pack_bf16x2(acc[c][4 * j + 2 * h], acc[c][4 * j + 2 * h + 1]);
            } else {
              *reinterpret_cast<float2*>(yb + c * TC_BM * 32 + r * 32 + (((cc >> 2) ^ g) << 2) + (cc & 3)) =
                  make_float2(acc[c][4 * j + 2 * h], acc[c][4 * j + 2 * h + 1]);
            }
          }
      fence_proxy_async_smem();
      named_barrier(1 + wg, 128);
      if (leader) {
        for (int c = 0; c < NC; c++) {
          if constexpr (fYb) tma_store_2d(&mapY, ybh + c * TC_BM * 32, n0 + 32 * c, (int)(tile * TC_BM) + 64 * wg);
          else tma_store_2d(&mapY, yb + c * TC_BM * 32, n0 + 32 * c, (int)(tile * TC_BM) + 64 * wg);
        }
        bulk_commit();
      }
      // The TMA store covers the columns below p.yCols, a multiple of 4 (8 for a bf16 Y): it writes whole 16-byte
      // units, so past a column count that is not such a multiple it would overwrite Y's padding.  The last columns go
      // directly.
#pragma unroll
      for (int c = 0; c < NC; c++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const int col = n0 + c * 32 + j * 8 + 2 * t;
          if (col >= p.yCols) {
            if constexpr (fYb) {
              tc_store_pair_bf16(p, row0, col, acc[c][4 * j], acc[c][4 * j + 1]);
              tc_store_pair_bf16(p, row1, col, acc[c][4 * j + 2], acc[c][4 * j + 3]);
            } else {
              tc_store_pair(p, false, row0, col, acc[c][4 * j], acc[c][4 * j + 1]);
              tc_store_pair(p, false, row1, col, acc[c][4 * j + 2], acc[c][4 * j + 3]);
            }
          }
        }
    } else {
#pragma unroll
      for (int c = 0; c < NC; c++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const int col = n0 + c * 32 + j * 8 + 2 * t;
          if constexpr (fYb) {
            tc_store_pair_bf16(p, row0, col, acc[c][4 * j], acc[c][4 * j + 1]);
            tc_store_pair_bf16(p, row1, col, acc[c][4 * j + 2], acc[c][4 * j + 3]);
          } else {
            tc_store_pair(p, fAcc, row0, col, acc[c][4 * j], acc[c][4 * j + 1]);
            tc_store_pair(p, fAcc, row1, col, acc[c][4 * j + 2], acc[c][4 * j + 3]);
          }
        }
    }
  }
  if (NC <= 2 && p.ystage && (threadIdx.x & 127) == 0) bulk_wait();   // the last stores have landed
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
// takes the generic kernel (-1).  A bf16 Y (a forward) has its own for no epilogue and the norm, and a generic one.
static int tc_instance(int epi) {
  if (epi & EPI_YBF16) {
    const int b = epi & ~EPI_YBF16;
    return EPI_YBF16 | ((b == 0 || b == EPI_NORM) ? b : EPI_GEN);
  }
  return (epi == 0 || epi == EPI_NORM || epi == EPI_OMASK || epi == (EPI_OMASK | EPI_RELUOF | EPI_NORM)) ? epi : -1;
}

struct TcMaps { CUtensorMap A, Whi, Wlo, R, M, IM, Y; };

template <int NC, int EPI, class TA>
static int tc_launch_epi(dim3 grid, size_t smemBytes, const TcMaps& m, const TcParams& q, cudaStream_t st) {
  return launch_dyn<k_tc_linear<NC, EPI, TA>>(grid, TC_THREADS, smemBytes, st, m.A, m.Whi, m.Wlo, m.R, m.M, m.IM, m.Y,
                                              q);
}

template <int NC, class TA>
static int tc_launch(dim3 grid, size_t smemBytes, int epi, const TcMaps& m, const TcParams& q, cudaStream_t st) {
  constexpr int E1 = EPI_NORM, E2 = EPI_OMASK, E3 = EPI_OMASK | EPI_RELUOF | EPI_NORM;
  constexpr int Y0 = EPI_YBF16, Y1 = EPI_YBF16 | EPI_NORM, YG = EPI_YBF16 | EPI_GEN;
  switch (tc_instance(epi)) {   // a bf16 Y: a forward, of an fp32 or a bf16 A
    case Y0: return tc_launch_epi<NC, Y0, TA>(grid, smemBytes, m, q, st);
    case Y1: return tc_launch_epi<NC, Y1, TA>(grid, smemBytes, m, q, st);
    case YG: return tc_launch_epi<NC, YG, TA>(grid, smemBytes, m, q, st);
    default: break;
  }
  if constexpr (sizeof(TA) == 2) {
    // a bf16 A is a leaf X in a forward: its epilogues are relu and the norm, so the dX instantiations are not built
    switch (tc_instance(epi)) {
      case 0: return tc_launch_epi<NC, 0, TA>(grid, smemBytes, m, q, st);
      case E1: return tc_launch_epi<NC, E1, TA>(grid, smemBytes, m, q, st);
      default: return tc_launch_epi<NC, -1, TA>(grid, smemBytes, m, q, st);
    }
  } else {
    switch (tc_instance(epi)) {
      case 0: return tc_launch_epi<NC, 0, TA>(grid, smemBytes, m, q, st);
      case E1: return tc_launch_epi<NC, E1, TA>(grid, smemBytes, m, q, st);
      case E2: return tc_launch_epi<NC, E2, TA>(grid, smemBytes, m, q, st);
      case E3: return tc_launch_epi<NC, E3, TA>(grid, smemBytes, m, q, st);
      default: return tc_launch_epi<NC, -1, TA>(grid, smemBytes, m, q, st);
    }
  }
}

// Y[rows][N] (op)= A[rows][K] * B^T with B(n, k) taken from W as k_split_w describes; A is fp32, or bf16 (raw bits)
// when aBf16; Y likewise with yBf16 (written, never accumulated)
static int ts_gemm(int64_t rows, int K, int N, const void* A, bool aBf16, int64_t ldA, const float* W, int ldW,
                   int transposed, void* Y, bool yBf16, int64_t ldY, const DropMask* inMask, const TsEpilogue& e,
                   cudaStream_t st, roc_gemm_info* info) {
  if (K < 8 || N < 1 || rows < 1) return ROC_ERR_UNSUPPORTED;
  if ((ldA % (aBf16 ? 8 : 4)) || (ldY % (yBf16 ? 8 : 4)) || !aligned16(A) || !aligned16(Y)) return ROC_ERR_UNSUPPORTED;
  if (e.reluOf && ((e.ldR % 4) || !aligned16(e.reluOf))) return ROC_ERR_UNSUPPORTED;
  if (e.outMask && !aligned16(e.outMask->bits)) return ROC_ERR_UNSUPPORTED;   // TMA takes the words [128][4] per tile
  if (inMask && !aligned16(inMask->bits)) return ROC_ERR_UNSUPPORTED;         // and [128][4] per k-block
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

  TcMaps m;
  memset(&m, 0, sizeof(m));
  if (aBf16 ? !make_tmap_bf16_2d(&m.A, static_cast<const uint16_t*>(A), (uint64_t)rows, (uint64_t)K, (uint64_t)ldA,
                                 TC_BM, TC_BK)
            : !make_tmap_f32_2d(&m.A, static_cast<const float*>(A), (uint64_t)rows, (uint64_t)K, (uint64_t)ldA, TC_BM,
                                TC_BK))
    return ROC_ERR_UNSUPPORTED;
  if (!make_tmap_f32_2d(&m.Whi, Whi, (uint64_t)Npad, (uint64_t)Kpad, (uint64_t)Kpad, (uint32_t)BN, TC_BK)) return ROC_ERR_UNSUPPORTED;
  if (!make_tmap_f32_2d(&m.Wlo, Wlo, (uint64_t)Npad, (uint64_t)Kpad, (uint64_t)Kpad, (uint32_t)BN, TC_BK)) return ROC_ERR_UNSUPPORTED;
  if (e.reluOf && !make_tmap_f32_2d(&m.R, e.reluOf, (uint64_t)rows, (uint64_t)N, (uint64_t)e.ldR, TC_BM, 32))
    return ROC_ERR_UNSUPPORTED;
  if (e.outMask && !make_tmap_u32_2d(&m.M, e.outMask->bits, (uint64_t)rows, (uint64_t)e.outMask->ld,
                                     (uint64_t)e.outMask->ld, TC_BM, 4))
    return ROC_ERR_UNSUPPORTED;
  if (inMask && !make_tmap_u32_2d(&m.IM, inMask->bits, (uint64_t)rows, (uint64_t)inMask->ld, (uint64_t)inMask->ld,
                                  TC_BM, 4))
    return ROC_ERR_UNSUPPORTED;
  // Y leaves by TMA stores from a staging tile when it is written, not accumulated, and the tile is <= 64 columns wide
  // (the 128-wide tile keeps its shared memory for the ring).  A bf16 tile is [64][32] with 64-byte rows.
  const int yCols = N & (yBf16 ? ~7 : ~3);
  const bool ystage = !e.accumulate && NC <= 2 && yCols > 0;
  if (ystage && !(yBf16 ? make_tmap_bf16_2d(&m.Y, static_cast<const uint16_t*>(Y), (uint64_t)rows, (uint64_t)yCols,
                                            (uint64_t)ldY, TC_BM / 2, 32)
                        : make_tmap_f32_2d(&m.Y, static_cast<const float*>(Y), (uint64_t)rows, (uint64_t)yCols,
                                           (uint64_t)ldY, TC_BM / 2, 32)))
    return ROC_ERR_UNSUPPORTED;

  // Shared memory: W resident when its slice fits beside both epilogue buffers, the Y staging tile and a ring that
  // holds TC_RES_MIN_A_BYTES of A (4 fp32 stages, 8 bf16 ones); then two epilogue buffers when they leave a ring of 2,
  // else one.  A bf16 stage is half as large, so its ring may be deeper, up to the same bytes of A as fp32's 8 stages.
  const int numKb = Kpad / TC_BK;
  const size_t aBytes = (size_t)TC_BM * TC_BK * (aBf16 ? 2 : 4), bBytes = (size_t)BN * TC_BK * 4;
  const int maxStages = aBf16 ? TC_MAX_STAGES_BF16 : TC_MAX_STAGES;
  const int resMinStages = (int)(TC_RES_MIN_A_BYTES / aBytes);
  const size_t mBytes = inMask ? (size_t)TC_BM * 4 * 4 : 0;
  const size_t wBytes = 2 * (size_t)numKb * bBytes;
  const size_t eBytes = (e.reluOf ? (size_t)TC_BM * BN * 4 : 0) + (e.outMask ? (size_t)TC_BM * 4 * 4 : 0);
  const size_t yBytes = ystage ? (size_t)TC_BM * BN * (yBf16 ? 2 : 4) : 0;
  const size_t fixedBytes = 1024 /*align*/ + 256 /*barriers*/ + yBytes;
  const bool wres = ring_stages(aBytes + mBytes, fixedBytes + wBytes + 2 * eBytes, maxStages) >= resMinStages;
  const size_t stageBytes = aBytes + (wres ? 0 : 2 * bBytes) + mBytes;
  const size_t wUsed = wres ? wBytes : 0;
  const int eb = !eBytes ? 0 : ring_stages(stageBytes, fixedBytes + wUsed + 2 * eBytes, maxStages) ? 2 : 1;
  const int stages = ring_stages(stageBytes, fixedBytes + wUsed + eb * eBytes, maxStages);
  if (!stages) return ROC_ERR_UNSUPPORTED;
  TcParams q{};
  q.Y = static_cast<float*>(Y); q.ldY = ldY; q.rows = rows; q.outDim = N; q.numKb = numKb; q.stages = stages;
  q.accumulate = e.accumulate;
  if (inMask) { q.mask = inMask->bits; q.ldm = inMask->ld; q.mscale = inMask->scale; }
  q.relu = e.relu;
  if (e.outMask) { q.omask = e.outMask->bits; q.oscale = e.outMask->scale; }
  q.reluOf = e.reluOf;
  q.rowEnd = e.rowEnd; q.colLeft = e.colLeft;
  q.wres = wres;
  q.stageOff = (uint32_t)wUsed; q.stageBytes = (uint32_t)stageBytes; q.mOff = (uint32_t)(stageBytes - mBytes);
  q.eOff = q.stageOff + (uint32_t)(stages * stageBytes); q.eBytes = (uint32_t)eBytes; q.eb = eb;
  q.eMaskOff = e.reluOf ? (uint32_t)(TC_BM * BN * 4) : 0u;
  q.ystage = ystage; q.yCols = yCols; q.yOff = q.eOff + (uint32_t)(eb * eBytes);
  q.barOff = q.yOff + (uint32_t)yBytes;
  const size_t smemBytes = (size_t)q.barOff + fixedBytes - yBytes;
  const int64_t numTiles = (rows + TC_BM - 1) / TC_BM;
  int gx = sm_count() / nTiles;
  if (gx < 1) gx = 1;
  if (numTiles < gx) gx = (int)numTiles;
  dim3 grid((unsigned)gx, (unsigned)nTiles, 1);
  const int epi = (q.relu ? EPI_RELU : 0) | (q.omask ? EPI_OMASK : 0) | (q.reluOf ? EPI_RELUOF : 0) |
                  (q.rowEnd ? EPI_NORM : 0) | (q.accumulate ? EPI_ACC : 0) | (yBf16 ? EPI_YBF16 : 0);
  if (info) {
    info->nc = NC; info->epi = tc_instance(epi); info->grid_x = (int)grid.x; info->grid_y = (int)grid.y;
    info->stages = stages; info->w_resident = wres; info->epi_bufs = eb;
  }
  if (aBf16) {
    switch (NC) {
      case 1: return tc_launch<1, uint16_t>(grid, smemBytes, epi, m, q, st);
      case 2: return tc_launch<2, uint16_t>(grid, smemBytes, epi, m, q, st);
      default: return tc_launch<4, uint16_t>(grid, smemBytes, epi, m, q, st);
    }
  }
  switch (NC) {
    case 1: return tc_launch<1, float>(grid, smemBytes, epi, m, q, st);
    case 2: return tc_launch<2, float>(grid, smemBytes, epi, m, q, st);
    default: return tc_launch<4, float>(grid, smemBytes, epi, m, q, st);
  }
}

// X is fp32, or bf16 (raw bits) when xBf16; Y likewise with yBf16
int tc_linear_fwd(int64_t rows, int inDim, int outDim, const void* X, bool xBf16, int64_t ldX, const float* W,
                  void* Y, bool yBf16, int64_t ldY, int relu, const uint64_t* rowEnd, uint64_t colLeft,
                  const DropMask* dm, cudaStream_t st, roc_gemm_info* info) {
  TsEpilogue e;
  e.relu = relu; e.rowEnd = rowEnd; e.colLeft = colLeft;
  return ts_gemm(rows, inDim, outDim, X, xBf16, ldX, W, inDim, 0, Y, yBf16, ldY, dm, e, st, info);
}

// dX (+)= dY W, optionally followed in the epilogue by the dropout backward of X's producer
int tc_linear_dx(int64_t rows, int inDim, int outDim, const float* dY, int64_t ldDY, const float* W, float* dX,
                 int64_t ldDX, int accumulate, const DropMask* dm, const float* reluOf, int64_t ldR,
                 const uint64_t* rowEnd, uint64_t colLeft, cudaStream_t st, roc_gemm_info* info) {
  TsEpilogue e;
  e.outMask = dm; e.accumulate = accumulate;
  e.reluOf = reluOf; e.ldR = ldR; e.rowEnd = rowEnd; e.colLeft = colLeft;
  return ts_gemm(rows, outDim, inDim, dY, false, ldDY, W, inDim, 1, dX, false, ldDX, nullptr, e, st, info);
}

}  // namespace roc
