// layernorm.cu — layer normalisation over the columns of each row of a [rows][H] node tensor for sm_90a
// (roc_layernorm_*): a one-pass forward (with an optional fused relu) and a one-pass backward that also reduces the
// gamma / beta gradients.
//
// A row is held in registers by a row group of S lanes (S a power of two <= 32; 32 / S rows per warp), lane l of the
// group holding the float4 groups l + S j, j < J.  The dispatch on H4 = ceil(H / 4):
//   H4 <= 32         J = 1, S = the smallest power of two >= H4
//   32 < H4 <= 224   S = 32, J = ceil(H4 / 32)                      (H <= 896)
//   H4 > 224         the wide path: one CTA per row, columns looped from memory
// J stops at 7: the backward keeps the row's xhat and gh (8 J floats) and its fp64 column partials (16 J registers)
// live, and at J = 8 that no longer fits in 255 registers without spilling.
// Every row statistic is an fp32 sum taken lane-local in column order and then over the group by an xor butterfly, so
// every lane holds the same bits and the backward recomputes the forward's mean, rstd, xhat and relu mask exactly.
// The gamma / beta partials are fp64 over fixed blocks of LN_BLOCK_ROWS rows, added in block order by bn_column_sum.
// Nothing depends on the grid or the SM count, and nothing uses atomics.
#include "common.cuh"

namespace roc {
namespace {

constexpr int LN_T = 256;                 // threads per CTA
constexpr int LN_WARPS = LN_T / 32;
constexpr int64_t LN_BLOCK_ROWS = 1024;   // rows of one gamma / beta partial: 4 / 1024 of the matrix bytes
constexpr int LN_WIDE_H4 = 224;           // float4 groups a register-held row may have

// rows a row group keeps in flight
template <int J> struct LnUnroll { static constexpr int U = J == 1 ? 4 : J == 2 ? 2 : 1; };

__device__ __forceinline__ float ln_rsqrt(float var, float eps) {
  return __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var, eps)));   // correctly rounded, never rsqrtf
}
__device__ __forceinline__ float ln_xhat(float x, float mu, float rstd) { return __fmul_rn(__fsub_rn(x, mu), rstd); }
// the forward's value before any relu, and the backward's relu test
__device__ __forceinline__ float ln_pre(float xhat, float gamma, float beta) { return __fmaf_rn(xhat, gamma, beta); }

template <int S>
__device__ __forceinline__ float group_sum(float s) {
#pragma unroll
  for (int o = S / 2; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  return s;
}

// The row statistics of a register-held row: mu = sum x / H, var = sum (x - mu)^2 / H, rstd = 1 / sqrt(var + eps).
// li: the lane's index in its group.  Every lane of the group returns the same bits.
template <int S, int J>
__device__ __forceinline__ float2 ln_row_stats(const float4 (&v)[J], int li, int H, float eps) {
  float s = 0.0f;
#pragma unroll
  for (int j = 0; j < J; j++)
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (4 * (li + S * j) + k < H) s = __fadd_rn(s, lane(v[j], k));
  const float mu = __fdiv_rn(group_sum<S>(s), (float)H);
  float q = 0.0f;
#pragma unroll
  for (int j = 0; j < J; j++)
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (4 * (li + S * j) + k < H) {
        const float d = __fsub_rn(lane(v[j], k), mu);
        q = __fmaf_rn(d, d, q);
      }
  return make_float2(mu, ln_rsqrt(__fdiv_rn(group_sum<S>(q), (float)H), eps));
}

// The lane's gamma / beta (0 beyond H): held in registers up to J = 4, re-read (L1-resident) per row beyond, where
// the registers go to the row and the partials.
template <int S, int J>
struct LnAffine {
  static constexpr bool HELD = J <= 4;
  float ga[HELD ? J : 1][4], be[HELD ? J : 1][4];
  const float *gamma, *beta;
  int li, H;
  __device__ __forceinline__ LnAffine(const float* g, const float* b, int l, int h) : gamma(g), beta(b), li(l), H(h) {
    if (HELD)
#pragma unroll
      for (int j = 0; j < (HELD ? J : 1); j++) { load_coef(gamma, li + S * j, H, ga[j]); load_coef(beta, li + S * j, H, be[j]); }
  }
  __device__ __forceinline__ void get(int j, float (&g)[4], float (&b)[4]) const {
    if (HELD) {
#pragma unroll
      for (int k = 0; k < 4; k++) { g[k] = ga[HELD ? j : 0][k]; b[k] = be[HELD ? j : 0][k]; }
    } else {
      load_coef(gamma, li + S * j, H, g);
      load_coef(beta, li + S * j, H, b);
    }
  }
};

// The lane's groups of row r (zeros for a row past the end or a group past H4; pad columns are loaded as they are)
template <int S, int J>
__device__ __forceinline__ void ln_load_row(const float* __restrict__ base, int64_t ld, int64_t r, int64_t rows, int li,
                                            int H4, float4 (&v)[J]) {
#pragma unroll
  for (int j = 0; j < J; j++)
    v[j] = (r < rows && li + S * j < H4) ? ld_stream4(reinterpret_cast<const float4*>(base + r * ld + 4 * (li + S * j)))
                                         : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

// y = relu?(xhat gamma + beta), grid-stride over the rows a warp takes U * 32 / S at a time
template <int S, int J, bool RELU>
__global__ void __launch_bounds__(LN_T, 1)
k_ln_fwd(int64_t rows, int H, const float* __restrict__ x, int64_t ldX, const float* __restrict__ gamma,
         const float* __restrict__ beta, float eps, float* __restrict__ y, int64_t ldY) {
  constexpr int U = LnUnroll<J>::U, RW = 32 / S;   // rows per warp step: U * RW
  const int H4 = (H + 3) / 4, li = threadIdx.x % S, gw = (threadIdx.x % 32) / S, warp = threadIdx.x / 32;
  const LnAffine<S, J> aff(gamma, beta, li, H);
  const int64_t step = (int64_t)gridDim.x * LN_WARPS * U * RW;
  for (int64_t rw = ((int64_t)blockIdx.x * LN_WARPS + warp) * U * RW; rw < rows; rw += step) {
    float4 v[U][J];
#pragma unroll
    for (int u = 0; u < U; u++) ln_load_row<S, J>(x, ldX, rw + u * RW + gw, rows, li, H4, v[u]);
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int64_t r = rw + u * RW + gw;
      const float2 st = ln_row_stats<S, J>(v[u], li, H, eps);
      if (r >= rows) continue;
#pragma unroll
      for (int j = 0; j < J; j++) {
        const int c4 = li + S * j;
        if (c4 >= H4) continue;
        float ga[4], be[4], o[4];
        aff.get(j, ga, be);
#pragma unroll
        for (int k = 0; k < 4; k++) {
          o[k] = ln_pre(ln_xhat(lane(v[u][j], k), st.x, st.y), ga[k], be[k]);
          if (RELU) o[k] = relu_nanprop(o[k]);
        }
        store_group(y + r * ldY, c4, H, make_float4(o[0], o[1], o[2], o[3]));
      }
    }
  }
}

// One CTA per block of LN_BLOCK_ROWS rows.  Per row: g' = dY (masked by the forward's pre-relu value > 0 when RELU),
// gh = g' gamma, dx (+)= rstd (gh - mean gh - xhat mean(gh xhat)); per column, the block's fp64 sums of g' xhat and g'
// go to partial[blockIdx.x][c].  dx == NULL: the partials only.
template <int S, int J, bool RELU, bool ACC>
__global__ void __launch_bounds__(LN_T, 1)
k_ln_bwd(int64_t rows, int H, const float* __restrict__ x, int64_t ldX, const float* __restrict__ g, int64_t ldG,
         const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float* __restrict__ dx,
         int64_t ldDX, double2* __restrict__ partial) {
  constexpr int U = LnUnroll<J>::U, RW = 32 / S;
  __shared__ double2 sh[LN_WARPS][32][4];
  const int H4 = (H + 3) / 4, li = threadIdx.x % S, gw = (threadIdx.x % 32) / S, warp = threadIdx.x / 32;
  const LnAffine<S, J> aff(gamma, beta, li, H);
  double pg[J][4], px[J][4];   // sums of g' and g' xhat over the rows this lane takes, in row order
#pragma unroll
  for (int j = 0; j < J; j++)
#pragma unroll
    for (int k = 0; k < 4; k++) { pg[j][k] = 0.0; px[j][k] = 0.0; }
  // rows relative to the block's first, whose base pointers these become
  const int64_t r0 = (int64_t)blockIdx.x * LN_BLOCK_ROWS;
  const int r1 = (int)min((int64_t)LN_BLOCK_ROWS, rows - r0);
  x += r0 * ldX;
  g += r0 * ldG;
  if (dx) dx += r0 * ldDX;
  for (int rw = warp * U * RW; rw < r1; rw += LN_WARPS * U * RW) {
    // PRE: dx's old values (ov) loaded with x and dY; wider rows load them at the store, short of registers
    constexpr bool PRE = ACC && J <= 4;
    float4 xv[U][J], gv[U][J], ov[PRE ? U : 1][J];
#pragma unroll
    for (int u = 0; u < U; u++) {
      ln_load_row<S, J>(x, ldX, rw + u * RW + gw, r1, li, H4, xv[u]);
      ln_load_row<S, J>(g, ldG, rw + u * RW + gw, r1, li, H4, gv[u]);
      if (PRE && dx)
#pragma unroll
        for (int j = 0; j < J; j++)
          ov[PRE ? u : 0][j] = (rw + u * RW + gw < r1 && li + S * j < H4)
                                   ? *reinterpret_cast<const float4*>(dx + (int64_t)(rw + u * RW + gw) * ldDX +
                                                                      4 * (li + S * j))
                                   : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int r = rw + u * RW + gw;
      const float2 st = ln_row_stats<S, J>(xv[u], li, H, eps);
      // gh and xhat in place of g and x; the row sums of gh and gh xhat
      float a = 0.0f, b = 0.0f;
#pragma unroll
      for (int j = 0; j < J; j++) {
        float xs[4], gs[4], ga[4], be[4];
        aff.get(j, ga, be);
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const bool in = 4 * (li + S * j) + k < H && r < r1;
          const float xh = ln_xhat(lane(xv[u][j], k), st.x, st.y);
          float gk = in ? lane(gv[u][j], k) : 0.0f;
          if (RELU && !(ln_pre(xh, ga[k], be[k]) > 0.0f)) gk = 0.0f;
          const float gh = __fmul_rn(gk, ga[k]);
          if (in) {
            a = __fadd_rn(a, gh);
            b = __fmaf_rn(gh, xh, b);
            pg[j][k] += (double)gk;
            px[j][k] = fma((double)gk, (double)xh, px[j][k]);
          }
          xs[k] = xh; gs[k] = gh;
        }
        xv[u][j] = make_float4(xs[0], xs[1], xs[2], xs[3]);
        gv[u][j] = make_float4(gs[0], gs[1], gs[2], gs[3]);
      }
      const float ma = __fdiv_rn(group_sum<S>(a), (float)H), mb = __fdiv_rn(group_sum<S>(b), (float)H);
      if (!dx || r >= r1) continue;
#pragma unroll
      for (int j = 0; j < J; j++) {
        const int c4 = li + S * j;
        if (c4 >= H4) continue;
        float4 old = PRE ? ov[PRE ? u : 0][j] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (ACC && !PRE) old = *reinterpret_cast<const float4*>(dx + (int64_t)r * ldDX + 4 * c4);
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
          o[k] = __fmul_rn(st.y, __fmaf_rn(-lane(xv[u][j], k), mb, __fsub_rn(lane(gv[u][j], k), ma)));
          if (ACC) o[k] = __fadd_rn(lane(old, k), o[k]);
        }
        store_group(dx + (int64_t)r * ldDX, c4, H, make_float4(o[0], o[1], o[2], o[3]));
      }
    }
  }
  // the block's column sums: the row groups of a warp by an xor butterfly over the lanes >= S, then the warps in order
#pragma unroll
  for (int j = 0; j < J; j++) {
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
      for (int o = S; o < 32; o <<= 1) {
        pg[j][k] += __shfl_xor_sync(0xffffffffu, pg[j][k], o);
        px[j][k] += __shfl_xor_sync(0xffffffffu, px[j][k], o);
      }
    if (threadIdx.x % 32 < S)
#pragma unroll
      for (int k = 0; k < 4; k++) sh[warp][li][k] = make_double2(px[j][k], pg[j][k]);
    __syncthreads();
    if (threadIdx.x < 4 * S) {
      const int l = threadIdx.x / 4, k = threadIdx.x % 4, c = 4 * (l + S * j) + k;
      double2 t = sh[0][l][k];
      for (int w = 1; w < LN_WARPS; w++) { t.x += sh[w][l][k].x; t.y += sh[w][l][k].y; }
      if (c < H) partial[(int64_t)blockIdx.x * H + c] = t;
    }
    __syncthreads();
  }
}

// ---- the wide path (H > 4 * LN_WIDE_H4): one CTA per row, thread t taking the float4 groups t, t + LN_T, ... from
//      memory in every pass; the row sums are lane-local in column order, a butterfly per warp, then the warps in order.
__device__ __forceinline__ float cta_sum(float s, float* red) {
  s = group_sum<32>(s);
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = s;
  __syncthreads();
  float t = red[0];
  for (int w = 1; w < LN_WARPS; w++) t = __fadd_rn(t, red[w]);
  __syncthreads();
  return t;
}
__device__ __forceinline__ float4 ld_group(const float* row, int c4) {
  return *reinterpret_cast<const float4*>(row + 4 * c4);
}
__device__ float2 ln_wide_stats(const float* row, int H, float eps, float* red) {
  const int H4 = (H + 3) / 4;
  float s = 0.0f;
  for (int c4 = threadIdx.x; c4 < H4; c4 += LN_T) {
    const float4 v = ld_group(row, c4);
    for (int k = 0; k < 4 && 4 * c4 + k < H; k++) s = __fadd_rn(s, lane(v, k));
  }
  const float mu = __fdiv_rn(cta_sum(s, red), (float)H);
  float q = 0.0f;
  for (int c4 = threadIdx.x; c4 < H4; c4 += LN_T) {
    const float4 v = ld_group(row, c4);
    for (int k = 0; k < 4 && 4 * c4 + k < H; k++) {
      const float d = __fsub_rn(lane(v, k), mu);
      q = __fmaf_rn(d, d, q);
    }
  }
  return make_float2(mu, ln_rsqrt(__fdiv_rn(cta_sum(q, red), (float)H), eps));
}

template <bool RELU>
__global__ void __launch_bounds__(LN_T)
k_ln_fwd_wide(int64_t rows, int H, const float* __restrict__ x, int64_t ldX, const float* __restrict__ gamma,
              const float* __restrict__ beta, float eps, float* __restrict__ y, int64_t ldY) {
  __shared__ float red[LN_WARPS];
  const int H4 = (H + 3) / 4;
  for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
    const float* row = x + r * ldX;
    const float2 st = ln_wide_stats(row, H, eps, red);
    for (int c4 = threadIdx.x; c4 < H4; c4 += LN_T) {
      const float4 v = ld_group(row, c4);
      float ga[4], be[4], o[4];
      load_coef(gamma, c4, H, ga);
      load_coef(beta, c4, H, be);
#pragma unroll
      for (int k = 0; k < 4; k++) {
        o[k] = ln_pre(ln_xhat(lane(v, k), st.x, st.y), ga[k], be[k]);
        if (RELU) o[k] = relu_nanprop(o[k]);
      }
      store_group(y + r * ldY, c4, H, make_float4(o[0], o[1], o[2], o[3]));
    }
  }
}

// One CTA per block of LN_BLOCK_ROWS rows; thread t keeps the partials of its own columns in partial[blockIdx.x].
template <bool RELU, bool ACC>
__global__ void __launch_bounds__(LN_T)
k_ln_bwd_wide(int64_t rows, int H, const float* __restrict__ x, int64_t ldX, const float* __restrict__ g, int64_t ldG,
              const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float* __restrict__ dx,
              int64_t ldDX, double2* __restrict__ partial) {
  __shared__ float red[LN_WARPS];
  const int H4 = (H + 3) / 4;
  double2* part = partial + (int64_t)blockIdx.x * H;
  for (int c4 = threadIdx.x; c4 < H4; c4 += LN_T)
    for (int k = 0; k < 4 && 4 * c4 + k < H; k++) part[4 * c4 + k] = make_double2(0.0, 0.0);
  const int64_t r0 = (int64_t)blockIdx.x * LN_BLOCK_ROWS;
  const int64_t r1 = min(r0 + LN_BLOCK_ROWS, rows);
  for (int64_t r = r0; r < r1; r++) {
    const float* row = x + r * ldX;
    const float* grow = g + r * ldG;
    const float2 st = ln_wide_stats(row, H, eps, red);
    float a = 0.0f, b = 0.0f;
    for (int c4 = threadIdx.x; c4 < H4; c4 += LN_T) {
      const float4 v = ld_group(row, c4), gv = ld_group(grow, c4);
      float ga[4], be[4];
      load_coef(gamma, c4, H, ga);
      load_coef(beta, c4, H, be);
      for (int k = 0; k < 4 && 4 * c4 + k < H; k++) {
        const float xh = ln_xhat(lane(v, k), st.x, st.y);
        float gk = lane(gv, k);
        if (RELU && !(ln_pre(xh, ga[k], be[k]) > 0.0f)) gk = 0.0f;
        const float gh = __fmul_rn(gk, ga[k]);
        a = __fadd_rn(a, gh);
        b = __fmaf_rn(gh, xh, b);
        double2 p = part[4 * c4 + k];
        p.x = fma((double)gk, (double)xh, p.x);
        p.y += (double)gk;
        part[4 * c4 + k] = p;
      }
    }
    const float ma = __fdiv_rn(cta_sum(a, red), (float)H), mb = __fdiv_rn(cta_sum(b, red), (float)H);
    if (!dx) continue;
    for (int c4 = threadIdx.x; c4 < H4; c4 += LN_T) {
      const float4 v = ld_group(row, c4), gv = ld_group(grow, c4);
      float4 old = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      if (ACC) old = ld_group(dx + r * ldDX, c4);
      float ga[4], be[4], o[4];
      load_coef(gamma, c4, H, ga);
      load_coef(beta, c4, H, be);
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const float xh = ln_xhat(lane(v, k), st.x, st.y);
        float gk = lane(gv, k);
        if (RELU && !(ln_pre(xh, ga[k], be[k]) > 0.0f)) gk = 0.0f;
        o[k] = __fmul_rn(st.y, __fmaf_rn(-xh, mb, __fsub_rn(__fmul_rn(gk, ga[k]), ma)));
        if (ACC) o[k] = __fadd_rn(lane(old, k), o[k]);
      }
      store_group(dx + r * ldDX, c4, H, make_float4(o[0], o[1], o[2], o[3]));
    }
  }
}

// dGamma[c], dBeta[c] from the partials of column blockIdx.x (rowBlocks = 0: zeros)
__global__ void __launch_bounds__(BN_FIN_T)
k_ln_finalize(int H, int64_t rowBlocks, const double2* __restrict__ partial, float* dGamma, float* dBeta) {
  const int c = blockIdx.x;
  const double2 t = bn_column_sum(partial, rowBlocks, H, c);
  if (threadIdx.x != 0) return;
  dGamma[c] = (float)t.x;
  dBeta[c] = (float)t.y;
}

struct LnShape {
  int S, J;   // J = 0: the wide path
};
LnShape ln_shape(int H) {
  const int H4 = (H + 3) / 4;
  if (H4 > LN_WIDE_H4) return {32, 0};
  if (H4 > 32) return {32, (H4 + 31) / 32};
  int S = 1;
  while (S < H4) S *= 2;
  return {S, 1};
}
int64_t ln_row_blocks(int64_t rows) { return (rows + LN_BLOCK_ROWS - 1) / LN_BLOCK_ROWS; }

// the forward's grid: rows / (rows per CTA step), at most 8 CTAs per SM
unsigned ln_fwd_grid(int64_t rows, int64_t rowsPerCta) {
  int64_t want = (rows + rowsPerCta - 1) / rowsPerCta;
  const int64_t cap = (int64_t)sm_count() * 8;
  return (unsigned)(want > cap ? cap : want < 1 ? 1 : want);
}

struct FwdArgs {
  int64_t rows; int H; const float* x; int64_t ldX; const float* gamma; const float* beta; float eps; float* y;
  int64_t ldY;
};
template <int S, int J, bool RELU>
void fwd_launch(const FwdArgs& a, cudaStream_t st) {
  constexpr int U = LnUnroll<J>::U;
  k_ln_fwd<S, J, RELU><<<ln_fwd_grid(a.rows, (int64_t)LN_T / S * U), LN_T, 0, st>>>(a.rows, a.H, a.x, a.ldX, a.gamma,
                                                                                   a.beta, a.eps, a.y, a.ldY);
}
template <bool RELU>
void fwd_dispatch(const LnShape& s, const FwdArgs& a, cudaStream_t st) {
  switch (s.J) {
    case 0: k_ln_fwd_wide<RELU><<<ln_fwd_grid(a.rows, 1), LN_T, 0, st>>>(a.rows, a.H, a.x, a.ldX, a.gamma, a.beta,
                                                                         a.eps, a.y, a.ldY); return;
    case 1:
      switch (s.S) {
        case 1: fwd_launch<1, 1, RELU>(a, st); return;
        case 2: fwd_launch<2, 1, RELU>(a, st); return;
        case 4: fwd_launch<4, 1, RELU>(a, st); return;
        case 8: fwd_launch<8, 1, RELU>(a, st); return;
        case 16: fwd_launch<16, 1, RELU>(a, st); return;
        default: fwd_launch<32, 1, RELU>(a, st); return;
      }
    case 2: fwd_launch<32, 2, RELU>(a, st); return;
    case 3: fwd_launch<32, 3, RELU>(a, st); return;
    case 4: fwd_launch<32, 4, RELU>(a, st); return;
    case 5: fwd_launch<32, 5, RELU>(a, st); return;
    case 6: fwd_launch<32, 6, RELU>(a, st); return;
    default: fwd_launch<32, 7, RELU>(a, st); return;
  }
}

struct BwdArgs {
  int64_t rows; int H; const float* x; int64_t ldX; const float* g; int64_t ldG; const float* gamma;
  const float* beta; float eps; float* dx; int64_t ldDX; double2* partial;
};
template <int S, int J, bool RELU, bool ACC>
void bwd_launch(const BwdArgs& a, cudaStream_t st) {
  k_ln_bwd<S, J, RELU, ACC><<<(unsigned)ln_row_blocks(a.rows), LN_T, 0, st>>>(
      a.rows, a.H, a.x, a.ldX, a.g, a.ldG, a.gamma, a.beta, a.eps, a.dx, a.ldDX, a.partial);
}
template <bool RELU, bool ACC>
void bwd_dispatch(const LnShape& s, const BwdArgs& a, cudaStream_t st) {
  switch (s.J) {
    case 0: k_ln_bwd_wide<RELU, ACC><<<(unsigned)ln_row_blocks(a.rows), LN_T, 0, st>>>(
                a.rows, a.H, a.x, a.ldX, a.g, a.ldG, a.gamma, a.beta, a.eps, a.dx, a.ldDX, a.partial); return;
    case 1:
      switch (s.S) {
        case 1: bwd_launch<1, 1, RELU, ACC>(a, st); return;
        case 2: bwd_launch<2, 1, RELU, ACC>(a, st); return;
        case 4: bwd_launch<4, 1, RELU, ACC>(a, st); return;
        case 8: bwd_launch<8, 1, RELU, ACC>(a, st); return;
        case 16: bwd_launch<16, 1, RELU, ACC>(a, st); return;
        default: bwd_launch<32, 1, RELU, ACC>(a, st); return;
      }
    case 2: bwd_launch<32, 2, RELU, ACC>(a, st); return;
    case 3: bwd_launch<32, 3, RELU, ACC>(a, st); return;
    case 4: bwd_launch<32, 4, RELU, ACC>(a, st); return;
    case 5: bwd_launch<32, 5, RELU, ACC>(a, st); return;
    case 6: bwd_launch<32, 6, RELU, ACC>(a, st); return;
    default: bwd_launch<32, 7, RELU, ACC>(a, st); return;
  }
}

inline bool rows16(const float* p, int64_t ld) { return aligned16(p) && ld % 4 == 0; }
inline bool eps_ok(float eps) { return eps >= 0.0f && eps <= 3.402823466e38f; }

}  // namespace
}  // namespace roc

using namespace roc;

extern "C" size_t roc_layernorm_workspace_bytes(int64_t rows, int H) {
  if (rows < 0 || H <= 0) return 0;
  const int64_t blocks = ln_row_blocks(rows);
  return (size_t)(blocks > 0 ? blocks : 1) * (size_t)H * sizeof(double2);
}

extern "C" int roc_layernorm_fwd(int64_t rows, int H, const float* x, int64_t ldX, const float* gamma,
                                 const float* beta, float eps, int relu, float* y, int64_t ldY, roc_stream_t stream) {
  if (!x || !gamma || !beta || !y || rows < 0 || H <= 0 || ldX < H || ldY < H) return ROC_ERR_INVALID;
  if (!rows16(x, ldX) || !rows16(y, ldY) || !eps_ok(eps)) return ROC_ERR_INVALID;
  if (rows == 0) return ROC_OK;
  cudaStream_t st = as_stream(stream);
  const FwdArgs a{rows, H, x, ldX, gamma, beta, eps, y, ldY};
  if (relu) fwd_dispatch<true>(ln_shape(H), a, st);
  else fwd_dispatch<false>(ln_shape(H), a, st);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

extern "C" int roc_layernorm_bwd(int64_t rows, int H, const float* x, int64_t ldX, const float* dY, int64_t ldDY,
                                 int relu, const float* gamma, const float* beta, float eps, float* dGamma,
                                 float* dBeta, float* dX, int64_t ldDX, int accumulate, void* workspace,
                                 size_t workspaceBytes, roc_stream_t stream) {
  if (!x || !dY || !gamma || !beta || !dGamma || !dBeta || !workspace) return ROC_ERR_INVALID;
  if (rows < 0 || H <= 0 || ldX < H || ldDY < H || (dX && ldDX < H) || !eps_ok(eps)) return ROC_ERR_INVALID;
  if (!rows16(x, ldX) || !rows16(dY, ldDY) || (dX && !rows16(dX, ldDX)) || !aligned16(workspace)) return ROC_ERR_INVALID;
  if (workspaceBytes < roc_layernorm_workspace_bytes(rows, H)) return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  double2* partial = static_cast<double2*>(workspace);
  if (rows > 0) {
    const BwdArgs a{rows, H, x, ldX, dY, ldDY, gamma, beta, eps, dX, ldDX, partial};
    const LnShape s = ln_shape(H);
    if (relu && accumulate) bwd_dispatch<true, true>(s, a, st);
    else if (relu) bwd_dispatch<true, false>(s, a, st);
    else if (accumulate) bwd_dispatch<false, true>(s, a, st);
    else bwd_dispatch<false, false>(s, a, st);
    ROC_LAUNCH_CHECK();
  }
  k_ln_finalize<<<H, BN_FIN_T, 0, st>>>(H, ln_row_blocks(rows), partial, dGamma, dBeta);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}
