// batchnorm.cu — batch normalisation over the rows of a [rows][H] node tensor for sm_90a (roc_batchnorm_*):
// per-column statistics, the normalise pass (with an optional fused relu) and the backward.
//
// Every pass lays a CTA out as TX column groups of 4 columns (one 16-byte access each) by TY row lanes, TX * TY <= 256.
// The reductions cut the rows into fixed blocks of BN_ROWS_PER_LANE * TY rows, a function of (rows, H) only; a thread
// sums its rows in order, the CTA adds its lanes in lane order, and a finalize adds the blocks' fp64 partials in block
// order.  So the bits of every result depend on the inputs and the shape alone, never on the card or the launch.
#include "common.cuh"

namespace roc {
namespace {

constexpr int BN_T = 256;               // threads per CTA (at most)
constexpr int BN_MAX_TX = 64;           // column groups per CTA: 256 columns
constexpr int BN_ROWS_PER_LANE = 128;   // rows a thread sums in one reduction block
constexpr int BN_UNROLL = 4;            // rows in flight per thread

struct BnShape {
  int H4, TX, TY, colBlocks;
  int64_t blockRows, rowBlocks;
};
BnShape bn_shape(int64_t rows, int H) {
  BnShape s;
  s.H4 = (H + 3) / 4;
  s.TX = s.H4 < BN_MAX_TX ? s.H4 : BN_MAX_TX;
  s.TY = BN_T / s.TX;
  s.colBlocks = (s.H4 + s.TX - 1) / s.TX;
  s.blockRows = (int64_t)BN_ROWS_PER_LANE * s.TY;
  s.rowBlocks = rows > 0 ? (rows + s.blockRows - 1) / s.blockRows : 1;
  return s;
}
// workspace: 3 coefficient rows of round_up4(H) floats (the backward's A, B, C; inference's a, b), then the
// reduction partials, double2 [rowBlocks][H]
size_t bn_coef_bytes(int H) { return ((size_t)3 * ((H + 3) / 4 * 4) * sizeof(float) + 255) / 256 * 256; }

// One reduction block of rows per blockIdx.x, one group of TX column groups per blockIdx.y.
//  forward:  s = sum (x - K), q = sum (x - K)^2 with K = x[0][c]
//  backward: s = sum g', q = sum g' (x - mean), g' = g masked by fma(x, a, b) > 0 when RELU
// partial[blockIdx.x][c] = (s, q) for c < H.
template <bool BWD, bool RELU>
__global__ void __launch_bounds__(BN_T)
k_bn_reduce(int64_t rows, int H, int64_t blockRows, const float* __restrict__ x, int64_t ldX,
            const float* __restrict__ g, int64_t ldG, const float* __restrict__ sa, const float* __restrict__ sb,
            const double* __restrict__ mean, double2* __restrict__ partial) {
  extern __shared__ double sh[];   // [TY][TX][8]
  const int TX = blockDim.x, TY = blockDim.y, tx = threadIdx.x, ty = threadIdx.y;
  const int c4 = blockIdx.y * TX + tx;
  const bool active = 4 * c4 < H;
  const int64_t r0 = (int64_t)blockIdx.x * blockRows;
  const int64_t r1 = min(r0 + blockRows, rows);
  double K[4], s[4], q[4];
  float a[4], b[4];
#pragma unroll
  for (int k = 0; k < 4; k++) { s[k] = 0.0; q[k] = 0.0; K[k] = 0.0; a[k] = 0.0f; b[k] = 0.0f; }
  if (active) {
    if (BWD) {
#pragma unroll
      for (int k = 0; k < 4; k++) K[k] = (4 * c4 + k < H) ? mean[4 * c4 + k] : 0.0;
      if (RELU) { load_coef(sa, c4, H, a); load_coef(sb, c4, H, b); }
    } else {
      const float4 k0 = *reinterpret_cast<const float4*>(x + 4 * c4);
      K[0] = k0.x; K[1] = k0.y; K[2] = k0.z; K[3] = k0.w;
    }
    for (int64_t r = r0 + ty; r < r1; r += (int64_t)BN_UNROLL * TY) {
      float4 xv[BN_UNROLL], gv[BN_UNROLL];
#pragma unroll
      for (int u = 0; u < BN_UNROLL; u++) {
        const int64_t rr = r + (int64_t)u * TY;
        if (rr < r1) {
          xv[u] = ld_stream4(reinterpret_cast<const float4*>(x + rr * ldX + 4 * c4));
          if (BWD) gv[u] = ld_stream4(reinterpret_cast<const float4*>(g + rr * ldG + 4 * c4));
        }
      }
#pragma unroll
      for (int u = 0; u < BN_UNROLL; u++) {
        if (r + (int64_t)u * TY >= r1) break;
        if (BWD) {
          const float4 z = fma4(xv[u], a, b);
#pragma unroll
          for (int k = 0; k < 4; k++) {
            float gk = lane(gv[u], k);
            if (RELU) gk = lane(z, k) > 0.0f ? gk : 0.0f;
            const double d = (double)lane(xv[u], k) - K[k];
            s[k] += (double)gk;
            q[k] = fma((double)gk, d, q[k]);
          }
        } else {
#pragma unroll
          for (int k = 0; k < 4; k++) {
            const double d = (double)lane(xv[u], k) - K[k];
            s[k] += d;
            q[k] = fma(d, d, q[k]);
          }
        }
      }
    }
  }
  double* mine = sh + ((size_t)ty * TX + tx) * 8;
#pragma unroll
  for (int k = 0; k < 4; k++) { mine[k] = s[k]; mine[4 + k] = q[k]; }
  __syncthreads();
  if (ty != 0 || !active) return;
  for (int l = 1; l < TY; l++) {   // lanes in order
    const double* o = sh + ((size_t)l * TX + tx) * 8;
#pragma unroll
    for (int k = 0; k < 4; k++) { s[k] += o[k]; q[k] += o[4 + k]; }
  }
#pragma unroll
  for (int k = 0; k < 4; k++)
    if (4 * c4 + k < H) partial[(int64_t)blockIdx.x * H + 4 * c4 + k] = make_double2(s[k], q[k]);
}

// training forward: batch statistics of column blockIdx.x, running statistics, and the affine map a, b
__global__ void __launch_bounds__(BN_FIN_T)
k_bn_finalize_fwd(int64_t rows, int H, int64_t rowBlocks, const double2* __restrict__ partial,
                  const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                  double eps, double momentum, float* runMean, float* runVar, float* saveA, float* saveB,
                  double* saveMean, double* saveInvStd) {
  const int c = blockIdx.x;
  const double2 t = bn_column_sum(partial, rowBlocks, H, c);
  if (threadIdx.x != 0) return;
  const double n = (double)rows;
  const double dm = t.x / n;
  const double mean = (double)x[c] + dm;
  const double var = fmax(t.y / n - dm * dm, 0.0);
  const double invstd = 1.0 / sqrt(var + eps);
  const double a = (double)gamma[c] * invstd;
  saveA[c] = (float)a;
  saveB[c] = (float)((double)beta[c] - mean * a);
  saveMean[c] = mean;
  saveInvStd[c] = invstd;
  if (runMean) {
    runMean[c] = (float)((1.0 - momentum) * (double)runMean[c] + momentum * mean);
    runVar[c] = (float)((1.0 - momentum) * (double)runVar[c] + momentum * var * n / (n - 1.0));
  }
}

// inference: the affine map from the running statistics
__global__ void k_bn_finalize_infer(int H, const float* __restrict__ gamma, const float* __restrict__ beta, double eps,
                                    const float* __restrict__ runMean, const float* __restrict__ runVar,
                                    float* __restrict__ a, float* __restrict__ b) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  const double ac = (double)gamma[c] / sqrt((double)runVar[c] + eps);
  a[c] = (float)ac;
  b[c] = (float)((double)beta[c] - (double)runMean[c] * ac);
}

// backward: dgamma, dbeta of column blockIdx.x, and dx = A g' + B x + C
__global__ void __launch_bounds__(BN_FIN_T)
k_bn_finalize_bwd(int64_t rows, int H, int64_t rowBlocks, const double2* __restrict__ partial,
                  const float* __restrict__ gamma, const double* __restrict__ saveMean,
                  const double* __restrict__ saveInvStd, float* dGamma, float* dBeta, float* coefA, float* coefB,
                  float* coefC) {
  const int c = blockIdx.x;
  const double2 t = bn_column_sum(partial, rowBlocks, H, c);
  if (threadIdx.x != 0) return;
  const double n = (double)rows, s = saveInvStd[c];
  const double dbeta = t.x, dgamma = t.y * s;
  dGamma[c] = (float)dgamma;
  dBeta[c] = (float)dbeta;
  if (!coefA) return;
  const double A = (double)gamma[c] * s;
  const double B = -A * s * dgamma / n;
  coefA[c] = (float)A;
  coefB[c] = (float)B;
  coefC[c] = (float)(-A * dbeta / n - B * saveMean[c]);
}

// y = relu?(fma(x, a, b)), grid-stride over rows
template <bool RELU>
__global__ void __launch_bounds__(BN_T)
k_bn_normalise(int64_t rows, int H, const float* __restrict__ x, int64_t ldX, const float* __restrict__ pa,
               const float* __restrict__ pb, float* __restrict__ y, int64_t ldY) {
  const int TY = blockDim.y;
  const int c4 = blockIdx.y * blockDim.x + threadIdx.x;
  if (4 * c4 >= H) return;
  float a[4], b[4];
  load_coef(pa, c4, H, a);
  load_coef(pb, c4, H, b);
  const int64_t step = (int64_t)gridDim.x * TY;
  for (int64_t r = (int64_t)blockIdx.x * TY + threadIdx.y; r < rows; r += step * BN_UNROLL) {
    float4 xv[BN_UNROLL];
#pragma unroll
    for (int u = 0; u < BN_UNROLL; u++)
      if (r + u * step < rows) xv[u] = ld_stream4(reinterpret_cast<const float4*>(x + (r + u * step) * ldX + 4 * c4));
#pragma unroll
    for (int u = 0; u < BN_UNROLL; u++) {
      if (r + u * step >= rows) break;
      float4 v = fma4(xv[u], a, b);
      if (RELU) { v.x = relu_nanprop(v.x); v.y = relu_nanprop(v.y); v.z = relu_nanprop(v.z); v.w = relu_nanprop(v.w); }
      store_group(y + (r + u * step) * ldY, c4, H, v);
    }
  }
}

// dx (+)= fma(A, g', fma(B, x, C)), g' = g masked by fma(x, a, b) > 0 when RELU
template <bool RELU, bool ACC>
__global__ void __launch_bounds__(BN_T)
k_bn_backward_apply(int64_t rows, int H, const float* __restrict__ x, int64_t ldX, const float* __restrict__ g,
                    int64_t ldG, const float* __restrict__ sa, const float* __restrict__ sb,
                    const float* __restrict__ coef, int64_t ldCoef, float* __restrict__ dx, int64_t ldDX) {
  const int TY = blockDim.y;
  const int c4 = blockIdx.y * blockDim.x + threadIdx.x;
  if (4 * c4 >= H) return;
  float A[4], B[4], Cc[4], a[4], b[4];
  load_coef(coef, c4, H, A);
  load_coef(coef + ldCoef, c4, H, B);
  load_coef(coef + 2 * ldCoef, c4, H, Cc);
  if (RELU) { load_coef(sa, c4, H, a); load_coef(sb, c4, H, b); }
  const int64_t step = (int64_t)gridDim.x * TY;
  for (int64_t r = (int64_t)blockIdx.x * TY + threadIdx.y; r < rows; r += step * BN_UNROLL) {
    float4 xv[BN_UNROLL], gv[BN_UNROLL], ov[BN_UNROLL];
#pragma unroll
    for (int u = 0; u < BN_UNROLL; u++) {
      const int64_t rr = r + u * step;
      if (rr < rows) {
        xv[u] = ld_stream4(reinterpret_cast<const float4*>(x + rr * ldX + 4 * c4));
        gv[u] = ld_stream4(reinterpret_cast<const float4*>(g + rr * ldG + 4 * c4));
        if (ACC) ov[u] = *reinterpret_cast<const float4*>(dx + rr * ldDX + 4 * c4);
      }
    }
#pragma unroll
    for (int u = 0; u < BN_UNROLL; u++) {
      if (r + u * step >= rows) break;
      float o[4];
      const float4 z = fma4(xv[u], a, b);
#pragma unroll
      for (int k = 0; k < 4; k++) {
        float gk = lane(gv[u], k);
        if (RELU) gk = lane(z, k) > 0.0f ? gk : 0.0f;
        o[k] = __fmaf_rn(A[k], gk, __fmaf_rn(B[k], lane(xv[u], k), Cc[k]));
        if (ACC) o[k] += lane(ov[u], k);
      }
      store_group(dx + (r + u * step) * ldDX, c4, H, make_float4(o[0], o[1], o[2], o[3]));
    }
  }
}

inline bool rows16(const float* p, int64_t ld) { return aligned16(p) && ld % 4 == 0; }

// grid of the streaming passes: row lanes over blockIdx.x (grid-stride), column groups over blockIdx.y
dim3 stream_grid(const BnShape& s, int64_t rows) {
  int64_t want = (rows + (int64_t)s.TY * BN_UNROLL - 1) / ((int64_t)s.TY * BN_UNROLL);
  const int64_t cap = (int64_t)sm_count() * 8;
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  return dim3((unsigned)want, (unsigned)s.colBlocks);
}

template <bool BWD>
int launch_reduce(const BnShape& s, int64_t rows, int H, const float* x, int64_t ldX, const float* g, int64_t ldG,
                  int relu, const float* sa, const float* sb, const double* mean, double2* partial, cudaStream_t st) {
  const dim3 grid((unsigned)s.rowBlocks, (unsigned)s.colBlocks), block((unsigned)s.TX, (unsigned)s.TY);
  const size_t smem = (size_t)s.TX * s.TY * 8 * sizeof(double);
  if (BWD && relu)
    k_bn_reduce<true, true><<<grid, block, smem, st>>>(rows, H, s.blockRows, x, ldX, g, ldG, sa, sb, mean, partial);
  else
    k_bn_reduce<BWD, false><<<grid, block, smem, st>>>(rows, H, s.blockRows, x, ldX, g, ldG, sa, sb, mean, partial);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

}  // namespace
}  // namespace roc

using namespace roc;

extern "C" size_t roc_batchnorm_workspace_bytes(int64_t rows, int H) {
  if (rows < 0 || H <= 0) return 0;
  const BnShape s = bn_shape(rows, H);
  return bn_coef_bytes(H) + (size_t)s.rowBlocks * (size_t)H * sizeof(double2);
}

extern "C" int roc_batchnorm_fwd(int64_t rows, int H, const float* x, int64_t ldX, const float* gamma,
                                 const float* beta, double eps, double momentum, float* runMean, float* runVar,
                                 int training, int relu, float* y, int64_t ldY, float* saveA, float* saveB,
                                 double* saveMean, double* saveInvStd, void* workspace, size_t workspaceBytes,
                                 roc_stream_t stream) {
  if (!x || !gamma || !beta || !y || !workspace || rows < 0 || H <= 0 || ldX < H || ldY < H) return ROC_ERR_INVALID;
  if (!rows16(x, ldX) || !rows16(y, ldY) || !aligned16(workspace)) return ROC_ERR_INVALID;
  if (!(eps >= 0.0) || !(momentum >= 0.0 && momentum <= 1.0)) return ROC_ERR_INVALID;
  if ((runMean == nullptr) != (runVar == nullptr)) return ROC_ERR_INVALID;
  if (training && (rows < 2 || !saveA || !saveB || !saveMean || !saveInvStd)) return ROC_ERR_INVALID;
  if (!training && !runMean) return ROC_ERR_INVALID;
  if (workspaceBytes < roc_batchnorm_workspace_bytes(rows, H)) return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  const BnShape s = bn_shape(rows, H);
  float* coef = static_cast<float*>(workspace);
  double2* partial = reinterpret_cast<double2*>(static_cast<char*>(workspace) + bn_coef_bytes(H));
  const float *a = saveA, *b = saveB;
  if (training) {
    int rc = launch_reduce<false>(s, rows, H, x, ldX, nullptr, 0, 0, nullptr, nullptr, nullptr, partial, st);
    if (rc) return rc;
    k_bn_finalize_fwd<<<H, BN_FIN_T, 0, st>>>(rows, H, s.rowBlocks, partial, x, gamma, beta, eps, momentum, runMean,
                                              runVar, saveA, saveB, saveMean, saveInvStd);
    ROC_LAUNCH_CHECK();
  } else {
    const int64_t ld4 = (H + 3) / 4 * 4;
    k_bn_finalize_infer<<<(H + 127) / 128, 128, 0, st>>>(H, gamma, beta, eps, runMean, runVar, coef, coef + ld4);
    ROC_LAUNCH_CHECK();
    a = coef; b = coef + ld4;
  }
  if (rows == 0) return ROC_OK;
  const dim3 grid = stream_grid(s, rows), block((unsigned)s.TX, (unsigned)s.TY);
  if (relu) k_bn_normalise<true><<<grid, block, 0, st>>>(rows, H, x, ldX, a, b, y, ldY);
  else k_bn_normalise<false><<<grid, block, 0, st>>>(rows, H, x, ldX, a, b, y, ldY);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

extern "C" int roc_batchnorm_bwd(int64_t rows, int H, const float* x, int64_t ldX, const float* dY, int64_t ldDY,
                                 int relu, const float* gamma, const float* saveA, const float* saveB,
                                 const double* saveMean, const double* saveInvStd, float* dGamma, float* dBeta,
                                 float* dX, int64_t ldDX, int accumulate, void* workspace, size_t workspaceBytes,
                                 roc_stream_t stream) {
  if (!x || !dY || !gamma || !saveMean || !saveInvStd || !dGamma || !dBeta || !workspace) return ROC_ERR_INVALID;
  if (rows < 2 || H <= 0 || ldX < H || ldDY < H || (dX && ldDX < H)) return ROC_ERR_INVALID;
  if (relu && (!saveA || !saveB)) return ROC_ERR_INVALID;
  if (!rows16(x, ldX) || !rows16(dY, ldDY) || (dX && !rows16(dX, ldDX)) || !aligned16(workspace)) return ROC_ERR_INVALID;
  if (workspaceBytes < roc_batchnorm_workspace_bytes(rows, H)) return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  const BnShape s = bn_shape(rows, H);
  const int64_t ld4 = (H + 3) / 4 * 4;
  float* coef = static_cast<float*>(workspace);
  double2* partial = reinterpret_cast<double2*>(static_cast<char*>(workspace) + bn_coef_bytes(H));
  int rc = launch_reduce<true>(s, rows, H, x, ldX, dY, ldDY, relu, saveA, saveB, saveMean, partial, st);
  if (rc) return rc;
  k_bn_finalize_bwd<<<H, BN_FIN_T, 0, st>>>(rows, H, s.rowBlocks, partial, gamma, saveMean, saveInvStd, dGamma, dBeta,
                                            dX ? coef : nullptr, coef + ld4, coef + 2 * ld4);
  ROC_LAUNCH_CHECK();
  if (!dX) return ROC_OK;
  const dim3 grid = stream_grid(s, rows), block((unsigned)s.TX, (unsigned)s.TY);
  if (relu && accumulate)
    k_bn_backward_apply<true, true><<<grid, block, 0, st>>>(rows, H, x, ldX, dY, ldDY, saveA, saveB, coef, ld4, dX, ldDX);
  else if (relu)
    k_bn_backward_apply<true, false><<<grid, block, 0, st>>>(rows, H, x, ldX, dY, ldDY, saveA, saveB, coef, ld4, dX, ldDX);
  else if (accumulate)
    k_bn_backward_apply<false, true><<<grid, block, 0, st>>>(rows, H, x, ldX, dY, ldDY, saveA, saveB, coef, ld4, dX, ldDX);
  else
    k_bn_backward_apply<false, false><<<grid, block, 0, st>>>(rows, H, x, ldX, dY, ldDY, saveA, saveB, coef, ld4, dX, ldDX);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}
