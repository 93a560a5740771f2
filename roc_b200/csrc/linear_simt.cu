// linear_simt.cu — fp32 SIMT GEMM family for the Linear op (fallback / checker path).
//
// Replaces the three cublasSgemm calls of the reference Linear op
// (linear_kernel.cu:76-80 fwd, :220-224 dW, :227-231 dX).  This file is the
// exact-fp32 register-tiled version; linear_tc.cu holds the wgmma
// tensor-core version that the dispatcher in linear.cu prefers for large shapes.
//
//   FWD : Y[v][o]  = sum_i X[v][i]  * W[o*in+i]       (A K-contig, B K-contig)
//   DX  : dX[v][i] (+)= sum_o dY[v][o] * W[o*in+i]    (A K-contig, B N-contig)
//   DW  : dW[o][i] += sum_v dY[v][o] * X[v][i]        (A M-contig, B N-contig, split-K over v)
#include "common.cuh"

namespace roc {

constexpr int GB_M = 128, GB_N = 64, GB_K = 16, GT_M = 8, GT_N = 4;
constexpr int G_THREADS = (GB_M / GT_M) * (GB_N / GT_N);  // 256

struct GemmP {
  const float* A; int64_t lda;
  const float* B; int64_t ldb;
  float* C; int64_t ldc;
  int64_t M; int N; int64_t K;
  int64_t kPerSplit;      // K range per blockIdx.z
  int64_t splitStrideC;   // C offset per split (floats)
  int accumulate;         // C += (only when splits == 1)
  int relu;               // epilogue relu
  const uint64_t* rowEnd; // epilogue row scale 1/sqrtf(deg(m)) if non-NULL
  uint64_t colLeft;
  // fused dropout (NULL = none): maskOn 1 = A element (m, k) [fwd], 2 = B element (k, n) [dW],
  // 3 = C element (m, n) [dX: the dropout backward]
  const uint32_t* mask; int64_t ldm; float mscale; int maskOn;
  const float* reluOf; int64_t ldR;   // epilogue relu backward: reluOf(m, n) > 0 ? v : 0 (NULL = none)
};

template <bool A_KCONTIG, bool B_KCONTIG>
__global__ void __launch_bounds__(G_THREADS)
k_sgemm(const GemmP p) {
  __shared__ float As[GB_K][GB_M + 4];
  __shared__ float Bs[GB_K][GB_N + 4];
  const int tid = threadIdx.x;
  const int64_t m0 = (int64_t)blockIdx.x * GB_M;
  const int n0 = blockIdx.y * GB_N;
  const int64_t kBeg = (int64_t)blockIdx.z * p.kPerSplit;
  const int64_t kEnd = (kBeg + p.kPerSplit < p.K) ? kBeg + p.kPerSplit : p.K;
  const int ty = tid / (GB_N / GT_N), tx = tid % (GB_N / GT_N);
  float acc[GT_M][GT_N];
#pragma unroll
  for (int i = 0; i < GT_M; i++)
#pragma unroll
    for (int j = 0; j < GT_N; j++) acc[i][j] = 0.f;

  for (int64_t k0 = kBeg; k0 < kEnd; k0 += GB_K) {
    // A tile: GB_M x GB_K
#pragma unroll
    for (int it = 0; it < GB_M * GB_K / G_THREADS; it++) {
      int lin = it * G_THREADS + tid;
      int mm, kk;
      if (A_KCONTIG) { kk = lin % GB_K; mm = lin / GB_K; } else { mm = lin % GB_M; kk = lin / GB_M; }
      int64_t m = m0 + mm, k = k0 + kk;
      float v = 0.f;
      if (m < p.M && k < kEnd) {
        v = A_KCONTIG ? p.A[m * p.lda + k] : p.A[k * p.lda + m];
        if (p.maskOn == 1) v = drop_apply(p.mask, p.ldm, p.mscale, m, (int)k, v);
      }
      As[kk][mm] = v;
    }
#pragma unroll
    for (int it = 0; it < GB_N * GB_K / G_THREADS; it++) {
      int lin = it * G_THREADS + tid;
      int nn, kk;
      if (B_KCONTIG) { kk = lin % GB_K; nn = lin / GB_K; } else { nn = lin % GB_N; kk = lin / GB_N; }
      int n = n0 + nn; int64_t k = k0 + kk;
      float v = 0.f;
      if (n < p.N && k < kEnd) {
        v = B_KCONTIG ? p.B[(int64_t)n * p.ldb + k] : p.B[k * p.ldb + n];
        if (p.maskOn == 2) v = drop_apply(p.mask, p.ldm, p.mscale, k, n, v);
      }
      Bs[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GB_K; kk++) {
      float a[GT_M], b[GT_N];
#pragma unroll
      for (int i = 0; i < GT_M; i++) a[i] = As[kk][ty * GT_M + i];
#pragma unroll
      for (int j = 0; j < GT_N; j++) b[j] = Bs[kk][tx * GT_N + j];
#pragma unroll
      for (int i = 0; i < GT_M; i++)
#pragma unroll
        for (int j = 0; j < GT_N; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* C = p.C + (int64_t)blockIdx.z * p.splitStrideC;
#pragma unroll
  for (int i = 0; i < GT_M; i++) {
    int64_t m = m0 + ty * GT_M + i;
    if (m >= p.M) continue;
    float d = 1.0f;
    if (p.rowEnd) {
      uint64_t s = (m == 0) ? p.colLeft : p.rowEnd[m - 1];
      d = sqrtf((float)(uint32_t)(p.rowEnd[m] - s));
    }
#pragma unroll
    for (int j = 0; j < GT_N; j++) {
      int n = n0 + tx * GT_N + j;
      if (n >= p.N) continue;
      float v = acc[i][j];
      if (p.relu) v = relu_nanprop(v);   // reference order: sgemm -> relu (linear_kernel.cu:83-104)
      // dX only: dropout backward, relu backward, then indegree-norm backward (the ops upstream of X)
      if (p.maskOn == 3) v = drop_apply(p.mask, p.ldm, p.mscale, m, n, v);
      if (p.reluOf) v = (p.reluOf[m * p.ldR + n] > 0.f) ? v : 0.f;
      if (p.rowEnd) v = v / d;           // fwd: the model's indegree_norm (gnn.cc:82)
      float* dst = C + m * p.ldc + n;
      *dst = p.accumulate ? *dst + v : v;
    }
  }
}

// dW += sum over splits (fixed order => deterministic)
__global__ void __launch_bounds__(256)
k_splitk_reduce(int64_t count, int splits, const float* __restrict__ part, float* __restrict__ dW) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count;
       i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int z = 0; z < splits; z++) s += part[(int64_t)z * count + i];
    dW[i] += s;
  }
}

__global__ void __launch_bounds__(256)
k_relu_bwd_inplace(int64_t rows, int H, const float* __restrict__ y, int64_t ldy, float* __restrict__ dy, int64_t lddy) {
  const int64_t total = rows * (int64_t)H;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / H; int c = (int)(i - r * H);
    float g = dy[r * lddy + c];
    dy[r * lddy + c] = (y[r * ldy + c] > 0.0f) ? g : 0.f;   // reluBackward, linear_kernel.cu:120-127
  }
}

int simt_dw_splits(int64_t rows, int inDim, int outDim) {
  int tiles = ((outDim + GB_M - 1) / GB_M) * ((inDim + GB_N - 1) / GB_N);
  int want = (sm_count() * 4 + tiles - 1) / tiles;
  int64_t maxSplits = (rows + 4 * GB_K - 1) / (4 * GB_K);
  if (want > maxSplits) want = (int)maxSplits;
  if (want < 1) want = 1;
  if (want > 1024) want = 1024;
  return want;
}

static void set_mask(GemmP& p, const DropMask* dm, int on) {
  if (!dm) return;
  p.mask = dm->bits; p.ldm = dm->ld; p.mscale = dm->scale; p.maskOn = on;
}

int simt_linear_fwd(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX, const float* W, float* Y,
                    int64_t ldY, int relu, const uint64_t* rowEnd, uint64_t colLeft, const DropMask* dm,
                    cudaStream_t st) {
  GemmP p{};
  p.A = X; p.lda = ldX; p.B = W; p.ldb = inDim; p.C = Y; p.ldc = ldY;
  p.M = rows; p.N = outDim; p.K = inDim; p.kPerSplit = inDim; p.splitStrideC = 0;
  p.accumulate = 0; p.relu = relu; p.rowEnd = rowEnd; p.colLeft = colLeft;
  set_mask(p, dm, 1);
  dim3 grid((unsigned)((rows + GB_M - 1) / GB_M), (unsigned)((outDim + GB_N - 1) / GB_N), 1);
  k_sgemm<true, true><<<grid, G_THREADS, 0, st>>>(p);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

int simt_linear_dx(int64_t rows, int inDim, int outDim, const float* dY, int64_t ldDY, const float* W, float* dX,
                   int64_t ldDX, int accumulate, const DropMask* dm, const float* reluOf, int64_t ldR,
                   const uint64_t* rowEnd, uint64_t colLeft, cudaStream_t st) {
  GemmP p{};
  p.A = dY; p.lda = ldDY; p.B = W; p.ldb = inDim; p.C = dX; p.ldc = ldDX;
  p.M = rows; p.N = inDim; p.K = outDim; p.kPerSplit = outDim; p.accumulate = accumulate;
  set_mask(p, dm, 3);
  p.reluOf = reluOf; p.ldR = ldR; p.rowEnd = rowEnd; p.colLeft = colLeft;
  dim3 grid((unsigned)((rows + GB_M - 1) / GB_M), (unsigned)((inDim + GB_N - 1) / GB_N), 1);
  k_sgemm<true, false><<<grid, G_THREADS, 0, st>>>(p);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

int simt_linear_dw(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX, const float* dY, int64_t ldDY,
                   float* dW, float* workspace, size_t wsBytes, const DropMask* dm, cudaStream_t st,
                   roc_gemm_info* info) {
  int splits = simt_dw_splits(rows, inDim, outDim);
  int64_t count = (int64_t)inDim * outDim;
  if (wsBytes < (size_t)splits * count * sizeof(float)) return ROC_ERR_INVALID;
  GemmP p{};
  p.A = dY; p.lda = ldDY; p.B = X; p.ldb = ldX; p.C = workspace; p.ldc = inDim;
  p.M = outDim; p.N = inDim; p.K = rows;
  p.kPerSplit = ((rows + splits - 1) / splits + GB_K - 1) / GB_K * GB_K;
  p.splitStrideC = count; p.accumulate = 0;
  set_mask(p, dm, 2);
  if (info) { info->splits = splits; info->v_per_split = p.kPerSplit; }
  dim3 grid((unsigned)((outDim + GB_M - 1) / GB_M), (unsigned)((inDim + GB_N - 1) / GB_N), (unsigned)splits);
  k_sgemm<false, false><<<grid, G_THREADS, 0, st>>>(p);
  ROC_LAUNCH_CHECK();
  int64_t blocks = (count + 255) / 256;
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  k_splitk_reduce<<<(unsigned)blocks, 256, 0, st>>>(count, splits, workspace, dW);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

int relu_bwd_inplace(int64_t rows, int H, const float* Y, int64_t ldY, float* dY, int64_t ldDY, cudaStream_t st) {
  int64_t blocks = (rows * H + 255) / 256;
  if (blocks > sm_count() * 16) blocks = sm_count() * 16;
  if (blocks < 1) blocks = 1;
  k_relu_bwd_inplace<<<(unsigned)blocks, 256, 0, st>>>(rows, H, Y, ldY, dY, ldDY);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

}  // namespace roc
