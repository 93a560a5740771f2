// attn_scores.cu — per-head GAT attention scores for sm_90a (roc_attn_scores_*): S = [s_dst | s_src] from the
// features X[rows][H], H = heads * F, and the two learned vectors of every head, A[2 * heads][F].
//
// Column c of X belongs to head c / F.  Row k of A is a_dst of head k and row heads + k its a_src, so a_dst over all
// heads is A[0 .. H) and a_src is A[H .. 2H), each indexed by the column.
//
// Forward: a CTA stages a tile of rows in shared memory (coalesced loads, a pitch of odd length so that the threads of
// a warp, one row each, read different banks), then one thread per (row, head) sums its F products in order f = 0 ..
// F - 1 with fp32 FMAs.  Backward: the column-group x row-lane layout of batchnorm.cu.  One pass reads X and dS, writes
// dX = gd a_dst + gs a_src and sums gd x and gs x per column in fp64 over fixed row blocks; a finalize adds the blocks
// in block order.  Every result depends on the inputs and the shape alone.
#include "common.cuh"

namespace roc {
namespace {

constexpr int AS_T = 256;                // threads per CTA
constexpr int AS_MAX_H = 1024;
constexpr int AS_FWD_MAX_TR = 256;       // forward tile: rows staged per CTA (at most)
constexpr int AS_FWD_SMEM = 72 * 1024;   // forward tile: shared-memory budget for the staged rows
constexpr int AS_UNROLL = 4;             // groups / rows in flight per thread
constexpr int AS_MAX_TX = 64;            // backward: column groups per CTA
constexpr int AS_ROWS_PER_LANE = 128;    // backward: rows a thread sums in one reduction block (at most)
constexpr int AS_MIN_ROWS_PER_LANE = 16; // ... (at least)
constexpr int AS_ROW_BLOCKS = 1024;      // backward: row blocks wanted, when that leaves a lane 16 to 128 rows
constexpr int AS_FIN_T = 128;            // finalize: threads per column

__device__ __forceinline__ float lane4(const float (&v)[4], int k) {
  return k == 0 ? v[0] : k == 1 ? v[1] : k == 2 ? v[2] : v[3];
}

// columns [4 * c4, 4 * c4 + 4) of a row: one 16-byte (fp32) or 8-byte (bf16) load when VEC, else one load per column
// below H (0 beyond)
template <bool VEC>
__device__ __forceinline__ void load_group(const float* p, int c4, int H, float (&v)[4]) {
  if (VEC) {
    const float4 t = ld_stream4(reinterpret_cast<const float4*>(p + 4 * c4));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
#pragma unroll
    for (int k = 0; k < 4; k++) v[k] = 4 * c4 + k < H ? p[4 * c4 + k] : 0.0f;
  }
}
template <bool VEC>
__device__ __forceinline__ void load_group(const uint16_t* p, int c4, int H, float (&v)[4]) {
  if (VEC) {
    const uint2 t = __ldcs(reinterpret_cast<const uint2*>(p + 4 * c4));
    v[0] = __uint_as_float(t.x << 16); v[1] = __uint_as_float(t.x & 0xFFFF0000u);
    v[2] = __uint_as_float(t.y << 16); v[3] = __uint_as_float(t.y & 0xFFFF0000u);
  } else {
#pragma unroll
    for (int k = 0; k < 4; k++) v[k] = 4 * c4 + k < H ? to_f32(p[4 * c4 + k]) : 0.0f;
  }
}

// ------------------------------------------------------------------------------------------------- forward ---
struct FwdShape {
  int TR, P;       // rows per tile, shared-memory pitch (odd)
  size_t smem;
};
FwdShape fwd_shape(int H, int heads) {
  FwdShape s;
  s.P = H | 1;
  int tr = (AS_T / heads + 31) / 32 * 32;                     // enough (row, head) items for every thread
  if (tr > AS_FWD_MAX_TR) tr = AS_FWD_MAX_TR;
  if (tr < 32) tr = 32;
  while (tr > 32 && (size_t)tr * s.P * sizeof(float) > (size_t)AS_FWD_SMEM) tr -= 32;
  s.TR = tr;
  s.smem = ((size_t)2 * H + (size_t)tr * s.P) * sizeof(float);
  return s;
}

// S[r][k] = sum_f A[k][f] X[r][kF + f], S[r][heads + k] = sum_f A[heads + k][f] X[r][kF + f], f in order
template <typename T, bool VEC>
__global__ void __launch_bounds__(AS_T)
k_attn_scores_fwd(int64_t rows, int H, int heads, int F, int TR, int P, const T* __restrict__ X, int64_t ldX,
                  const float* __restrict__ A, float* __restrict__ S, int64_t ldS) {
  extern __shared__ float sm[];
  float2* a2 = reinterpret_cast<float2*>(sm);   // [H]: (a_dst, a_src) of column c
  float* xs = sm + 2 * H;                       // [TR][P]
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int c = tid; c < H; c += nt) a2[c] = make_float2(A[c], A[H + c]);
  // loading: thread (tx, ty) takes column group tx (+ TX, ...) of rows ty, ty + TY, ...
  const int H4 = (H + 3) / 4;
  const int TX = H4 < nt ? H4 : nt, TY = nt / TX;
  const int tx = tid % TX, ty = tid / TX;
  for (int64_t t0 = (int64_t)blockIdx.x * TR; t0 < rows; t0 += (int64_t)gridDim.x * TR) {
    const int nr = (int)min((int64_t)TR, rows - t0);
    __syncthreads();   // the previous tile is consumed (and a2 is written)
    if (ty < TY) {
      for (int c4 = tx; c4 < H4; c4 += TX) {
        // the 4 stores of a group start at a lane-dependent column, so lanes 8 groups apart hit different banks
        const int rot = (c4 >> 3) & 3;
        for (int r = ty; r < nr; r += AS_UNROLL * TY) {
          float v[AS_UNROLL][4];
#pragma unroll
          for (int u = 0; u < AS_UNROLL; u++)
            if (r + u * TY < nr) load_group<VEC>(X + (t0 + r + u * TY) * ldX, c4, H, v[u]);
#pragma unroll
          for (int u = 0; u < AS_UNROLL; u++) {
            if (r + u * TY >= nr) break;
            float* row = xs + (size_t)(r + u * TY) * P + 4 * c4;
#pragma unroll
            for (int j = 0; j < 4; j++) {
              const int k = (j + rot) & 3;
              if (4 * c4 + k < H) row[k] = lane4(v[u], k);
            }
          }
        }
      }
    }
    __syncthreads();
    // one (row, head) per item, rows fastest: a warp shares its head, so the A reads are broadcasts
    for (int i = tid; i < TR * heads; i += nt) {
      const int k = i / TR, r = i - k * TR;
      if (r >= nr) continue;
      const float* xr = xs + (size_t)r * P + k * F;
      const float2* ar = a2 + k * F;
      float sd = 0.0f, ss = 0.0f;
#pragma unroll 4
      for (int f = 0; f < F; f++) {
        const float x = xr[f];
        const float2 a = ar[f];
        sd = __fmaf_rn(a.x, x, sd);
        ss = __fmaf_rn(a.y, x, ss);
      }
      float* srow = S + (t0 + r) * ldS;
      srow[k] = sd;
      srow[heads + k] = ss;
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward ---
struct BwdShape {
  int H4, TX, TY, colBlocks;
  int64_t blockRows, rowBlocks;
};
BwdShape bwd_shape(int64_t rows, int H) {
  BwdShape s;
  s.H4 = (H + 3) / 4;
  s.TX = s.H4 < AS_MAX_TX ? s.H4 : AS_MAX_TX;
  s.TY = AS_T / s.TX;
  s.colBlocks = (s.H4 + s.TX - 1) / s.TX;
  // a narrow H has many row lanes per CTA: shorter lanes keep the grid at about AS_ROW_BLOCKS CTAs there
  int64_t perLane = (rows + (int64_t)s.TY * AS_ROW_BLOCKS - 1) / ((int64_t)s.TY * AS_ROW_BLOCKS);
  if (perLane < AS_MIN_ROWS_PER_LANE) perLane = AS_MIN_ROWS_PER_LANE;
  if (perLane > AS_ROWS_PER_LANE) perLane = AS_ROWS_PER_LANE;
  s.blockRows = perLane * s.TY;
  s.rowBlocks = rows > 0 ? (rows + s.blockRows - 1) / s.blockRows : 1;
  return s;
}

// One reduction block of rows per blockIdx.x, one set of TX column groups per blockIdx.y.  Per column c of head k:
//   dX[r][c] (+)= fma(gs, a_src[c], gd * a_dst[c])        with gd = dS[r][k], gs = dS[r][heads + k]
//   partial[blockIdx.x][c] = (sum_r gd x, sum_r gs x)       in fp64, rows in order, then the lanes in order
template <typename T, bool VEC>
__global__ void __launch_bounds__(AS_T)
k_attn_scores_bwd(int64_t rows, int H, int heads, int F, int64_t blockRows, const T* __restrict__ X, int64_t ldX,
                  const float* __restrict__ A, const float* __restrict__ dS, int64_t ldDS, float* __restrict__ dX,
                  int64_t ldDX, int accumulate, int dxVec, double2* __restrict__ partial) {
  extern __shared__ double shd[];   // [TY][TX][8]
  const int TX = blockDim.x, TY = blockDim.y, tx = threadIdx.x, ty = threadIdx.y;
  const int c4 = blockIdx.y * TX + tx;
  const bool active = 4 * c4 < H;
  const int64_t r0 = (int64_t)blockIdx.x * blockRows;
  const int64_t r1 = min(r0 + blockRows, rows);
  double s[4], q[4];
  float ad[4], as[4];
  int hd[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    s[k] = 0.0; q[k] = 0.0;
    const int c = 4 * c4 + k;
    const bool in = active && c < H;
    ad[k] = in ? A[c] : 0.0f;
    as[k] = in ? A[H + c] : 0.0f;
    // a padding column takes the head of the row's last column, so that the one-head test below sees every head the
    // group's in-range columns belong to
    hd[k] = active ? min(c, H - 1) / F : 0;
  }
  const bool oneHead = hd[0] == hd[3];   // the group lies in one head: two dS loads per row
  if (active) {
    for (int64_t r = r0 + ty; r < r1; r += (int64_t)AS_UNROLL * TY) {
      float xv[AS_UNROLL][4], gd[AS_UNROLL][4], gs[AS_UNROLL][4];
#pragma unroll
      for (int u = 0; u < AS_UNROLL; u++) {
        const int64_t rr = r + (int64_t)u * TY;
        if (rr >= r1) break;
        load_group<VEC>(X + rr * ldX, c4, H, xv[u]);
        const float* g = dS + rr * ldDS;
        if (oneHead) {
          const float d = g[hd[0]], e = g[heads + hd[0]];
#pragma unroll
          for (int k = 0; k < 4; k++) { gd[u][k] = d; gs[u][k] = e; }
        } else {
#pragma unroll
          for (int k = 0; k < 4; k++) { gd[u][k] = g[hd[k]]; gs[u][k] = g[heads + hd[k]]; }
        }
      }
#pragma unroll
      for (int u = 0; u < AS_UNROLL; u++) {
        const int64_t rr = r + (int64_t)u * TY;
        if (rr >= r1) break;
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const double x = (double)xv[u][k];
          s[k] = fma((double)gd[u][k], x, s[k]);
          q[k] = fma((double)gs[u][k], x, q[k]);
        }
        if (dX) {
          float* drow = dX + rr * ldDX + 4 * c4;
          float o[4];
#pragma unroll
          for (int k = 0; k < 4; k++) o[k] = __fmaf_rn(gs[u][k], as[k], __fmul_rn(gd[u][k], ad[k]));
          if (dxVec && 4 * c4 + 4 <= H) {
            float4* p = reinterpret_cast<float4*>(drow);
            if (accumulate) {
              const float4 old = *p;
              o[0] += old.x; o[1] += old.y; o[2] += old.z; o[3] += old.w;
            }
            st_stream4(p, make_float4(o[0], o[1], o[2], o[3]));
          } else {
#pragma unroll
            for (int k = 0; k < 4; k++)
              if (4 * c4 + k < H) drow[k] = accumulate ? drow[k] + o[k] : o[k];
          }
        }
      }
    }
  }
  double* mine = shd + ((size_t)ty * TX + tx) * 8;
#pragma unroll
  for (int k = 0; k < 4; k++) { mine[k] = s[k]; mine[4 + k] = q[k]; }
  __syncthreads();
  if (ty != 0 || !active) return;
  for (int l = 1; l < TY; l++) {   // lanes in order
    const double* o = shd + ((size_t)l * TX + tx) * 8;
#pragma unroll
    for (int k = 0; k < 4; k++) { s[k] += o[k]; q[k] += o[4 + k]; }
  }
#pragma unroll
  for (int k = 0; k < 4; k++)
    if (4 * c4 + k < H) partial[(int64_t)blockIdx.x * H + 4 * c4 + k] = make_double2(s[k], q[k]);
}

// dA of column blockIdx.x: thread t adds blocks t, t + AS_FIN_T, ... in order, then a fixed tree
__global__ void __launch_bounds__(AS_FIN_T)
k_attn_scores_finalize(int H, int64_t rowBlocks, const double2* __restrict__ partial, float* __restrict__ dA) {
  __shared__ double2 red[AS_FIN_T];
  const int c = blockIdx.x;
  double2 acc = make_double2(0.0, 0.0);
  for (int64_t i = threadIdx.x; i < rowBlocks; i += AS_FIN_T) {
    const double2 p = partial[i * H + c];
    acc.x += p.x; acc.y += p.y;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int w = AS_FIN_T / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) {
      red[threadIdx.x].x += red[threadIdx.x + w].x;
      red[threadIdx.x].y += red[threadIdx.x + w].y;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    dA[c] = (float)red[0].x;
    dA[H + c] = (float)red[0].y;
  }
}

inline bool vec_rows(const float* p, int64_t ld) { return aligned16(p) && ld % 4 == 0; }
inline bool vec_rows(const uint16_t* p, int64_t ld) {
  return (reinterpret_cast<uintptr_t>(p) & 7u) == 0 && ld % 4 == 0;
}

int check_shape(int64_t rows, int H, int heads) {
  if (rows < 0 || H <= 0 || heads <= 0) return ROC_ERR_INVALID;
  if (H % heads || H > AS_MAX_H) return ROC_ERR_UNSUPPORTED;
  return ROC_OK;
}

template <typename T>
int scores_fwd(int64_t rows, int H, int heads, const T* X, int64_t ldX, const float* A, float* S, int64_t ldS,
               roc_stream_t stream) {
  if (!X || !A || !S || ldX < H || ldS < 2 * (int64_t)heads) return ROC_ERR_INVALID;
  if (int rc = check_shape(rows, H, heads)) return rc;
  if (rows == 0) return ROC_OK;
  const FwdShape s = fwd_shape(H, heads);
  const int64_t tiles = (rows + s.TR - 1) / s.TR;
  int64_t perSm = (int64_t)(200 * 1024) / (int64_t)s.smem;
  if (perSm < 1) perSm = 1;
  if (perSm > 8) perSm = 8;
  const int64_t grid = std::min<int64_t>(tiles, (int64_t)sm_count() * perSm);
  const int F = H / heads;
  cudaStream_t st = as_stream(stream);
  if (vec_rows(X, ldX))
    return launch_dyn<k_attn_scores_fwd<T, true>>(dim3((unsigned)grid), AS_T, s.smem, st, rows, H, heads, F, s.TR,
                                                  s.P, X, ldX, A, S, ldS);
  return launch_dyn<k_attn_scores_fwd<T, false>>(dim3((unsigned)grid), AS_T, s.smem, st, rows, H, heads, F, s.TR, s.P,
                                                 X, ldX, A, S, ldS);
}

template <typename T>
int scores_bwd(int64_t rows, int H, int heads, const T* X, int64_t ldX, const float* A, const float* dS, int64_t ldDS,
               float* dX, int64_t ldDX, int accumulate, float* dA, void* workspace, size_t workspaceBytes,
               roc_stream_t stream) {
  if (!X || !A || !dS || !dA || !workspace || ldX < H || ldDS < 2 * (int64_t)heads || (dX && ldDX < H))
    return ROC_ERR_INVALID;
  if (int rc = check_shape(rows, H, heads)) return rc;
  if (!aligned16(workspace) || workspaceBytes < roc_attn_scores_workspace_bytes(rows, H, heads)) return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  const BwdShape s = bwd_shape(rows, H);
  double2* partial = static_cast<double2*>(workspace);
  const dim3 grid((unsigned)s.rowBlocks, (unsigned)s.colBlocks), block((unsigned)s.TX, (unsigned)s.TY);
  const size_t smem = (size_t)s.TX * s.TY * 8 * sizeof(double);
  const int F = H / heads, dxVec = dX ? (int)vec_rows(dX, ldDX) : 0;
  if (vec_rows(X, ldX))
    k_attn_scores_bwd<T, true><<<grid, block, smem, st>>>(rows, H, heads, F, s.blockRows, X, ldX, A, dS, ldDS, dX,
                                                          ldDX, accumulate, dxVec, partial);
  else
    k_attn_scores_bwd<T, false><<<grid, block, smem, st>>>(rows, H, heads, F, s.blockRows, X, ldX, A, dS, ldDS, dX,
                                                           ldDX, accumulate, dxVec, partial);
  ROC_LAUNCH_CHECK();
  k_attn_scores_finalize<<<H, AS_FIN_T, 0, st>>>(H, s.rowBlocks, partial, dA);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

}  // namespace
}  // namespace roc

using namespace roc;

extern "C" size_t roc_attn_scores_workspace_bytes(int64_t rows, int H, int heads) {
  if (check_shape(rows, H, heads)) return 0;
  return (size_t)bwd_shape(rows, H).rowBlocks * (size_t)H * sizeof(double2);
}

extern "C" int roc_attn_scores_fwd(int64_t rows, int H, int heads, const float* X, int64_t ldX, const float* A,
                                   float* S, int64_t ldS, roc_stream_t stream) {
  return scores_fwd(rows, H, heads, X, ldX, A, S, ldS, stream);
}
extern "C" int roc_attn_scores_fwd_bf16(int64_t rows, int H, int heads, const uint16_t* X, int64_t ldX, const float* A,
                                        float* S, int64_t ldS, roc_stream_t stream) {
  return scores_fwd(rows, H, heads, X, ldX, A, S, ldS, stream);
}
extern "C" int roc_attn_scores_bwd(int64_t rows, int H, int heads, const float* X, int64_t ldX, const float* A,
                                   const float* dS, int64_t ldDS, float* dX, int64_t ldDX, int accumulate, float* dA,
                                   void* workspace, size_t workspaceBytes, roc_stream_t stream) {
  return scores_bwd(rows, H, heads, X, ldX, A, dS, ldDS, dX, ldDX, accumulate, dA, workspace, workspaceBytes, stream);
}
extern "C" int roc_attn_scores_bwd_bf16(int64_t rows, int H, int heads, const uint16_t* X, int64_t ldX, const float* A,
                                        const float* dS, int64_t ldDS, float* dX, int64_t ldDX, int accumulate,
                                        float* dA, void* workspace, size_t workspaceBytes, roc_stream_t stream) {
  return scores_bwd(rows, H, heads, X, ldX, A, dS, ldDS, dX, ldDX, accumulate, dA, workspace, workspaceBytes, stream);
}
