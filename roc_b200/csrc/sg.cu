// sg.cu — ScatterGather (CSR row-parallel SpMM: sum, min / max and attention aggregation) for sm_90a.
//
// Replaces aggre_coop_kernel + ScatterGather::{forward,backward}_task
// (reference scattergather_kernel.cu:20-76, 78-170).  The reference walks one
// edge per H-thread group per iteration and accumulates with shared-memory
// float atomics; this is a different algorithm built for HBM3e:
//
//  * edge-balanced schedule ("plan"): the partition's edge array is cut into
//    CH = 64-edge chunks; one WORKER owns chunk c.  A row is owned by the chunk
//    its first edge lies in.  Rows no longer than CH are always finished by their
//    owner (so a worker does at most 2*CH-1 edges); a longer ("heavy") row is cut
//    at chunk boundaries: the owner stores its raw partial, every later chunk
//    stores its part into a carry slot and a second small kernel adds partial +
//    carries in chunk order.  No atomics anywhere => bit-reproducible sums (the
//    reference is not: smem atomicAdd, scattergather_kernel.cu:66).  The plan also
//    holds a 32-byte start record per chunk (k_chunk_desc) so a worker begins with
//    one load instead of a three-deep dependent walk.
//  * the store applies the ops the model puts right after scatter_gather
//    (indegree_norm, relu; gnn.cc:83-85) so the N x H result is written once.
//  * the main kernel, sg_chunk_kernel, gathers the neighbour rows in registers.  A row is Q T-columns (float4
//    when the rows are 16-byte aligned, else float); a worker is L = 4, 8, 16 or 32 lanes, the fewest that cover
//    Q, and each lane loads its NCH = ceil(Q / L) columns of U rows per group.  A launch covers up to 256
//    T-columns (1024 floats vectorised, 256 scalar); wider rows are split into column blocks.  with_shape picks L
//    and NCH; one row per reduction of the table SG_REDS gives its widest row, its gathers in flight and CTAs per SM,
//    the fix-ups and carries it needs, and whether it has a ring form.  One launcher (launch) runs the main kernel
//    and the fix-ups the row names.
//  * vectorised rows of 65..256 floats run on sg_chunk_kernel_t instead, which fetches them with cp.async.bulk
//    copies into a shared-memory ring: it was faster there on a products-shaped graph (DESIGN.md §3.1).  It
//    shares the plan and the per-row summation order, so its results are bit-identical to sg_chunk_kernel's.
//  * min / max aggregation (roc_sg_minmax_*) runs the same kernel and fix-ups templated on the reduction; its
//    backward is the sum schedule with a second gathered row and a predicated add, finished by the sum's fix-ups.
//    The sum and min / max entry points check their arguments and share one column-block driver (run_planned).
//  * attention aggregation (roc_sg_attn_*) is more reductions of the same kernel: a stats pass and an a-weighted
//    sum forward; a per-node record kernel and two gathers backward.  Both entry points share attn_setup.
//  * edge-weighted aggregation (roc_sg_weighted_*, roc_sg_edge_dot_planned) is two more: WSUM, a sum with one FMA by
//    each edge's weight, finished by the sum's fix-ups; EDOT, one dot product G[i] . X[j] per edge, which carries
//    nothing.  The exact backward runs WSUM over a transposed CSR (roc_sg_transpose) with the weights permuted.
//  * the exact backwards of the other aggregations run over the same transpose (roc_sg_transpose_*_backward,
//    roc_sg_attn_backward_exact): TSUM is the sum whose NORM epilogue divides by the original graph's in-degree,
//    TMASK the min / max backward that skips a repeated destination (a duplicate edge), and the attention input
//    gradient is the ASRC gather itself, run over the transposed plan.
//  * the sum over bf16 rows (roc_sg_forward_planned_bf16) is BSUM: SUM's row of the table with half-width loads,
//    widened in registers, on both the register and the ring kernel.
//  * the max / min, weighted, edge-dot and attention calls over bf16 feature rows (roc_sg_*_bf16) are those
//    reductions plus SG_RED_BF16: the same row of the table and the same fix-ups, with the feature rows loaded at half
//    width and widened in registers as BSUM's are.  Their bytes per gathered row fall from 4H to 2H.
//  * attention dropout (roc_sg_attn_*_dropout_*) is SG_RED_DROP on ATTN, ADST and ASRC: each pass loads one keep byte
//    per edge beside its source id and weighs a dropped head's term by 0.  k_attn_keep writes those bytes from Philox,
//    keyed by the (destination, source) pair, in any plan's edge order.
//  * the teleport sum (roc_sg_forward_teleport_planned, APPNP / GCNII's hop) is TELE: SUM's row of the table, column
//    blocks and sum fix-ups, with a row store (tele_store) that also reads the row of t and applies
//    post(fmaf(alpha, pre(sum), beta * t)) wherever a row is finally stored.  It runs every width on sg_chunk_kernel.
//  * edge dropout (roc_sg_forward_dropout_planned, roc_sg_forward_teleport_dropout_planned,
//    roc_sg_transpose_sum_backward_dropout) is SG_RED_DROP on SUM, TELE and TSUM: the keep bytes attention dropout
//    uses, bit 0 per edge, loaded beside the source ids; a dropped edge's row is not gathered, a kept one is added as
//    fmaf(s, x, acc).  Every width runs on sg_chunk_kernel, with the sum's column blocks and fix-ups.
//  * dynamic attention (roc_sg_attn_v2_*, GATv2) runs on its own kernel, sg_v2_kernel (end of file): one warp per
//    chunk of the same plan, finished by the attention stats fix-up and the sum's fix-ups.
//  * softmax aggregation (roc_sg_softmax_*, PyG's SoftmaxAggregation) runs on its own kernel, sg_smx_kernel (end of
//    file), with the schedule of sg_v2_kernel: a one-pass online softmax per column forward, finished by its own
//    rescale-and-add fix-ups (sg_smx_fixup), and a record pass and a source pass backward, finished by the sum's.
//  * dot-product attention (roc_sg_attn_dot_*, the graph transformer's) runs on its own kernel, sg_dot_kernel (end of
//    file), with the same schedule: a one-pass online softmax per head forward, finished by sg_dot_fixup, and
//    GATv2's record pass, a destination pass and a source pass backward, finished by the sum's fix-ups.
//
// Algorithmic bytes per launch (DESIGN.md): E*(4H+4) + Nloc*(4H+8); min / max forward E*(4H+4) + Nloc*(8H+8),
// backward E*(8H+4) + Nloc*(4H+8); the sum over bf16 rows E*(2H+4) + Nloc*(4H+8); weighted forward E*(4H+8) + Nloc*(4H+8), edge dot E*(4H+8) + Nloc*4H; attention
// in DESIGN.md §3.1.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <initializer_list>
#include <new>
#include <type_traits>
#include "common.cuh"
#include "tc_common.cuh"

namespace roc {

constexpr int SG_CH = 64;          // edges per chunk
constexpr int SG_THREADS = 256;    // threads per CTA

}  // namespace roc

struct roc_sg_plan {
  uint32_t nloc = 0, E = 0, numChunks = 0, numCarries = 0, numHeavy = 0, numBig = 0;
  uint32_t* rs = nullptr;         // [nloc+1]   local row starts (rs[r+1] = rowEnd[r]-colLeft)
  uint32_t* firstRow = nullptr;   // [numChunks+1] first row whose start >= c*CH
  uint32_t* carryIdx = nullptr;   // [numChunks+1] exclusive scan of carry-in flags
  uint32_t* heavyRows = nullptr;  // [numHeavy]  rows with degree > CH and <= 32 carries (one worker each)
  uint32_t* bigRows = nullptr;    // [numBig]    rows with more carries (one CTA each)
  const uint32_t* col = nullptr;  // caller's colSrc
  // Grown on demand (grow); each *Bytes is its buffer's capacity.
  float* carry = nullptr;         // [numCarries][carryLd]
  size_t carryBytes = 0, carryLd = 0;
  uint32_t* carryArg = nullptr;   // [numCarries][carryLd] indices of the min / max carries
  size_t carryArgBytes = 0;
  float* carry2 = nullptr;        // [numCarries][16] attention: the heads-wide partials
  size_t carry2Bytes = 0;
  float4* attnRec = nullptr;      // attention backward: {s_dst, m, 1/Z, D} per (node id, head)
  size_t attnRecBytes = 0;
  char* smxWs = nullptr;          // softmax aggregation: the backward's records, R and dt's block sums; the inference
  size_t smxWsBytes = 0;          // forward's (m, s) of cut rows

  uint64_t idEnd = 0;             // 1 + the largest id in col (found by the first attention backward)
  bool idEndKnown = false;
  uint32_t* desc = nullptr;       // [numChunks][8] per-chunk start state of a worker (k_chunk_desc)
  int device = 0;
};

namespace roc {

// ------------------------------------------------------------ plan kernels ---

__global__ void k_build_rs(uint32_t nloc, uint64_t colLeft, const uint64_t* __restrict__ rowEnd,
                           uint32_t* __restrict__ rs) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) rs[0] = 0;
  if (i < nloc) rs[i + 1] = (uint32_t)(rowEnd[i] - colLeft);
}

__global__ void k_first_row(uint32_t nloc, uint32_t numChunks, const uint32_t* __restrict__ rs,
                            uint32_t* __restrict__ firstRow) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > numChunks) return;
  if (c == numChunks) { firstRow[c] = nloc; return; }
  uint32_t target = c * (uint32_t)SG_CH;
  uint32_t lo = 0, hi = nloc;  // first r in [0,nloc) with rs[r] >= target, else nloc
  while (lo < hi) {
    uint32_t mid = lo + ((hi - lo) >> 1);
    if (rs[mid] >= target) hi = mid; else lo = mid + 1;
  }
  firstRow[c] = lo;
}

__global__ void k_carry_flag(uint32_t numChunks, const uint32_t* __restrict__ rs,
                             const uint32_t* __restrict__ firstRow, uint32_t* __restrict__ flag) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > numChunks) return;
  uint32_t f = 0;
  if (c < numChunks) {
    uint32_t r0 = firstRow[c];
    if (r0 > 0) {
      uint32_t pe = rs[r0], ps = rs[r0 - 1];
      f = (pe > c * (uint32_t)SG_CH && pe - ps > (uint32_t)SG_CH) ? 1u : 0u;
    }
  }
  flag[c] = f;
}

__global__ void k_heavy_flag(uint32_t nloc, const uint32_t* __restrict__ rs, uint8_t* __restrict__ flag,
                             uint8_t* __restrict__ bigFlag) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nloc) return;
  const uint32_t s = rs[r], t = rs[r + 1];
  const bool heavy = t - s > (uint32_t)SG_CH;
  const uint32_t carries = heavy ? (t - 1) / SG_CH - s / SG_CH : 0;
  flag[r] = (heavy && carries <= 32u) ? 1 : 0;      // 32 == SG_BIG
  bigFlag[r] = (carries > 32u) ? 1 : 0;
}

// Start state of the worker that owns chunk c, so that it reads ONE 32-byte record instead
// of walking firstRow -> rs -> rs (three dependent global loads per chunk):
//   [0] eb  first edge the worker processes     [1] ee  one past its last edge
//   [2] cur first row it accumulates into        [3] curS = rs[cur]   [4] curT = rs[cur + 1]
//   [5] r1  one past its last owned row          [6] flags: 1 = carry-in (cur is a heavy row owned by an
//       earlier chunk), 2 = nothing to do        [7] carry slot of a carry-in part
__global__ void k_chunk_desc(uint32_t numChunks, uint32_t E, const uint32_t* __restrict__ rs,
                             const uint32_t* __restrict__ firstRow, const uint32_t* __restrict__ carryIdx,
                             uint32_t* __restrict__ desc) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= numChunks) return;
  constexpr uint32_t CH = SG_CH;
  const uint32_t cb = w * CH, ce = min(cb + CH, E);
  const uint32_t r0 = firstRow[w], r1 = firstRow[w + 1];
  uint32_t eb = cb, ee = cb, cur = r0, curS = 0, curT = 0, flags = 0, segEnd = cb;
  bool carryIn = false;
  if (r0 > 0) {
    const uint32_t pe = rs[r0], ps = rs[r0 - 1];
    if (pe > cb && pe - ps > CH) {
      carryIn = true; cur = r0 - 1; curS = ps; curT = pe; eb = cb; segEnd = min(pe, ce); flags = 1u;
    }
  }
  if (!carryIn) {
    if (r0 >= r1) { flags = 2u; }
    else {
      cur = r0; curS = rs[r0]; curT = rs[r0 + 1]; eb = curS;
      segEnd = (curT - curS > CH) ? min(curT, ce) : curT;
    }
  }
  if (r1 > r0) {
    const uint32_t s = rs[r1 - 1], t = rs[r1];
    ee = (t - s > CH) ? min(t, ce) : t;
  } else {
    ee = segEnd;
  }
  if (flags & 2u) { eb = cb; ee = cb; }
  uint4* d = reinterpret_cast<uint4*>(desc + (size_t)w * 8);
  d[0] = make_uint4(eb, ee, cur, curS);
  d[1] = make_uint4(curT, r1, flags, carryIdx[w]);
}

// bad = 1 if some row's sources are not strictly increasing (one thread per row; an init-time check)
__global__ void k_rows_sorted(uint32_t nloc, const uint32_t* __restrict__ rs, const uint32_t* __restrict__ col,
                              uint32_t* __restrict__ bad) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nloc) return;
  const uint32_t t = rs[r + 1];
  for (uint32_t e = rs[r] + 1; e < t; e++)
    if (col[e] <= col[e - 1]) { *bad = 1u; return; }
}

// ----------------------------------------------------------- vector helper ---

template <int VEC> struct V;
template <> struct V<4> {
  typedef float4 T;
  typedef uint4 I;           // the index of each float (min / max aggregation)
  static __device__ __forceinline__ T zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
  static __device__ __forceinline__ T ld(const T* p) { return __ldg(p); }
  static __device__ __forceinline__ T ld_plain(const T* p) { return *p; }
  static __device__ __forceinline__ void st(T* p, const T& v) { *p = v; }
  static __device__ __forceinline__ void add(T& a, const T& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
  static __device__ __forceinline__ void fma(T& a, float w, const T& b) {
    a.x = fmaf(w, b.x, a.x); a.y = fmaf(w, b.y, a.y); a.z = fmaf(w, b.z, a.z); a.w = fmaf(w, b.w, a.w);
  }
  static __device__ __forceinline__ T rdiv(const T& a, const RowDiv& r) {
    float v[4] = {a.x, a.y, a.z, a.w};
    rowdiv4(v, r);          // one safety test for the four quotients
    return make_float4(v[0], v[1], v[2], v[3]);
  }
  static __device__ __forceinline__ T relu(const T& a) {
    return make_float4(relu_nanprop(a.x), relu_nanprop(a.y), relu_nanprop(a.z), relu_nanprop(a.w));
  }
};
template <> struct V<1> {
  typedef float T;
  typedef uint32_t I;
  static __device__ __forceinline__ T zero() { return 0.f; }
  static __device__ __forceinline__ T ld(const T* p) { return __ldg(p); }
  static __device__ __forceinline__ T ld_plain(const T* p) { return *p; }
  static __device__ __forceinline__ void st(T* p, const T& v) { *p = v; }
  static __device__ __forceinline__ void add(T& a, const T& b) { a += b; }
  static __device__ __forceinline__ void fma(T& a, float w, const T& b) { a = fmaf(w, b, a); }
  static __device__ __forceinline__ T rdiv(const T& a, const RowDiv& r) { return rowdiv(a, r); }
  static __device__ __forceinline__ T relu(const T& a) { return relu_nanprop(a); }
};

// One T-column of a bf16 row (BSUM): VEC bf16 values (2 * VEC bytes, element 0 in the low half of the first word),
// each widened exactly, as to_f32 does.
__device__ __forceinline__ float4 widen_bf16x4(uint2 u) {
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xFFFF0000u));
}
template <int VEC>
__device__ __forceinline__ typename V<VEC>::T ld_bf16(const char* p) {
  if constexpr (VEC == 4) return widen_bf16x4(__ldg(reinterpret_cast<const uint2*>(p)));
  else return to_f32(__ldg(reinterpret_cast<const unsigned short*>(p)));
}

// ------------------------------------------------------- min / max reduction ---
// What a kernel does with each gathered row.  SUM adds it; MAX / MIN keep, per float, the value and the source id of
// the first edge in CSR order that holds the extreme (roc_sg_minmax_forward_planned); MASK is the backward of those:
// it adds the gathered gradient only where the gathered index names the row being computed.
// The attention passes (roc_sg_attn_*): ASTAT gives each row's (m, Z) per head, ATTN the a-weighted sum, ADST the
// destination-score gradient (heads wide), ASRC the input gradient and the source-score gradient.
// The edge-weighted passes (roc_sg_weighted_*, roc_sg_edge_dot_planned): WSUM the w-weighted sum, EDOT the per-edge
// dot product G[i] . X[j] (the gradient of the edge weights).
// The exact backwards over a transposed plan (roc_sg_transpose_*_backward): TSUM is the sum whose NORM epilogue
// divides by the in-degree of the original graph (its row ends in p.xrow) instead of the plan's row length; TMASK is
// MASK where an entry whose destination repeats the previous entry's in the same row (a duplicate edge) adds nothing.
// BSUM is the sum over bf16 rows (roc_sg_forward_planned_bf16): only its loads differ from SUM's, each T-column of VEC
// bf16 values widened exactly in registers, so it adds the same floats in the same order.
// SG_RED_BF16 added to MAX, MIN, ATTN, ADST, ASRC, WSUM or EDOT is that reduction's bf16 form (the roc_sg_*_bf16
// calls): the feature rows X it reads (gathered, or ASRC's own row i) are bf16, loaded and widened as BSUM's are, and
// everything else is the fp32 reduction's, its row of SG_REDS included.
// TELE is the sum whose row store is the teleport of roc_sg_forward_teleport_planned (tele_store): it adds what SUM adds
// in SUM's order, and only what a finished row stores differs.
enum { SG_RED_SUM = 0, SG_RED_MAX = ROC_SG_AGGR_MAX, SG_RED_MIN = ROC_SG_AGGR_MIN, SG_RED_MASK = 3,
       SG_RED_ASTAT = 4, SG_RED_ATTN = 5, SG_RED_ADST = 6, SG_RED_ASRC = 7, SG_RED_WSUM = 8, SG_RED_EDOT = 9,
       SG_RED_TSUM = 10, SG_RED_TMASK = 11, SG_RED_BSUM = 12, SG_RED_TELE = 13 };
constexpr int SG_RED_BF16 = 16;
// SG_RED_DROP added to ATTN, ADST or ASRC (with or without SG_RED_BF16) is that pass with attention dropout
// (roc_sg_attn_*_dropout): it loads each edge's keep byte (p.keep) beside its source id, the way WSUM loads its weight,
// and weighs a dropped head's term by 0 and a kept one's by p.keepScale; everything else, its row of SG_REDS included,
// is the pass without dropout's.
// SG_RED_DROP added to SUM, TSUM or TELE is that sum with edge dropout (roc_sg_forward_dropout_planned,
// roc_sg_transpose_sum_backward_dropout, roc_sg_forward_teleport_dropout_planned): it loads each edge's keep byte the
// same way, gathers the source row only where bit 0 is set and adds it as fmaf(p.dropScale, x, acc); a dropped edge's
// row is never loaded.  Its column blocks, row shapes, fix-ups and row store are the sum's, but every width runs on
// sg_chunk_kernel (no ring form).
constexpr int SG_RED_DROP = 32;
__host__ __device__ constexpr int sg_red_base(int RF) { return RF & (SG_RED_BF16 - 1); }
// the rows gathered as `in` are bf16 (every bf16 form but ASRC's, which gathers fp32 gradients)
__host__ __device__ constexpr bool sg_bf16_in(int RF) {
  return RF == SG_RED_BSUM || ((RF & SG_RED_BF16) && sg_red_base(RF) != SG_RED_ASRC);
}
constexpr uint32_t SG_NOARG = 0xFFFFFFFFu;   // index of a row that has no edge yet

// The ordering rule: the candidate v replaces the current a iff it is strictly greater (smaller) or it is NaN and a
// is not.  `!(v <= a || a != a)` is exactly that for max.  A current index of SG_NOARG means "no edge yet": the
// first edge always wins.  Taking the partials of consecutive edge ranges in order with the same rule gives the
// result of one sequential pass (the rule picks the leftmost maximal element of a total preorder).
template <int RED>
__device__ __forceinline__ void mm_take(float& a, uint32_t& ai, float v, uint32_t vi) {
  const bool better = (RED == SG_RED_MAX) ? !(v <= a || a != a) : !(v >= a || a != a);
  if (ai == SG_NOARG || better) { a = v; ai = vi; }
}
// one edge: every float of the row has the same source id
template <int RED>
__device__ __forceinline__ void mm_add(float4& a, uint4& ai, const float4& v, uint32_t src) {
  mm_take<RED>(a.x, ai.x, v.x, src); mm_take<RED>(a.y, ai.y, v.y, src);
  mm_take<RED>(a.z, ai.z, v.z, src); mm_take<RED>(a.w, ai.w, v.w, src);
}
template <int RED>
__device__ __forceinline__ void mm_add(float& a, uint32_t& ai, float v, uint32_t src) { mm_take<RED>(a, ai, v, src); }
// a partial of a later edge range (fix-ups): one with no edge is skipped
template <int RED>
__device__ __forceinline__ void mm_combine1(float& a, uint32_t& ai, float v, uint32_t vi) {
  if (vi != SG_NOARG) mm_take<RED>(a, ai, v, vi);
}
template <int RED>
__device__ __forceinline__ void mm_combine(float4& a, uint4& ai, const float4& v, const uint4& vi) {
  mm_combine1<RED>(a.x, ai.x, v.x, vi.x); mm_combine1<RED>(a.y, ai.y, v.y, vi.y);
  mm_combine1<RED>(a.z, ai.z, v.z, vi.z); mm_combine1<RED>(a.w, ai.w, v.w, vi.w);
}
template <int RED>
__device__ __forceinline__ void mm_combine(float& a, uint32_t& ai, float v, uint32_t vi) { mm_combine1<RED>(a, ai, v, vi); }
// a row with no edge stores 0 (its index stays SG_NOARG)
__device__ __forceinline__ float mm_value1(float a, uint32_t ai) { return ai == SG_NOARG ? 0.f : a; }
__device__ __forceinline__ float4 mm_value(const float4& a, const uint4& ai) {
  return make_float4(mm_value1(a.x, ai.x), mm_value1(a.y, ai.y), mm_value1(a.z, ai.z), mm_value1(a.w, ai.w));
}
__device__ __forceinline__ float mm_value(float a, uint32_t ai) { return mm_value1(a, ai); }
__device__ __forceinline__ uint4 mm_noarg(uint4*) { return make_uint4(SG_NOARG, SG_NOARG, SG_NOARG, SG_NOARG); }
__device__ __forceinline__ uint32_t mm_noarg(uint32_t*) { return SG_NOARG; }
// backward: acc += (arg == me) ? g : 0
__device__ __forceinline__ void mask_add(float4& acc, const float4& g, const uint4& a, uint32_t me) {
  acc.x += (a.x == me) ? g.x : 0.f; acc.y += (a.y == me) ? g.y : 0.f;
  acc.z += (a.z == me) ? g.z : 0.f; acc.w += (a.w == me) ? g.w : 0.f;
}
__device__ __forceinline__ void mask_add(float& acc, float g, uint32_t a, uint32_t me) { acc += (a == me) ? g : 0.f; }

// ------------------------------------------------------- attention helpers ---
__device__ __forceinline__ float leaky(float z, float slope) { return z > 0.f ? z : slope * z; }
// a = exp(y - m) / Z from the row's stats; a row of degree 0 (1/Z = 0) gives 0 whatever y is
__device__ __forceinline__ float attn_alpha(float y, float m, float iz) { return iz == 0.f ? 0.f : expf(y - m) * iz; }
// the product of two T-columns over their first nv floats (the rest of a partial last float4 is padding)
__device__ __forceinline__ float dot_t(const float4& a, const float4& b, int nv) {
  float s = a.x * b.x;
  s += (nv > 1) ? a.y * b.y : 0.f;
  s += (nv > 2) ? a.z * b.z : 0.f;
  s += (nv > 3) ? a.w * b.w : 0.f;
  return nv > 0 ? s : 0.f;
}
__device__ __forceinline__ float dot_t(float a, float b, int nv) { return nv > 0 ? a * b : 0.f; }
__device__ __forceinline__ float4 attn_scale(float a, const float4& v) { return make_float4(a * v.x, a * v.y, a * v.z, a * v.w); }
__device__ __forceinline__ float attn_scale(float a, float v) { return a * v; }
// attention dropout: x scaled by s where bit k of the edge's keep byte is set, else 0
__device__ __forceinline__ float keep_mul(uint32_t kb, uint32_t k, float s, float x) { return ((kb >> k) & 1u) ? x * s : 0.f; }
// Per-head sums of d[ch] (lane `lane` holds T-column lane + ch*L; a head is 2^ftShift consecutive T-columns): first
// across the chunks of one head in the lane (a pairwise tree), then across the head's lanes (an xor butterfly, whose
// two operands are added in either order to the same bits, so every lane of the head ends with identical sums).
// Every branch is uniform across the worker, as the shuffles need.
template <int L, int NCH>
__device__ __forceinline__ void head_sum(float (&d)[NCH], uint32_t ftShift, unsigned wmask) {
  constexpr int LS = L == 4 ? 2 : L == 8 ? 3 : L == 16 ? 4 : 5;
  const int gs = ftShift > (uint32_t)LS ? (int)min(ftShift - LS, 3u) : 0;     // log2 of the chunks per head
#pragma unroll
  for (int s = 0; (1 << s) < NCH; s++)
#pragma unroll
    for (int ch = 0; ch + (1 << s) < NCH; ch += 2 << s)
      if (s < gs) d[ch] += d[ch + (1 << s)];
  const int span = 1 << min((int)ftShift, LS);                               // lanes per head
#pragma unroll
  for (int ch = 0; ch < NCH; ch++)
    if ((ch & ((1 << gs) - 1)) == 0)
      for (int o = 1; o < span; o <<= 1) d[ch] += __shfl_xor_sync(wmask, d[ch], o, L);
#pragma unroll
  for (int ch = 1; ch < NCH; ch++) {            // every chunk takes its group's sum (indices resolved at compile time)
    float v = d[ch];
#pragma unroll
    for (int g = 1; g <= 3; g++)
      if (gs == g) v = d[ch & ~((1 << g) - 1)];
    d[ch] = v;
  }
}

struct SgParams {
  const uint32_t* rs;
  const uint32_t* firstRow;
  const uint32_t* carryIdx;
  const uint32_t* heavyRows;
  const uint32_t* bigRows;
  const uint32_t* col;
  const void* in;      // [*][ldIn]  (in units of T)
  void* out;           // [nloc][ldOut]
  void* carry;         // [numCarries][ldC]
  size_t ldIn, ldOut, ldC;   // in units of T (float4 or float)
  uint32_t Q;          // valid T-columns per row
  uint32_t E, numChunks, numHeavy, numBig;
  int epi;
  const uint32_t* desc; // [numChunks][8] chunk start records (k_chunk_desc)
  // min / max aggregation
  // The attention dropout passes (SG_RED_DROP) take the arg and dwAdd slots, which no attention pass uses, so that the
  // struct keeps its size: the record kernel's arguments after it keep their offsets, and so its code.
  union {
    void* arg;          // MAX / MIN: [nloc][ldArg] indices written; MASK: [*][ldArg] indices gathered like `in`
    const uint8_t* keep;  // attention dropout: [E] one keep byte per local edge (bit k keeps head k)
  };
  void* carryArg;       // MAX / MIN: [numCarries][ldC] indices of the carry partials
  size_t ldArg;         // in units of T
  uint32_t selfBase;    // MASK, attention: id of local row 0 in the id space of col
  union {
    int dwAdd;          // EDOT: add to dw instead of overwriting it
    float keepScale;    // attention dropout: the scale of a kept weight
    float teleBeta;     // TELE: beta, the coefficient of t
  };
  // attention (units of float unless stated).  The edge-weighted passes use two of its slots (score, out2), so that
  // the struct, every kernel's parameter block, keeps its layout (a union there changed the attention kernels' code).
  const float* score;   // [*][ldS]  s_dst | s_src, indexed like `in`;  WSUM: [E] each local edge's weight
  const float* stats;   // ATTN: [nloc][ldStats] m | 1/Z of the local rows
  const float4* rec;    // ADST / ASRC: [*][heads] {s_dst, m, 1/Z, D}, indexed like `in`
  const void* xrow;     // ADST, EDOT: G, ASRC: X, the local row's own row (units of T, ldX); EDOT: indexed by plan
                        // row, else like `in`.  TSUM: the original graph's rowEnd (u64), for in_degree.  TELE: t, fp32
                        // rows indexed by plan row with leading dimension ldS (in floats), and alpha in `slope`
  float* out2;          // ASTAT: unused; ADST / ASRC: heads-wide output [nloc][ldOut2];  EDOT: [E] dw of each local edge
  float* carry2;        // [numCarries][SG_LDC2] heads-wide partials (ASTAT: m | Z)
  size_t ldS, ldStats, ldX, ldOut2;
  uint32_t heads;
  union {
    uint32_t ftShift;   // log2 of the T-columns per head (31 for one head)
    float dropScale;    // edge dropout (SG_RED_DROP on SUM, TSUM, TELE): the scale of a kept row
  };
  uint32_t H;           // EDOT, TELE: H floats per row
  float slope;
};
constexpr int SG_LDC2 = 16;     // 2 * the most heads

// The lanes of the calling thread's L-lane worker within its warp: the mask of the worker's sub-warp shuffles.
template <int L>
__device__ __forceinline__ unsigned worker_mask() {
  return (L == 32) ? 0xffffffffu : (((1u << L) - 1u) << (((threadIdx.x & 31) / L) * L));
}
// Attention: the floats of T-column c that hold features (the rest of a partial last float4 is padding; none past Q).
template <int VEC>
__device__ __forceinline__ int t_floats(uint32_t c, const SgParams& p) {
  return (VEC == 4) ? max(0, min(4, (int)p.H - 4 * (int)c)) : (c < p.Q ? 1 : 0);
}
// Attention: the bits of a T-column's index within its head.  Column c is the head's first, whose lane stores the
// head's sums, when c < Q and (c & head_mask(p)) == 0.
__device__ __forceinline__ uint32_t head_mask(const SgParams& p) {
  return (p.ftShift >= 31u) ? 0x7FFFFFFFu : ((1u << p.ftShift) - 1u);
}

// out[v] = relu?(acc / sqrtf(deg)) — what the model applies right after
// scatter_gather (gnn.cc:84-85), IEEE sqrt and divide like graphnorm_kernel.cu:49-51.
// The divisor is uniform over the row, so the divide is the row-uniform form of common.cuh
// (one refined reciprocal, 3 FMAs per element, bit-identical to div.rn), cheaper than the plain `/`
// (zero pad lanes take its slow path).
template <int VEC>
__device__ __forceinline__ void epi_store(typename V<VEC>::T v, typename V<VEC>::T* dst, uint32_t deg, int epi) {
  if (epi & ROC_SG_EPI_NORM) {
    const RowDiv rd = rowdiv_make(sqrtf((float)deg));
    v = V<VEC>::rdiv(v, rd);
  }
  if (epi & ROC_SG_EPI_RELU) v = V<VEC>::relu(v);
  V<VEC>::st(dst, v);
}

// TSUM: the in-degree of node r in the original whole graph, from its row ends (what roc_indegree_norm divides by).
__device__ __forceinline__ uint32_t in_degree(const SgParams& p, uint32_t r) {
  const uint64_t* re = static_cast<const uint64_t*>(p.xrow);
  return (uint32_t)(__ldg(re + r) - (r ? __ldg(re + r - 1) : 0ull));
}
// What the NORM epilogue of plan row r, of `len` edges, divides by the square root of.
template <int RED>
__device__ __forceinline__ uint32_t norm_deg(const SgParams& p, uint32_t r, uint32_t len) {
  if constexpr (RED == SG_RED_TSUM) return in_degree(p, r);
  else return len;
}

// TELE's row store: out[v] = post(fmaf(alpha, pre(acc), beta * t[v])), pre and post the divide by sqrtf(deg) of
// ROC_SG_EPI_NORM and ROC_SG_EPI_NORM_OUT, each in epi_store's row-uniform form (== the IEEE divide).  That is, float
// for float, roc_sg_forward_planned (NORM or NONE), then roc_scaled_add_fwd (beta * t rounded first), then
// roc_indegree_norm.  t is read one float at a time, so that any pitch and alignment of t takes the row form `in` and
// `out` chose; the pad floats of a partial last float4 take t = 0.  Column c (in T-columns) of plan row `row`.
__device__ __forceinline__ float tele_axpby(float a, float x, float b, float t) { return fmaf(a, x, __fmul_rn(b, t)); }
__device__ __forceinline__ float4 tele_axpby(float a, const float4& x, float b, const float4& t) {
  return make_float4(tele_axpby(a, x.x, b, t.x), tele_axpby(a, x.y, b, t.y), tele_axpby(a, x.z, b, t.z),
                     tele_axpby(a, x.w, b, t.w));
}
template <int VEC>
__device__ __forceinline__ void tele_store(const SgParams& p, typename V<VEC>::T v, typename V<VEC>::T* dst, uint32_t row,
                                           uint32_t c, uint32_t deg) {
  const float* tr = static_cast<const float*>(p.xrow) + (uint64_t)row * p.ldS + (uint64_t)c * VEC;
  typename V<VEC>::T t;
  if constexpr (VEC == 4) {
    const int nv = min(4, (int)p.H - 4 * (int)c);
    t = make_float4(__ldg(tr), nv > 1 ? __ldg(tr + 1) : 0.f, nv > 2 ? __ldg(tr + 2) : 0.f, nv > 3 ? __ldg(tr + 3) : 0.f);
  } else {
    t = __ldg(tr);
  }
  const bool pre = (p.epi & ROC_SG_EPI_NORM) != 0, post = (p.epi & ROC_SG_EPI_NORM_OUT) != 0;
  const RowDiv rd = rowdiv_make((pre || post) ? sqrtf((float)deg) : 1.f);
  if (pre) v = V<VEC>::rdiv(v, rd);
  v = tele_axpby(p.slope, v, p.teleBeta, t);
  if (post) v = V<VEC>::rdiv(v, rd);
  V<VEC>::st(dst, v);
}

// ------------------------------------------------------------- main kernel ---
// One worker (L lanes) per chunk.  Lane `lane` owns T-columns lane + ch*L.
// RED (SG_RED_*) changes only what is done with a gathered row and what the row store writes; the schedule, the
// gathers and the single store site are the same for every reduction.  RF is RED, plus SG_RED_BF16 for its bf16 form.
template <int VEC, int L, int NCH, int U, int MINB, int RF = SG_RED_SUM>
__global__ void __launch_bounds__(SG_THREADS, MINB)
sg_chunk_kernel(const SgParams p) {
  typedef typename V<VEC>::T T;
  typedef typename V<VEC>::I I;
  constexpr int RED = sg_red_base(RF);
  constexpr bool MM = RED == SG_RED_MAX || RED == SG_RED_MIN;
  constexpr bool AT = RED >= SG_RED_ASTAT && RED <= SG_RED_ASRC; // an attention pass
  constexpr bool SV = RED == SG_RED_ATTN || RED == SG_RED_ADST;  // gathers s_src[j] beside in[j]
  constexpr bool XI = RED == SG_RED_ADST || RED == SG_RED_ASRC;  // holds a row of its own row i, and heads-wide sums
  constexpr bool WS = RED == SG_RED_WSUM;                        // loads each edge's weight beside its source id
  constexpr bool ED = RED == SG_RED_EDOT;                        // holds G[i], stores one dot product per edge
  constexpr bool MK = RED == SG_RED_MASK || RED == SG_RED_TMASK; // gathers an index row beside each gradient row
  constexpr bool BX = (RF & SG_RED_BF16) && RED == SG_RED_ASRC;  // its own row X[i] (xrow) is bf16
  constexpr bool BF = sg_bf16_in(RF);                            // gathers bf16 rows
  constexpr bool DR = (RF & SG_RED_DROP) != 0;                   // attention or edge dropout: loads each edge's keep byte
  constexpr bool DS = DR && (RED == SG_RED_SUM || RED == SG_RED_TSUM || RED == SG_RED_TELE);   // edge dropout of a sum
  static_assert(!DR || DS || RED == SG_RED_ATTN || RED == SG_RED_ADST || RED == SG_RED_ASRC,
                "dropout of an attention gather or a sum");
  static_assert(!DR || !(RF & SG_RED_BF16) || !DS, "no edge dropout over bf16 rows");
  constexpr uint32_t TB = BF ? 2 * VEC : sizeof(T);              // bytes of one T-column of `in`
  constexpr int WPB = SG_THREADS / L;
  constexpr uint32_t CH = SG_CH;
  const int lane = threadIdx.x % L;
  const uint32_t w = blockIdx.x * WPB + threadIdx.x / L;
  if (w >= p.numChunks) return;
  const unsigned wmask = worker_mask<L>();
  (void)wmask;

  const uint32_t* __restrict__ rs = p.rs;
  const uint32_t* __restrict__ col = p.col;
  const T* __restrict__ in = reinterpret_cast<const T*>(p.in);
  T* __restrict__ out = reinterpret_cast<T*>(p.out);

  bool act[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) act[ch] = (uint32_t)(lane + ch * L) < p.Q;

  const uint32_t cb = w * CH;
  const uint32_t ce = min(cb + CH, p.E);

  // The worker's start state comes from the plan's 32-byte chunk record (k_chunk_desc) — one load instead of
  // the dependent walk firstRow[w] -> rs[r0], rs[r0 - 1] -> ... that cost every worker three round trips
  // before its first gather.
  const uint4 dA = __ldg(reinterpret_cast<const uint4*>(p.desc) + 2 * (size_t)w);
  const uint4 dB = __ldg(reinterpret_cast<const uint4*>(p.desc) + 2 * (size_t)w + 1);
  if (dB.z & 2u) return;           // nothing owned, nothing carried
  uint32_t cur = dA.z;             // row id of the current segment
  uint32_t curS = dA.w, curT = dB.x;   // its [start, end) in the edge array
  uint32_t e = dA.x;               // next edge
  const uint32_t ee = dA.y;        // end of this worker's whole edge range
  const uint32_t r1 = dB.y;
  const uint32_t carrySlot = dB.w;
  int kind = (dB.z & 1u) ? 0 : ((curT - curS > CH) ? 2 : 1);   // 0 = carry-in part of a heavy row, 1 = complete row, 2 = cut heavy row
  uint32_t segEnd = (kind == 1) ? curT : min(curT, ce);        // where this worker stops accumulating into it

  T acc[NCH];
  I aidx[NCH];          // MAX / MIN: source id behind each float of acc
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) {
    acc[ch] = V<VEC>::zero();
    if constexpr (MM) aidx[ch] = mm_noarg((I*)nullptr);
  }

  // Attention: the head of each column chunk, its valid floats, and the current row's state (row_state).
  constexpr int NA = (AT || ED) ? NCH : 1;
  uint32_t kh[NA];
  int nv[NA];
  float accS[NA];       // ASTAT: Z (acc holds m); ADST / ASRC: the heads-wide sums
  float r0s[NA], r1s[NA], r2s[NA];   // ASTAT: s_dst[i]; ATTN: s_dst[i], m[i], 1/Z[i]; ASRC: s_src[i]
  float4 rrec[RED == SG_RED_ADST ? NCH : 1];   // ADST: the record of row i
  T xi[(XI || ED) ? NCH : 1];   // ADST, EDOT: G[i], ASRC: X[i]
  if constexpr (ED) {
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) nv[ch] = t_floats<VEC>((uint32_t)(lane + ch * L), p);
  }
  if constexpr (AT) {
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) {
      const uint32_t c = (uint32_t)(lane + ch * L);
      kh[ch] = min(c, p.Q - 1u) >> p.ftShift;
      nv[ch] = t_floats<VEC>(c, p);
      accS[ch] = 0.f;
      if constexpr (RED == SG_RED_ASTAT) acc[ch] = -INFINITY;
    }
  }
  auto row_state = [&]() {
    if constexpr (AT) {
      const uint64_t gi = (uint64_t)(p.selfBase + cur);
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        if constexpr (RED == SG_RED_ASTAT || RED == SG_RED_ATTN) r0s[ch] = __ldg(p.score + gi * p.ldS + kh[ch]);
        if constexpr (RED == SG_RED_ATTN) {
          r1s[ch] = __ldg(p.stats + (uint64_t)cur * p.ldStats + kh[ch]);
          r2s[ch] = __ldg(p.stats + (uint64_t)cur * p.ldStats + p.heads + kh[ch]);
        }
        if constexpr (RED == SG_RED_ASRC) r0s[ch] = __ldg(p.score + gi * p.ldS + p.heads + kh[ch]);
        if constexpr (RED == SG_RED_ADST) rrec[ch] = __ldg(p.rec + gi * p.heads + kh[ch]);
        if constexpr (BX)
          xi[ch] = ld_bf16<VEC>(static_cast<const char*>(p.xrow) +
                                (gi * p.ldX + min((uint32_t)(lane + ch * L), p.Q - 1u)) * (2 * VEC));
        else if constexpr (XI)
          xi[ch] = V<VEC>::ld(reinterpret_cast<const T*>(p.xrow) + gi * p.ldX + min((uint32_t)(lane + ch * L), p.Q - 1u));
      }
    }
    if constexpr (ED) {
#pragma unroll
      for (int ch = 0; ch < NCH; ch++)
        xi[ch] = V<VEC>::ld(reinterpret_cast<const T*>(p.xrow) + (uint64_t)cur * p.ldX + min((uint32_t)(lane + ch * L), p.Q - 1u));
    }
  };
  row_state();

  // Row store.  The epilogue (IEEE sqrt + divides) lives in ONE out-of-line copy:
  // inlining it at every edge position made the kernel 4096 SASS instructions and
  // instruction-fetch bound.
  auto flush = [&]() {
    if constexpr (ED) return;           // its outputs are per edge, stored as it goes
    char* dstb = (kind == 0)
        ? reinterpret_cast<char*>(reinterpret_cast<T*>(p.carry) + lane) + (uint64_t)carrySlot * ((uint32_t)p.ldC * (uint32_t)sizeof(T))
        : reinterpret_cast<char*>(out + lane) + (uint64_t)cur * ((uint32_t)p.ldOut * (uint32_t)sizeof(T));
    T* dst = reinterpret_cast<T*>(dstb);
    if constexpr (MM) {
      // the owner of a cut row stores its partial to out / arg, a later chunk to its carry slot
      char* ib = (kind == 0)
          ? reinterpret_cast<char*>(reinterpret_cast<I*>(p.carryArg) + lane) + (uint64_t)carrySlot * ((uint32_t)p.ldC * (uint32_t)sizeof(I))
          : reinterpret_cast<char*>(reinterpret_cast<I*>(p.arg) + lane) + (uint64_t)cur * ((uint32_t)p.ldArg * (uint32_t)sizeof(I));
      I* idst = reinterpret_cast<I*>(ib);
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        if (act[ch]) {
          V<VEC>::st(dst + ch * L, mm_value(acc[ch], aidx[ch]));
          idst[ch * L] = aidx[ch];
        }
        acc[ch] = V<VEC>::zero();
        aidx[ch] = mm_noarg((I*)nullptr);
      }
      return;
    }
    if constexpr (RED == SG_RED_ASTAT) {
      // lane k holds head k's (m, Z): a complete row stores m and 1/Z (0 and 0 with no edge), a cut row's parts their
      // raw (m, Z) for sg_attn_stat_fixup
      float* sdst = (kind == 0) ? p.carry2 + (uint64_t)carrySlot * SG_LDC2 : reinterpret_cast<float*>(p.out) + (uint64_t)cur * p.ldOut;
      if (act[0]) {
        const float m = acc[0], z = accS[0];
        const bool done = kind == 1;
        sdst[lane] = (done && !(z > 0.f)) ? 0.f : m;
        sdst[p.heads + lane] = !done ? z : (z > 0.f ? 1.f / z : 0.f);
      }
      acc[0] = -INFINITY; accS[0] = 0.f;
      return;
    }
    if constexpr (XI) {
      // the heads-wide sums: the lane of a head's first column stores them
      float* d2 = (kind == 0) ? p.carry2 + (uint64_t)carrySlot * SG_LDC2 : p.out2 + (uint64_t)cur * p.ldOut2;
      const uint32_t ftMask = head_mask(p);
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        const uint32_t c = (uint32_t)(lane + ch * L);
        if (c < p.Q && (c & ftMask) == 0) d2[kh[ch]] = accS[ch];
        accS[ch] = 0.f;
      }
      if constexpr (RED == SG_RED_ADST) return;
    }
    if constexpr (RED == SG_RED_TELE) {
      // a complete row takes the teleport whatever p.epi is; a cut row's parts store raw partials for the fix-ups
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        if (act[ch]) {
          if (kind == 1) tele_store<VEC>(p, acc[ch], dst + ch * L, cur, (uint32_t)(lane + ch * L), curT - curS);
          else V<VEC>::st(dst + ch * L, acc[ch]);
        }
        acc[ch] = V<VEC>::zero();
      }
      return;
    }
    const int epi = (kind == 1) ? p.epi : 0;
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) {
      if (act[ch]) {
        if (epi) epi_store<VEC>(acc[ch], dst + ch * L, norm_deg<RED>(p, cur, curT - curS), epi);
        else V<VEC>::st(dst + ch * L, acc[ch]);
      }
      acc[ch] = V<VEC>::zero();
    }
  };
  auto advance = [&]() {  // move to the next owned row
    cur += 1; curS = curT; curT = rs[cur + 1];
    bool heavy = curT - curS > CH;
    segEnd = heavy ? min(curT, ce) : curT;
    kind = heavy ? 2 : 1;
    row_state();
  };

  // Every lane reads the source ids itself (same address across the worker: one broadcast
  // transaction from L1); sub-warp shuffles with a runtime mask cost a MATCH.ANY sequence each.
  // Gathers are unpredicated: a group that runs past the worker's last edge re-reads that edge's
  // source (index clamped; an L1 hit) and the tail values are simply never added.  With the tail
  // predicates (16 ISETP + 20 zero-inits per group) and a 64 x 64-bit address multiply the group
  // preamble was 146 SASS instructions for 8 gathers; now one VIMNMX + LDG + IMAD.WIDE
  // + LDG.128 per edge.
  // lanes beyond the row's last column gather that last column instead (same sector, no extra
  // traffic): their sums are never stored (flush tests act[]), and no load needs a predicate
  const char* inl[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) {
    if constexpr (BF)
      inl[ch] = reinterpret_cast<const char*>(p.in) + (size_t)min((uint32_t)(lane + ch * L), p.Q - 1u) * TB;
    else
      inl[ch] = reinterpret_cast<const char*>(in + min((uint32_t)(lane + ch * L), p.Q - 1u));
  }
  const uint32_t rowBytes = (uint32_t)p.ldIn * TB;
  // MASK: the index row of each edge's source is gathered next to its gradient row
  const char* argl[MK ? NCH : 1];
  uint32_t argRowBytes = 0;
  if constexpr (MK) {
#pragma unroll
    for (int ch = 0; ch < NCH; ch++)
      argl[ch] = reinterpret_cast<const char*>(reinterpret_cast<const I*>(p.arg) + min((uint32_t)(lane + ch * L), p.Q - 1u));
    argRowBytes = (uint32_t)p.ldArg * (uint32_t)sizeof(I);
  }
  const uint32_t eLast = ee - 1u;
#pragma unroll 1
  for (uint32_t base = e; base < ee; base += U) {
    const uint32_t cnt = min((uint32_t)U, ee - base);
    uint32_t srcs[U];
    float wv[WS ? U : 1];                      // WSUM: each edge's weight, loaded like its source id
    uint32_t kb[DR ? U : 1];                   // attention dropout: each edge's keep byte, likewise
    if (cnt == (uint32_t)U) {
      const uint32_t* colp = col + base;       // full group: one address, immediate offsets
#pragma unroll
      for (int u = 0; u < U; u++) srcs[u] = __ldg(colp + u);
      if constexpr (WS) {
#pragma unroll
        for (int u = 0; u < U; u++) wv[u] = __ldg(p.score + base + u);
      }
      if constexpr (DR) {
#pragma unroll
        for (int u = 0; u < U; u++) kb[u] = __ldg(p.keep + base + u);
      }
    } else {
#pragma unroll
      for (int u = 0; u < U; u++) srcs[u] = __ldg(col + min(base + (uint32_t)u, eLast));
      if constexpr (WS) {
#pragma unroll
        for (int u = 0; u < U; u++) wv[u] = __ldg(p.score + min(base + (uint32_t)u, eLast));
      }
      if constexpr (DR) {
#pragma unroll
        for (int u = 0; u < U; u++) kb[u] = __ldg(p.keep + min(base + (uint32_t)u, eLast));
      }
    }
    // TMASK: bit u is set when edge base + u has the destination of the edge before it (for u = 0 the edge before the
    // group, which may lie in an earlier chunk of the same row); whether that edge is in the same row is checked when
    // the edge is added
    [[maybe_unused]] uint32_t repeat = 0;
    if constexpr (RED == SG_RED_TMASK) {
      uint32_t prev = __ldg(col + (base ? base - 1u : 0u));
#pragma unroll
      for (int u = 0; u < U; u++) {
        repeat |= (srcs[u] == prev ? 1u : 0u) << u;
        prev = srcs[u];
      }
    }
    T v[U][NCH];
    I av[MK ? U : 1][MK ? NCH : 1];
    float sv[SV ? U : 1][SV ? NCH : 1];                              // ATTN / ADST: s_src[j] of each chunk's head
    float4 rv[RED == SG_RED_ASRC ? U : 1][RED == SG_RED_ASRC ? NCH : 1];   // ASRC: the record of j
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint64_t off = (uint64_t)srcs[u] * rowBytes;
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        if constexpr (BF) v[u][ch] = ld_bf16<VEC>(inl[ch] + off);
        else if constexpr (DS)   // edge dropout: a dropped edge's row is not loaded, and adds fmaf(s, 0, acc) == acc
          v[u][ch] = (kb[u] & 1u) ? V<VEC>::ld(reinterpret_cast<const T*>(inl[ch] + off)) : V<VEC>::zero();
        else v[u][ch] = V<VEC>::ld(reinterpret_cast<const T*>(inl[ch] + off));
      }
      if constexpr (MK) {
        const uint64_t aoff = (uint64_t)srcs[u] * argRowBytes;
#pragma unroll
        for (int ch = 0; ch < NCH; ch++) av[u][ch] = __ldg(reinterpret_cast<const I*>(argl[ch] + aoff));
      }
      if constexpr (SV) {
#pragma unroll
        for (int ch = 0; ch < NCH; ch++) sv[u][ch] = __ldg(p.score + (uint64_t)srcs[u] * p.ldS + p.heads + kh[ch]);
      }
      if constexpr (RED == SG_RED_ASRC) {
#pragma unroll
        for (int ch = 0; ch < NCH; ch++) rv[u][ch] = __ldg(p.rec + (uint64_t)srcs[u] * p.heads + kh[ch]);
      }
    }
    {
      // One rolled loop over the row segments of the group (predicated adds of the edges [pos, lim)
      // of the current segment, then ONE copy of the row store).  A separate branch-free path for
      // groups inside one row did not pay: the two 16-lane workers of a warp rarely agree, so the
      // warp ran both paths in most iterations.  The
      // unrolled per-edge `while (edge == segEnd) { flush; advance; }` had 8 inlined copies of the
      // store and cost ~180 SASS instructions per row.
      uint32_t pos = 0;
      for (;;) {
        const uint32_t lim = min(cnt, segEnd - base);
#pragma unroll
        for (int u = 0; u < U; u++) {
          if ((uint32_t)u >= pos && (uint32_t)u < lim) {
            if constexpr (RED == SG_RED_ASTAT) {
              // online (m, Z) of head `lane`: the running max is exact, Z is rescaled when it grows
              const float y = leaky(r0s[0] + v[u][0], p.slope);
              float& m = acc[0];
              if (y > m) { accS[0] = accS[0] * expf(m - y) + 1.f; m = y; }
              else accS[0] += expf(y - m);
            } else if constexpr (RED == SG_RED_ATTN) {
#pragma unroll
              for (int ch = 0; ch < NCH; ch++) {
                const float a = attn_alpha(leaky(r0s[ch] + sv[u][ch], p.slope), r1s[ch], r2s[ch]);
                // dropout: a' = keep ? a s : 0
                V<VEC>::add(acc[ch], attn_scale(DR ? keep_mul(kb[u], kh[ch], p.keepScale, a) : a, v[u][ch]));
              }
            } else if constexpr (RED == SG_RED_ADST) {
              // dz(i<-j) = a(i<-j) (G[i].X[j] - D[i]) l: v is X[j], xi is G[i], rrec is {s_dst, m, 1/Z, D} of i;
              // dropout: a(i<-j) (M G[i].X[j] - D[i]) l, M = keep ? s : 0, with D over the dropped output
              float d[NCH];
#pragma unroll
              for (int ch = 0; ch < NCH; ch++) d[ch] = dot_t(xi[ch], v[u][ch], nv[ch]);
              head_sum<L, NCH>(d, p.ftShift, wmask);
#pragma unroll
              for (int ch = 0; ch < NCH; ch++) {
                const float z = rrec[ch].x + sv[u][ch];
                const float a = attn_alpha(leaky(z, p.slope), rrec[ch].y, rrec[ch].z);
                const float md = DR ? keep_mul(kb[u], kh[ch], p.keepScale, d[ch]) : d[ch];
                accS[ch] += a * (md - rrec[ch].w) * (z > 0.f ? 1.f : p.slope);
              }
            } else if constexpr (RED == SG_RED_ASRC) {
              // a(j<-i) G[j] and dz(j<-i) = a(j<-i) (G[j].X[i] - D[j]) l: v is G[j], xi is X[i], rv the record of j;
              // dropout: a'(j<-i) G[j] and a(j<-i) (M G[j].X[i] - D[j]) l, with the keep byte of the pair (j<-i)
              float d[NCH];
#pragma unroll
              for (int ch = 0; ch < NCH; ch++) d[ch] = dot_t(v[u][ch], xi[ch], nv[ch]);
              head_sum<L, NCH>(d, p.ftShift, wmask);
#pragma unroll
              for (int ch = 0; ch < NCH; ch++) {
                const float4 r = rv[u][ch];
                const float z = r.x + r0s[ch];
                const float a = attn_alpha(leaky(z, p.slope), r.y, r.z);
                V<VEC>::add(acc[ch], attn_scale(DR ? keep_mul(kb[u], kh[ch], p.keepScale, a) : a, v[u][ch]));
                const float md = DR ? keep_mul(kb[u], kh[ch], p.keepScale, d[ch]) : d[ch];
                accS[ch] += a * (md - r.w) * (z > 0.f ? 1.f : p.slope);
              }
            } else if constexpr (WS) {
#pragma unroll
              for (int ch = 0; ch < NCH; ch++) V<VEC>::fma(acc[ch], wv[u], v[u][ch]);
            } else if constexpr (ED) {
              // dw(e) = G[i] . X[j]: v is X[j], xi is G[i]; the whole row reduced like one attention head
              float d[NCH];
#pragma unroll
              for (int ch = 0; ch < NCH; ch++) d[ch] = dot_t(xi[ch], v[u][ch], nv[ch]);
              head_sum<L, NCH>(d, 31u, wmask);
              if (lane == 0) {
                float* q = p.out2 + base + (uint32_t)u;
                *q = p.dwAdd ? *q + d[0] : d[0];
              }
            } else if constexpr (RED == SG_RED_TMASK) {
              // a duplicate edge j -> i sits right after its twin in transposed row j (the sort is stable): only the
              // first of them adds, so each distinct destination's gradient is taken once
              if (base + (uint32_t)u == curS || !((repeat >> u) & 1u)) {
#pragma unroll
                for (int ch = 0; ch < NCH; ch++) mask_add(acc[ch], v[u][ch], av[u][ch], p.selfBase + cur);
              }
            } else {
#pragma unroll
              for (int ch = 0; ch < NCH; ch++) {
                if constexpr (DS) V<VEC>::fma(acc[ch], p.dropScale, v[u][ch]);
                else if constexpr (RED == SG_RED_SUM || RED == SG_RED_TSUM || RED == SG_RED_BSUM || RED == SG_RED_TELE)
                  V<VEC>::add(acc[ch], v[u][ch]);
                else if constexpr (RED == SG_RED_MASK) mask_add(acc[ch], v[u][ch], av[u][ch], p.selfBase + cur);
                else mm_add<RED>(acc[ch], aidx[ch], v[u][ch], srcs[u]);
              }
            }
          }
        }
        pos = lim;
        if (pos >= cnt) break;
        flush();
        advance();
      }
    }
  }
  flush();
  while (cur + 1 < r1) { advance(); flush(); }  // trailing zero-degree rows
}

// -------------------------------------- main kernel, 65..256 floats (U and T) ---
// Same schedule and the same per-row summation order as sg_chunk_kernel, but the neighbour rows are fetched by
// the TMA unit: four `cp.async.bulk` row copies per four edges (one unit) land 4 x rowBytes in the
// worker's shared-memory ring and
// completes on an mbarrier; the lanes then add with LDS.128 + FADD.  What this buys over the
// register kernel: (1) bytes in flight are bounded by the ring (P stages x S units per
// worker, ~100 KB per SM) instead of by the register file — the register kernel holds up to 8 rows per lane in
// registers, issues them as a burst, waits for all of them and only then adds, so its *average*
// bytes in flight are well under half of its peak; the ring is refilled stage by stage, so it
// stays full.  (2) the copies are issued by one lane instead of an index load + IMAD.WIDE +
// LDG.128 per lane group.  MODE 0 (T) loads the source ids of a stage when it issues it; MODE 2 (U) holds them in
// the lanes that issue them.  MODE bit 4 makes it TSUM (the NORM epilogue divides by in_degree); bit 8 makes it
// BSUM: the copies carry bf16 rows (8 bytes per T-column, rounded up to whole 16-byte units, which stay inside a row
// whose leading dimension is a multiple of 8 elements), and each lane widens its T-column as it reads it.
// A row slot is L*NCH*16 bytes (8 for bf16; the worker's whole lane span), so the shared-memory row pitch is a
// compile-time constant and the adds are unpredicated; lanes past the row's end add stale slot
// contents they never store.
__device__ __forceinline__ float4 lds128(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr) : "memory");
  return v;
}
__device__ __forceinline__ float4 lds_bf16x4(uint32_t saddr) {
  uint2 u;
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(u.x), "=r"(u.y) : "r"(saddr) : "memory");
  return widen_bf16x4(u);
}
__device__ __forceinline__ void mbar_init_a(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx_a(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "SG_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra SG_DONE;\n\t"
      "bra SG_WAIT;\n\t"
      "SG_DONE:\n\t}"
      ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_row(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// four rows (source ids r0..r3) into consecutive slots of slotB bytes: one bulk copy of rowB bytes per row
__device__ __forceinline__ void bulk_rows4(uint32_t dst, const char* inB, uint32_t strideB, uint32_t rowB, uint32_t slotB,
                                           uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3, uint32_t bar) {
  bulk_row(dst, inB + (size_t)r0 * strideB, rowB, bar);
  bulk_row(dst + slotB, inB + (size_t)r1 * strideB, rowB, bar);
  bulk_row(dst + 2 * slotB, inB + (size_t)r2 * strideB, rowB, bar);
  bulk_row(dst + 3 * slotB, inB + (size_t)r3 * strideB, rowB, bar);
}

template <int L, int NCH, int S, int P, int NT, int MINB, int MODE>
__global__ void __launch_bounds__(NT, MINB)
sg_chunk_kernel_t(const SgParams p) {
  typedef float4 T;
  constexpr int WPB = NT / L;
  constexpr uint32_t CH = SG_CH;
  constexpr int G = 4 * S;                       // edges per stage
  constexpr bool BF = (MODE & 8) != 0;           // bf16 rows
  constexpr uint32_t CB = BF ? 8 : 16;           // bytes of one T-column
  constexpr uint32_t SLOTB = NCH * L * CB;       // shared-memory bytes per gathered row
  constexpr uint32_t G4B = 4 * SLOTB;            // one four-row unit
  constexpr uint32_t STAGEB = S * G4B;
  constexpr uint32_t RINGB = P * STAGEB;
  extern __shared__ __align__(128) unsigned char sg_smem_t[];
  const int lane = threadIdx.x % L;
  const int wi = threadIdx.x / L;
  const uint32_t w = blockIdx.x * WPB + wi;
  if (w >= p.numChunks) return;
  const unsigned wmask = worker_mask<L>();
  const uint32_t smem0 = (uint32_t)__cvta_generic_to_shared(sg_smem_t);
  const uint32_t ring = smem0 + wi * RINGB;
  const uint32_t bars = smem0 + WPB * RINGB + wi * (P * 8);
  const uint32_t* __restrict__ rs = p.rs;
  const uint32_t* __restrict__ col = p.col;
  bool act[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) act[ch] = (uint32_t)(lane + ch * L) < p.Q;

  const uint32_t cb = w * CH;
  const uint32_t ce = min(cb + CH, p.E);
  const uint32_t r0 = p.firstRow[w], r1 = p.firstRow[w + 1];
  uint32_t cur, curS, curT, segEnd, e;
  int kind;
  bool carryIn = false;
  if (r0 > 0) {
    uint32_t pe = rs[r0], ps = rs[r0 - 1];
    if (pe > cb && pe - ps > CH) {
      carryIn = true;
      cur = r0 - 1; curS = ps; curT = pe; kind = 0; e = cb; segEnd = min(pe, ce);
    }
  }
  if (!carryIn) {
    if (r0 >= r1) return;
    cur = r0; curS = rs[r0]; curT = rs[r0 + 1]; e = curS;
    bool heavy = curT - curS > CH;
    segEnd = heavy ? min(curT, ce) : curT;
    kind = heavy ? 2 : 1;
  }
  uint32_t ee;
  if (r1 > r0) {
    uint32_t s = rs[r1 - 1], t = rs[r1];
    ee = (t - s > CH) ? min(t, ce) : t;
  } else {
    ee = segEnd;
  }
  const uint32_t eb = e;
  const uint32_t nE = ee - eb;
  const uint32_t nStages = (nE + G - 1) / G;

  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < P; s++) mbar_init_a(bars + 8 * s, 1);
    tc::fence_barrier_init();
  }
  __syncwarp(wmask);

  T acc[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) acc[ch] = make_float4(0.f, 0.f, 0.f, 0.f);

  auto flush = [&]() {
    T* dst = (kind == 0) ? reinterpret_cast<T*>(p.carry) + (size_t)p.carryIdx[w] * p.ldC
                         : reinterpret_cast<T*>(p.out) + (size_t)cur * p.ldOut;
    dst += lane;
    const int epi = (kind == 1) ? p.epi : 0;
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) {
      if (act[ch]) {
        if (epi)
          epi_store<4>(acc[ch], dst + ch * L, norm_deg<(MODE & 4) ? SG_RED_TSUM : SG_RED_SUM>(p, cur, curT - curS), epi);
        else *(dst + ch * L) = acc[ch];
      }
      acc[ch] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto advance = [&]() {
    cur += 1; curS = curT; curT = rs[cur + 1];
    bool heavy = curT - curS > CH;
    segEnd = heavy ? min(curT, ce) : curT;
    kind = heavy ? 2 : 1;
  };

  // stage k -> ring slot `slot`: issued by the worker's first lane.  A stage that runs past the
  // worker's last edge repeats that edge's source (a duplicate row, L2-resident; never added).
  const char* inB = reinterpret_cast<const char*>(p.in);
  const uint32_t strideB = (uint32_t)p.ldIn * CB;
  const uint32_t rowB = BF ? (p.Q * 8u + 15u) & ~15u : p.Q * 16u;
  // MODE 2: the source ids never sit in front of the issue.  Lane j of the worker loads, once and up front, the
  // ids of units j, j + L, ... of the worker's edge range (a worker has at most 127 edges = 32 units) and
  // issues those units itself when their ring slot frees (on MODE 0 the id load of the stage about to be issued
  // is a large share of the stalls).
  constexpr int NU = (MODE & 2) ? (32 / L) : 1;
  uint4 ids[NU];
  if ((MODE & 2) && nE) {
#pragma unroll
    for (int n = 0; n < NU; n++) {
      const uint32_t e4 = 4u * ((uint32_t)lane + (uint32_t)n * L);
      const uint32_t last = nE - 1u;
      const uint32_t* cp = col + eb;
      ids[n] = make_uint4(__ldg(cp + min(e4, last)), __ldg(cp + min(e4 + 1u, last)), __ldg(cp + min(e4 + 2u, last)),
                          __ldg(cp + min(e4 + 3u, last)));
    }
  }
  auto issue = [&](uint32_t k, uint32_t slot) {
    if (MODE & 2) {
      if (k < nStages) {
        const uint32_t off = k * G;
        const uint32_t bar = bars + slot * 8;
        const uint32_t dst = ring + slot * STAGEB;
        const uint32_t nv = min((uint32_t)G, nE - off);
        const uint32_t n4 = (nv + 3u) >> 2;
        if ((uint32_t)lane == (k * S) % (uint32_t)L) mbar_expect_tx_a(bar, n4 * 4u * rowB);
#pragma unroll
        for (int s = 0; s < S; s++) {
          const uint32_t g = k * S + (uint32_t)s;              // unit within the worker's range
          if ((uint32_t)s < n4 && (uint32_t)lane == g % (uint32_t)L) {
            uint4 id = ids[0];
#pragma unroll
            for (int n = 1; n < NU; n++) if (g / (uint32_t)L == (uint32_t)n) id = ids[n];
            bulk_rows4(dst + s * G4B, inB, strideB, rowB, SLOTB, id.x, id.y, id.z, id.w, bar);
          }
        }
      }
      return;
    }
    if (k < nStages && lane == 0) {      // MODE 0
      const uint32_t off = k * G;
      const uint32_t* cp = col + eb + off;
      const uint32_t bar = bars + slot * 8;
      const uint32_t dst = ring + slot * STAGEB;
      const uint32_t nv = min((uint32_t)G, nE - off);
      const uint32_t n4 = (nv + 3u) >> 2;
      mbar_expect_tx_a(bar, n4 * 4u * rowB);
#pragma unroll
      for (int s = 0; s < S; s++) {
        if ((uint32_t)s < n4) {
          uint32_t i0, i1, i2, i3;
          if ((uint32_t)(4 * s + 4) <= nv) {
            i0 = __ldg(cp + 4 * s); i1 = __ldg(cp + 4 * s + 1); i2 = __ldg(cp + 4 * s + 2); i3 = __ldg(cp + 4 * s + 3);
          } else {
            const uint32_t last = nv - 1u;
            i0 = __ldg(cp + min((uint32_t)(4 * s), last)); i1 = __ldg(cp + min((uint32_t)(4 * s + 1), last));
            i2 = __ldg(cp + min((uint32_t)(4 * s + 2), last)); i3 = __ldg(cp + min((uint32_t)(4 * s + 3), last));
          }
          bulk_rows4(dst + s * G4B, inB, strideB, rowB, SLOTB, i0, i1, i2, i3, bar);
        }
      }
    }
  };
#pragma unroll 1
  for (uint32_t k = 0; k < (uint32_t)P; k++) issue(k, k);
  uint32_t slot = 0, parity = 0;
#pragma unroll 1
  for (uint32_t k = 0; k < nStages; k++) {
    mbar_wait_a(bars + slot * 8, parity);
    const uint32_t e0 = eb + k * G;
    const uint32_t sa = ring + slot * STAGEB + lane * CB;
    auto lds = [&](int u, int ch) {
      if constexpr (BF) return lds_bf16x4(sa + u * SLOTB + ch * L * CB);
      else return lds128(sa + u * SLOTB + ch * L * 16);
    };
    if (segEnd - e0 >= (uint32_t)G) {
      // the whole stage lies inside the current row segment
#pragma unroll
      for (int u = 0; u < G; u++)
#pragma unroll
        for (int ch = 0; ch < NCH; ch++) {
          const float4 v = lds(u, ch);
          acc[ch].x += v.x; acc[ch].y += v.y; acc[ch].z += v.z; acc[ch].w += v.w;
        }
    } else {
      // one rolled loop over the row segments of the stage, ONE row-store site
      const uint32_t cnt = min((uint32_t)G, ee - e0);
      uint32_t pos = 0;
      for (;;) {
        const uint32_t lim = min(cnt, segEnd - e0);
#pragma unroll
        for (int u = 0; u < G; u++) {
          if ((uint32_t)u >= pos && (uint32_t)u < lim) {
#pragma unroll
            for (int ch = 0; ch < NCH; ch++) {
              const float4 v = lds(u, ch);
              acc[ch].x += v.x; acc[ch].y += v.y; acc[ch].z += v.z; acc[ch].w += v.w;
            }
          }
        }
        pos = lim;
        if (pos >= cnt) break;
        flush();
        advance();
      }
    }
    __syncwarp(wmask);          // every lane has read the slot before the TMA unit rewrites it
    issue(k + P, slot);
    slot += 1;
    if (slot == (uint32_t)P) { slot = 0; parity ^= 1u; }
  }
  flush();
  while (cur + 1 < r1) { advance(); flush(); }
}

// ---------------------------------------------------------- fix-up kernels ---
// A row cut at chunk boundaries is finished from its owner's partial (out[R]; arg[R] for MAX / MIN) and its carries,
// taken in chunk order: added for the sum (whose partials include the min / max backward's), combined by the
// ordering rule for MAX / MIN.  Only the sum has an epilogue.
// U carries are loaded per batch.  The carries are taken in chunk order whatever U is, so U never changes a result;
// MAX / MIN take fewer per batch where their index carries would otherwise spill.
__host__ __device__ constexpr int sg_fixup_u(int L, int NCH, int RED) {
  return (RED == SG_RED_SUM || RED == SG_RED_TSUM || RED == SG_RED_TELE) ? (NCH == 1 ? (L == 4 ? 4 : 8) : 8 / NCH) : (NCH <= 2 ? 4 : 1);
}

// One worker per heavy row.
template <int VEC, int L, int NCH, int RED>
__global__ void __launch_bounds__(SG_THREADS)
sg_fixup_kernel(const SgParams p) {
  typedef typename V<VEC>::T T;
  typedef typename V<VEC>::I I;
  constexpr bool MM = RED == SG_RED_MAX || RED == SG_RED_MIN;
  constexpr int U = sg_fixup_u(L, NCH, RED);
  constexpr int WPB = SG_THREADS / L;
  constexpr uint32_t CH = SG_CH;
  const int lane = threadIdx.x % L;
  const uint32_t w = blockIdx.x * WPB + threadIdx.x / L;
  if (w >= p.numHeavy) return;
  const uint32_t R = p.heavyRows[w];
  const uint32_t s = p.rs[R], t = p.rs[R + 1];
  const uint32_t c0 = s / CH, cLast = (t - 1) / CH;
  const uint32_t n = cLast - c0;
  const uint32_t slot0 = p.carryIdx[c0 + 1];
  T* dst = reinterpret_cast<T*>(p.out) + (size_t)R * p.ldOut;
  const T* cbase = reinterpret_cast<const T*>(p.carry) + (size_t)slot0 * p.ldC;
  I* adst = reinterpret_cast<I*>(p.arg) + (size_t)R * p.ldArg;
  const I* abase = reinterpret_cast<const I*>(p.carryArg) + (size_t)slot0 * p.ldC;
  bool act[NCH];
  T acc[NCH];
  I ai[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) {
    act[ch] = (uint32_t)(lane + ch * L) < p.Q;
    acc[ch] = act[ch] ? V<VEC>::ld_plain(dst + lane + ch * L) : V<VEC>::zero();
    if constexpr (MM) ai[ch] = act[ch] ? adst[lane + ch * L] : mm_noarg((I*)nullptr);
  }
  for (uint32_t k = 0; k < n; k += U) {
    T v[U][NCH];
    I vi[MM ? U : 1][MM ? NCH : 1];
#pragma unroll
    for (int u = 0; u < U; u++)
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        if constexpr (MM) {
          const bool ok = k + u < n && act[ch];
          v[u][ch] = ok ? V<VEC>::ld_plain(cbase + (size_t)(k + u) * p.ldC + lane + ch * L) : V<VEC>::zero();
          vi[u][ch] = ok ? abase[(size_t)(k + u) * p.ldC + lane + ch * L] : mm_noarg((I*)nullptr);
        } else {
          v[u][ch] = (k + u < n && act[ch]) ? V<VEC>::ld_plain(cbase + (size_t)(k + u) * p.ldC + lane + ch * L)
                                            : V<VEC>::zero();
        }
      }
#pragma unroll
    for (int u = 0; u < U; u++)
      if (MM || k + u < n)          // MAX / MIN: a carry past n has no index and is skipped
#pragma unroll
        for (int ch = 0; ch < NCH; ch++) {
          if constexpr (MM) mm_combine<RED>(acc[ch], ai[ch], v[u][ch], vi[u][ch]);
          else V<VEC>::add(acc[ch], v[u][ch]);
        }
  }
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) {
    if (act[ch]) {
      if constexpr (MM) { V<VEC>::st(dst + lane + ch * L, acc[ch]); adst[lane + ch * L] = ai[ch]; }
      else if constexpr (RED == SG_RED_TELE) tele_store<VEC>(p, acc[ch], dst + lane + ch * L, R, (uint32_t)(lane + ch * L), t - s);
      else epi_store<VEC>(acc[ch], dst + lane + ch * L, norm_deg<RED>(p, R, t - s), p.epi);
    }
  }
}

// Rows with more than SG_BIG carries (hubs: R-MAT-22's largest row spans 1 524 chunks) get a
// whole CTA: each of the 256/L lane groups reduces a contiguous block of the carries, then group 0
// takes the owner's partial and the groups' results in group order — chunk order again.  With one
// worker per row the hubs' serial chains set the kernel's duration.
constexpr uint32_t SG_BIG = 32;

template <int VEC, int L, int NCH, int RED>
__global__ void __launch_bounds__(SG_THREADS)
sg_fixup_big_kernel(const SgParams p) {
  typedef typename V<VEC>::T T;
  typedef typename V<VEC>::I I;
  constexpr bool MM = RED == SG_RED_MAX || RED == SG_RED_MIN;
  constexpr int U = sg_fixup_u(L, NCH, RED);
  constexpr int WPB = SG_THREADS / L;
  constexpr uint32_t CH = SG_CH;
  __shared__ __align__(16) float part[WPB * NCH * L * VEC];
  __shared__ __align__(16) uint32_t parti[MM ? WPB * NCH * L * VEC : 1];   // MAX / MIN: the partials' indices
  const int lane = threadIdx.x % L;
  const int g = threadIdx.x / L;
  const uint32_t R = p.bigRows[blockIdx.x];
  const uint32_t s = p.rs[R], t = p.rs[R + 1];
  const uint32_t c0 = s / CH, cLast = (t - 1) / CH;
  const uint32_t n = cLast - c0;
  const uint32_t slot0 = p.carryIdx[c0 + 1];
  const T* cbase = reinterpret_cast<const T*>(p.carry) + (size_t)slot0 * p.ldC;
  const I* abase = reinterpret_cast<const I*>(p.carryArg) + (size_t)slot0 * p.ldC;
  const uint32_t per = (n + WPB - 1) / WPB;
  const uint32_t k0 = min(n, (uint32_t)g * per), k1 = min(n, k0 + per);
  bool act[NCH];
  T acc[NCH];
  I ai[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) {
    act[ch] = (uint32_t)(lane + ch * L) < p.Q; acc[ch] = V<VEC>::zero();
    if constexpr (MM) ai[ch] = mm_noarg((I*)nullptr);
  }
  for (uint32_t k = k0; k < k1; k += U) {
    T v[U][NCH];
    I vi[MM ? U : 1][MM ? NCH : 1];
#pragma unroll
    for (int u = 0; u < U; u++)
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        if constexpr (MM) {
          const bool ok = k + u < k1 && act[ch];
          v[u][ch] = ok ? V<VEC>::ld_plain(cbase + (size_t)(k + u) * p.ldC + lane + ch * L) : V<VEC>::zero();
          vi[u][ch] = ok ? abase[(size_t)(k + u) * p.ldC + lane + ch * L] : mm_noarg((I*)nullptr);
        } else {
          v[u][ch] = (k + u < k1 && act[ch]) ? V<VEC>::ld_plain(cbase + (size_t)(k + u) * p.ldC + lane + ch * L)
                                            : V<VEC>::zero();
        }
      }
#pragma unroll
    for (int u = 0; u < U; u++)
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        if constexpr (MM) mm_combine<RED>(acc[ch], ai[ch], v[u][ch], vi[u][ch]);
        else V<VEC>::add(acc[ch], v[u][ch]);
      }
  }
  T* sp = reinterpret_cast<T*>(part);
  I* spi = reinterpret_cast<I*>(parti);
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) {
    sp[(g * NCH + ch) * L + lane] = acc[ch];
    if constexpr (MM) spi[(g * NCH + ch) * L + lane] = ai[ch];
  }
  __syncthreads();
  if (g == 0) {
    T* dst = reinterpret_cast<T*>(p.out) + (size_t)R * p.ldOut;
    I* adst = reinterpret_cast<I*>(p.arg) + (size_t)R * p.ldArg;
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) {
      if (!act[ch]) continue;
      T a = V<VEC>::ld_plain(dst + lane + ch * L);      // the owner chunk's partial
      if constexpr (MM) {
        I ia = adst[lane + ch * L];
        for (int gg = 0; gg < WPB; gg++) mm_combine<RED>(a, ia, sp[(gg * NCH + ch) * L + lane], spi[(gg * NCH + ch) * L + lane]);
        V<VEC>::st(dst + lane + ch * L, a);
        adst[lane + ch * L] = ia;
      } else {
        for (int gg = 0; gg < WPB; gg++) V<VEC>::add(a, sp[(gg * NCH + ch) * L + lane]);
        if constexpr (RED == SG_RED_TELE) tele_store<VEC>(p, a, dst + lane + ch * L, R, (uint32_t)(lane + ch * L), t - s);
        else epi_store<VEC>(a, dst + lane + ch * L, norm_deg<RED>(p, R, t - s), p.epi);
      }
    }
  }
}

// ------------------------------------------------------- attention kernels ---
// (m, Z) partials of one head merged: the max is exact, each Z rescaled to it.  merge(a, b) and merge(b, a) give the
// same bits, which the butterfly below relies on.  A partial with Z = 0 has no edge.
__device__ __forceinline__ void attn_merge(float& m, float& z, float m2, float z2) {
  if (!(z2 > 0.f)) return;
  if (!(z > 0.f)) { m = m2; z = z2; return; }
  const float M = fmaxf(m, m2);
  z = z * expf(m - M) + z2 * expf(m2 - M);
  m = M;
}

// Finishes the stats of every row the ASTAT pass cut (heavy and big rows alike): one warp per row, lane l merging
// carries l, l + 32, ... in order, then an xor butterfly, then the owner's partial; stores m and 1/Z.  The order is
// fixed by the plan, so the result is reproducible.
__global__ void __launch_bounds__(SG_THREADS)
sg_attn_stat_fixup(const SgParams p) {
  constexpr uint32_t CH = SG_CH;
  const uint32_t w = (blockIdx.x * SG_THREADS + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (w >= p.numHeavy + p.numBig) return;
  const uint32_t R = w < p.numHeavy ? p.heavyRows[w] : p.bigRows[w - p.numHeavy];
  const uint32_t s = p.rs[R], t = p.rs[R + 1];
  const uint32_t c0 = s / CH, n = (t - 1) / CH - c0;
  const float* cb = p.carry2 + (uint64_t)p.carryIdx[c0 + 1] * SG_LDC2;
  float* dst = reinterpret_cast<float*>(p.out) + (uint64_t)R * p.ldOut;
  for (uint32_t k = 0; k < p.heads; k++) {
    float m = 0.f, z = 0.f;
    for (uint32_t i = lane; i < n; i += 32) attn_merge(m, z, cb[(uint64_t)i * SG_LDC2 + k], cb[(uint64_t)i * SG_LDC2 + p.heads + k]);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m, o), z2 = __shfl_xor_sync(0xffffffffu, z, o);
      attn_merge(m, z, m2, z2);
    }
    if (lane == 0) {
      float mo = dst[k], zo = dst[p.heads + k];
      attn_merge(mo, zo, m, z);
      dst[k] = mo;
      dst[p.heads + k] = 1.f / zo;
    }
  }
}

// The backward's per-node record {s_dst, m, 1/Z, D} of ids [0, n): one worker of L lanes per node, D[k] = G[k] . O[k]
// reduced per head like the gathers' dot products.
template <int VEC, int L, int NCH>
__global__ void __launch_bounds__(SG_THREADS)
sg_attn_rec_kernel(const SgParams p, const void* G, size_t ldG, const void* O, size_t ldO, uint32_t n) {
  typedef typename V<VEC>::T T;
  constexpr int WPB = SG_THREADS / L;
  const int lane = threadIdx.x % L;
  const uint32_t v = blockIdx.x * WPB + threadIdx.x / L;
  if (v >= n) return;
  const unsigned wmask = worker_mask<L>();
  const T* g = reinterpret_cast<const T*>(G) + (uint64_t)v * ldG;
  const T* o = reinterpret_cast<const T*>(O) + (uint64_t)v * ldO;
  float d[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) {
    const uint32_t c = (uint32_t)(lane + ch * L);
    const int nv = t_floats<VEC>(c, p);
    const uint32_t cc = min(c, p.Q - 1u);
    d[ch] = dot_t(V<VEC>::ld(g + cc), V<VEC>::ld(o + cc), nv);
  }
  head_sum<L, NCH>(d, p.ftShift, wmask);
  const uint32_t ftMask = head_mask(p);
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) {
    const uint32_t c = (uint32_t)(lane + ch * L);
    if (c < p.Q && (c & ftMask) == 0) {
      const uint32_t k = c >> p.ftShift;
      const_cast<float4*>(p.rec)[(uint64_t)v * p.heads + k] =
          make_float4(p.score[(uint64_t)v * p.ldS + k], p.stats[(uint64_t)v * p.ldStats + k],
                      p.stats[(uint64_t)v * p.ldStats + p.heads + k], d[ch]);
    }
  }
}

// ------------------------------------------------------------------ launches ---
// The launches of the calling thread's last planned call (roc_sg_last_call_info): every planned entry point clears the
// list, and every launch site below appends what it launched.
static thread_local roc_sg_call_info t_call = {};
static void clear_launches() { t_call.count = 0; }
static void note_launch(int kind, int red, int vec, int lanes, int nch, uint32_t grid) {
  if (t_call.count < ROC_SG_MAX_LAUNCHES) t_call.launch[t_call.count] = roc_sg_launch{kind, red, vec, lanes, nch, (int64_t)grid};
  t_call.count++;
}

// ----------------------------------------------------------- reduction table ---
// Everything the host needs to know to launch a reduction: one row per SG_RED_* value.
enum SgFix {
  SG_FIX_NONE,    // nothing carried (EDOT's outputs are per edge), or only heads-wide partials (ADST)
  SG_FIX_OWN,     // the fix-ups instantiated for the reduction itself
  SG_FIX_SUM,     // the H-wide partials are plain sums, finished by the sum's fix-ups
  SG_FIX_STATS    // sg_attn_stat_fixup
};
enum SgCarry {
  SG_CARRY_NONE,
  SG_CARRY_FLOAT,
  SG_CARRY_INDEX  // the float carries plus the min / max index carries
};
struct SgRed {
  int red;          // the SG_RED_* value this row describes
  // The widest row, in T-columns, one launch takes, on float4 rows and on scalar rows; run_planned cuts wider rows
  // into column blocks of VEC * maxQ floats.
  int maxQ4, maxQ1;
  // -1: every row runs on sg_chunk_kernel.  Otherwise vectorised rows at L = 32, NCH <= 2 run on sg_chunk_kernel_t,
  // and this is the MODE bit the reduction adds there (4: TSUM's NORM epilogue divides by in_degree; 8: bf16 rows).
  int ring;
  SgFix fix;        // the fix-up of the H-wide partials of the rows the main kernel cut
  bool headsFix;    // the heads-wide partials (out2 / carry2) also go through the sum's fix-ups
  SgCarry carry;
  int u4;           // sg_chunk_kernel's gathers in flight (U) at L = 4
  int u[4];         // U at NCH = 1 (L = 8..32), 2, 4, 8 chunks per lane
  int minb[4];      // CTAs per SM at NCH = 1, 2, 4, 8
};

// maxQ: 256 T-columns (1024 floats vectorised, 256 scalar), but 128 on float4 rows for every reduction except the sums
// (min / max: the big-row fix-up keeps values and indices of every lane group in static shared memory).  The weighted
// sum and TSUM take the sum's column blocks, so that with all-ones weights (on a symmetric graph) they give the sum's
// bits at every width (the big-row fix-up groups a row's carries by the block's lane count).  ASTAT's row is one
// score per head, on scalar rows only.
// U and MINB are lower than the sum's where a second value held or gathered per float (the min / max index, the
// min / max backward's index row, s_src, the record, the local row's own row) would otherwise spill under the
// occupancy.  WSUM keeps the sum's U and holds U weights beside them, so at one chunk per lane it runs three CTAs per
// SM.  TSUM and TMASK take the shapes of SUM and MASK, but TMASK, which also holds each group's repeated-destination
// bits, runs three CTAs per SM at one chunk per lane.  BSUM is SUM's row with bf16 loads (ring MODE bit 8): the same
// column blocks, shapes and sum fix-ups, so that its results are SUM's bits on the widened rows.  The other bf16 forms
// (SG_RED_BF16) have no row of their own: they take their reduction's, fix-ups included, for the same reason.  TELE is
// SUM's row without the ring (its row store needs the row of t, which the ring kernel does not load), with its own
// fix-ups (the sum's, storing through tele_store): the same column blocks, row shapes and carry order, hence SUM's sums.
// Its row store holds a row of t and the coefficients while a group's gathered rows are live, so it runs three CTAs
// per SM at one chunk per lane and one gather in flight at four, where SUM's occupancy and U would spill.
constexpr SgRed SG_REDS[] = {
    // red           maxQ4 maxQ1 ring fix           heads  carry           u4  u             minb
    {SG_RED_SUM,     256,  256,  0,   SG_FIX_SUM,   false, SG_CARRY_FLOAT, 4, {8, 4, 2, 1}, {4, 3, 3, 2}},
    {SG_RED_MAX,     128,  256,  -1,  SG_FIX_OWN,   false, SG_CARRY_INDEX, 4, {4, 4, 1, 1}, {4, 3, 3, 2}},
    {SG_RED_MIN,     128,  256,  -1,  SG_FIX_OWN,   false, SG_CARRY_INDEX, 4, {4, 4, 1, 1}, {4, 3, 3, 2}},
    {SG_RED_MASK,    128,  256,  -1,  SG_FIX_SUM,   false, SG_CARRY_FLOAT, 4, {4, 2, 1, 1}, {4, 3, 3, 2}},
    {SG_RED_ASTAT,   0,    SG_LDC2 / 2, -1, SG_FIX_STATS, false, SG_CARRY_FLOAT, 8, {8, 0, 0, 0}, {4, 0, 0, 0}},
    {SG_RED_ATTN,    128,  256,  -1,  SG_FIX_SUM,   false, SG_CARRY_FLOAT, 4, {4, 2, 1, 1}, {4, 3, 2, 2}},
    {SG_RED_ADST,    128,  256,  -1,  SG_FIX_NONE,  true,  SG_CARRY_FLOAT, 4, {4, 2, 1, 1}, {4, 3, 2, 1}},
    {SG_RED_ASRC,    128,  256,  -1,  SG_FIX_SUM,   true,  SG_CARRY_FLOAT, 2, {2, 2, 1, 1}, {4, 2, 2, 1}},
    {SG_RED_WSUM,    256,  256,  -1,  SG_FIX_SUM,   false, SG_CARRY_FLOAT, 8, {8, 4, 2, 1}, {3, 3, 3, 2}},
    {SG_RED_EDOT,    128,  256,  -1,  SG_FIX_NONE,  false, SG_CARRY_NONE,  4, {4, 2, 1, 1}, {4, 3, 2, 1}},
    {SG_RED_TSUM,    256,  256,  4,   SG_FIX_OWN,   false, SG_CARRY_FLOAT, 4, {8, 4, 2, 1}, {4, 3, 3, 2}},
    {SG_RED_TMASK,   128,  256,  -1,  SG_FIX_SUM,   false, SG_CARRY_FLOAT, 4, {4, 2, 1, 1}, {3, 3, 3, 2}},
    {SG_RED_BSUM,    256,  256,  8,   SG_FIX_SUM,   false, SG_CARRY_FLOAT, 4, {8, 4, 2, 1}, {4, 3, 3, 2}},
    {SG_RED_TELE,    256,  256,  -1,  SG_FIX_OWN,   false, SG_CARRY_FLOAT, 4, {8, 4, 1, 1}, {3, 3, 3, 2}}};
constexpr bool sg_reds_in_order() {
  for (int i = 0; i < (int)(sizeof(SG_REDS) / sizeof(SG_REDS[0])); i++)
    if (SG_REDS[i].red != i) return false;
  return sizeof(SG_REDS) / sizeof(SG_REDS[0]) == SG_RED_TELE + 1;
}
static_assert(sg_reds_in_order(), "SG_REDS has one row per SG_RED_* value, in order");

// A bf16 form (SG_RED_BF16) takes its reduction's row.
constexpr const SgRed& sg_red(int RF) { return SG_REDS[sg_red_base(RF)]; }
constexpr int sg_max_q(int VEC, int RED) { return VEC == 4 ? sg_red(RED).maxQ4 : sg_red(RED).maxQ1; }
constexpr int sg_nch_index(int NCH) { return NCH == 1 ? 0 : NCH == 2 ? 1 : NCH == 4 ? 2 : 3; }
constexpr int sg_chunk_u(int RED, int L, int NCH) { return L == 4 ? sg_red(RED).u4 : sg_red(RED).u[sg_nch_index(NCH)]; }
// The dropped sums (SG_RED_DROP on SUM, TSUM and TELE) take their sum's row, holding U keep bytes beside the gathered
// rows.  On float4 rows at eight chunks per lane that pushes TELE's, whose store also holds a row of t, past two CTAs'
// registers: it runs one CTA per SM there rather than spill.
constexpr int sg_chunk_minb(int VEC, int RED, int NCH) {
  return (VEC == 4 && RED == (SG_RED_TELE | SG_RED_DROP) && NCH == 8) ? 1 : sg_red(RED).minb[sg_nch_index(NCH)];
}

// sg_chunk_kernel_t's two shapes, the measured defaults (DESIGN.md §3.1), four workers per CTA: rows of 65..128 floats
// (one float4 per lane) with lane-held ids and two stages of two four-row units per worker; rows of 129..256 floats
// with the ids loaded per stage and two stages of one unit.
template <int NCH, int RED>
static int launch_ring(const SgParams& p, cudaStream_t st) {
  constexpr int L = 32, P = 2, NT = 128;
  constexpr int S = NCH == 1 ? 2 : 1, MINB = NCH == 1 ? 4 : 6, MODE = (NCH == 1 ? 2 : 0) | SG_REDS[RED].ring;
  constexpr int WPB = NT / L;
  constexpr size_t smem = (size_t)WPB * P * S * 4 * NCH * L * ((MODE & 8) ? 8 : 16) + (size_t)WPB * P * 8;
  static std::atomic<uint64_t> configured{0};
  ROC_CUDA(once_per_device(configured, [] {
    return cudaFuncSetAttribute(sg_chunk_kernel_t<L, NCH, S, P, NT, MINB, MODE>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }));
  const uint32_t grid = (p.numChunks + WPB - 1) / WPB;
  sg_chunk_kernel_t<L, NCH, S, P, NT, MINB, MODE><<<grid, NT, smem, st>>>(p);
  ROC_LAUNCH_CHECK();
  note_launch(ROC_SG_LAUNCH_RING, RED, 4, L, NCH, grid);
  return ROC_OK;
}

// The row shape of every launch: calls f(L, NCH), as std::integral_constants, for rows of Q T-columns.  L is the
// fewest of 4, 8, 16 or 32 lanes that cover Q; past 32 T-columns each lane takes NCH = 2, 4 or 8 chunks:
// Q <= 4 -> (4, 1), <= 8 -> (8, 1), <= 16 -> (16, 1), <= 32 -> (32, 1), <= 64 -> (32, 2), <= 128 -> (32, 4),
// <= 256 -> (32, 8).  Rows wider than QMAX are ROC_ERR_UNSUPPORTED.
template <int QMAX, int QC = 4, class F>
static int with_shape(uint32_t Q, F&& f) {
  if constexpr (QC > QMAX) {
    return ROC_ERR_UNSUPPORTED;
  } else {
    if (Q <= (uint32_t)QC)
      return f(std::integral_constant<int, (QC < 32 ? QC : 32)>{}, std::integral_constant<int, (QC < 32 ? 1 : QC / 32)>{});
    return with_shape<QMAX, 2 * QC>(Q, f);
  }
}

// The fix-ups of the rows a main kernel cut, reduced by FIX over p's out / carry: one worker per heavy row, one CTA
// per big row.  `heads`: p holds an attention gather's heads-wide partials.
template <int VEC, int L, int NCH, int FIX>
static int launch_fixups(const SgParams& p, cudaStream_t st, bool heads = false) {
  constexpr int WPB = SG_THREADS / L;
  if (p.numHeavy) {
    const uint32_t grid = (p.numHeavy + WPB - 1) / WPB;
    sg_fixup_kernel<VEC, L, NCH, FIX><<<grid, SG_THREADS, 0, st>>>(p);
    ROC_LAUNCH_CHECK();
    note_launch(heads ? ROC_SG_LAUNCH_HEADS_FIXUP : ROC_SG_LAUNCH_FIXUP, FIX, VEC, L, NCH, grid);
  }
  if (p.numBig) {
    sg_fixup_big_kernel<VEC, L, NCH, FIX><<<p.numBig, SG_THREADS, 0, st>>>(p);
    ROC_LAUNCH_CHECK();
    note_launch(heads ? ROC_SG_LAUNCH_HEADS_BIG_FIXUP : ROC_SG_LAUNCH_BIG_FIXUP, FIX, VEC, L, NCH, p.numBig);
  }
  return ROC_OK;
}

// One ScatterGather launch: the main kernel (sg_chunk_kernel_t for the ring reductions' vectorised rows of 17..64
// T-columns, where it is faster on a products-shaped graph, DESIGN.md §3.1), then the fix-ups of the rows it cut, as
// the reduction's row of SG_REDS says.  Heads-wide partials are finished by the sum's fix-ups on p2, p with
// out2 / carry2 as a VEC = 1, Q = heads output.
template <int VEC, int RED, int L, int NCH>
static int launch(const SgParams& p, cudaStream_t st) {
  constexpr SgRed R = sg_red(RED);
  constexpr int WPB = SG_THREADS / L;
  int rc = ROC_OK;
  if (p.numChunks) {
    if constexpr (VEC == 4 && R.ring >= 0 && !(RED & SG_RED_DROP) && L == 32 && NCH <= 2) {
      if ((rc = launch_ring<NCH, RED>(p, st)) != ROC_OK) return rc;
    } else {
      const uint32_t grid = (p.numChunks + WPB - 1) / WPB;
      sg_chunk_kernel<VEC, L, NCH, sg_chunk_u(RED, L, NCH), sg_chunk_minb(VEC, RED, NCH), RED><<<grid, SG_THREADS, 0, st>>>(p);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_MAIN, RED, VEC, L, NCH, grid);
    }
  }
  if constexpr (R.fix == SG_FIX_STATS) {
    const uint32_t rows = p.numHeavy + p.numBig;
    if (rows) {
      const uint32_t grid = (rows + SG_THREADS / 32 - 1) / (SG_THREADS / 32);
      sg_attn_stat_fixup<<<grid, SG_THREADS, 0, st>>>(p);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_STAT_FIXUP, RED, 1, 32, 1, grid);
    }
  } else if constexpr (R.fix != SG_FIX_NONE) {
    if ((rc = launch_fixups<VEC, L, NCH, R.fix == SG_FIX_OWN ? R.red : SG_RED_SUM>(p, st)) != ROC_OK) return rc;
  }
  if constexpr (R.headsFix) {
    SgParams p2 = p;
    p2.out = p.out2; p2.ldOut = p.ldOut2; p2.carry = p.carry2; p2.ldC = SG_LDC2; p2.Q = p.heads;
    rc = launch_fixups<1, 8, 1, SG_RED_SUM>(p2, st, true);
  }
  return rc;
}

// Reduction RED over rows of p.Q T-columns of VEC floats.
template <int VEC, int RED>
static int dispatch(const SgParams& p, cudaStream_t st) {
  return with_shape<sg_max_q(VEC, RED)>(p.Q, [&](auto L, auto NCH) { return launch<VEC, RED, L, NCH>(p, st); });
}

// The attention backward's node records of ids [0, n), in the shape of its H-wide passes, from G = p.in (leading
// dimension p.ldIn) and O = p.xrow (p.ldX).
template <int VEC>
static int launch_rec(const SgParams& p, uint32_t n, cudaStream_t st) {
  return with_shape<sg_max_q(VEC, SG_RED_ATTN)>(p.Q, [&](auto L, auto NCH) {
    if (n) {
      constexpr int WPB = SG_THREADS / L;
      const uint32_t grid = (n + WPB - 1) / WPB;
      sg_attn_rec_kernel<VEC, L, NCH><<<grid, SG_THREADS, 0, st>>>(p, p.in, p.ldIn, p.xrow, p.ldX, n);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_RECORD, -1, VEC, L, NCH, grid);
    }
    return ROC_OK;
  });
}

// A plan buffer of at least `bytes`, `cap` its size in bytes.  roc_sg_plan_reserve sizes the carries up front (plain
// cudaMalloc, an init-time call).  A launch that still finds a buffer too small grows it on its own stream with
// stream-ordered allocation: the old buffer is returned in stream order, after the launches that used it — no device
// synchronisation in the middle of a step.  A failed allocation leaves the buffer null with zero capacity.
template <class T>
static int grow(T*& buf, size_t& cap, size_t bytes, cudaStream_t st, bool inStream = true) {
  if (bytes <= cap) return ROC_OK;
  if (buf) {
    if (inStream) ROC_CUDA(cudaFreeAsync(buf, st));
    else { ROC_CUDA(cudaDeviceSynchronize()); ROC_CUDA(cudaFree(buf)); }
    buf = nullptr; cap = 0;
  }
  cudaError_t e = inStream ? cudaMallocAsync((void**)&buf, bytes, st) : cudaMalloc((void**)&buf, bytes);
  if (e != cudaSuccess) { buf = nullptr; return (int)e; }
  cap = bytes;
  return ROC_OK;
}

// The carry slots of rows cut at chunk boundaries: [numCarries][carryLd] floats, carryLd at least `cols` rounded up
// to float4 rows.
static int grow_carries(roc_sg_plan* pl, int cols, cudaStream_t st, bool inStream = true) {
  const size_t n = pl->numCarries, ld = ((size_t)cols + 3) / 4 * 4;
  const int rc = grow(pl->carry, pl->carryBytes, n * ld * sizeof(float), st, inStream);
  pl->carryLd = n ? pl->carryBytes / (n * sizeof(float)) : 0;
  return rc;
}

// 1 + the largest id in col, found once (one reduction and one synchronisation of the stream) and kept in the plan.
static int find_id_end(roc_sg_plan* plan, cudaStream_t st) {
  if (plan->idEndKnown) return ROC_OK;
  uint64_t idEnd = 0;
  if (plan->E) {
    uint32_t* dmax = nullptr;
    void* tmp = nullptr;
    size_t tb = 0;
    uint32_t h = 0;
    cudaError_t e = cub::DeviceReduce::Max(nullptr, tb, plan->col, dmax, (int)plan->E, st);
    if (e == cudaSuccess) e = cudaMallocAsync((void**)&dmax, 16 + (tb ? tb : 16), st);   // the max, then cub's scratch
    if (e == cudaSuccess) {
      tmp = reinterpret_cast<char*>(dmax) + 16;
      e = cub::DeviceReduce::Max(tmp, tb, plan->col, dmax, (int)plan->E, st);
      count_launch();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h, dmax, sizeof(uint32_t), cudaMemcpyDeviceToHost, st);
    if (dmax) { cudaError_t f = cudaFreeAsync(dmax, st); if (e == cudaSuccess) e = f; }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return (int)e;
    idEnd = (uint64_t)h + 1;
  }
  plan->idEnd = idEnd;
  plan->idEndKnown = true;
  return ROC_OK;
}

// ------------------------------------------------------- transposed CSR ---
// From the stable sort of (colSrc, edge index): perm[t] is the original edge of transposed edge t, srcSorted[t] its
// source.  Transposed row v (node v's out-edges) is [rowEndT[v - 1], rowEndT[v]); colT[t] is the destination of
// perm[t], the row whose [start, end) holds it.
__global__ void k_iota(uint32_t n, uint32_t* __restrict__ a) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = i;
}

__global__ void k_transpose_col(uint32_t E, uint32_t N, const uint64_t* __restrict__ rowEnd,
                                const uint32_t* __restrict__ perm, uint32_t* __restrict__ colT) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= E) return;
  const uint64_t e = perm[t];
  uint32_t lo = 0, hi = N;        // the first row r with rowEnd[r] > e
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (rowEnd[mid] > e) hi = mid; else lo = mid + 1;
  }
  colT[t] = lo;
}

__global__ void k_transpose_row_end(uint32_t N, uint32_t E, const uint32_t* __restrict__ srcSorted,
                                    uint64_t* __restrict__ rowEndT) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  uint32_t lo = 0, hi = E;        // the number of sources <= v
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (srcSorted[mid] <= v) lo = mid + 1; else hi = mid;
  }
  rowEndT[v] = lo;
}

// wT[t] = w[perm[t]]: the weights in the transposed plan's edge order
__global__ void k_permute(uint32_t E, const uint32_t* __restrict__ perm, const float* __restrict__ w,
                          float* __restrict__ wT) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < E) wT[t] = __ldg(w + perm[t]);
}

// Attention dropout's keep bytes in a plan's edge order (roc_sg_attn_keep_mask): one thread and one Philox block per
// edge.  The edge's row is the last row starting at or before it; only the rows from the one before chunk c's first
// owned row up to chunk c + 1's first owned row can hold it, so the search touches a few adjacent rs entries.
__global__ void k_attn_keep(uint32_t E, const uint32_t* __restrict__ rs, const uint32_t* __restrict__ firstRow,
                            const uint32_t* __restrict__ col, uint32_t selfBase, int rowIsSource, uint32_t thresh16,
                            uint32_t seedLo, uint32_t seedHi, uint32_t step, uint8_t* __restrict__ keep) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const uint32_t c = e / (uint32_t)SG_CH;
  uint32_t lo = __ldg(firstRow + c), hi = __ldg(firstRow + c + 1);
  lo = lo ? lo - 1 : 0;           // rs[lo] <= e < rs[hi]
  while (hi - lo > 1) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(rs + mid) <= e) lo = mid; else hi = mid;
  }
  const uint32_t self = selfBase + lo, other = __ldg(col + e);
  const uint32_t i = rowIsSource ? other : self, j = rowIsSource ? self : other;    // the pair (i <- j)
  keep[e] = (uint8_t)dropout_keep8(((uint64_t)j << 32) | i, 0u, step, seedLo, seedHi, thresh16);
}

}  // namespace roc

struct roc_sg_transpose {
  uint32_t N = 0, E = 0;
  uint64_t* rowEndT = nullptr;    // [N]
  uint32_t* colT = nullptr;       // [E]
  uint32_t* perm = nullptr;       // [E]
  roc_sg_plan* planT = nullptr;   // the plan over (rowEndT, colT)
  float* wT = nullptr;            // [E] the permuted weights of the last backward, grown on demand (grow)
  size_t wTBytes = 0;
};

using namespace roc;

extern "C" int roc_sg_plan_create(roc_vid_t rowLeft, roc_vid_t rowRight, roc_eid_t colLeft,
                                  const roc_eid_t* rowEnd, const roc_vid_t* colSrc,
                                  roc_stream_t stream, roc_sg_plan** planOut) {
  if (!planOut || !rowEnd || rowRight < rowLeft) return ROC_ERR_INVALID;
  if (roc_device_count() <= 0) return ROC_ERR_NO_DEVICE;
  cudaStream_t st = as_stream(stream);
  uint64_t nloc64 = (uint64_t)rowRight - rowLeft + 1;
  if (nloc64 >= 0xFFFFFFF0ull) return ROC_ERR_UNSUPPORTED;
  uint32_t nloc = (uint32_t)nloc64;
  uint64_t lastEnd = 0;
  ROC_CUDA(cudaMemcpyAsync(&lastEnd, rowEnd + (nloc - 1), sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  ROC_CUDA(cudaStreamSynchronize(st));
  if (lastEnd < colLeft) return ROC_ERR_INVALID;
  uint64_t E64 = lastEnd - colLeft;
  if (E64 >= 0xFFFFFF00ull) return ROC_ERR_UNSUPPORTED;  // local edge offsets are u32
  if (E64 > 0 && !colSrc) return ROC_ERR_INVALID;

  roc_sg_plan* pl = new (std::nothrow) roc_sg_plan();
  if (!pl) return ROC_ERR_NOMEM;
  cudaGetDevice(&pl->device);
  pl->nloc = nloc; pl->E = (uint32_t)E64; pl->col = colSrc;
  pl->numChunks = pl->E / SG_CH + 1;
  uint32_t* flag = nullptr; uint8_t* hflag = nullptr; uint8_t* bflag = nullptr; void* tmp = nullptr; uint32_t* dcount = nullptr;
  int rc = ROC_OK;
  auto fail = [&](int code) { rc = code; };
#define PL_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fail((int)e_); goto done; } } while (0)
  {
    PL_CUDA(cudaMalloc(&pl->rs, sizeof(uint32_t) * ((size_t)nloc + 1)));
    PL_CUDA(cudaMalloc(&pl->firstRow, sizeof(uint32_t) * ((size_t)pl->numChunks + 1)));
    PL_CUDA(cudaMalloc(&pl->carryIdx, sizeof(uint32_t) * ((size_t)pl->numChunks + 1)));
    PL_CUDA(cudaMalloc(&flag, sizeof(uint32_t) * ((size_t)pl->numChunks + 1)));
    PL_CUDA(cudaMalloc(&hflag, (size_t)nloc));
    PL_CUDA(cudaMalloc(&pl->heavyRows, sizeof(uint32_t) * (size_t)nloc));
    PL_CUDA(cudaMalloc(&dcount, sizeof(uint32_t)));
    const int T = 256;
    k_build_rs<<<(nloc + T) / T, T, 0, st>>>(nloc, colLeft, rowEnd, pl->rs);
    count_launch();
    k_first_row<<<(pl->numChunks + 1 + T - 1) / T, T, 0, st>>>(nloc, pl->numChunks, pl->rs, pl->firstRow);
    count_launch();
    k_carry_flag<<<(pl->numChunks + 1 + T - 1) / T, T, 0, st>>>(pl->numChunks, pl->rs, pl->firstRow, flag);
    count_launch();
    PL_CUDA(cudaMalloc(&bflag, (size_t)nloc));
    PL_CUDA(cudaMalloc(&pl->bigRows, sizeof(uint32_t) * (size_t)nloc));
    k_heavy_flag<<<(nloc + T - 1) / T, T, 0, st>>>(nloc, pl->rs, hflag, bflag);
    count_launch();
    PL_CUDA(cudaGetLastError());
    size_t tb1 = 0, tb2 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb1, flag, pl->carryIdx, (int)(pl->numChunks + 1), st);
    thrust::counting_iterator<uint32_t> cnt(0);
    cub::DeviceSelect::Flagged(nullptr, tb2, cnt, hflag, pl->heavyRows, dcount, (int)nloc, st);
    size_t tb = tb1 > tb2 ? tb1 : tb2;
    PL_CUDA(cudaMalloc(&tmp, tb ? tb : 16));
    PL_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb1, flag, pl->carryIdx, (int)(pl->numChunks + 1), st));
    PL_CUDA(cub::DeviceSelect::Flagged(tmp, tb2, cnt, hflag, pl->heavyRows, dcount, (int)nloc, st));
    PL_CUDA(cudaMemcpyAsync(&pl->numHeavy, dcount, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    PL_CUDA(cub::DeviceSelect::Flagged(tmp, tb2, cnt, bflag, pl->bigRows, dcount, (int)nloc, st));
    count_launch(6);
    PL_CUDA(cudaMemcpyAsync(&pl->numCarries, pl->carryIdx + pl->numChunks, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    PL_CUDA(cudaMemcpyAsync(&pl->numBig, dcount, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    PL_CUDA(cudaMalloc(&pl->desc, sizeof(uint32_t) * 8 * (size_t)pl->numChunks));
    k_chunk_desc<<<(pl->numChunks + T - 1) / T, T, 0, st>>>(pl->numChunks, pl->E, pl->rs, pl->firstRow, pl->carryIdx, pl->desc);
    count_launch();
    PL_CUDA(cudaGetLastError());
    PL_CUDA(cudaStreamSynchronize(st));
  }
done:
#undef PL_CUDA
  cudaFree(flag); cudaFree(hflag); cudaFree(bflag); cudaFree(tmp); cudaFree(dcount);
  if (rc != ROC_OK) { roc_sg_plan_destroy(pl); return rc; }
  *planOut = pl;
  return ROC_OK;
}

extern "C" void roc_sg_plan_destroy(roc_sg_plan* pl) {
  if (!pl) return;
  cudaFree(pl->rs); cudaFree(pl->firstRow); cudaFree(pl->carryIdx); cudaFree(pl->heavyRows); cudaFree(pl->bigRows); cudaFree(pl->carry); cudaFree(pl->desc);
  cudaFree(pl->carryArg); cudaFree(pl->carry2); cudaFree(pl->attnRec); cudaFree(pl->smxWs);
  delete pl;
}

extern "C" int roc_sg_plan_reserve(roc_sg_plan* pl, int maxH) {
  if (!pl || maxH <= 0) return ROC_ERR_INVALID;
  return grow_carries(pl, maxH, nullptr, false);
}

extern "C" int roc_sg_plan_info(const roc_sg_plan* pl, uint64_t* numChunks, uint64_t* numCarries,
                                uint64_t* numHeavyRows) {
  if (!pl) return ROC_ERR_INVALID;
  if (numChunks) *numChunks = pl->numChunks;
  if (numCarries) *numCarries = pl->numCarries;
  if (numHeavyRows) *numHeavyRows = (uint64_t)pl->numHeavy + pl->numBig;
  return ROC_OK;
}

// The plan parameters shared by every launch, with the carries' leading dimension in floats like the caller's.
static SgParams plan_params(const roc_sg_plan* pl) {
  SgParams p;
  memset(&p, 0, sizeof(p));
  p.rs = pl->rs; p.firstRow = pl->firstRow; p.carryIdx = pl->carryIdx; p.heavyRows = pl->heavyRows; p.bigRows = pl->bigRows;
  p.col = pl->col; p.carry = pl->carry; p.carryArg = pl->carryArg; p.ldC = pl->carryLd;
  p.E = pl->E; p.numChunks = pl->numChunks; p.numHeavy = pl->numHeavy; p.numBig = pl->numBig; p.epi = 0;
  p.desc = pl->desc;
  return p;
}

// Whether rows can be read as float4 T-columns: every row pointer 16-byte aligned, every leading dimension a multiple
// of 4 floats.
static bool float4_rows(std::initializer_list<const void*> rows, std::initializer_list<int64_t> lds) {
  for (const void* r : rows)
    if (!aligned16(r)) return false;
  for (int64_t ld : lds)
    if (ld % 4) return false;
  return true;
}

// Converts the leading dimensions of p's T-column rows (in, out, arg, xrow and the carries) from floats to T-columns
// of vw floats, and sets Q for rows of `cols` floats.
static void t_units(SgParams& p, int vw, int cols) {
  p.ldIn /= vw; p.ldOut /= vw; p.ldArg /= vw; p.ldX /= vw; p.ldC /= vw;
  p.Q = ((uint32_t)cols + vw - 1) / vw;
}

// The operands of run_planned only some reductions take: WSUM's weights, EDOT's G rows (indexed by plan row) and its
// output, TSUM's row ends of the original graph, TELE's t (indexed by plan row) and coefficients.
struct SgEdge {
  const float* w = nullptr;
  const float* g = nullptr;
  int64_t ldG = 0;
  float* dw = nullptr;
  bool accumulate = false;
  const roc_eid_t* rowEnd = nullptr;
  const float* t = nullptr;
  int64_t ldT = 0;
  float alpha = 1.f, beta = 1.f;
  const uint8_t* keep = nullptr;   // edge dropout (SG_RED_DROP): one keep byte per edge of the plan, and a kept row's scale
  float dropScale = 1.f;
};

// Reduction RED over the columns [0, H) of every row, in column blocks of the widest row one launch takes (SG_REDS),
// on float4 rows when every leading dimension and pointer allows them.  `arg` holds the min / max indices
// (written by the forward, gathered by the backward); the sum passes none.  EDOT's column blocks add their partial
// dot products to dw in block order: the first overwrites it (or adds, with ed.accumulate), the later ones add.
// `in` holds fp32 rows, bf16 ones (raw bits) for BSUM and the bf16 forms; its leading dimension is in elements either
// way.
template <int RED>
static int run_planned(roc_sg_plan* pl, int H, const void* in, int64_t ldIn, float* out, int64_t ldOut,
                       const roc_vid_t* arg, int64_t ldArg, int epilogue, roc_vid_t selfBase, cudaStream_t st,
                       const SgEdge& ed = SgEdge()) {
  constexpr SgCarry CARRY = sg_red(RED).carry;
  const bool vec = float4_rows({in, out, arg, ed.g}, {ldIn, ldOut, ldArg, ed.ldG});
  const int blockCols = vec ? 4 * sg_max_q(4, RED) : sg_max_q(1, RED);
  int rc = CARRY == SG_CARRY_NONE ? ROC_OK : grow_carries(pl, std::min(H, blockCols), st);
  // the min / max forward's index carries, which the kernels address with the float carries' leading dimension
  if (rc == ROC_OK && CARRY == SG_CARRY_INDEX)
    rc = grow(pl->carryArg, pl->carryArgBytes, (size_t)pl->numCarries * pl->carryLd * sizeof(uint32_t), st);
  if (rc != ROC_OK) return rc;
  for (int c0 = 0; c0 < H; c0 += blockCols) {
    SgParams p = plan_params(pl);
    p.in = static_cast<const char*>(in) + (size_t)c0 * (sg_bf16_in(RED) ? 2 : 4);
    p.out = out ? out + c0 : nullptr; p.epi = epilogue; p.selfBase = selfBase;
    if (arg) p.arg = const_cast<roc_vid_t*>(arg) + c0;
    p.ldIn = (size_t)ldIn; p.ldOut = (size_t)ldOut; p.ldArg = (size_t)ldArg;
    p.score = ed.w; p.out2 = ed.dw; p.dwAdd = (ed.accumulate || c0 > 0) ? 1 : 0;
    if (ed.g) { p.xrow = ed.g + c0; p.ldX = (size_t)ed.ldG; }
    if (ed.rowEnd) p.xrow = ed.rowEnd;
    if (ed.t) { p.xrow = ed.t + c0; p.ldS = (size_t)ed.ldT; p.slope = ed.alpha; p.teleBeta = ed.beta; }
    if (ed.keep) { p.keep = ed.keep; p.dropScale = ed.dropScale; }
    p.H = (uint32_t)std::min(H - c0, blockCols);
    t_units(p, vec ? 4 : 1, std::min(H - c0, blockCols));
    rc = vec ? dispatch<4, RED>(p, st) : dispatch<1, RED>(p, st);
    if (rc != ROC_OK) return rc;
  }
  return ROC_OK;
}

// The input rule of every bf16 feature input `in` (a NULL one is left to the call's own checks): 16-byte aligned, with
// a leading dimension that is a multiple of 8 elements, so that it takes float4 rows exactly when its fp32 twin does.
static bool bf16_rows_bad(const void* in, int64_t ldIn) { return in && ((ldIn % 8) || !aligned16(in)); }

extern "C" int roc_sg_forward_planned(const roc_sg_plan* plc, int H, const float* in, int64_t ldIn,
                                      float* out, int64_t ldOut, int epilogue, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || H <= 0 || !in || !out || ldIn < H || ldOut < H) return ROC_ERR_INVALID;
  return run_planned<SG_RED_SUM>(pl, H, in, ldIn, out, ldOut, nullptr, 0, epilogue, 0, as_stream(stream));
}

// A 16-byte aligned `in` with ldIn a multiple of 8 is read as float4 T-columns whenever `out` allows it, as the fp32
// call does for the widened copy of `in` (roc_bf16_to_f32 into any 16-byte aligned buffer whose leading dimension is
// a multiple of 4): the same column blocks and row shapes, hence the same bits.
extern "C" int roc_sg_forward_planned_bf16(const roc_sg_plan* plc, int H, const uint16_t* in, int64_t ldIn,
                                           float* out, int64_t ldOut, int epilogue, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || H <= 0 || !in || !out || ldIn < H || ldOut < H || (ldIn % 8) || !aligned16(in)) return ROC_ERR_INVALID;
  return run_planned<SG_RED_BSUM>(pl, H, in, ldIn, out, ldOut, nullptr, 0, epilogue, 0, as_stream(stream));
}

extern "C" int roc_sg_forward_teleport_planned(const roc_sg_plan* plc, int H, const float* in, int64_t ldIn,
                                               float alpha, const float* t, int64_t ldT, float beta, float* out,
                                               int64_t ldOut, int epilogue, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || H <= 0 || !in || !t || !out || out == t || ldIn < H || ldT < H || ldOut < H ||
      (epilogue & ~(ROC_SG_EPI_NORM | ROC_SG_EPI_NORM_OUT)) || !std::isfinite(alpha) || !std::isfinite(beta))
    return ROC_ERR_INVALID;
  SgEdge ed;
  ed.t = t; ed.ldT = ldT; ed.alpha = alpha; ed.beta = beta;
  return run_planned<SG_RED_TELE>(pl, H, in, ldIn, out, ldOut, nullptr, 0, epilogue, 0, as_stream(stream), ed);
}

extern "C" int roc_sg_plan_rows_sorted(const roc_sg_plan* pl, int* sorted, roc_stream_t stream) {
  if (!pl || !sorted) return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  uint32_t* bad = nullptr;
  uint32_t h = 0;
  ROC_CUDA(cudaMallocAsync((void**)&bad, sizeof(uint32_t), st));
  cudaError_t e = cudaMemsetAsync(bad, 0, sizeof(uint32_t), st);
  if (e == cudaSuccess && pl->nloc && pl->E) {
    k_rows_sorted<<<(pl->nloc + 255) / 256, 256, 0, st>>>(pl->nloc, pl->rs, pl->col, bad);
    count_launch();
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&h, bad, sizeof(uint32_t), cudaMemcpyDeviceToHost, st);
  cudaError_t f = cudaFreeAsync(bad, st);
  if (e == cudaSuccess) e = f;
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return (int)e;
  *sorted = h ? 0 : 1;
  return ROC_OK;
}

template <int BF>
static int minmax_forward(const roc_sg_plan* plc, int aggr, int H, const void* in, int64_t ldIn, float* out,
                          int64_t ldOut, roc_vid_t* arg, int64_t ldArg, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || (aggr != ROC_SG_AGGR_MAX && aggr != ROC_SG_AGGR_MIN) || H <= 0 || !in || !out || !arg || ldIn < H ||
      ldOut < H || ldArg < H || (BF && bf16_rows_bad(in, ldIn)))
    return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  return aggr == ROC_SG_AGGR_MAX ? run_planned<SG_RED_MAX | BF>(pl, H, in, ldIn, out, ldOut, arg, ldArg, 0, 0, st)
                                 : run_planned<SG_RED_MIN | BF>(pl, H, in, ldIn, out, ldOut, arg, ldArg, 0, 0, st);
}

extern "C" int roc_sg_minmax_forward_planned(const roc_sg_plan* plc, int aggr, int H, const float* in, int64_t ldIn,
                                             float* out, int64_t ldOut, roc_vid_t* arg, int64_t ldArg,
                                             roc_stream_t stream) {
  return minmax_forward<0>(plc, aggr, H, in, ldIn, out, ldOut, arg, ldArg, stream);
}

extern "C" int roc_sg_minmax_forward_planned_bf16(const roc_sg_plan* plc, int aggr, int H, const uint16_t* in,
                                                  int64_t ldIn, float* out, int64_t ldOut, roc_vid_t* arg,
                                                  int64_t ldArg, roc_stream_t stream) {
  return minmax_forward<SG_RED_BF16>(plc, aggr, H, in, ldIn, out, ldOut, arg, ldArg, stream);
}

extern "C" int roc_sg_minmax_backward_planned(const roc_sg_plan* plc, int H, roc_vid_t selfBase, const float* outGrad,
                                              int64_t ldG, const roc_vid_t* arg, int64_t ldArg, float* inGrad,
                                              int64_t ldIn, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || H <= 0 || !outGrad || !arg || !inGrad || ldG < H || ldArg < H || ldIn < H) return ROC_ERR_INVALID;
  return run_planned<SG_RED_MASK>(pl, H, outGrad, ldG, inGrad, ldIn, arg, ldArg, 0, selfBase, as_stream(stream));
}

// What both attention entry points do once their own arguments are checked: ROC_ERR_INVALID for a bad slope,
// ROC_ERR_UNSUPPORTED for a head layout the kernels do not take, then the carries of the H-wide and the heads-wide
// partials.  *ftShift = log2 of the T-columns per head.
static int attn_setup(roc_sg_plan* pl, int heads, int H, float slope, bool vec, cudaStream_t st, uint32_t* ftShift) {
  if (!(slope >= 0.f) || !std::isfinite(slope)) return ROC_ERR_INVALID;
  if ((heads != 1 && heads != 2 && heads != 4 && heads != 8) || H % heads) return ROC_ERR_UNSUPPORTED;
  const int F = H / heads;
  if (heads > 1 && (F < 4 || (F & (F - 1)))) return ROC_ERR_UNSUPPORTED;
  if (H > (vec ? 512 : 256)) return ROC_ERR_UNSUPPORTED;
  uint32_t fs = 0;
  while ((1 << fs) < F / (vec ? 4 : 1)) fs++;
  *ftShift = heads == 1 ? 31u : fs;
  int rc = grow_carries(pl, H, st);
  if (rc == ROC_OK) rc = grow(pl->carry2, pl->carry2Bytes, (size_t)pl->numCarries * SG_LDC2 * sizeof(float), st);
  return rc;
}

// The parameters every attention pass shares (leading dimensions of T-column rows set by the pass, in floats).
static SgParams attn_params(const roc_sg_plan* pl, int heads, int H, float slope, roc_vid_t selfBase,
                            const float* score, int64_t ldS, const float* stats, int64_t ldStats, uint32_t ftShift) {
  SgParams p = plan_params(pl);
  p.carry2 = pl->carry2; p.rec = pl->attnRec;
  p.selfBase = selfBase; p.score = score; p.ldS = (size_t)ldS; p.stats = stats; p.ldStats = (size_t)ldStats;
  p.heads = (uint32_t)heads; p.H = (uint32_t)H; p.slope = slope; p.ftShift = ftShift;
  return p;
}

// The attention passes RF (with SG_RED_BF16 as the call's rows are) on float4 or scalar rows, with dropout
// (SG_RED_DROP) when `drop`.
template <int RF>
static int dispatch_attn(const SgParams& p, bool vec, bool drop, cudaStream_t st) {
  if (drop) return vec ? dispatch<4, RF | SG_RED_DROP>(p, st) : dispatch<1, RF | SG_RED_DROP>(p, st);
  return vec ? dispatch<4, RF>(p, st) : dispatch<1, RF>(p, st);
}

// Attention and edge dropout's arguments: ROC_ERR_INVALID for a rate outside [0, 1); *drop when there is a mask and
// rate > 0 (rate 0 or no mask: the calls without dropout).  The scale is roc_dropout_fwd's.
static int attn_drop_args(const void* keep, float rate, bool* drop, float* scale) {
  if (!(rate >= 0.f && rate < 1.f)) return ROC_ERR_INVALID;
  *drop = keep != nullptr && rate > 0.f;
  *scale = 1.0f / (1.0f - rate);
  return ROC_OK;
}

// The attention backward's passes once its arguments are checked and both plans' carries grown: the node records of
// ids [0, n) and B1 (d s_dst) over `pl`, B2 (inGrad, d s_src) over `plB2`.  With plB2 = pl, B2 is the gather over the
// same CSR (quirk Q1); over the transposed plan its row j gathers the destinations i of j's out-edges, where the same
// formula, a(i<-j) G[i] against the record of i, is the true adjoint.
// BF = SG_RED_BF16: `in` holds bf16 rows, gathered by B1 and read as each row's own row by B2.  With `drop`, B1 reads
// the keep bytes `keep` in pl's edge order and B2 `keep2` in plB2's, each byte the pair's that pass weighs.
template <int BF>
static int attn_backward_passes(roc_sg_plan* pl, roc_sg_plan* plB2, uint32_t n, int heads, int H, float slope,
                                roc_vid_t selfBase, uint32_t fs, bool vec, const void* in, int64_t ldIn,
                                const float* score, int64_t ldS, const float* out, int64_t ldOut, const float* stats,
                                int64_t ldStats, const float* outGrad, int64_t ldG, float* inGrad, int64_t ldInG,
                                float* scoreGrad, int64_t ldSG, bool drop, const uint8_t* keep, const uint8_t* keep2,
                                float keepScale, cudaStream_t st) {
  int rc = grow(pl->attnRec, pl->attnRecBytes, (size_t)n * heads * sizeof(float4), st);
  if (rc != ROC_OK) return rc;
  const int vw = vec ? 4 : 1;
  SgParams p = attn_params(pl, heads, H, slope, selfBase, score, ldS, stats, ldStats, fs);
  p.keepScale = keepScale;
  // the node records {s_dst, m, 1/Z, D}, from G and O
  SgParams r = p;
  r.in = outGrad; r.ldIn = (size_t)ldG; r.xrow = out; r.ldX = (size_t)ldOut;
  t_units(r, vw, H);
  rc = vec ? launch_rec<4>(r, n, st) : launch_rec<1>(r, n, st);
  if (rc != ROC_OK) return rc;
  // B1: d s_dst, gathering X[j] and s_src[j] against G[i]
  SgParams b1 = p;
  b1.in = in; b1.ldIn = (size_t)ldIn; b1.xrow = outGrad; b1.ldX = (size_t)ldG;
  b1.out = nullptr; b1.out2 = scoreGrad; b1.ldOut2 = (size_t)ldSG; b1.keep = keep;
  t_units(b1, vw, H);
  rc = dispatch_attn<SG_RED_ADST | BF>(b1, vec, drop, st);
  if (rc != ROC_OK) return rc;
  // B2: inGrad and d s_src, gathering G[j] and the record of j against X[i]
  SgParams b2 = attn_params(plB2, heads, H, slope, selfBase, score, ldS, stats, ldStats, fs);
  b2.rec = pl->attnRec;
  b2.in = outGrad; b2.ldIn = (size_t)ldG; b2.xrow = in; b2.ldX = (size_t)ldIn;
  b2.out = inGrad; b2.ldOut = (size_t)ldInG; b2.out2 = scoreGrad + heads; b2.ldOut2 = (size_t)ldSG;
  b2.keep = keep2; b2.keepScale = keepScale;
  t_units(b2, vw, H);
  return dispatch_attn<SG_RED_ASRC | BF>(b2, vec, drop, st);
}

template <int BF>
static int attn_forward(const roc_sg_plan* plc, int heads, int H, float slope, roc_vid_t selfBase, const void* in,
                        int64_t ldIn, const float* score, int64_t ldS, float* out, int64_t ldOut, float* stats,
                        int64_t ldStats, const uint8_t* keep, float rate, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  bool drop = false;
  float keepScale = 1.f;
  if (!pl || !in || !score || !out || !stats || heads <= 0 || H <= 0 || ldIn < H || ldOut < H ||
      ldS < 2 * (int64_t)heads || ldStats < 2 * (int64_t)heads || (BF && bf16_rows_bad(in, ldIn)) ||
      attn_drop_args(keep, rate, &drop, &keepScale) != ROC_OK)
    return ROC_ERR_INVALID;
  const bool vec = float4_rows({in, out}, {ldIn, ldOut});
  cudaStream_t st = as_stream(stream);
  uint32_t fs = 0;
  int rc = attn_setup(pl, heads, H, slope, vec, st, &fs);
  if (rc != ROC_OK) return rc;
  // pass 1: (m, 1/Z) per row and head from the scores alone, one float per head (dropout does not change them)
  SgParams a = attn_params(pl, heads, H, slope, selfBase, score, ldS, stats, ldStats, 0);
  a.in = score + heads; a.ldIn = (size_t)ldS; a.out = stats; a.ldOut = (size_t)ldStats;
  t_units(a, 1, heads);
  if ((rc = dispatch<1, SG_RED_ASTAT>(a, st)) != ROC_OK) return rc;
  // pass 2: the a-weighted sum of the feature rows
  SgParams b = attn_params(pl, heads, H, slope, selfBase, score, ldS, stats, ldStats, fs);
  b.in = in; b.ldIn = (size_t)ldIn; b.out = out; b.ldOut = (size_t)ldOut;
  b.keep = keep; b.keepScale = keepScale;
  t_units(b, vec ? 4 : 1, H);
  return dispatch_attn<SG_RED_ATTN | BF>(b, vec, drop, st);
}

extern "C" int roc_sg_attn_forward_planned(const roc_sg_plan* plc, int heads, int H, float slope, roc_vid_t selfBase,
                                           const float* in, int64_t ldIn, const float* score, int64_t ldS,
                                           float* out, int64_t ldOut, float* stats, int64_t ldStats,
                                           roc_stream_t stream) {
  return attn_forward<0>(plc, heads, H, slope, selfBase, in, ldIn, score, ldS, out, ldOut, stats, ldStats, nullptr,
                         0.f, stream);
}

extern "C" int roc_sg_attn_forward_planned_bf16(const roc_sg_plan* plc, int heads, int H, float slope,
                                                roc_vid_t selfBase, const uint16_t* in, int64_t ldIn,
                                                const float* score, int64_t ldS, float* out, int64_t ldOut,
                                                float* stats, int64_t ldStats, roc_stream_t stream) {
  return attn_forward<SG_RED_BF16>(plc, heads, H, slope, selfBase, in, ldIn, score, ldS, out, ldOut, stats, ldStats,
                                   nullptr, 0.f, stream);
}

extern "C" int roc_sg_attn_forward_dropout_planned(const roc_sg_plan* plc, int heads, int H, float slope,
                                                   roc_vid_t selfBase, const float* in, int64_t ldIn,
                                                   const float* score, int64_t ldS, float* out, int64_t ldOut,
                                                   float* stats, int64_t ldStats, const uint8_t* keep, float rate,
                                                   roc_stream_t stream) {
  return attn_forward<0>(plc, heads, H, slope, selfBase, in, ldIn, score, ldS, out, ldOut, stats, ldStats, keep, rate,
                         stream);
}

extern "C" int roc_sg_attn_forward_dropout_planned_bf16(const roc_sg_plan* plc, int heads, int H, float slope,
                                                        roc_vid_t selfBase, const uint16_t* in, int64_t ldIn,
                                                        const float* score, int64_t ldS, float* out, int64_t ldOut,
                                                        float* stats, int64_t ldStats, const uint8_t* keep, float rate,
                                                        roc_stream_t stream) {
  return attn_forward<SG_RED_BF16>(plc, heads, H, slope, selfBase, in, ldIn, score, ldS, out, ldOut, stats, ldStats,
                                   keep, rate, stream);
}

// The backward's keep bytes: both or neither (ROC_ERR_INVALID otherwise), then attn_drop_args.
static int attn_drop_args2(const uint8_t* keep, const uint8_t* keep2, float rate, bool* drop, float* scale) {
  if ((keep == nullptr) != (keep2 == nullptr)) return ROC_ERR_INVALID;
  return attn_drop_args(keep, rate, drop, scale);
}

template <int BF>
static int attn_backward(const roc_sg_plan* plc, int heads, int H, float slope, roc_vid_t selfBase, const void* in,
                         int64_t ldIn, const float* score, int64_t ldS, const float* out, int64_t ldOut,
                         const float* stats, int64_t ldStats, const float* outGrad, int64_t ldG, float* inGrad,
                         int64_t ldInG, float* scoreGrad, int64_t ldSG, const uint8_t* keep, const uint8_t* keepRev,
                         float rate, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  bool drop = false;
  float keepScale = 1.f;
  if (!pl || !in || !score || !out || !stats || !outGrad || !inGrad || !scoreGrad || heads <= 0 || H <= 0 ||
      ldIn < H || ldOut < H || ldG < H || ldInG < H || ldS < 2 * (int64_t)heads || ldStats < 2 * (int64_t)heads ||
      ldSG < 2 * (int64_t)heads || (BF && bf16_rows_bad(in, ldIn)) ||
      attn_drop_args2(keep, keepRev, rate, &drop, &keepScale) != ROC_OK)
    return ROC_ERR_INVALID;
  const bool vec = float4_rows({in, out, outGrad, inGrad}, {ldIn, ldOut, ldG, ldInG});
  cudaStream_t st = as_stream(stream);
  uint32_t fs = 0;
  int rc = attn_setup(pl, heads, H, slope, vec, st, &fs);
  if (rc != ROC_OK) return rc;
  if ((rc = find_id_end(pl, st)) != ROC_OK) return rc;
  const uint64_t n64 = std::max<uint64_t>(pl->idEnd, (uint64_t)selfBase + pl->nloc);
  if (n64 >= 0xFFFFFFF0ull) return ROC_ERR_UNSUPPORTED;
  return attn_backward_passes<BF>(pl, pl, (uint32_t)n64, heads, H, slope, selfBase, fs, vec, in, ldIn, score, ldS, out,
                                  ldOut, stats, ldStats, outGrad, ldG, inGrad, ldInG, scoreGrad, ldSG, drop, keep,
                                  keepRev, keepScale, st);
}

extern "C" int roc_sg_attn_backward_planned(const roc_sg_plan* plc, int heads, int H, float slope, roc_vid_t selfBase,
                                            const float* in, int64_t ldIn, const float* score, int64_t ldS,
                                            const float* out, int64_t ldOut, const float* stats, int64_t ldStats,
                                            const float* outGrad, int64_t ldG, float* inGrad, int64_t ldInG,
                                            float* scoreGrad, int64_t ldSG, roc_stream_t stream) {
  return attn_backward<0>(plc, heads, H, slope, selfBase, in, ldIn, score, ldS, out, ldOut, stats, ldStats, outGrad,
                          ldG, inGrad, ldInG, scoreGrad, ldSG, nullptr, nullptr, 0.f, stream);
}

extern "C" int roc_sg_attn_backward_planned_bf16(const roc_sg_plan* plc, int heads, int H, float slope,
                                                 roc_vid_t selfBase, const uint16_t* in, int64_t ldIn,
                                                 const float* score, int64_t ldS, const float* out, int64_t ldOut,
                                                 const float* stats, int64_t ldStats, const float* outGrad,
                                                 int64_t ldG, float* inGrad, int64_t ldInG, float* scoreGrad,
                                                 int64_t ldSG, roc_stream_t stream) {
  return attn_backward<SG_RED_BF16>(plc, heads, H, slope, selfBase, in, ldIn, score, ldS, out, ldOut, stats, ldStats,
                                    outGrad, ldG, inGrad, ldInG, scoreGrad, ldSG, nullptr, nullptr, 0.f, stream);
}

extern "C" int roc_sg_attn_backward_dropout_planned(const roc_sg_plan* plc, int heads, int H, float slope,
                                                    roc_vid_t selfBase, const float* in, int64_t ldIn,
                                                    const float* score, int64_t ldS, const float* out, int64_t ldOut,
                                                    const float* stats, int64_t ldStats, const float* outGrad,
                                                    int64_t ldG, float* inGrad, int64_t ldInG, float* scoreGrad,
                                                    int64_t ldSG, const uint8_t* keep, const uint8_t* keepRev,
                                                    float rate, roc_stream_t stream) {
  return attn_backward<0>(plc, heads, H, slope, selfBase, in, ldIn, score, ldS, out, ldOut, stats, ldStats, outGrad,
                          ldG, inGrad, ldInG, scoreGrad, ldSG, keep, keepRev, rate, stream);
}

extern "C" int roc_sg_attn_backward_dropout_planned_bf16(const roc_sg_plan* plc, int heads, int H, float slope,
                                                         roc_vid_t selfBase, const uint16_t* in, int64_t ldIn,
                                                         const float* score, int64_t ldS, const float* out,
                                                         int64_t ldOut, const float* stats, int64_t ldStats,
                                                         const float* outGrad, int64_t ldG, float* inGrad,
                                                         int64_t ldInG, float* scoreGrad, int64_t ldSG,
                                                         const uint8_t* keep, const uint8_t* keepRev, float rate,
                                                         roc_stream_t stream) {
  return attn_backward<SG_RED_BF16>(plc, heads, H, slope, selfBase, in, ldIn, score, ldS, out, ldOut, stats, ldStats,
                                    outGrad, ldG, inGrad, ldInG, scoreGrad, ldSG, keep, keepRev, rate, stream);
}

template <int BF>
static int attn_backward_exact(const roc_sg_plan* plc, roc_sg_transpose* tr, int heads, int H, float slope,
                               const void* in, int64_t ldIn, const float* score, int64_t ldS, const float* out,
                               int64_t ldOut, const float* stats, int64_t ldStats, const float* outGrad, int64_t ldG,
                               float* inGrad, int64_t ldInG, float* scoreGrad, int64_t ldSG, const uint8_t* keep,
                               const uint8_t* keepT, float rate, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  bool drop = false;
  float keepScale = 1.f;
  if (!pl || !tr || !in || !score || !out || !stats || !outGrad || !inGrad || !scoreGrad || heads <= 0 || H <= 0 ||
      ldIn < H || ldOut < H || ldG < H || ldInG < H || ldS < 2 * (int64_t)heads || ldStats < 2 * (int64_t)heads ||
      ldSG < 2 * (int64_t)heads || pl->nloc != tr->N || pl->E != tr->E || (BF && bf16_rows_bad(in, ldIn)) ||
      attn_drop_args2(keep, keepT, rate, &drop, &keepScale) != ROC_OK)
    return ROC_ERR_INVALID;
  const bool vec = float4_rows({in, out, outGrad, inGrad}, {ldIn, ldOut, ldG, ldInG});
  cudaStream_t st = as_stream(stream);
  uint32_t fs = 0;
  int rc = attn_setup(pl, heads, H, slope, vec, st, &fs);
  if (rc == ROC_OK) rc = attn_setup(tr->planT, heads, H, slope, vec, st, &fs);
  if (rc != ROC_OK) return rc;
  // a whole graph: every id is below N, so the records cover [0, N) with no id scan
  return attn_backward_passes<BF>(pl, tr->planT, tr->N, heads, H, slope, 0, fs, vec, in, ldIn, score, ldS, out, ldOut,
                                  stats, ldStats, outGrad, ldG, inGrad, ldInG, scoreGrad, ldSG, drop, keep, keepT,
                                  keepScale, st);
}

extern "C" int roc_sg_attn_backward_exact(const roc_sg_plan* plc, roc_sg_transpose* tr, int heads, int H, float slope,
                                          const float* in, int64_t ldIn, const float* score, int64_t ldS,
                                          const float* out, int64_t ldOut, const float* stats, int64_t ldStats,
                                          const float* outGrad, int64_t ldG, float* inGrad, int64_t ldInG,
                                          float* scoreGrad, int64_t ldSG, roc_stream_t stream) {
  return attn_backward_exact<0>(plc, tr, heads, H, slope, in, ldIn, score, ldS, out, ldOut, stats, ldStats, outGrad,
                                ldG, inGrad, ldInG, scoreGrad, ldSG, nullptr, nullptr, 0.f, stream);
}

extern "C" int roc_sg_attn_backward_exact_bf16(const roc_sg_plan* plc, roc_sg_transpose* tr, int heads, int H,
                                               float slope, const uint16_t* in, int64_t ldIn, const float* score,
                                               int64_t ldS, const float* out, int64_t ldOut, const float* stats,
                                               int64_t ldStats, const float* outGrad, int64_t ldG, float* inGrad,
                                               int64_t ldInG, float* scoreGrad, int64_t ldSG, roc_stream_t stream) {
  return attn_backward_exact<SG_RED_BF16>(plc, tr, heads, H, slope, in, ldIn, score, ldS, out, ldOut, stats, ldStats,
                                          outGrad, ldG, inGrad, ldInG, scoreGrad, ldSG, nullptr, nullptr, 0.f, stream);
}

extern "C" int roc_sg_attn_backward_dropout_exact(const roc_sg_plan* plc, roc_sg_transpose* tr, int heads, int H,
                                                  float slope, const float* in, int64_t ldIn, const float* score,
                                                  int64_t ldS, const float* out, int64_t ldOut, const float* stats,
                                                  int64_t ldStats, const float* outGrad, int64_t ldG, float* inGrad,
                                                  int64_t ldInG, float* scoreGrad, int64_t ldSG, const uint8_t* keep,
                                                  const uint8_t* keepT, float rate, roc_stream_t stream) {
  return attn_backward_exact<0>(plc, tr, heads, H, slope, in, ldIn, score, ldS, out, ldOut, stats, ldStats, outGrad,
                                ldG, inGrad, ldInG, scoreGrad, ldSG, keep, keepT, rate, stream);
}

extern "C" int roc_sg_attn_backward_dropout_exact_bf16(const roc_sg_plan* plc, roc_sg_transpose* tr, int heads, int H,
                                                       float slope, const uint16_t* in, int64_t ldIn,
                                                       const float* score, int64_t ldS, const float* out,
                                                       int64_t ldOut, const float* stats, int64_t ldStats,
                                                       const float* outGrad, int64_t ldG, float* inGrad,
                                                       int64_t ldInG, float* scoreGrad, int64_t ldSG,
                                                       const uint8_t* keep, const uint8_t* keepT, float rate,
                                                       roc_stream_t stream) {
  return attn_backward_exact<SG_RED_BF16>(plc, tr, heads, H, slope, in, ldIn, score, ldS, out, ldOut, stats, ldStats,
                                          outGrad, ldG, inGrad, ldInG, scoreGrad, ldSG, keep, keepT, rate, stream);
}

extern "C" int roc_sg_attn_keep_mask(const roc_sg_plan* plc, roc_vid_t selfBase, int rowIsSource, float rate,
                                     uint64_t seed, uint32_t step, uint8_t* keep, roc_stream_t stream) {
  clear_launches();
  if (!plc || (plc->E && !keep) || (rowIsSource != 0 && rowIsSource != 1) || !(rate >= 0.f && rate < 1.f))
    return ROC_ERR_INVALID;
  if (plc->E == 0) return ROC_OK;
  const uint32_t grid = (plc->E + 255) / 256;
  k_attn_keep<<<grid, 256, 0, as_stream(stream)>>>(plc->E, plc->rs, plc->firstRow, plc->col, selfBase, rowIsSource,
                                                   dropout_thresh16(rate), (uint32_t)seed, (uint32_t)(seed >> 32),
                                                   step, keep);
  ROC_LAUNCH_CHECK();
  note_launch(ROC_SG_LAUNCH_KEEP_MASK, -1, 1, 1, 1, grid);
  return ROC_OK;
}

template <int BF>
static int weighted_forward(const roc_sg_plan* plc, int H, const void* in, int64_t ldIn, const float* w, float* out,
                            int64_t ldOut, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || H <= 0 || !in || !w || !out || ldIn < H || ldOut < H || (BF && bf16_rows_bad(in, ldIn)))
    return ROC_ERR_INVALID;
  SgEdge ed;
  ed.w = w;
  return run_planned<SG_RED_WSUM | BF>(pl, H, in, ldIn, out, ldOut, nullptr, 0, 0, 0, as_stream(stream), ed);
}

extern "C" int roc_sg_weighted_forward_planned(const roc_sg_plan* plc, int H, const float* in, int64_t ldIn,
                                               const float* w, float* out, int64_t ldOut, roc_stream_t stream) {
  return weighted_forward<0>(plc, H, in, ldIn, w, out, ldOut, stream);
}

extern "C" int roc_sg_weighted_forward_planned_bf16(const roc_sg_plan* plc, int H, const uint16_t* in, int64_t ldIn,
                                                    const float* w, float* out, int64_t ldOut, roc_stream_t stream) {
  return weighted_forward<SG_RED_BF16>(plc, H, in, ldIn, w, out, ldOut, stream);
}

template <int BF>
static int edge_dot(const roc_sg_plan* plc, int H, const float* outGrad, int64_t ldG, const void* in, int64_t ldIn,
                    float* dw, int accumulate, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || H <= 0 || !outGrad || !in || !dw || ldG < H || ldIn < H || (BF && bf16_rows_bad(in, ldIn)))
    return ROC_ERR_INVALID;
  SgEdge ed;
  ed.g = outGrad; ed.ldG = ldG; ed.dw = dw; ed.accumulate = accumulate != 0;
  return run_planned<SG_RED_EDOT | BF>(pl, H, in, ldIn, nullptr, 0, nullptr, 0, 0, 0, as_stream(stream), ed);
}

extern "C" int roc_sg_edge_dot_planned(const roc_sg_plan* plc, int H, const float* outGrad, int64_t ldG,
                                       const float* in, int64_t ldIn, float* dw, int accumulate, roc_stream_t stream) {
  return edge_dot<0>(plc, H, outGrad, ldG, in, ldIn, dw, accumulate, stream);
}

extern "C" int roc_sg_edge_dot_planned_bf16(const roc_sg_plan* plc, int H, const float* outGrad, int64_t ldG,
                                            const uint16_t* in, int64_t ldIn, float* dw, int accumulate,
                                            roc_stream_t stream) {
  return edge_dot<SG_RED_BF16>(plc, H, outGrad, ldG, in, ldIn, dw, accumulate, stream);
}

extern "C" void roc_sg_transpose_destroy(roc_sg_transpose* tr) {
  if (!tr) return;
  roc_sg_plan_destroy(tr->planT);
  cudaFree(tr->rowEndT); cudaFree(tr->colT); cudaFree(tr->perm); cudaFree(tr->wT);
  delete tr;
}

extern "C" int roc_sg_transpose_create(roc_vid_t numNodes, const roc_eid_t* rowEnd, const roc_vid_t* colSrc,
                                       roc_stream_t stream, roc_sg_transpose** out) {
  if (!out || !rowEnd || numNodes == 0) return ROC_ERR_INVALID;
  if (roc_device_count() <= 0) return ROC_ERR_NO_DEVICE;
  if (numNodes >= 0xFFFFFFF0u) return ROC_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  uint64_t E64 = 0;
  ROC_CUDA(cudaMemcpyAsync(&E64, rowEnd + (numNodes - 1), sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  ROC_CUDA(cudaStreamSynchronize(st));
  if (E64 > 0x7FFFFFFFull) return ROC_ERR_UNSUPPORTED;   // cub's sort counts items in an int
  if (E64 > 0 && !colSrc) return ROC_ERR_INVALID;
  roc_sg_transpose* tr = new (std::nothrow) roc_sg_transpose();
  if (!tr) return ROC_ERR_NOMEM;
  tr->N = numNodes; tr->E = (uint32_t)E64;
  const uint32_t N = tr->N, E = tr->E;
  uint32_t* iota = nullptr; uint32_t* srcSorted = nullptr; void* tmp = nullptr;
  uint32_t maxSrc = 0;
  int rc = ROC_OK;
#define TR_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { rc = (int)e_; goto done; } } while (0)
  {
    const int T = 256;
    TR_CUDA(cudaMalloc(&tr->rowEndT, sizeof(uint64_t) * (size_t)N));
    TR_CUDA(cudaMalloc(&tr->colT, sizeof(uint32_t) * std::max<size_t>(E, 1)));
    TR_CUDA(cudaMalloc(&tr->perm, sizeof(uint32_t) * std::max<size_t>(E, 1)));
    if (E) {
      TR_CUDA(cudaMalloc(&iota, sizeof(uint32_t) * (size_t)E));
      TR_CUDA(cudaMalloc(&srcSorted, sizeof(uint32_t) * (size_t)E));
      k_iota<<<(E + T - 1) / T, T, 0, st>>>(E, iota);
      count_launch();
      size_t tb = 0;
      TR_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, colSrc, srcSorted, iota, tr->perm, (int)E, 0, 32, st));
      TR_CUDA(cudaMalloc(&tmp, tb ? tb : 16));
      TR_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb, colSrc, srcSorted, iota, tr->perm, (int)E, 0, 32, st));
      count_launch(4);
      TR_CUDA(cudaMemcpyAsync(&maxSrc, srcSorted + (E - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      TR_CUDA(cudaStreamSynchronize(st));
      if (maxSrc >= N) { rc = ROC_ERR_UNSUPPORTED; goto done; }   // a slice (global ids) or a bad id
      k_transpose_col<<<(E + T - 1) / T, T, 0, st>>>(E, N, rowEnd, tr->perm, tr->colT);
      count_launch();
    }
    k_transpose_row_end<<<(N + T - 1) / T, T, 0, st>>>(N, E, srcSorted, tr->rowEndT);
    count_launch();
    TR_CUDA(cudaGetLastError());
    rc = roc_sg_plan_create(0, N - 1, 0, tr->rowEndT, tr->colT, stream, &tr->planT);
  }
done:
#undef TR_CUDA
  cudaFree(iota); cudaFree(srcSorted); cudaFree(tmp);
  if (rc != ROC_OK) { roc_sg_transpose_destroy(tr); return rc; }
  *out = tr;
  return ROC_OK;
}

extern "C" int roc_sg_transpose_info(const roc_sg_transpose* tr, const roc_eid_t** rowEndT, const roc_vid_t** colT,
                                     const uint32_t** perm, const roc_sg_plan** planT) {
  if (!tr) return ROC_ERR_INVALID;
  if (rowEndT) *rowEndT = tr->rowEndT;
  if (colT) *colT = tr->colT;
  if (perm) *perm = tr->perm;
  if (planT) *planT = tr->planT;
  return ROC_OK;
}

extern "C" int roc_sg_weighted_backward_planned(roc_sg_transpose* tr, int H, const float* outGrad, int64_t ldG,
                                                const float* w, float* inGrad, int64_t ldIn, roc_stream_t stream) {
  clear_launches();
  if (!tr || H <= 0 || !outGrad || !w || !inGrad || ldG < H || ldIn < H) return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  int rc = grow(tr->wT, tr->wTBytes, sizeof(float) * std::max<size_t>(tr->E, 1), st);
  if (rc != ROC_OK) return rc;
  if (tr->E) {
    const uint32_t grid = (tr->E + 255) / 256;
    k_permute<<<grid, 256, 0, st>>>(tr->E, tr->perm, w, tr->wT);
    ROC_LAUNCH_CHECK();
    note_launch(ROC_SG_LAUNCH_PERMUTE, -1, 1, 1, 1, grid);
  }
  SgEdge ed;
  ed.w = tr->wT;
  return run_planned<SG_RED_WSUM>(tr->planT, H, outGrad, ldG, inGrad, ldIn, nullptr, 0, 0, 0, st, ed);
}

extern "C" int roc_sg_transpose_sum_backward(roc_sg_transpose* tr, int H, const float* outGrad, int64_t ldG,
                                             float* inGrad, int64_t ldIn, int epilogue, const roc_eid_t* rowEnd,
                                             roc_stream_t stream) {
  clear_launches();
  if (!tr || H <= 0 || !outGrad || !inGrad || ldG < H || ldIn < H || ((epilogue & ROC_SG_EPI_NORM) && !rowEnd))
    return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  // without NORM the transposed plan's own sum is the whole computation
  if (!(epilogue & ROC_SG_EPI_NORM))
    return run_planned<SG_RED_SUM>(tr->planT, H, outGrad, ldG, inGrad, ldIn, nullptr, 0, epilogue, 0, st);
  SgEdge ed;
  ed.rowEnd = rowEnd;
  return run_planned<SG_RED_TSUM>(tr->planT, H, outGrad, ldG, inGrad, ldIn, nullptr, 0, epilogue, 0, st, ed);
}

// ------------------------------------------------------------ edge dropout ---
// The sums above with edge dropout (SG_RED_DROP): each checks its arguments as its plain call does, plus the rate
// (attn_drop_args: rate 0 or no mask runs the plain call itself).
extern "C" int roc_sg_forward_dropout_planned(const roc_sg_plan* plc, int H, const float* in, int64_t ldIn, float* out,
                                              int64_t ldOut, int epilogue, const uint8_t* keep, float rate,
                                              roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  bool drop = false;
  SgEdge ed;
  if (attn_drop_args(keep, rate, &drop, &ed.dropScale) != ROC_OK) return ROC_ERR_INVALID;
  if (!drop) return roc_sg_forward_planned(plc, H, in, ldIn, out, ldOut, epilogue, stream);
  if (!pl || H <= 0 || !in || !out || ldIn < H || ldOut < H) return ROC_ERR_INVALID;
  ed.keep = keep;
  return run_planned<SG_RED_SUM | SG_RED_DROP>(pl, H, in, ldIn, out, ldOut, nullptr, 0, epilogue, 0, as_stream(stream),
                                               ed);
}

extern "C" int roc_sg_forward_teleport_dropout_planned(const roc_sg_plan* plc, int H, const float* in, int64_t ldIn,
                                                       float alpha, const float* t, int64_t ldT, float beta, float* out,
                                                       int64_t ldOut, int epilogue, const uint8_t* keep, float rate,
                                                       roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  bool drop = false;
  SgEdge ed;
  if (attn_drop_args(keep, rate, &drop, &ed.dropScale) != ROC_OK) return ROC_ERR_INVALID;
  if (!drop)
    return roc_sg_forward_teleport_planned(plc, H, in, ldIn, alpha, t, ldT, beta, out, ldOut, epilogue, stream);
  if (!pl || H <= 0 || !in || !t || !out || out == t || ldIn < H || ldT < H || ldOut < H ||
      (epilogue & ~(ROC_SG_EPI_NORM | ROC_SG_EPI_NORM_OUT)) || !std::isfinite(alpha) || !std::isfinite(beta))
    return ROC_ERR_INVALID;
  ed.t = t; ed.ldT = ldT; ed.alpha = alpha; ed.beta = beta; ed.keep = keep;
  return run_planned<SG_RED_TELE | SG_RED_DROP>(pl, H, in, ldIn, out, ldOut, nullptr, 0, epilogue, 0,
                                                as_stream(stream), ed);
}

extern "C" int roc_sg_transpose_sum_backward_dropout(roc_sg_transpose* tr, int H, const float* outGrad, int64_t ldG,
                                                     float* inGrad, int64_t ldIn, int epilogue, const roc_eid_t* rowEnd,
                                                     const uint8_t* keep, float rate, roc_stream_t stream) {
  clear_launches();
  bool drop = false;
  SgEdge ed;
  if (attn_drop_args(keep, rate, &drop, &ed.dropScale) != ROC_OK) return ROC_ERR_INVALID;
  if (!drop) return roc_sg_transpose_sum_backward(tr, H, outGrad, ldG, inGrad, ldIn, epilogue, rowEnd, stream);
  if (!tr || H <= 0 || !outGrad || !inGrad || ldG < H || ldIn < H || ((epilogue & ROC_SG_EPI_NORM) && !rowEnd))
    return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  ed.keep = keep;
  if (!(epilogue & ROC_SG_EPI_NORM))
    return run_planned<SG_RED_SUM | SG_RED_DROP>(tr->planT, H, outGrad, ldG, inGrad, ldIn, nullptr, 0, epilogue, 0, st,
                                                 ed);
  ed.rowEnd = rowEnd;
  return run_planned<SG_RED_TSUM | SG_RED_DROP>(tr->planT, H, outGrad, ldG, inGrad, ldIn, nullptr, 0, epilogue, 0, st,
                                                ed);
}

extern "C" int roc_sg_transpose_minmax_backward(roc_sg_transpose* tr, int H, const float* outGrad, int64_t ldG,
                                                const roc_vid_t* arg, int64_t ldArg, float* inGrad, int64_t ldIn,
                                                roc_stream_t stream) {
  clear_launches();
  if (!tr || H <= 0 || !outGrad || !arg || !inGrad || ldG < H || ldArg < H || ldIn < H) return ROC_ERR_INVALID;
  return run_planned<SG_RED_TMASK>(tr->planT, H, outGrad, ldG, inGrad, ldIn, arg, ldArg, 0, 0, as_stream(stream));
}

extern "C" int roc_sg_forward(roc_vid_t rowLeft, roc_vid_t rowRight, roc_eid_t colLeft, int H,
                              const roc_eid_t* rowEnd, const roc_vid_t* colSrc, const float* in,
                              float* out, roc_stream_t stream) {
  roc_sg_plan* pl = nullptr;
  int rc = roc_sg_plan_create(rowLeft, rowRight, colLeft, rowEnd, colSrc, stream, &pl);
  if (rc != ROC_OK) return rc;
  rc = roc_sg_forward_planned(pl, H, in, H, out, H, ROC_SG_EPI_NONE, stream);
  cudaError_t e = cudaStreamSynchronize(as_stream(stream));
  roc_sg_plan_destroy(pl);
  if (rc != ROC_OK) return rc;
  return (int)e;
}

extern "C" int roc_sg_backward(roc_vid_t rowLeft, roc_vid_t rowRight, roc_eid_t colLeft, int H,
                               const roc_eid_t* rowEnd, const roc_vid_t* colSrc, const float* outGrad,
                               float* inGrad, roc_stream_t stream) {
  // Forward and backward do exactly the same thing (scattergather_kernel.cu:168-169).
  return roc_sg_forward(rowLeft, rowRight, colLeft, H, rowEnd, colSrc, outGrad, inGrad, stream);
}

extern "C" int roc_sg_last_call_info(roc_sg_call_info* info) {
  if (!info) return ROC_ERR_INVALID;
  *info = t_call;
  return ROC_OK;
}

// ------------------------------------------------- dynamic attention (GATv2) ---
// roc_sg_attn_v2_*: GATv2's logit e(v<-u, k) = sum_f a[k][f] LeakyReLU(xl[u][kF+f] + xr[v][kF+f]) needs both endpoint
// rows of every edge, so every pass recomputes it from the rows.  The passes run on their own kernel, sg_v2_kernel, over
// the plan's chunks, chunk records and carry slots, and are finished by the attention stats fix-up and the sum's
// fix-ups, as ASTAT and ATTN are.  One worker is a whole warp: lane l holds columns l + 32 j, j < J = ceil(H / 32), of
// every row, scalar, so a head's F columns may start anywhere.  A per-head sum (v2_head_sums) adds the lane's columns of
// the head in column order, then runs an xor butterfly over the warp; both depend on (H, heads) only, and every lane
// ends with the same bits.  e is computed by v2_logits alone, with the products and sums rounded one by one, so the
// forward and both backward passes see the same bits for every e (and the backward passes the same d).
namespace roc {

enum { SG_V2_STAT = 0, SG_V2_SUM = 1, SG_V2_DST = 2, SG_V2_SRC = 3 };
constexpr int SG_RED_V2 = 64;                 // the `red` sg_last_call_info reports for pass P is SG_RED_V2 + P
constexpr int SG_V2_HEADS = SG_LDC2 / 2;      // the most heads (the stats carries hold m | Z of each)
constexpr uint32_t SG_V2_RB = 512;            // rows per block of da's fp64 column sums

struct V2Params {
  const uint32_t* rs;
  const uint32_t* col;
  const uint32_t* desc;
  uint32_t E, numChunks, H, heads;
  float slope;
  const float* a;                 // [F][heads]: a[k][f] at f * heads + k
  const float* g;  size_t ldG;    // gathered rows (by col id): STAT, SUM, DST xl; SRC xr; the record kernel: gy
  const float* g2; size_t ldG2;   // SRC: gy, gathered beside xr
  const float* o;  size_t ldO;    // the row's own row (by plan row): STAT, SUM, DST xr; SRC xl; the record kernel: y
  const float* o2; size_t ldO2;   // DST: gy of the row
  const float* stats; size_t ldStats;   // SUM, the record kernel: m | 1/Z per head
  float4* rec;                    // DST, SRC: {m, 1/Z, c, 0} per (id, head)
  float* out;  size_t ldOut;      // STAT: m | 1/Z (a cut row's owner: m | Z); SUM: y; DST: dxr; SRC: dxl
  float* out2; size_t ldOut2;     // DST: R
  float* carry; size_t ldC;       // H-wide partials (DST: out's at [0, H), out2's at [H, 2H))
  float* carry2;                  // STAT: [numCarries][SG_LDC2] m | Z
};

// s[k] = sum over the warp of t over the columns of head k (hj: the head of each of the lane's columns, -1 for none)
template <int J>
__device__ __forceinline__ void v2_head_sums(const float (&t)[J], const int (&hj)[J], uint32_t heads,
                                             float (&s)[SG_V2_HEADS]) {
#pragma unroll
  for (int k = 0; k < SG_V2_HEADS; k++) {
    float x = 0.f;
    if ((uint32_t)k < heads) {
#pragma unroll
      for (int j = 0; j < J; j++) x = __fadd_rn(x, hj[j] == k ? t[j] : 0.f);
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) x = __fadd_rn(x, __shfl_xor_sync(0xffffffffu, x, o));
    }
    s[k] = x;
  }
}
// s[h] without indexing a register array at run time
__device__ __forceinline__ float v2_pick(const float (&s)[SG_V2_HEADS], int h) {
  float r = s[0];
#pragma unroll
  for (int k = 1; k < SG_V2_HEADS; k++) r = h == k ? s[k] : r;
  return r;
}
// The one computation of e: z = xl + xr per column, e[k] the head sums of a * LeakyReLU(z).
template <int J>
__device__ __forceinline__ void v2_logits(const float (&xl)[J], const float (&xr)[J], const float (&a)[J],
                                          const int (&hj)[J], uint32_t heads, float slope, float (&z)[J],
                                          float (&e)[SG_V2_HEADS]) {
  float t[J];
#pragma unroll
  for (int j = 0; j < J; j++) {
    z[j] = __fadd_rn(xl[j], xr[j]);
    t[j] = __fmul_rn(a[j], leaky(z[j], slope));
  }
  v2_head_sums<J>(t, hj, heads, e);
}
// g[k] = gy_k . x_k, the backward's dot products (the record's c and each edge's gy[v] . xl[u])
template <int J>
__device__ __forceinline__ void v2_dots(const float (&gy)[J], const float (&x)[J], const int (&hj)[J], uint32_t heads,
                                        float (&g)[SG_V2_HEADS]) {
  float t[J];
#pragma unroll
  for (int j = 0; j < J; j++) t[j] = __fmul_rn(gy[j], x[j]);
  v2_head_sums<J>(t, hj, heads, g);
}
template <int J>
__device__ __forceinline__ void v2_load_row(const float* row, int lane, const bool (&vj)[J], float (&x)[J]) {
#pragma unroll
  for (int j = 0; j < J; j++) x[j] = vj[j] ? __ldg(row + lane + 32 * j) : 0.f;
}

// One warp per chunk of the plan, the schedule of sg_chunk_kernel (a row cut at chunk boundaries: its owner stores a raw
// partial, every later chunk a carry).  Per edge (row v's edge from u in the forward plan):
//   STAT  online (m, Z) of e per head;                    SUM  y[v] += p xl[u], p = exp(e - m) / Z;
//   DST   d = p (gy[v] . xl[u] - c[v]) per head, dxr[v] += d a LeakyReLU'(z), R[v] += d LeakyReLU(z);
//   SRC   (row u, gathering v) dxl[u] += p gy[v] + d a LeakyReLU'(z).
// __launch_bounds__(SG_THREADS, 1) asks for at least one resident CTA per SM, which lets ptxas use up to 255 registers
// per thread: with no minimum it held J = 3 sums and J = 5 destination passes to fewer registers and gave them a stack
// frame.  It does not fix the occupancy, which follows each instantiation's registers (about four CTAs per SM for the
// J = 1 stats pass, one for the J = 8 destination pass).
template <int J, int PASS>
__global__ void __launch_bounds__(SG_THREADS, 1)
sg_v2_kernel(const V2Params p) {
  constexpr bool SRC = PASS == SG_V2_SRC, DST = PASS == SG_V2_DST;
  constexpr int U = SRC ? (J <= 2 ? 2 : 1) : (J <= 2 ? 4 : J <= 4 ? 2 : 1);   // edges in flight
  constexpr int WPB = SG_THREADS / 32;
  constexpr uint32_t CH = SG_CH;
  const int lane = threadIdx.x % 32;
  const uint32_t w = blockIdx.x * WPB + threadIdx.x / 32;
  if (w >= p.numChunks) return;
  // the chunk record (k_chunk_desc), read field by field: held as two uint4 it took a stack frame at some J
  const uint32_t* dsc = p.desc + 8 * (size_t)w;
  const uint32_t flags = __ldg(dsc + 6);
  if (flags & 2u) return;
  const uint32_t ce = min(w * CH + CH, p.E);
  uint32_t cur = __ldg(dsc + 2), curS = __ldg(dsc + 3), curT = __ldg(dsc + 4);
  const uint32_t e0 = __ldg(dsc), ee = __ldg(dsc + 1), r1 = __ldg(dsc + 5), carrySlot = __ldg(dsc + 7);
  int kind = (flags & 1u) ? 0 : ((curT - curS > CH) ? 2 : 1);   // 0 carry-in part, 1 complete row, 2 cut row's owner
  uint32_t segEnd = (kind == 1) ? curT : min(curT, ce);

  const uint32_t heads = p.heads, F = p.H / heads;
  int hj[J];
  bool vj[J];
  float a[J];
#pragma unroll
  for (int j = 0; j < J; j++) {
    const uint32_t c = (uint32_t)(lane + 32 * j);
    vj[j] = c < p.H;
    hj[j] = vj[j] ? (int)(c / F) : -1;
    a[j] = vj[j] ? __ldg(p.a + (c % F) * heads + c / F) : 0.f;
  }
  float xo[J], yo[DST ? J : 1];                 // the row's own row (and DST: its gy)
  float sm[SG_V2_HEADS], sz[SG_V2_HEADS], sc[SG_V2_HEADS];   // STAT: running m, Z; SUM, DST: m, 1/Z (DST: c)
  float acc[J], acc2[DST ? J : 1];
#pragma unroll
  for (int k = 0; k < SG_V2_HEADS; k++) { sm[k] = PASS == SG_V2_STAT ? -INFINITY : 0.f; sz[k] = 0.f; sc[k] = 0.f; }
#pragma unroll
  for (int j = 0; j < J; j++) { acc[j] = 0.f; if constexpr (DST) acc2[j] = 0.f; }

  auto row_state = [&]() {
    v2_load_row<J>(p.o + (uint64_t)cur * p.ldO, lane, vj, xo);
    if constexpr (DST) v2_load_row<J>(p.o2 + (uint64_t)cur * p.ldO2, lane, vj, yo);
    if constexpr (PASS == SG_V2_SUM) {
#pragma unroll
      for (int k = 0; k < SG_V2_HEADS; k++)
        if ((uint32_t)k < heads) {
          sm[k] = __ldg(p.stats + (uint64_t)cur * p.ldStats + k);
          sz[k] = __ldg(p.stats + (uint64_t)cur * p.ldStats + heads + k);
        }
    }
    if constexpr (DST) {
#pragma unroll
      for (int k = 0; k < SG_V2_HEADS; k++)
        if ((uint32_t)k < heads) {
          const float4 r = __ldg(p.rec + (uint64_t)cur * heads + k);
          sm[k] = r.x; sz[k] = r.y; sc[k] = r.z;
        }
    }
  };
  row_state();

  auto flush = [&]() {
    if constexpr (PASS == SG_V2_STAT) {
      // as ASTAT's store: a complete row stores m and 1/Z (0 and 0 with no edge), a cut row's parts their raw (m, Z)
      float* sdst = (kind == 0) ? p.carry2 + (uint64_t)carrySlot * SG_LDC2 : p.out + (uint64_t)cur * p.ldOut;
      if ((uint32_t)lane < heads) {
        const float m = v2_pick(sm, lane), z = v2_pick(sz, lane);
        const bool done = kind == 1;
        sdst[lane] = (done && !(z > 0.f)) ? 0.f : m;
        sdst[heads + lane] = !done ? z : (z > 0.f ? 1.f / z : 0.f);
      }
#pragma unroll
      for (int k = 0; k < SG_V2_HEADS; k++) { sm[k] = -INFINITY; sz[k] = 0.f; }
    } else {
      float* d1 = (kind == 0) ? p.carry + (uint64_t)carrySlot * p.ldC : p.out + (uint64_t)cur * p.ldOut;
      float* d2 = (kind == 0) ? d1 + p.H : p.out2 + (uint64_t)cur * p.ldOut2;
      (void)d2;
#pragma unroll
      for (int j = 0; j < J; j++) {
        if (vj[j]) {
          d1[lane + 32 * j] = acc[j];
          if constexpr (DST) d2[lane + 32 * j] = acc2[j];
        }
        acc[j] = 0.f;
        if constexpr (DST) acc2[j] = 0.f;
      }
    }
  };
  auto advance = [&]() {
    cur += 1; curS = curT; curT = p.rs[cur + 1];
    const bool heavy = curT - curS > CH;
    segEnd = heavy ? min(curT, ce) : curT;
    kind = heavy ? 2 : 1;
    row_state();
  };

  const uint32_t eLast = ee - 1u;
#pragma unroll 1
  for (uint32_t base = e0; base < ee; base += U) {
    const uint32_t cnt = min((uint32_t)U, ee - base);
    uint32_t srcs[U];
#pragma unroll
    for (int u = 0; u < U; u++) srcs[u] = __ldg(p.col + min(base + (uint32_t)u, eLast));
    float gv[U][J], gv2[SRC ? U : 1][SRC ? J : 1];
    float4 gr[SRC ? U : 1];
#pragma unroll
    for (int u = 0; u < U; u++) {
      v2_load_row<J>(p.g + (uint64_t)srcs[u] * p.ldG, lane, vj, gv[u]);
      if constexpr (SRC) {
        v2_load_row<J>(p.g2 + (uint64_t)srcs[u] * p.ldG2, lane, vj, gv2[u]);
        gr[u] = __ldg(p.rec + (uint64_t)srcs[u] * heads + min((uint32_t)lane, heads - 1u));
      }
    }
    uint32_t pos = 0;
    for (;;) {
      const uint32_t lim = min(cnt, segEnd - base);
#pragma unroll
      for (int u = 0; u < U; u++) {
        if ((uint32_t)u >= pos && (uint32_t)u < lim) {
          float z[J], e[SG_V2_HEADS];
          if constexpr (SRC) v2_logits<J>(xo, gv[u], a, hj, heads, p.slope, z, e);
          else v2_logits<J>(gv[u], xo, a, hj, heads, p.slope, z, e);
          if constexpr (PASS == SG_V2_STAT) {
#pragma unroll
            for (int k = 0; k < SG_V2_HEADS; k++)
              if ((uint32_t)k < heads) {
                if (e[k] > sm[k]) { sz[k] = sz[k] * expf(sm[k] - e[k]) + 1.f; sm[k] = e[k]; }
                else sz[k] += expf(e[k] - sm[k]);
              }
          } else if constexpr (PASS == SG_V2_SUM) {
            float pk[SG_V2_HEADS];
#pragma unroll
            for (int k = 0; k < SG_V2_HEADS; k++) pk[k] = attn_alpha(e[k], sm[k], sz[k]);
#pragma unroll
            for (int j = 0; j < J; j++) acc[j] = fmaf(v2_pick(pk, hj[j]), gv[u][j], acc[j]);
          } else {
            // DST: v's own m, 1/Z, c and gy; SRC: those of the gathered v, its record's heads spread over the lanes
            float m[SG_V2_HEADS], iz[SG_V2_HEADS], c[SG_V2_HEADS], g[SG_V2_HEADS];
            if constexpr (SRC) {
#pragma unroll
              for (int k = 0; k < SG_V2_HEADS; k++) {
                m[k] = __shfl_sync(0xffffffffu, gr[u].x, k);
                iz[k] = __shfl_sync(0xffffffffu, gr[u].y, k);
                c[k] = __shfl_sync(0xffffffffu, gr[u].z, k);
              }
              v2_dots<J>(gv2[u], xo, hj, heads, g);
            } else {
#pragma unroll
              for (int k = 0; k < SG_V2_HEADS; k++) { m[k] = sm[k]; iz[k] = sz[k]; c[k] = sc[k]; }
              v2_dots<J>(yo, gv[u], hj, heads, g);
            }
            float pk[SG_V2_HEADS], dk[SG_V2_HEADS];
#pragma unroll
            for (int k = 0; k < SG_V2_HEADS; k++) {
              pk[k] = attn_alpha(e[k], m[k], iz[k]);
              dk[k] = __fmul_rn(pk[k], __fsub_rn(g[k], c[k]));
            }
#pragma unroll
            for (int j = 0; j < J; j++) {
              const float d = v2_pick(dk, hj[j]);
              const float da = __fmul_rn(a[j], z[j] > 0.f ? 1.f : p.slope);
              if constexpr (SRC) {
                acc[j] = fmaf(v2_pick(pk, hj[j]), gv2[u][j], acc[j]);
                acc[j] = fmaf(d, da, acc[j]);
              } else {
                acc[j] = fmaf(d, da, acc[j]);
                acc2[j] = fmaf(d, leaky(z[j], p.slope), acc2[j]);
              }
            }
          }
        }
      }
      pos = lim;
      if (pos >= cnt) break;
      flush();
      advance();
    }
  }
  flush();
  while (cur + 1 < r1) { advance(); flush(); }   // trailing zero-degree rows
}

// The backward's record {m, 1/Z, c, 0} of nodes [0, n), c[k] = gy[v]_k . y[v]_k: one warp per node (g = gy, o = y).
template <int J>
__global__ void __launch_bounds__(SG_THREADS)
sg_v2_rec_kernel(const V2Params p, uint32_t n) {
  const int lane = threadIdx.x % 32;
  const uint32_t v = blockIdx.x * (SG_THREADS / 32) + threadIdx.x / 32;
  if (v >= n) return;
  const uint32_t F = p.H / p.heads;
  int hj[J];
  bool vj[J];
#pragma unroll
  for (int j = 0; j < J; j++) {
    const uint32_t c = (uint32_t)(lane + 32 * j);
    vj[j] = c < p.H;
    hj[j] = vj[j] ? (int)(c / F) : -1;
  }
  float gy[J], y[J], c[SG_V2_HEADS];
  v2_load_row<J>(p.g + (uint64_t)v * p.ldG, lane, vj, gy);
  v2_load_row<J>(p.o + (uint64_t)v * p.ldO, lane, vj, y);
  v2_dots<J>(gy, y, hj, p.heads, c);
  if ((uint32_t)lane < p.heads)
    p.rec[(uint64_t)v * p.heads + lane] = make_float4(p.stats[(uint64_t)v * p.ldStats + lane],
                                                      p.stats[(uint64_t)v * p.ldStats + p.heads + lane], v2_pick(c, lane), 0.f);
}

// da, the column sums of R [n][H] (ld ldR), in the layout of a: fp64 sums over blocks of SG_V2_RB rows, one thread per
// column, then the blocks' sums added in block order.  The blocks depend on (n, H) only.
__global__ void __launch_bounds__(SG_THREADS)
sg_v2_colsum_part(uint32_t n, uint32_t H, const float* __restrict__ R, size_t ldR, double* __restrict__ part) {
  const uint32_t c = threadIdx.x, r0 = blockIdx.x * SG_V2_RB, r1 = min(n, r0 + SG_V2_RB);
  if (c >= H) return;
  double s = 0.0;
  for (uint32_t r = r0; r < r1; r++) s += (double)__ldg(R + (uint64_t)r * ldR + c);
  part[(uint64_t)blockIdx.x * H + c] = s;
}
__global__ void __launch_bounds__(SG_THREADS)
sg_v2_colsum_final(uint32_t nb, uint32_t H, uint32_t heads, const double* __restrict__ part, float* __restrict__ da) {
  const uint32_t c = threadIdx.x;
  if (c >= H) return;
  double s = 0.0;
  for (uint32_t b = 0; b < nb; b++) s += part[(uint64_t)b * H + c];
  const uint32_t F = H / heads;
  da[(c % F) * heads + c / F] = (float)s;
}

// J = ceil(H / 32) as a std::integral_constant
template <class Fn>
static int v2_with_j(uint32_t H, Fn&& f) {
  switch ((H + 31) / 32) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 3: return f(std::integral_constant<int, 3>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 5: return f(std::integral_constant<int, 5>{});
    case 6: return f(std::integral_constant<int, 6>{});
    case 7: return f(std::integral_constant<int, 7>{});
    case 8: return f(std::integral_constant<int, 8>{});
    default: return ROC_ERR_UNSUPPORTED;
  }
}

static V2Params v2_params(const roc_sg_plan* pl, int heads, int H, float slope, const float* a) {
  V2Params p;
  memset(&p, 0, sizeof(p));
  p.rs = pl->rs; p.col = pl->col; p.desc = pl->desc; p.E = pl->E; p.numChunks = pl->numChunks;
  p.H = (uint32_t)H; p.heads = (uint32_t)heads; p.slope = slope; p.a = a;
  p.carry = pl->carry; p.ldC = pl->carryLd; p.carry2 = pl->carry2;
  return p;
}

// The sum's fix-ups of the H-wide partials `carryOff` floats into pl's carry slots, into out.
static int v2_fixups(const roc_sg_plan* pl, int H, float* out, int64_t ldOut, size_t carryOff, cudaStream_t st) {
  SgParams sp = plan_params(pl);
  sp.out = out; sp.ldOut = (size_t)ldOut; sp.carry = pl->carry + carryOff; sp.ldC = pl->carryLd; sp.Q = (uint32_t)H;
  return with_shape<256>((uint32_t)H, [&](auto L, auto NCH) { return launch_fixups<1, L, NCH, SG_RED_SUM>(sp, st); });
}

// One pass of sg_v2_kernel over pl, then its fix-ups: the stats fix-up (STAT), or the sum's over out (and DST: out2).
template <int PASS>
static int v2_pass(const roc_sg_plan* pl, const V2Params& p, cudaStream_t st) {
  int rc = v2_with_j(p.H, [&](auto J) {
    if (p.numChunks) {
      constexpr int WPB = SG_THREADS / 32;
      const uint32_t grid = (p.numChunks + WPB - 1) / WPB;
      sg_v2_kernel<J, PASS><<<grid, SG_THREADS, 0, st>>>(p);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_MAIN, SG_RED_V2 + PASS, 1, 32, J, grid);
    }
    return ROC_OK;
  });
  if (rc != ROC_OK) return rc;
  if constexpr (PASS == SG_V2_STAT) {
    const uint32_t rows = pl->numHeavy + pl->numBig;
    if (rows) {
      SgParams sp = plan_params(pl);
      sp.carry2 = pl->carry2; sp.out = p.out; sp.ldOut = p.ldOut; sp.heads = p.heads;
      const uint32_t grid = (rows + SG_THREADS / 32 - 1) / (SG_THREADS / 32);
      sg_attn_stat_fixup<<<grid, SG_THREADS, 0, st>>>(sp);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_STAT_FIXUP, SG_RED_V2 + PASS, 1, 32, 1, grid);
    }
    return ROC_OK;
  } else {
    rc = v2_fixups(pl, (int)p.H, p.out, (int64_t)p.ldOut, 0, st);
    if (rc == ROC_OK && PASS == SG_V2_DST) rc = v2_fixups(pl, (int)p.H, p.out2, (int64_t)p.ldOut2, p.H, st);
    return rc;
  }
}

// The checks every dynamic attention call shares once its pointers and leading dimensions are checked: a bad slope is
// ROC_ERR_INVALID; H % heads, H > 256, heads > SG_V2_HEADS and a plan whose ids are not all its own rows (a graph slice)
// are ROC_ERR_UNSUPPORTED.  Then the carries: `cols` floats per slot, and the stats slots.
static int v2_setup(roc_sg_plan* pl, int heads, int H, float slope, int cols, cudaStream_t st) {
  if (!(slope >= 0.f) || !std::isfinite(slope)) return ROC_ERR_INVALID;
  if (H > 256 || H % heads || heads > SG_V2_HEADS) return ROC_ERR_UNSUPPORTED;
  int rc = find_id_end(pl, st);
  if (rc != ROC_OK) return rc;
  if (pl->idEnd > pl->nloc) return ROC_ERR_UNSUPPORTED;
  rc = grow_carries(pl, cols, st);
  if (rc == ROC_OK) rc = grow(pl->carry2, pl->carry2Bytes, (size_t)pl->numCarries * SG_LDC2 * sizeof(float), st);
  return rc;
}

// da from R [n][H]: the blocks' fp64 column sums, then their sum in block order (da = 0 with no rows).
static int v2_colsum(uint32_t n, uint32_t nb, int H, int heads, const float* R, double* part, float* da,
                     cudaStream_t st) {
  if (!nb) {
    ROC_CUDA(cudaMemsetAsync(da, 0, (size_t)H * sizeof(float), st));
    return ROC_OK;
  }
  sg_v2_colsum_part<<<nb, SG_THREADS, 0, st>>>(n, (uint32_t)H, R, (size_t)H, part);
  ROC_LAUNCH_CHECK();
  note_launch(ROC_SG_LAUNCH_COLSUM, -1, 1, SG_THREADS, 1, nb);
  sg_v2_colsum_final<<<1, SG_THREADS, 0, st>>>(nb, (uint32_t)H, (uint32_t)heads, part, da);
  ROC_LAUNCH_CHECK();
  note_launch(ROC_SG_LAUNCH_COLSUM, -1, 1, SG_THREADS, 1, 1);
  return ROC_OK;
}

// The backward once its arguments are checked: the records over pl's rows, the destination pass over pl, the source
// pass over plB (pl itself, or the transposed plan), and da from R, a workspace of this call.
static int v2_backward(roc_sg_plan* pl, roc_sg_plan* plB, int heads, int H, float slope, const float* xl, int64_t ldXl,
                       const float* xr, int64_t ldXr, const float* a, const float* out, int64_t ldOut,
                       const float* stats, int64_t ldStats, const float* outGrad, int64_t ldG, float* dxl,
                       int64_t ldDxl, float* dxr, int64_t ldDxr, float* da, cudaStream_t st) {
  int rc = v2_setup(pl, heads, H, slope, 2 * H, st);
  if (rc == ROC_OK && plB != pl) rc = v2_setup(plB, heads, H, slope, H, st);
  if (rc != ROC_OK) return rc;
  const uint32_t n = pl->nloc;
  if ((rc = grow(pl->attnRec, pl->attnRecBytes, (size_t)n * heads * sizeof(float4), st)) != ROC_OK) return rc;
  const uint32_t nb = (n + SG_V2_RB - 1) / SG_V2_RB;
  const size_t rBytes = ((size_t)n * H * sizeof(float) + 15) / 16 * 16;
  char* ws = nullptr;
  ROC_CUDA(cudaMallocAsync((void**)&ws, rBytes + (size_t)std::max(nb, 1u) * H * sizeof(double), st));
  float* R = reinterpret_cast<float*>(ws);
  double* part = reinterpret_cast<double*>(ws + rBytes);
  // the records {m, 1/Z, c}
  V2Params r = v2_params(pl, heads, H, slope, a);
  r.g = outGrad; r.ldG = (size_t)ldG; r.o = out; r.ldO = (size_t)ldOut; r.stats = stats; r.ldStats = (size_t)ldStats;
  r.rec = pl->attnRec;
  rc = v2_with_j((uint32_t)H, [&](auto J) {
    if (n) {
      const uint32_t grid = (n + SG_THREADS / 32 - 1) / (SG_THREADS / 32);
      sg_v2_rec_kernel<J><<<grid, SG_THREADS, 0, st>>>(r, n);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_RECORD, -1, 1, 32, J, grid);
    }
    return ROC_OK;
  });
  // destination pass: dxr and R
  if (rc == ROC_OK) {
    V2Params d = v2_params(pl, heads, H, slope, a);
    d.g = xl; d.ldG = (size_t)ldXl; d.o = xr; d.ldO = (size_t)ldXr; d.o2 = outGrad; d.ldO2 = (size_t)ldG;
    d.rec = pl->attnRec; d.out = dxr; d.ldOut = (size_t)ldDxr; d.out2 = R; d.ldOut2 = (size_t)H;
    rc = v2_pass<SG_V2_DST>(pl, d, st);
  }
  // source pass: dxl
  if (rc == ROC_OK) {
    V2Params s = v2_params(plB, heads, H, slope, a);
    s.g = xr; s.ldG = (size_t)ldXr; s.g2 = outGrad; s.ldG2 = (size_t)ldG; s.o = xl; s.ldO = (size_t)ldXl;
    s.rec = pl->attnRec; s.out = dxl; s.ldOut = (size_t)ldDxl;
    rc = v2_pass<SG_V2_SRC>(plB, s, st);
  }
  if (rc == ROC_OK) rc = v2_colsum(n, nb, H, heads, R, part, da, st);
  // every path after the allocation ends here, so the workspace is always returned
  const cudaError_t e = cudaFreeAsync(ws, st);
  if (rc == ROC_OK && e != cudaSuccess) rc = (int)e;
  return rc;
}

}  // namespace roc

extern "C" int roc_sg_attn_v2_forward_planned(const roc_sg_plan* plc, int heads, int H, float slope, const float* xl,
                                              int64_t ldXl, const float* xr, int64_t ldXr, const float* a, float* out,
                                              int64_t ldOut, float* stats, int64_t ldStats, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || !xl || !xr || !a || !out || !stats || heads <= 0 || H <= 0 || ldXl < H || ldXr < H || ldOut < H ||
      ldStats < 2 * (int64_t)heads)
    return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  int rc = v2_setup(pl, heads, H, slope, H, st);
  if (rc != ROC_OK) return rc;
  // pass 1: m and 1/Z per row and head
  V2Params s = v2_params(pl, heads, H, slope, a);
  s.g = xl; s.ldG = (size_t)ldXl; s.o = xr; s.ldO = (size_t)ldXr; s.out = stats; s.ldOut = (size_t)ldStats;
  if ((rc = v2_pass<SG_V2_STAT>(pl, s, st)) != ROC_OK) return rc;
  // pass 2: the p-weighted sum of the xl rows
  V2Params b = v2_params(pl, heads, H, slope, a);
  b.g = xl; b.ldG = (size_t)ldXl; b.o = xr; b.ldO = (size_t)ldXr; b.stats = stats; b.ldStats = (size_t)ldStats;
  b.out = out; b.ldOut = (size_t)ldOut;
  return v2_pass<SG_V2_SUM>(pl, b, st);
}

extern "C" int roc_sg_attn_v2_backward_planned(const roc_sg_plan* plc, int heads, int H, float slope, const float* xl,
                                               int64_t ldXl, const float* xr, int64_t ldXr, const float* a,
                                               const float* out, int64_t ldOut, const float* stats, int64_t ldStats,
                                               const float* outGrad, int64_t ldG, float* dxl, int64_t ldDxl,
                                               float* dxr, int64_t ldDxr, float* da, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || !xl || !xr || !a || !out || !stats || !outGrad || !dxl || !dxr || !da || dxl == dxr || heads <= 0 ||
      H <= 0 || ldXl < H || ldXr < H || ldOut < H || ldG < H || ldDxl < H || ldDxr < H || ldStats < 2 * (int64_t)heads)
    return ROC_ERR_INVALID;
  return v2_backward(pl, pl, heads, H, slope, xl, ldXl, xr, ldXr, a, out, ldOut, stats, ldStats, outGrad, ldG, dxl,
                     ldDxl, dxr, ldDxr, da, as_stream(stream));
}

extern "C" int roc_sg_attn_v2_backward_exact(const roc_sg_plan* plc, roc_sg_transpose* tr, int heads, int H,
                                             float slope, const float* xl, int64_t ldXl, const float* xr, int64_t ldXr,
                                             const float* a, const float* out, int64_t ldOut, const float* stats,
                                             int64_t ldStats, const float* outGrad, int64_t ldG, float* dxl,
                                             int64_t ldDxl, float* dxr, int64_t ldDxr, float* da, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || !tr || !xl || !xr || !a || !out || !stats || !outGrad || !dxl || !dxr || !da || dxl == dxr ||
      heads <= 0 || H <= 0 || ldXl < H || ldXr < H || ldOut < H || ldG < H || ldDxl < H || ldDxr < H ||
      ldStats < 2 * (int64_t)heads || pl->nloc != tr->N || pl->E != tr->E)
    return ROC_ERR_INVALID;
  return v2_backward(pl, tr->planT, heads, H, slope, xl, ldXl, xr, ldXr, a, out, ldOut, stats, ldStats, outGrad, ldG,
                     dxl, ldDxl, dxr, ldDxr, da, as_stream(stream));
}

// ------------------------------------------------------ softmax aggregation ---
// roc_sg_softmax_*: PyG's SoftmaxAggregation with one temperature t.  Per destination v and column f over v's in-edges
// u: z = t x[u][f], p = softmax_u(z), y[v][f] = sum_u p x[u][f].  Every column is its own softmax, so a lane owns its
// columns outright: one warp per chunk of the plan, lane l holding columns l + 32 j (j < J = ceil(Hb / 32)) of a column
// block of Hb <= 256 columns, scalar, as sg_v2_kernel.  The forward is one pass with an online softmax per column,
// (m, s, w) = (max z, sum exp(z - m), sum exp(z - m) x); a cut row's parts are merged by sg_smx_fixup in chunk order.
// The backward is a record pass per destination and a source pass per row, whose cut rows are plain sums finished by
// the sum's fix-ups; dt is the fp64 sum of the source pass's R.  t is read from device memory (a learned t is updated
// there by Adam).  expf throughout, never exp(t x) exp(-m): each factor can overflow where the product cannot.
namespace roc {

enum { SG_SMX_FWD = 0, SG_SMX_SRC = 1, SG_SMX_SRC_DT = 2 };
constexpr int SG_RED_SMX = 72;                // the `red` sg_last_call_info reports for pass P is SG_RED_SMX + P
constexpr int SG_SMX_COLS = 256;              // columns per block (J <= 8)
constexpr uint32_t SG_SMX_RB = 512;           // rows per block of dt's fp64 sums

struct SmxParams {
  const uint32_t* rs;
  const uint32_t* col;
  const uint32_t* desc;
  const uint32_t* carryIdx;
  const uint32_t* heavyRows;
  const uint32_t* bigRows;
  uint32_t E, numChunks, numHeavy, numBig, H;   // H: the block's columns
  const float* t;
  const float* g;  size_t ldG;    // gathered rows: FWD x; SRC the records {m | r | y} (3H floats per id)
  const float* o;  size_t ldO;    // SRC: x of the row itself
  float* out;  size_t ldOut;      // FWD: y; SRC: dx
  float* m;    float* z; size_t ldMZ;   // FWD: m and 1/Z of a complete row (when `stats`); a cut row's owner: raw m, s
  float* out2; size_t ldOut2;     // SRC_DT: R
  float* carry; size_t ldC;       // FWD: [m | s | w]; SRC: [dx | R]
  int stats;                      // FWD: complete rows store m and 1/Z
};

// Two (m, s, w) partials of one column merged, the first one earlier in chunk order.  s = 0: no edge (w = 0), which
// leaves the other partial as it is.  Selects rather than branches, so that the unrolled merges of a row stay in
// registers.
__device__ __forceinline__ void smx_merge(float& m, float& s, float& w, float m2, float s2, float w2) {
  const bool h1 = s > 0.f, h2 = s2 > 0.f;
  const float M = h2 ? (h1 ? fmaxf(m, m2) : m2) : m;
  const float a = h1 ? expf(m - M) : 0.f, b = h2 ? expf(m2 - M) : 0.f;
  s = fmaf(s, a, __fmul_rn(s2, b));
  w = fmaf(w, a, __fmul_rn(w2, b));
  m = M;
}

// A finished column: y = w / s, m and 1/Z (0, 0 and 0 for a row with no edge).
__device__ __forceinline__ void smx_store(float m, float s, float w, float* y, float* mo, float* zo, bool stats) {
  const bool any = s > 0.f;
  *y = any ? __fdiv_rn(w, s) : 0.f;
  if (stats) { *mo = any ? m : 0.f; *zo = any ? __frcp_rn(s) : 0.f; }
}

// One warp per chunk of the plan, the schedule of sg_v2_kernel.  Per edge (row v's edge from u):
//   FWD  online (m, s, w) of z = t x[u] per column;
//   SRC  (row u, gathering v's record {m, r = gy / Z, y}) e = exp(t x[u] - m), q = r e, d = x[u] - y[v]:
//        dx[u] += q (1 + t d); SRC_DT also R[u] += q d d.
template <int J, int PASS>
__global__ void __launch_bounds__(SG_THREADS, 2)
sg_smx_kernel(const SmxParams p) {
  constexpr bool SRC = PASS != SG_SMX_FWD, DT = PASS == SG_SMX_SRC_DT;
  constexpr int U = SRC ? (J <= 2 ? 4 : J <= 4 ? 2 : 1) : (J <= 2 ? 8 : J <= 4 ? 4 : 2);   // edges in flight
  constexpr int NG = SRC ? 3 : 1;                 // floats gathered per column and edge
  constexpr int WPB = SG_THREADS / 32;
  constexpr uint32_t CH = SG_CH;
  const int lane = threadIdx.x % 32;
  const uint32_t w = blockIdx.x * WPB + threadIdx.x / 32;
  if (w >= p.numChunks) return;
  const uint32_t* dsc = p.desc + 8 * (size_t)w;
  const uint32_t flags = __ldg(dsc + 6);
  if (flags & 2u) return;
  const uint32_t ce = min(w * CH + CH, p.E);
  uint32_t cur = __ldg(dsc + 2), curS = __ldg(dsc + 3), curT = __ldg(dsc + 4);
  const uint32_t e0 = __ldg(dsc), ee = __ldg(dsc + 1), r1 = __ldg(dsc + 5), carrySlot = __ldg(dsc + 7);
  int kind = (flags & 1u) ? 0 : ((curT - curS > CH) ? 2 : 1);   // 0 carry-in part, 1 complete row, 2 cut row's owner
  uint32_t segEnd = (kind == 1) ? curT : min(curT, ce);

  const float t = __ldg(p.t);
  const uint32_t H = p.H;
  bool vj[J];
#pragma unroll
  for (int j = 0; j < J; j++) vj[j] = (uint32_t)(lane + 32 * j) < H;
  float xo[SRC ? J : 1], zo[SRC ? J : 1];         // SRC: the row's own x and t x
  float sm[SRC ? 1 : J], ss[SRC ? 1 : J];         // FWD: running m, s (acc: w)
  float acc[J], acc2[DT ? J : 1];
#pragma unroll
  for (int j = 0; j < J; j++) {
    acc[j] = 0.f;
    if constexpr (DT) acc2[j] = 0.f;
    if constexpr (!SRC) { sm[j] = -INFINITY; ss[j] = 0.f; }
  }
  auto row_state = [&]() {
    if constexpr (SRC) {
#pragma unroll
      for (int j = 0; j < J; j++) {
        xo[j] = vj[j] ? __ldg(p.o + (uint64_t)cur * p.ldO + lane + 32 * j) : 0.f;
        zo[j] = __fmul_rn(t, xo[j]);
      }
    }
  };
  row_state();

  auto flush = [&]() {
    if constexpr (!SRC) {
      if (kind == 0) {
        float* c = p.carry + (uint64_t)carrySlot * p.ldC;
#pragma unroll
        for (int j = 0; j < J; j++)
          if (vj[j]) { c[lane + 32 * j] = sm[j]; c[H + lane + 32 * j] = ss[j]; c[2 * H + lane + 32 * j] = acc[j]; }
      } else {
        float* y = p.out + (uint64_t)cur * p.ldOut;
        float* mo = p.m + (uint64_t)cur * p.ldMZ;
        float* zr = p.z + (uint64_t)cur * p.ldMZ;
#pragma unroll
        for (int j = 0; j < J; j++) {
          if (!vj[j]) continue;
          const int c = lane + 32 * j;
          if (kind == 2) { y[c] = acc[j]; mo[c] = sm[j]; zr[c] = ss[j]; }   // the raw partial, for sg_smx_fixup
          else smx_store(sm[j], ss[j], acc[j], y + c, mo + c, zr + c, p.stats != 0);
        }
      }
#pragma unroll
      for (int j = 0; j < J; j++) { sm[j] = -INFINITY; ss[j] = 0.f; acc[j] = 0.f; }
    } else {
      float* d1 = (kind == 0) ? p.carry + (uint64_t)carrySlot * p.ldC : p.out + (uint64_t)cur * p.ldOut;
      float* d2 = (kind == 0) ? d1 + H : p.out2 + (uint64_t)cur * p.ldOut2;
      (void)d2;
#pragma unroll
      for (int j = 0; j < J; j++) {
        if (vj[j]) {
          d1[lane + 32 * j] = acc[j];
          if constexpr (DT) d2[lane + 32 * j] = acc2[j];
        }
        acc[j] = 0.f;
        if constexpr (DT) acc2[j] = 0.f;
      }
    }
  };
  auto advance = [&]() {
    cur += 1; curS = curT; curT = p.rs[cur + 1];
    const bool heavy = curT - curS > CH;
    segEnd = heavy ? min(curT, ce) : curT;
    kind = heavy ? 2 : 1;
    row_state();
  };

  const uint32_t eLast = ee - 1u;
#pragma unroll 1
  for (uint32_t base = e0; base < ee; base += U) {
    const uint32_t cnt = min((uint32_t)U, ee - base);
    float gv[U][NG][J];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const float* row = p.g + (uint64_t)__ldg(p.col + min(base + (uint32_t)u, eLast)) * p.ldG;
#pragma unroll
      for (int k = 0; k < NG; k++)
#pragma unroll
        for (int j = 0; j < J; j++) gv[u][k][j] = vj[j] ? __ldg(row + k * H + lane + 32 * j) : 0.f;
    }
    uint32_t pos = 0;
    for (;;) {
      const uint32_t lim = min(cnt, segEnd - base);
#pragma unroll
      for (int u = 0; u < U; u++) {
        if ((uint32_t)u >= pos && (uint32_t)u < lim) {
#pragma unroll
          for (int j = 0; j < J; j++) {
            if constexpr (!SRC) {
              const float x = gv[u][0][j], z = __fmul_rn(t, x);
              if (z > sm[j]) {
                const float c = expf(sm[j] - z);
                ss[j] = fmaf(ss[j], c, 1.f); acc[j] = fmaf(acc[j], c, x); sm[j] = z;
              } else {
                const float e = expf(z - sm[j]);
                ss[j] = __fadd_rn(ss[j], e); acc[j] = fmaf(e, x, acc[j]);
              }
            } else {
              const float q = __fmul_rn(gv[u][1][j], expf(__fsub_rn(zo[j], gv[u][0][j])));
              const float d = __fsub_rn(xo[j], gv[u][2][j]);
              acc[j] = fmaf(q, fmaf(t, d, 1.f), acc[j]);
              if constexpr (DT) acc2[j] = fmaf(__fmul_rn(q, d), d, acc2[j]);
            }
          }
        }
      }
      pos = lim;
      if (pos >= cnt) break;
      flush();
      advance();
    }
  }
  flush();
  while (cur + 1 < r1) { advance(); flush(); }   // trailing zero-degree rows
}

// Finishes the forward's cut rows: the owner's raw partial (y: w, m, z: s), then the carries in chunk order, stored as
// y, m and 1/Z.  Heavy rows (at most 32 carries): one warp each.  BIG rows: one CTA each, whose warps merge contiguous
// blocks of the carries, then warp 0 the owner's partial and the blocks' in block order.  The grouping depends on the
// plan only, so the result is reproducible.
template <int J, bool BIG>
__global__ void __launch_bounds__(SG_THREADS)
sg_smx_fixup(const SmxParams p) {
  constexpr uint32_t CH = SG_CH;
  constexpr int WPB = SG_THREADS / 32;
  const int lane = threadIdx.x % 32, g = threadIdx.x / 32;
  const uint32_t w = BIG ? blockIdx.x : blockIdx.x * WPB + g;
  if (w >= (BIG ? p.numBig : p.numHeavy)) return;
  const uint32_t R = BIG ? p.bigRows[w] : p.heavyRows[w];
  const uint32_t s = p.rs[R], t = p.rs[R + 1];
  const uint32_t c0 = s / CH, n = (t - 1) / CH - c0;
  const float* cb = p.carry + (uint64_t)p.carryIdx[c0 + 1] * p.ldC;
  const uint32_t H = p.H;
  uint32_t k0 = 0, k1 = n;
  if constexpr (BIG) { const uint32_t per = (n + WPB - 1) / WPB; k0 = min(n, g * per); k1 = min(n, k0 + per); }
  float m[J], z[J], a[J];
#pragma unroll
  for (int j = 0; j < J; j++) { m[j] = -INFINITY; z[j] = 0.f; a[j] = 0.f; }
  if (!BIG) {   // a heavy row starts from its owner's partial
#pragma unroll
    for (int j = 0; j < J; j++) {
      const uint32_t c = lane + 32 * j;
      if (c < H) { m[j] = p.m[(uint64_t)R * p.ldMZ + c]; z[j] = p.z[(uint64_t)R * p.ldMZ + c]; a[j] = p.out[(uint64_t)R * p.ldOut + c]; }
    }
  }
  for (uint32_t k = k0; k < k1; k++) {
    const float* ck = cb + (uint64_t)k * p.ldC;
#pragma unroll
    for (int j = 0; j < J; j++) {
      const uint32_t c = lane + 32 * j;
      if (c < H) smx_merge(m[j], z[j], a[j], ck[c], ck[H + c], ck[2 * H + c]);
    }
  }
  float* y = p.out + (uint64_t)R * p.ldOut;
  float* mo = p.m + (uint64_t)R * p.ldMZ;
  float* zo = p.z + (uint64_t)R * p.ldMZ;
  if constexpr (BIG) {
    __shared__ float part[WPB][3][32 * J];
#pragma unroll
    for (int j = 0; j < J; j++) { part[g][0][lane + 32 * j] = m[j]; part[g][1][lane + 32 * j] = z[j]; part[g][2][lane + 32 * j] = a[j]; }
    __syncthreads();
    if (g != 0) return;
#pragma unroll
    for (int j = 0; j < J; j++) {
      const uint32_t c = lane + 32 * j;
      if (c >= H) continue;
      float mm = mo[c], zz = zo[c], aa = y[c];
      for (int gg = 0; gg < WPB; gg++) smx_merge(mm, zz, aa, part[gg][0][c], part[gg][1][c], part[gg][2][c]);
      smx_store(mm, zz, aa, y + c, mo + c, zo + c, true);
    }
  } else {
#pragma unroll
    for (int j = 0; j < J; j++) {
      const uint32_t c = lane + 32 * j;
      if (c < H) smx_store(m[j], z[j], a[j], y + c, mo + c, zo + c, true);
    }
  }
}

// The backward's records of ids [0, n) over one column block, one warp per id: {m | r | y}, 3H floats, with
// r = gy / Z = gy * (1/Z); a row with no in-edge records m = +inf, so that exp(t x - m) = 0 for any finite t x.
template <int J>
__global__ void __launch_bounds__(SG_THREADS)
sg_smx_rec_kernel(uint32_t n, uint32_t H, const float* __restrict__ M, const float* __restrict__ IZ, size_t ldS,
                  const float* __restrict__ gy, size_t ldG, const float* __restrict__ y, size_t ldY,
                  float* __restrict__ rec) {
  const int lane = threadIdx.x % 32;
  const uint32_t v = blockIdx.x * (SG_THREADS / 32) + threadIdx.x / 32;
  if (v >= n) return;
  float* r = rec + (uint64_t)v * 3 * H;
#pragma unroll
  for (int j = 0; j < J; j++) {
    const uint32_t c = lane + 32 * j;
    if (c >= H) continue;
    const float iz = __ldg(IZ + (uint64_t)v * ldS + c);
    r[c] = iz > 0.f ? __ldg(M + (uint64_t)v * ldS + c) : INFINITY;
    r[H + c] = __fmul_rn(__ldg(gy + (uint64_t)v * ldG + c), iz);
    r[2 * H + c] = __ldg(y + (uint64_t)v * ldY + c);
  }
}

// dt = the sum of R [n][H] (packed): fp64 sums over blocks of SG_SMX_RB rows (each thread its columns, then the CTA's
// threads in a fixed tree), then the blocks' sums added in block order.  The blocks depend on (n, H) only.
__global__ void __launch_bounds__(SG_THREADS)
sg_smx_dt_part(uint32_t n, uint32_t H, const float* __restrict__ R, double* __restrict__ part) {
  __shared__ double sh[SG_THREADS];
  const uint32_t r0 = blockIdx.x * SG_SMX_RB, r1 = min(n, r0 + SG_SMX_RB);
  double s = 0.0;
  for (uint32_t r = r0; r < r1; r++)
    for (uint32_t c = threadIdx.x; c < H; c += SG_THREADS) s += (double)__ldg(R + (uint64_t)r * H + c);
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int k = SG_THREADS / 2; k > 0; k >>= 1) {
    if ((int)threadIdx.x < k) sh[threadIdx.x] += sh[threadIdx.x + k];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}
__global__ void sg_smx_dt_final(uint32_t nb, const double* __restrict__ part, float* __restrict__ dt) {
  const int lane = threadIdx.x;
  double s = 0.0;
  for (uint32_t b0 = 0; b0 < nb; b0 += 32) {
    const double v = b0 + lane < nb ? part[b0 + lane] : 0.0;
    for (int k = 0; k < 32 && b0 + k < nb; k++) s += __shfl_sync(0xffffffffu, v, k);
  }
  if (lane == 0) *dt = (float)s;
}

static SmxParams smx_params(const roc_sg_plan* pl, const float* t, int Hb) {
  SmxParams p;
  memset(&p, 0, sizeof(p));
  p.rs = pl->rs; p.col = pl->col; p.desc = pl->desc; p.carryIdx = pl->carryIdx; p.heavyRows = pl->heavyRows;
  p.bigRows = pl->bigRows; p.E = pl->E; p.numChunks = pl->numChunks; p.numHeavy = pl->numHeavy; p.numBig = pl->numBig;
  p.H = (uint32_t)Hb; p.t = t; p.carry = pl->carry; p.ldC = pl->carryLd;
  return p;
}

// One pass of sg_smx_kernel over pl, then its fix-ups: sg_smx_fixup (FWD), or the sum's over dx (and SRC_DT: R).
template <int PASS>
static int smx_pass(const roc_sg_plan* pl, const SmxParams& p, cudaStream_t st) {
  return v2_with_j(p.H, [&](auto J) {
    constexpr int WPB = SG_THREADS / 32;
    if (p.numChunks) {
      const uint32_t grid = (p.numChunks + WPB - 1) / WPB;
      sg_smx_kernel<J, PASS><<<grid, SG_THREADS, 0, st>>>(p);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_MAIN, SG_RED_SMX + PASS, 1, 32, J, grid);
    }
    if constexpr (PASS == SG_SMX_FWD) {
      if (p.numHeavy) {
        const uint32_t grid = (p.numHeavy + WPB - 1) / WPB;
        sg_smx_fixup<J, false><<<grid, SG_THREADS, 0, st>>>(p);
        ROC_LAUNCH_CHECK();
        note_launch(ROC_SG_LAUNCH_FIXUP, SG_RED_SMX + PASS, 1, 32, J, grid);
      }
      if (p.numBig) {
        sg_smx_fixup<J, true><<<p.numBig, SG_THREADS, 0, st>>>(p);
        ROC_LAUNCH_CHECK();
        note_launch(ROC_SG_LAUNCH_BIG_FIXUP, SG_RED_SMX + PASS, 1, 32, J, p.numBig);
      }
      return ROC_OK;
    } else {
      int rc = v2_fixups(pl, (int)p.H, p.out, (int64_t)p.ldOut, 0, st);
      if (rc == ROC_OK && PASS == SG_SMX_SRC_DT) rc = v2_fixups(pl, (int)p.H, p.out2, (int64_t)p.ldOut2, p.H, st);
      return rc;
    }
  });
}

// A plan whose ids are not all its own rows (a graph slice) is ROC_ERR_UNSUPPORTED; then the carries, `cols` floats.
static int smx_setup(roc_sg_plan* pl, int cols, cudaStream_t st) {
  int rc = find_id_end(pl, st);
  if (rc != ROC_OK) return rc;
  if (pl->idEnd > pl->nloc) return ROC_ERR_UNSUPPORTED;
  return grow_carries(pl, cols, st);
}

static int smx_forward(roc_sg_plan* pl, int H, const float* t, const float* x, int64_t ldX, float* y, int64_t ldY,
                       float* stats, int64_t ldStats, cudaStream_t st) {
  const int bc = std::min(H, SG_SMX_COLS);
  int rc = smx_setup(pl, 3 * bc, st);
  if (rc != ROC_OK) return rc;
  // without stats, a cut row's owner keeps its raw (m, s) in the plan's workspace
  float* ws = nullptr;
  if (!stats && pl->numHeavy + pl->numBig) {
    if ((rc = grow(pl->smxWs, pl->smxWsBytes, (size_t)pl->nloc * 2 * bc * sizeof(float), st)) != ROC_OK) return rc;
    ws = reinterpret_cast<float*>(pl->smxWs);
  }
  for (int c0 = 0; c0 < H && rc == ROC_OK; c0 += SG_SMX_COLS) {
    const int Hb = std::min(H - c0, SG_SMX_COLS);
    SmxParams p = smx_params(pl, t, Hb);
    p.g = x + c0; p.ldG = (size_t)ldX; p.out = y + c0; p.ldOut = (size_t)ldY;
    if (stats) { p.m = stats + c0; p.z = stats + H + c0; p.ldMZ = (size_t)ldStats; p.stats = 1; }
    else { p.m = ws; p.z = ws + bc; p.ldMZ = 2 * (size_t)bc; }
    rc = smx_pass<SG_SMX_FWD>(pl, p, st);
  }
  return rc;
}

// The backward once its arguments are checked: per column block the records over pl's rows and the source pass over
// plB (pl itself, or the transposed plan); then dt from R.  The records, R and dt's block sums live in pl's workspace,
// grown on demand (grow) and kept, so that a training step does not allocate and map gigabytes per call.
static int smx_backward(roc_sg_plan* pl, roc_sg_plan* plB, int H, const float* t, const float* x, int64_t ldX,
                        const float* y, int64_t ldY, const float* stats, int64_t ldStats, const float* gy, int64_t ldG,
                        float* dx, int64_t ldDx, float* dt, cudaStream_t st) {
  const int bc = std::min(H, SG_SMX_COLS);
  int rc = find_id_end(pl, st);
  if (rc == ROC_OK && pl->idEnd > pl->nloc) rc = ROC_ERR_UNSUPPORTED;
  if (rc == ROC_OK) rc = smx_setup(plB, (dt ? 2 : 1) * bc, st);
  if (rc != ROC_OK) return rc;
  const uint32_t n = pl->nloc, nb = (n + SG_SMX_RB - 1) / SG_SMX_RB;
  const size_t recBytes = ((size_t)n * 3 * bc * sizeof(float) + 15) / 16 * 16;
  const size_t rBytes = dt ? ((size_t)n * H * sizeof(float) + 15) / 16 * 16 : 0;
  rc = grow(pl->smxWs, pl->smxWsBytes, recBytes + rBytes + (dt ? (size_t)std::max(nb, 1u) * sizeof(double) : 0), st);
  if (rc != ROC_OK) return rc;
  char* ws = pl->smxWs;
  float* rec = reinterpret_cast<float*>(ws);
  float* R = dt ? reinterpret_cast<float*>(ws + recBytes) : nullptr;
  double* part = dt ? reinterpret_cast<double*>(ws + recBytes + rBytes) : nullptr;
  for (int c0 = 0; c0 < H && rc == ROC_OK; c0 += SG_SMX_COLS) {
    const int Hb = std::min(H - c0, SG_SMX_COLS);
    rc = v2_with_j((uint32_t)Hb, [&](auto J) {
      if (n) {
        const uint32_t grid = (n + SG_THREADS / 32 - 1) / (SG_THREADS / 32);
        sg_smx_rec_kernel<J><<<grid, SG_THREADS, 0, st>>>(n, (uint32_t)Hb, stats + c0, stats + H + c0, (size_t)ldStats,
                                                          gy + c0, (size_t)ldG, y + c0, (size_t)ldY, rec);
        ROC_LAUNCH_CHECK();
        note_launch(ROC_SG_LAUNCH_RECORD, -1, 1, 32, J, grid);
      }
      return ROC_OK;
    });
    if (rc != ROC_OK) break;
    SmxParams p = smx_params(plB, t, Hb);
    p.g = rec; p.ldG = 3 * (size_t)Hb; p.o = x + c0; p.ldO = (size_t)ldX; p.out = dx + c0; p.ldOut = (size_t)ldDx;
    if (dt) { p.out2 = R + c0; p.ldOut2 = (size_t)H; rc = smx_pass<SG_SMX_SRC_DT>(plB, p, st); }
    else rc = smx_pass<SG_SMX_SRC>(plB, p, st);
  }
  if (rc == ROC_OK && dt) {
    if (!nb) {
      const cudaError_t e = cudaMemsetAsync(dt, 0, sizeof(float), st);
      if (e != cudaSuccess) rc = (int)e;
    } else {
      sg_smx_dt_part<<<nb, SG_THREADS, 0, st>>>(n, (uint32_t)H, R, part);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_COLSUM, -1, 1, SG_THREADS, 1, nb);
      sg_smx_dt_final<<<1, 32, 0, st>>>(nb, part, dt);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_COLSUM, -1, 1, 32, 1, 1);
    }
  }
  return rc;
}

// dx may alias none of the inputs, nor dt t.
static bool smx_backward_args_bad(int H, const float* t, const float* x, int64_t ldX, const float* y, int64_t ldY,
                                  const float* stats, int64_t ldStats, const float* gy, int64_t ldG, const float* dx,
                                  int64_t ldDx, const float* dt) {
  return !t || !x || !y || !stats || !gy || !dx || H <= 0 || ldX < H || ldY < H || ldStats < 2 * (int64_t)H ||
         ldG < H || ldDx < H || dx == x || dx == y || dx == stats || dx == gy || dx == t || (dt && dt == t);
}

}  // namespace roc

extern "C" int roc_sg_softmax_forward_planned(const roc_sg_plan* plc, int H, const float* t, const float* x,
                                              int64_t ldX, float* y, int64_t ldY, float* stats, int64_t ldStats,
                                              roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || !t || !x || !y || H <= 0 || ldX < H || ldY < H || y == x || (stats && ldStats < 2 * (int64_t)H))
    return ROC_ERR_INVALID;
  return smx_forward(pl, H, t, x, ldX, y, ldY, stats, ldStats, as_stream(stream));
}

extern "C" int roc_sg_softmax_backward_planned(const roc_sg_plan* plc, int H, const float* t, const float* x,
                                               int64_t ldX, const float* y, int64_t ldY, const float* stats,
                                               int64_t ldStats, const float* gy, int64_t ldG, float* dx, int64_t ldDx,
                                               float* dt, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || smx_backward_args_bad(H, t, x, ldX, y, ldY, stats, ldStats, gy, ldG, dx, ldDx, dt)) return ROC_ERR_INVALID;
  return smx_backward(pl, pl, H, t, x, ldX, y, ldY, stats, ldStats, gy, ldG, dx, ldDx, dt, as_stream(stream));
}

extern "C" int roc_sg_softmax_backward_exact(const roc_sg_plan* plc, roc_sg_transpose* tr, int H, const float* t,
                                             const float* x, int64_t ldX, const float* y, int64_t ldY,
                                             const float* stats, int64_t ldStats, const float* gy, int64_t ldG,
                                             float* dx, int64_t ldDx, float* dt, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || !tr || smx_backward_args_bad(H, t, x, ldX, y, ldY, stats, ldStats, gy, ldG, dx, ldDx, dt) ||
      pl->nloc != tr->N || pl->E != tr->E)
    return ROC_ERR_INVALID;
  return smx_backward(pl, tr->planT, H, t, x, ldX, y, ldY, stats, ldStats, gy, ldG, dx, ldDx, dt, as_stream(stream));
}

// ------------------------------------------------ dot-product attention ---
// roc_sg_attn_dot_*: the graph transformer's attention (PyG TransformerConv, UniMP): s(v<-u, k) = scale q[v]_k . k[u]_k
// and out[v]_k = sum_u softmax_u(s) v[u]_k.  The passes run on their own kernel, sg_dot_kernel, over the plan's chunks,
// chunk records and carry slots, one warp per chunk with lane l holding columns l + 32 j (j < J = ceil(H / 32)),
// scalar, as sg_v2_kernel.  Unlike sg_v2_kernel, every per-head quantity is held per column, replicated over the head's
// columns, so that the row walk needs no shuffle and no per-head select:
//  * dot_head_sums reduces a group's U edges' products together, before the row walk.  Where F divides 32 a head's
//    columns sit at one lane each within an aligned group of F lanes, and each is reduced over those lanes alone
//    (log2 F xor levels); otherwise each head is summed over the lane's columns in column order, then over the warp by
//    an xor butterfly.  The order depends on (H, heads) only and every lane of a head ends with the same bits, so the
//    forward and both backward passes see the same s.
//  * the forward is one pass with an online softmax per head, kept per column as (m, s, w) = (max s, sum exp(s - m),
//    sum exp(s - m) v): the softmax aggregation's scheme, whose merge (smx_merge) and store (smx_store) it reuses.
//    A cut row's owner stores w and its per-head (m, s); the carries hold [m | s | w] per column; sg_dot_fixup merges
//    them in chunk order.
//  * the backward is the record pass of GATv2 (sg_v2_rec_kernel: {m, 1/Z, c} per head), a destination pass (dq) and a
//    source pass (dk, dv), finished by the sum's fix-ups.
namespace roc {

enum { SG_DOT_FWD = 0, SG_DOT_DST = 1, SG_DOT_SRC = 2 };
constexpr int SG_RED_DOT = 80;                // the `red` sg_last_call_info reports for pass P is SG_RED_DOT + P

struct DotParams {
  const uint32_t* rs;
  const uint32_t* col;
  const uint32_t* desc;
  const uint32_t* carryIdx;
  const uint32_t* heavyRows;
  const uint32_t* bigRows;
  uint32_t E, numChunks, numHeavy, numBig, H, heads;
  float scale;
  const float* g;  size_t ldG;    // gathered rows (by col id): FWD, DST k; SRC q
  const float* g2; size_t ldG2;   // FWD, DST v; SRC gy
  const float* o;  size_t ldO;    // the row's own row: FWD, DST q; SRC k
  const float* o2; size_t ldO2;   // DST gy; SRC v
  const float4* rec;              // DST, SRC: {m, 1/Z, c, 0} per (id, head)
  float* out;  size_t ldOut;      // FWD y (a cut row's owner: w); DST dq; SRC dk
  float* out2; size_t ldOut2;     // SRC dv
  float* stats; size_t ldStats;   // FWD: m | 1/Z per head of finished rows (nullptr: none)
  float* raw;  size_t ldRaw;      // FWD: a cut row's owner's raw m | s per head (stats, or a workspace)
  float* carry; size_t ldC;       // FWD [m | s | w]; DST dq; SRC [dk | dv]
};

// r[n][j] = the sum over the warp of t[n] over the columns of head hj[j] (the fixed order described above); N rows of
// products reduced together, each xor level issued for all of them at once.
template <int N, int J>
__device__ __forceinline__ void dot_head_sums(const float (&t)[N][J], const int (&hj)[J], uint32_t heads, uint32_t F,
                                              float (&r)[N][J]) {
  if (32u % F == 0u) {
#pragma unroll
    for (int n = 0; n < N; n++)
#pragma unroll
      for (int j = 0; j < J; j++) r[n][j] = t[n][j];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1)
      if ((uint32_t)o < F) {
#pragma unroll
        for (int n = 0; n < N; n++)
#pragma unroll
          for (int j = 0; j < J; j++) r[n][j] = __fadd_rn(r[n][j], __shfl_xor_sync(0xffffffffu, r[n][j], o));
      }
  } else {
#pragma unroll
    for (int n = 0; n < N; n++)
#pragma unroll
      for (int j = 0; j < J; j++) r[n][j] = 0.f;
#pragma unroll
    for (int k = 0; k < SG_V2_HEADS; k++) {
      if ((uint32_t)k < heads) {
        float x[N];
#pragma unroll
        for (int n = 0; n < N; n++) {
          x[n] = 0.f;
#pragma unroll
          for (int j = 0; j < J; j++) x[n] = __fadd_rn(x[n], hj[j] == k ? t[n][j] : 0.f);
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1)
#pragma unroll
          for (int n = 0; n < N; n++) x[n] = __fadd_rn(x[n], __shfl_xor_sync(0xffffffffu, x[n], o));
#pragma unroll
        for (int n = 0; n < N; n++)
#pragma unroll
          for (int j = 0; j < J; j++) r[n][j] = hj[j] == k ? x[n] : r[n][j];
      }
    }
  }
}

// One warp per chunk of the plan, the schedule of sg_v2_kernel.  Per edge (row v's edge from u in the forward plan),
// with s = scale q[v] . k[u] per head:
//   FWD  online (m, s, w) per column of s and v[u];
//   DST  p = exp(s - m) / Z, d = p (gy[v] . v[u] - c[v]), dq[v] += scale d k[u];
//   SRC  (row u, gathering v and v's record) dk[u] += scale d q[v], dv[u] += p gy[v].
// The dot products of a group of U edges are taken together with the current row's own row, before the walk over the
// rows the group spans; a row that starts inside the group takes them again for the whole group.  The per-edge branch
// of the walk holds no shuffle.  __launch_bounds__(SG_THREADS, 1) as sg_v2_kernel: it lets ptxas use up to 255
// registers, so that no instantiation needs local memory.
template <int J, int PASS>
__global__ void __launch_bounds__(SG_THREADS, 1)
sg_dot_kernel(const DotParams p) {
  constexpr bool FWD = PASS == SG_DOT_FWD, DST = PASS == SG_DOT_DST, SRC = PASS == SG_DOT_SRC;
  constexpr int ND = FWD ? 1 : 2;               // dot products per edge and head
  constexpr int U = FWD ? (J <= 2 ? 8 : J <= 4 ? 4 : 2) : (J <= 2 ? 4 : J <= 4 ? 2 : 1);   // edges in flight
  constexpr int WPB = SG_THREADS / 32;
  constexpr uint32_t CH = SG_CH;
  const int lane = threadIdx.x % 32;
  const uint32_t w = blockIdx.x * WPB + threadIdx.x / 32;
  if (w >= p.numChunks) return;
  const uint32_t* dsc = p.desc + 8 * (size_t)w;
  const uint32_t flags = __ldg(dsc + 6);
  if (flags & 2u) return;
  const uint32_t ce = min(w * CH + CH, p.E);
  uint32_t cur = __ldg(dsc + 2), curS = __ldg(dsc + 3), curT = __ldg(dsc + 4);
  const uint32_t e0 = __ldg(dsc), ee = __ldg(dsc + 1), r1 = __ldg(dsc + 5), carrySlot = __ldg(dsc + 7);
  int kind = (flags & 1u) ? 0 : ((curT - curS > CH) ? 2 : 1);   // 0 carry-in part, 1 complete row, 2 cut row's owner
  uint32_t segEnd = (kind == 1) ? curT : min(curT, ce);

  const uint32_t H = p.H, heads = p.heads, F = H / heads;
  const float scale = p.scale;
  int hj[J];
  bool vj[J], lead[J];          // lead: the head's first column, which stores its per-head values
#pragma unroll
  for (int j = 0; j < J; j++) {
    const uint32_t c = (uint32_t)(lane + 32 * j);
    vj[j] = c < H;
    hj[j] = vj[j] ? (int)(c / F) : -1;
    lead[j] = vj[j] && c % F == 0u;
  }
  float xo[J], yo[FWD ? 1 : J];               // the row's own rows: FWD q; DST q, gy; SRC k, v
  float rm[DST ? J : 1], ri[DST ? J : 1], rc[DST ? J : 1];   // DST: the row's m, 1/Z and c per column
  float sm[FWD ? J : 1], ss[FWD ? J : 1];     // FWD: running m, s (acc: w)
  float acc[J], acc2[SRC ? J : 1];
#pragma unroll
  for (int j = 0; j < J; j++) {
    acc[j] = 0.f;
    if constexpr (SRC) acc2[j] = 0.f;
    if constexpr (FWD) { sm[j] = -INFINITY; ss[j] = 0.f; }
  }

  auto row_state = [&]() {
    v2_load_row<J>(p.o + (uint64_t)cur * p.ldO, lane, vj, xo);
    if constexpr (!FWD) v2_load_row<J>(p.o2 + (uint64_t)cur * p.ldO2, lane, vj, yo);
    if constexpr (DST) {
#pragma unroll
      for (int j = 0; j < J; j++) {
        const float4 r = vj[j] ? __ldg(p.rec + (uint64_t)cur * heads + hj[j]) : make_float4(0.f, 0.f, 0.f, 0.f);
        rm[j] = r.x; ri[j] = r.y; rc[j] = r.z;
      }
    }
  };
  row_state();

  auto flush = [&]() {
    if constexpr (FWD) {
      if (kind == 0) {
        float* c = p.carry + (uint64_t)carrySlot * p.ldC;
#pragma unroll
        for (int j = 0; j < J; j++)
          if (vj[j]) { c[lane + 32 * j] = sm[j]; c[H + lane + 32 * j] = ss[j]; c[2 * H + lane + 32 * j] = acc[j]; }
      } else {
        float* y = p.out + (uint64_t)cur * p.ldOut;
#pragma unroll
        for (int j = 0; j < J; j++) {
          if (!vj[j]) continue;
          const uint32_t c = lane + 32 * j, h = (uint32_t)hj[j];
          if (kind == 2) {    // the raw partial, for sg_dot_fixup
            y[c] = acc[j];
            if (lead[j]) { p.raw[(uint64_t)cur * p.ldRaw + h] = sm[j]; p.raw[(uint64_t)cur * p.ldRaw + heads + h] = ss[j]; }
          } else {
            float* st = p.stats + (uint64_t)cur * p.ldStats;
            smx_store(sm[j], ss[j], acc[j], y + c, st + h, st + heads + h, p.stats && lead[j]);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < J; j++) { sm[j] = -INFINITY; ss[j] = 0.f; acc[j] = 0.f; }
    } else {
      float* d1 = (kind == 0) ? p.carry + (uint64_t)carrySlot * p.ldC : p.out + (uint64_t)cur * p.ldOut;
      float* d2 = (kind == 0) ? d1 + H : p.out2 + (uint64_t)cur * p.ldOut2;
      (void)d2;
#pragma unroll
      for (int j = 0; j < J; j++) {
        if (vj[j]) {
          d1[lane + 32 * j] = acc[j];
          if constexpr (SRC) d2[lane + 32 * j] = acc2[j];
        }
        acc[j] = 0.f;
        if constexpr (SRC) acc2[j] = 0.f;
      }
    }
  };
  auto advance = [&]() {
    cur += 1; curS = curT; curT = p.rs[cur + 1];
    const bool heavy = curT - curS > CH;
    segEnd = heavy ? min(curT, ce) : curT;
    kind = heavy ? 2 : 1;
    row_state();
  };

  const uint32_t eLast = ee - 1u;
#pragma unroll 1
  for (uint32_t base = e0; base < ee; base += U) {
    const uint32_t cnt = min((uint32_t)U, ee - base);
    float ga[U][J], gb[U][J];        // FWD, DST: k[u], v[u]; SRC: q[v], gy[v]
    float4 gr[SRC ? U : 1][SRC ? J : 1];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint32_t id = __ldg(p.col + min(base + (uint32_t)u, eLast));
      v2_load_row<J>(p.g + (uint64_t)id * p.ldG, lane, vj, ga[u]);
      v2_load_row<J>(p.g2 + (uint64_t)id * p.ldG2, lane, vj, gb[u]);
      if constexpr (SRC) {
#pragma unroll
        for (int j = 0; j < J; j++)
          gr[u][j] = vj[j] ? __ldg(p.rec + (uint64_t)id * heads + hj[j]) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    uint32_t pos = 0;
    for (;;) {
      const uint32_t lim = min(cnt, segEnd - base);
      if (lim > pos) {
        // the group's dot products with this row: q . k (and gy . v) per edge and head, all U edges together
        float t[ND * U][J], d[ND * U][J];
#pragma unroll
        for (int u = 0; u < U; u++)
#pragma unroll
          for (int j = 0; j < J; j++) {
            t[ND * u][j] = __fmul_rn(xo[j], ga[u][j]);
            if constexpr (DST) t[ND * u + 1][j] = __fmul_rn(yo[j], gb[u][j]);
            if constexpr (SRC) t[ND * u + 1][j] = __fmul_rn(gb[u][j], yo[j]);
          }
        dot_head_sums<ND * U, J>(t, hj, heads, F, d);
#pragma unroll
        for (int u = 0; u < U; u++) {
          if ((uint32_t)u >= pos && (uint32_t)u < lim) {
#pragma unroll
            for (int j = 0; j < J; j++) {
              const float e = __fmul_rn(scale, d[ND * u][j]);
              if constexpr (FWD) {
                const float x = gb[u][j];
                if (e > sm[j]) {
                  const float c = expf(sm[j] - e);
                  ss[j] = fmaf(ss[j], c, 1.f); acc[j] = fmaf(acc[j], c, x); sm[j] = e;
                } else {
                  const float q = expf(e - sm[j]);
                  ss[j] = __fadd_rn(ss[j], q); acc[j] = fmaf(q, x, acc[j]);
                }
              } else {
                const float m = SRC ? gr[u][j].x : rm[j], iz = SRC ? gr[u][j].y : ri[j];
                const float c = SRC ? gr[u][j].z : rc[j];
                const float pk = attn_alpha(e, m, iz);
                const float ds = __fmul_rn(scale, __fmul_rn(pk, __fsub_rn(d[ND * u + 1][j], c)));
                acc[j] = fmaf(ds, ga[u][j], acc[j]);
                if constexpr (SRC) acc2[j] = fmaf(pk, gb[u][j], acc2[j]);
              }
            }
          }
        }
      }
      pos = lim;
      if (pos >= cnt) break;
      flush();
      advance();
    }
  }
  flush();
  while (cur + 1 < r1) { advance(); flush(); }   // trailing zero-degree rows
}

// Finishes the forward's cut rows, as sg_smx_fixup with the owner's (m, s) per head: the owner's raw partial (y: w,
// raw: m | s per head), then the carries in chunk order, stored as y and, with stats, m | 1/Z per head.  Heavy rows (at
// most 32 carries): one warp each.  BIG rows: one CTA each, whose warps merge contiguous blocks of the carries, then
// warp 0 the owner's partial and the blocks' in block order.  The grouping depends on the plan only.
template <int J, bool BIG>
__global__ void __launch_bounds__(SG_THREADS, 1)
sg_dot_fixup(const DotParams p) {
  constexpr uint32_t CH = SG_CH;
  constexpr int WPB = SG_THREADS / 32;
  const int lane = threadIdx.x % 32, g = threadIdx.x / 32;
  const uint32_t w = BIG ? blockIdx.x : blockIdx.x * WPB + g;
  if (w >= (BIG ? p.numBig : p.numHeavy)) return;
  const uint32_t R = BIG ? p.bigRows[w] : p.heavyRows[w];
  const uint32_t s = p.rs[R], t = p.rs[R + 1];
  const uint32_t c0 = s / CH, n = (t - 1) / CH - c0;
  const float* cb = p.carry + (uint64_t)p.carryIdx[c0 + 1] * p.ldC;
  const uint32_t H = p.H, heads = p.heads, F = H / heads;
  float* y = p.out + (uint64_t)R * p.ldOut;
  const float* raw = p.raw + (uint64_t)R * p.ldRaw;
  uint32_t hc[J];               // the head of each of the lane's columns
  bool vj[J];
#pragma unroll
  for (int j = 0; j < J; j++) { vj[j] = (uint32_t)(lane + 32 * j) < H; hc[j] = vj[j] ? (lane + 32 * j) / F : 0u; }
  uint32_t k0 = 0, k1 = n;
  if constexpr (BIG) { const uint32_t per = (n + WPB - 1) / WPB; k0 = min(n, g * per); k1 = min(n, k0 + per); }
  float m[J], z[J], a[J];
#pragma unroll
  for (int j = 0; j < J; j++) { m[j] = -INFINITY; z[j] = 0.f; a[j] = 0.f; }
  if (!BIG) {   // a heavy row starts from its owner's partial
#pragma unroll
    for (int j = 0; j < J; j++)
      if (vj[j]) { m[j] = raw[hc[j]]; z[j] = raw[heads + hc[j]]; a[j] = y[lane + 32 * j]; }
  }
  for (uint32_t k = k0; k < k1; k++) {
    const float* ck = cb + (uint64_t)k * p.ldC;
#pragma unroll
    for (int j = 0; j < J; j++) {
      const uint32_t c = lane + 32 * j;
      if (vj[j]) smx_merge(m[j], z[j], a[j], ck[c], ck[H + c], ck[2 * H + c]);
    }
  }
  if constexpr (BIG) {
    __shared__ float part[WPB][3][32 * J];
#pragma unroll
    for (int j = 0; j < J; j++) { part[g][0][lane + 32 * j] = m[j]; part[g][1][lane + 32 * j] = z[j]; part[g][2][lane + 32 * j] = a[j]; }
    __syncthreads();
    if (g != 0) return;
#pragma unroll
    for (int j = 0; j < J; j++) {
      const uint32_t c = lane + 32 * j;
      if (vj[j]) {
        m[j] = raw[hc[j]]; z[j] = raw[heads + hc[j]]; a[j] = y[c];
#pragma unroll
        for (int gg = 0; gg < WPB; gg++) smx_merge(m[j], z[j], a[j], part[gg][0][c], part[gg][1][c], part[gg][2][c]);
      }
    }
  }
  __syncwarp();   // every lane of a head has read the owner's (m, s) before its first column overwrites them
  float* st = p.stats ? p.stats + (uint64_t)R * p.ldStats : nullptr;
#pragma unroll
  for (int j = 0; j < J; j++) {
    const uint32_t c = lane + 32 * j;
    if (vj[j]) smx_store(m[j], z[j], a[j], y + c, st + hc[j], st + heads + hc[j], st && c % F == 0u);
  }
}

static DotParams dot_params(const roc_sg_plan* pl, int heads, int H, float scale) {
  DotParams p;
  memset(&p, 0, sizeof(p));
  p.rs = pl->rs; p.col = pl->col; p.desc = pl->desc; p.carryIdx = pl->carryIdx; p.heavyRows = pl->heavyRows;
  p.bigRows = pl->bigRows; p.E = pl->E; p.numChunks = pl->numChunks; p.numHeavy = pl->numHeavy; p.numBig = pl->numBig;
  p.H = (uint32_t)H; p.heads = (uint32_t)heads; p.scale = scale; p.carry = pl->carry; p.ldC = pl->carryLd;
  return p;
}

// One pass of sg_dot_kernel over pl, then its fix-ups: sg_dot_fixup (FWD), or the sum's over out (and SRC: out2).
template <int PASS>
static int dot_pass(const roc_sg_plan* pl, const DotParams& p, cudaStream_t st) {
  return v2_with_j(p.H, [&](auto J) {
    constexpr int WPB = SG_THREADS / 32;
    if (p.numChunks) {
      const uint32_t grid = (p.numChunks + WPB - 1) / WPB;
      sg_dot_kernel<J, PASS><<<grid, SG_THREADS, 0, st>>>(p);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_MAIN, SG_RED_DOT + PASS, 1, 32, J, grid);
    }
    if constexpr (PASS == SG_DOT_FWD) {
      if (p.numHeavy) {
        const uint32_t grid = (p.numHeavy + WPB - 1) / WPB;
        sg_dot_fixup<J, false><<<grid, SG_THREADS, 0, st>>>(p);
        ROC_LAUNCH_CHECK();
        note_launch(ROC_SG_LAUNCH_FIXUP, SG_RED_DOT + PASS, 1, 32, J, grid);
      }
      if (p.numBig) {
        sg_dot_fixup<J, true><<<p.numBig, SG_THREADS, 0, st>>>(p);
        ROC_LAUNCH_CHECK();
        note_launch(ROC_SG_LAUNCH_BIG_FIXUP, SG_RED_DOT + PASS, 1, 32, J, p.numBig);
      }
      return ROC_OK;
    } else {
      int rc = v2_fixups(pl, (int)p.H, p.out, (int64_t)p.ldOut, 0, st);
      if (rc == ROC_OK && PASS == SG_DOT_SRC) rc = v2_fixups(pl, (int)p.H, p.out2, (int64_t)p.ldOut2, p.H, st);
      return rc;
    }
  });
}

// The checks every dot-product attention call shares once its pointers and leading dimensions are checked: a scale of
// 0 or not finite is ROC_ERR_INVALID; H % heads, H > 256, heads > SG_V2_HEADS and a plan whose ids are not all its own
// rows (a graph slice) are ROC_ERR_UNSUPPORTED.  Then the carries, `cols` floats per slot.
static int dot_setup(roc_sg_plan* pl, int heads, int H, float scale, int cols, cudaStream_t st) {
  if (scale == 0.f || !std::isfinite(scale)) return ROC_ERR_INVALID;
  if (H > 256 || H % heads || heads > SG_V2_HEADS) return ROC_ERR_UNSUPPORTED;
  int rc = find_id_end(pl, st);
  if (rc != ROC_OK) return rc;
  if (pl->idEnd > pl->nloc) return ROC_ERR_UNSUPPORTED;
  return grow_carries(pl, cols, st);
}

static int dot_forward(roc_sg_plan* pl, int heads, int H, float scale, const float* q, int64_t ldQ, const float* k,
                       int64_t ldK, const float* v, int64_t ldV, float* out, int64_t ldOut, float* stats,
                       int64_t ldStats, cudaStream_t st) {
  int rc = dot_setup(pl, heads, H, scale, 3 * H, st);
  if (rc != ROC_OK) return rc;
  DotParams p = dot_params(pl, heads, H, scale);
  p.g = k; p.ldG = (size_t)ldK; p.g2 = v; p.ldG2 = (size_t)ldV; p.o = q; p.ldO = (size_t)ldQ;
  p.out = out; p.ldOut = (size_t)ldOut;
  if (stats) {
    p.stats = p.raw = stats; p.ldStats = p.ldRaw = (size_t)ldStats;
  } else if (pl->numHeavy + pl->numBig) {
    // without stats, a cut row's owner keeps its raw (m, s) in the plan's workspace (the softmax aggregation's)
    if ((rc = grow(pl->smxWs, pl->smxWsBytes, (size_t)pl->nloc * 2 * heads * sizeof(float), st)) != ROC_OK) return rc;
    p.raw = reinterpret_cast<float*>(pl->smxWs); p.ldRaw = 2 * (size_t)heads;
  }
  return dot_pass<SG_DOT_FWD>(pl, p, st);
}

// The backward once its arguments are checked: the records over pl's rows (the GATv2 record kernel), the destination
// pass over pl, and the source pass over plB (pl itself, or the transposed plan).
static int dot_backward(roc_sg_plan* pl, roc_sg_plan* plB, int heads, int H, float scale, const float* q, int64_t ldQ,
                        const float* k, int64_t ldK, const float* v, int64_t ldV, const float* out, int64_t ldOut,
                        const float* stats, int64_t ldStats, const float* gy, int64_t ldG, float* dq, int64_t ldDq,
                        float* dk, int64_t ldDk, float* dv, int64_t ldDv, cudaStream_t st) {
  int rc = dot_setup(pl, heads, H, scale, plB == pl ? 2 * H : H, st);
  if (rc == ROC_OK && plB != pl) rc = dot_setup(plB, heads, H, scale, 2 * H, st);
  if (rc != ROC_OK) return rc;
  const uint32_t n = pl->nloc;
  if ((rc = grow(pl->attnRec, pl->attnRecBytes, (size_t)n * heads * sizeof(float4), st)) != ROC_OK) return rc;
  V2Params r = v2_params(pl, heads, H, 0.f, nullptr);
  r.g = gy; r.ldG = (size_t)ldG; r.o = out; r.ldO = (size_t)ldOut; r.stats = stats; r.ldStats = (size_t)ldStats;
  r.rec = pl->attnRec;
  rc = v2_with_j((uint32_t)H, [&](auto J) {
    if (n) {
      const uint32_t grid = (n + SG_THREADS / 32 - 1) / (SG_THREADS / 32);
      sg_v2_rec_kernel<J><<<grid, SG_THREADS, 0, st>>>(r, n);
      ROC_LAUNCH_CHECK();
      note_launch(ROC_SG_LAUNCH_RECORD, -1, 1, 32, J, grid);
    }
    return ROC_OK;
  });
  if (rc == ROC_OK) {   // destination pass: dq
    DotParams d = dot_params(pl, heads, H, scale);
    d.g = k; d.ldG = (size_t)ldK; d.g2 = v; d.ldG2 = (size_t)ldV; d.o = q; d.ldO = (size_t)ldQ;
    d.o2 = gy; d.ldO2 = (size_t)ldG; d.rec = pl->attnRec; d.out = dq; d.ldOut = (size_t)ldDq;
    rc = dot_pass<SG_DOT_DST>(pl, d, st);
  }
  if (rc == ROC_OK) {   // source pass: dk and dv
    DotParams s = dot_params(plB, heads, H, scale);
    s.g = q; s.ldG = (size_t)ldQ; s.g2 = gy; s.ldG2 = (size_t)ldG; s.o = k; s.ldO = (size_t)ldK;
    s.o2 = v; s.ldO2 = (size_t)ldV; s.rec = pl->attnRec; s.out = dk; s.ldOut = (size_t)ldDk;
    s.out2 = dv; s.ldOut2 = (size_t)ldDv;
    rc = dot_pass<SG_DOT_SRC>(plB, s, st);
  }
  return rc;
}

// NULL pointers, bad leading dimensions, and outputs that alias each other or an input.
static bool dot_backward_args_bad(int heads, int H, const float* q, int64_t ldQ, const float* k, int64_t ldK,
                                  const float* v, int64_t ldV, const float* out, int64_t ldOut, const float* stats,
                                  int64_t ldStats, const float* gy, int64_t ldG, const float* dq, int64_t ldDq,
                                  const float* dk, int64_t ldDk, const float* dv, int64_t ldDv) {
  if (!q || !k || !v || !out || !stats || !gy || !dq || !dk || !dv || heads <= 0 || H <= 0 || ldQ < H || ldK < H ||
      ldV < H || ldOut < H || ldG < H || ldDq < H || ldDk < H || ldDv < H || ldStats < 2 * (int64_t)heads)
    return true;
  if (dq == dk || dq == dv || dk == dv) return true;
  for (const float* o : {dq, dk, dv})
    if (o == q || o == k || o == v || o == out || o == stats || o == gy) return true;
  return false;
}

}  // namespace roc

extern "C" int roc_sg_attn_dot_forward_planned(const roc_sg_plan* plc, int heads, int H, float scale, const float* q,
                                               int64_t ldQ, const float* k, int64_t ldK, const float* v, int64_t ldV,
                                               float* out, int64_t ldOut, float* stats, int64_t ldStats,
                                               roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || !q || !k || !v || !out || heads <= 0 || H <= 0 || ldQ < H || ldK < H || ldV < H || ldOut < H ||
      (stats && ldStats < 2 * (int64_t)heads) || out == q || out == k || out == v ||
      (stats && (stats == out || stats == q || stats == k || stats == v)))
    return ROC_ERR_INVALID;
  return dot_forward(pl, heads, H, scale, q, ldQ, k, ldK, v, ldV, out, ldOut, stats, ldStats, as_stream(stream));
}

extern "C" int roc_sg_attn_dot_backward_planned(const roc_sg_plan* plc, int heads, int H, float scale, const float* q,
                                                int64_t ldQ, const float* k, int64_t ldK, const float* v, int64_t ldV,
                                                const float* out, int64_t ldOut, const float* stats, int64_t ldStats,
                                                const float* outGrad, int64_t ldG, float* dq, int64_t ldDq, float* dk,
                                                int64_t ldDk, float* dv, int64_t ldDv, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || dot_backward_args_bad(heads, H, q, ldQ, k, ldK, v, ldV, out, ldOut, stats, ldStats, outGrad, ldG, dq, ldDq,
                                   dk, ldDk, dv, ldDv))
    return ROC_ERR_INVALID;
  return dot_backward(pl, pl, heads, H, scale, q, ldQ, k, ldK, v, ldV, out, ldOut, stats, ldStats, outGrad, ldG, dq,
                      ldDq, dk, ldDk, dv, ldDv, as_stream(stream));
}

extern "C" int roc_sg_attn_dot_backward_exact(const roc_sg_plan* plc, roc_sg_transpose* tr, int heads, int H,
                                              float scale, const float* q, int64_t ldQ, const float* k, int64_t ldK,
                                              const float* v, int64_t ldV, const float* out, int64_t ldOut,
                                              const float* stats, int64_t ldStats, const float* outGrad, int64_t ldG,
                                              float* dq, int64_t ldDq, float* dk, int64_t ldDk, float* dv,
                                              int64_t ldDv, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  clear_launches();
  if (!pl || !tr || dot_backward_args_bad(heads, H, q, ldQ, k, ldK, v, ldV, out, ldOut, stats, ldStats, outGrad, ldG,
                                          dq, ldDq, dk, ldDk, dv, ldDv) ||
      pl->nloc != tr->N || pl->E != tr->E)
    return ROC_ERR_INVALID;
  return dot_backward(pl, tr->planT, heads, H, scale, q, ldQ, k, ldK, v, ldV, out, ldOut, stats, ldStats, outGrad, ldG,
                      dq, ldDq, dk, ldDk, dv, ldDv, as_stream(stream));
}
