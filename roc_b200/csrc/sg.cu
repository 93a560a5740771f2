// sg.cu — ScatterGather (CSR row-parallel SpMM, sum aggregation) for sm_90a.
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
//  * FIVE main kernels share that plan and the per-row summation order — they are
//    bit-identical to each other — and differ in how the neighbour rows travel:
//      A  sg_chunk_kernel      registers: L = min(32, H/4) lanes per worker, one LDG.128 per lane and row,
//                              8 rows in flight per lane (default up to 64 floats per row)
//      C  sg_chunk_kernel_c2   cp.async (LDGSTS) ring per worker (rows wider than 256 floats)
//      T  sg_chunk_kernel_t    TMA: cp.async.bulk row copies, four per 4-edge unit, into a shared-memory
//                              ring per worker, mbarrier completion (default for 129..256 floats)
//      U  (T, MODE 2)          the same with the source ids held by the lanes that issue them (65..128 floats)
//      b  (T, MODE 1)          one plain cp.async.bulk per row (measurement only)
//      R  sg_ring_kernel       producer / consumer ring: producer warps issue the row copies for whole chunks into a
//                              two-slot ring, two worker warps consume (the structure the measured gather ceilings
//                              ask for; not yet faster — DESIGN.md §3.1)
//    The choice per width is by measurement (pick_variant); ROC_SG_VARIANT forces one.
//  * min / max aggregation (roc_sg_minmax_*) runs kernel A templated on the reduction, with its own fix-ups
//    for the forward; its backward is the sum schedule with a second gathered row and a predicated add.
//
// Algorithmic bytes per launch (DESIGN.md): E*(4H+4) + Nloc*(4H+8); min / max forward E*(4H+4) + Nloc*(8H+8),
// backward E*(8H+4) + Nloc*(4H+8).
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <cstdlib>
#include <cstring>
#include <new>
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
  float* carry = nullptr;         // [numCarries][carryLd]
  size_t carryLd = 0;
  uint32_t* carryArg = nullptr;   // [numCarries][carryLd] indices of the min / max carries (first use)
  size_t carryArgLd = 0;
  uint32_t* desc = nullptr;       // [numChunks][8] per-chunk start state of the ring kernel (k_chunk_desc)
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

// Start state of the worker that owns chunk c, so that the ring kernel reads ONE 32-byte record instead
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
  // IEEE divide.  A zero numerator sends nvcc's div.rn sequence down its slow path (FCHK flags
  // zero operands) and one such lane drags the whole warp along: gradients and pad columns are
  // full of zeros.  0/d == 0 (same
  // sign) for d != 0, so those lanes skip the divide; d == 0 (degree 0) still yields NaN/Inf.
  static __device__ __forceinline__ float div1(float a, float d) { return (a != 0.0f || d == 0.0f) ? a / d : a; }
  static __device__ __forceinline__ T div(const T& a, float d) {
    return make_float4(div1(a.x, d), div1(a.y, d), div1(a.z, d), div1(a.w, d));
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
  static __device__ __forceinline__ T div(const T& a, float d) { return (a != 0.0f || d == 0.0f) ? a / d : a; }
  static __device__ __forceinline__ T rdiv(const T& a, const RowDiv& r) { return rowdiv(a, r); }
  static __device__ __forceinline__ T relu(const T& a) { return relu_nanprop(a); }
};

// ------------------------------------------------------- min / max reduction ---
// What a kernel does with each gathered row.  SUM adds it; MAX / MIN keep, per float, the value and the source id of
// the first edge in CSR order that holds the extreme (roc_sg_minmax_forward_planned); MASK is the backward of those:
// it adds the gathered gradient only where the gathered index names the row being computed.
enum { SG_RED_SUM = 0, SG_RED_MAX = ROC_SG_AGGR_MAX, SG_RED_MIN = ROC_SG_AGGR_MIN, SG_RED_MASK = 3 };
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
  int dense;           // mean degree >= chunk size: nearly every row is cut at chunk boundaries
  const uint32_t* desc; // [numChunks][8] chunk start records (ring kernel)
  uint32_t nloc;        // rows of the partition (rs has nloc + 1 entries)
  // min / max aggregation (kernel A only)
  void* arg;            // MAX / MIN: [nloc][ldArg] indices written; MASK: [*][ldArg] indices gathered like `in`
  void* carryArg;       // MAX / MIN: [numCarries][ldC] indices of the carry partials
  size_t ldArg;         // in units of T
  uint32_t selfBase;    // MASK: id of local row 0 in the id space of col
};

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

// ------------------------------------------------------------- main kernel ---
// One worker (L lanes) per chunk.  Lane `lane` owns T-columns lane + ch*L.
// RED (SG_RED_*) changes only what is done with a gathered row and what the row store writes; the schedule, the
// gathers and the single store site are the same for every reduction.
template <int VEC, int L, int NCH, int U, int MINB, int RED = SG_RED_SUM>
__global__ void __launch_bounds__(SG_THREADS, MINB)
sg_chunk_kernel(const SgParams p) {
  typedef typename V<VEC>::T T;
  typedef typename V<VEC>::I I;
  constexpr bool MM = RED == SG_RED_MAX || RED == SG_RED_MIN;
  constexpr int WPB = SG_THREADS / L;
  constexpr uint32_t CH = SG_CH;
  const int lane = threadIdx.x % L;
  const uint32_t w = blockIdx.x * WPB + threadIdx.x / L;
  if (w >= p.numChunks) return;
  const unsigned wmask = (L == 32) ? 0xffffffffu
                                   : (((1u << L) - 1u) << (((threadIdx.x & 31) / L) * L));

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

  // Row store.  The epilogue (IEEE sqrt + divides) lives in ONE out-of-line copy:
  // inlining it at every edge position made the kernel 4096 SASS instructions and
  // instruction-fetch bound.
  auto flush = [&]() {
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
    const int epi = (kind == 1) ? p.epi : 0;
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) {
      if (act[ch]) {
        if (epi) epi_store<VEC>(acc[ch], dst + ch * L, curT - curS, epi);
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
  };

  // Every lane reads the source ids itself (same address across the worker: one broadcast
  // transaction from L1); sub-warp shuffles with a runtime mask cost a MATCH.ANY sequence each.
  (void)wmask;
  // Gathers are unpredicated: a group that runs past the worker's last edge re-reads that edge's
  // source (index clamped; an L1 hit) and the tail values are simply never added.  With the tail
  // predicates (16 ISETP + 20 zero-inits per group) and a 64 x 64-bit address multiply the group
  // preamble was 146 SASS instructions for 8 gathers; now one VIMNMX + LDG + IMAD.WIDE
  // + LDG.128 per edge.
  // lanes beyond the row's last column gather that last column instead (same sector, no extra
  // traffic): their sums are never stored (flush tests act[]), and no load needs a predicate
  const char* inl[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++)
    inl[ch] = reinterpret_cast<const char*>(in + min((uint32_t)(lane + ch * L), p.Q - 1u));
  const uint32_t rowBytes = (uint32_t)p.ldIn * (uint32_t)sizeof(T);
  // MASK: the index row of each edge's source is gathered next to its gradient row
  const char* argl[RED == SG_RED_MASK ? NCH : 1];
  uint32_t argRowBytes = 0;
  if constexpr (RED == SG_RED_MASK) {
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
    if (cnt == (uint32_t)U) {
      const uint32_t* colp = col + base;       // full group: one address, immediate offsets
#pragma unroll
      for (int u = 0; u < U; u++) srcs[u] = __ldg(colp + u);
    } else {
#pragma unroll
      for (int u = 0; u < U; u++) srcs[u] = __ldg(col + min(base + (uint32_t)u, eLast));
    }
    T v[U][NCH];
    I av[RED == SG_RED_MASK ? U : 1][RED == SG_RED_MASK ? NCH : 1];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint64_t off = (uint64_t)srcs[u] * rowBytes;
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) v[u][ch] = V<VEC>::ld(reinterpret_cast<const T*>(inl[ch] + off));
      if constexpr (RED == SG_RED_MASK) {
        const uint64_t aoff = (uint64_t)srcs[u] * argRowBytes;
#pragma unroll
        for (int ch = 0; ch < NCH; ch++) av[u][ch] = __ldg(reinterpret_cast<const I*>(argl[ch] + aoff));
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
#pragma unroll
            for (int ch = 0; ch < NCH; ch++) {
              if constexpr (RED == SG_RED_SUM) V<VEC>::add(acc[ch], v[u][ch]);
              else if constexpr (RED == SG_RED_MASK) mask_add(acc[ch], v[u][ch], av[u][ch], p.selfBase + cur);
              else mm_add<RED>(acc[ch], aidx[ch], v[u][ch], srcs[u]);
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

// ------------------------------------------------- main kernel, variant C ---
// Same schedule, same per-row summation order, but the gathered rows are staged in
// shared memory with cp.async (LDGSTS) instead of registers: every lane copies its
// own 16 bytes of each neighbour row into a per-worker ring of DEPTH = P*GROUP row
// slots and later adds exactly the bytes it copied (no cross-lane sharing, so no
// barrier — only cp.async.wait_group).  Bytes in flight per SM are bounded by the
// ring (~100 KB per CTA) rather than by the register file, and the per-edge
// instruction count drops (one LDGSTS + one LDS.128 + 4 FADD per 16-byte column).
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)),
               "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ------------------------------------------- main kernel, variant C (lean) ---
// Variant C with the instruction stream trimmed (a first version issued
// 34 instructions per edge — generic-address arithmetic and per-edge predicates —
// and was issue-bound once the latency was hidden): 32-bit shared addresses with
// immediate slot offsets, whole-group fast paths when the group is complete and no
// row boundary falls inside it.
__device__ __forceinline__ void cp_async16_s(uint32_t saddr, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(saddr), "l"(gsrc) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr) : "memory");
  return v;
}

template <int L, int NCH, int GROUP, int P>
__global__ void __launch_bounds__(SG_THREADS, 3)
sg_chunk_kernel_c2(const SgParams p) {
  typedef float4 T;
  constexpr int WPB = SG_THREADS / L;
  constexpr uint32_t CH = SG_CH;
  constexpr uint32_t ROWB = NCH * L * 16;          // bytes per ring slot
  constexpr uint32_t GRPB = GROUP * ROWB;          // bytes per group of slots
  constexpr uint32_t RINGB = P * GRPB;             // bytes per worker ring
  extern __shared__ __align__(16) float4 sg_ring[];
  const int lane = threadIdx.x % L;
  const uint32_t w = blockIdx.x * WPB + threadIdx.x / L;
  const uint32_t ringBase = (uint32_t)__cvta_generic_to_shared(sg_ring) + (threadIdx.x / L) * RINGB + lane * 16;
  if (w >= p.numChunks) return;
  const unsigned wmask = (L == 32) ? 0xffffffffu
                                   : (((1u << L) - 1u) << (((threadIdx.x & 31) / L) * L));
  const uint32_t* __restrict__ rs = p.rs;
  const uint32_t* __restrict__ col = p.col;
  const char* inB = reinterpret_cast<const char*>(p.in) + lane * 16;
  const uint32_t strideB = (uint32_t)p.ldIn * 16u;   // bytes between input rows (ldIn is in float4 units)
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
  const uint32_t nG = (nE + GROUP - 1) / GROUP;

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
        if (epi) epi_store<4>(acc[ch], dst + ch * L, curT - curS, epi);
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

  // issue group gi into the ring slots at byte offset slotOff (= (gi % P) * GRPB).
  // Every lane of the worker reads the source id itself (same address: one broadcast
  // transaction, L1-resident): a sub-warp __shfl_sync with a runtime mask costs a
  // MATCH.ANY sequence of ~11 instructions per edge.
  (void)wmask;
  auto issue = [&](uint32_t gi, uint32_t slotOff) {
    if (gi < nG) {
      const uint32_t off = gi * GROUP;
      const uint32_t* cp = col + eb + off;
      const uint32_t sa = ringBase + slotOff;
      if (off + GROUP <= nE) {
        uint32_t srcs[GROUP];
#pragma unroll
        for (int u = 0; u < GROUP; u++) srcs[u] = __ldg(cp + u);
#pragma unroll
        for (int u = 0; u < GROUP; u++) {
          const char* g = inB + (size_t)srcs[u] * strideB;
#pragma unroll
          for (int ch = 0; ch < NCH; ch++)
            if (act[ch]) cp_async16_s(sa + u * ROWB + ch * L * 16, g + ch * L * 16);
        }
      } else {
#pragma unroll
        for (int u = 0; u < GROUP; u++) {
          if (off + u < nE) {
            const uint32_t src = __ldg(cp + u);
            const char* g = inB + (size_t)src * strideB;
#pragma unroll
            for (int ch = 0; ch < NCH; ch++)
              if (act[ch]) cp_async16_s(sa + u * ROWB + ch * L * 16, g + ch * L * 16);
          }
        }
      }
    }
    cp_async_commit();
  };
#pragma unroll 1
  for (uint32_t g = 0; g < (uint32_t)P; g++) issue(g, g * GRPB);   // one code copy: keep the kernel in the I-cache
  uint32_t slotOff = 0;
#pragma unroll 1
  for (uint32_t g = 0; g < nG; g++) {
    cp_async_wait<P - 1>();
    const uint32_t e0 = eb + g * GROUP;
    const uint32_t sa = ringBase + slotOff;
    if (segEnd - e0 >= (uint32_t)GROUP) {
      // the whole group lies inside the current row segment: no boundary tests
#pragma unroll
      for (int u = 0; u < GROUP; u++)
#pragma unroll
        for (int ch = 0; ch < NCH; ch++)
          if (act[ch]) {
            const float4 v = lds128(sa + u * ROWB + ch * L * 16);
            acc[ch].x += v.x; acc[ch].y += v.y; acc[ch].z += v.z; acc[ch].w += v.w;
          }
    } else {
#pragma unroll
      for (int u = 0; u < GROUP; u++) {
        const uint32_t ecur = e0 + u;
        if (ecur < ee) {
          while (ecur == segEnd) { flush(); advance(); }
#pragma unroll
          for (int ch = 0; ch < NCH; ch++)
            if (act[ch]) {
              const float4 v = lds128(sa + u * ROWB + ch * L * 16);
              acc[ch].x += v.x; acc[ch].y += v.y; acc[ch].z += v.z; acc[ch].w += v.w;
            }
        }
      }
    }
    issue(g + P, slotOff);
    slotOff += GRPB;
    if (slotOff == RINGB) slotOff = 0;
  }
  flush();
  while (cur + 1 < r1) { advance(); flush(); }
}

// ------------------------------------------------- main kernel, variant T ---
// Same schedule and the same per-row summation order again, but the neighbour rows are fetched by
// the TMA unit: four `cp.async.bulk` row copies per four edges (one unit) land 4 x rowBytes in the
// worker's shared-memory ring and
// completes on an mbarrier; the lanes then add with LDS.128 + FADD.  What this buys over the
// register variant A: (1) bytes in flight are bounded by the ring (P stages x S units per
// worker, ~100 KB per SM) instead of by the register file — variant A holds 8 rows per lane in
// registers, issues them as a burst, waits for all of them and only then adds, so its *average*
// bytes in flight are well under half of its peak; the ring is refilled stage by stage, so it
// stays full.  (2) the copies are issued by one lane instead of an index load + IMAD.WIDE +
// LDG.128 per lane group.  MODE 1 issues the copies of a stage one row at a time (kept for
// measurement).
// A row slot is L*NCH*16 bytes (the worker's whole lane span), so the shared-memory row pitch is a
// compile-time constant and the adds are unpredicated; lanes past the row's end add stale slot
// contents they never store.
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
  constexpr uint32_t SLOTB = NCH * L * 16;       // shared-memory bytes per gathered row
  constexpr uint32_t G4B = 4 * SLOTB;            // one four-row unit
  constexpr uint32_t STAGEB = S * G4B;
  constexpr uint32_t RINGB = P * STAGEB;
  extern __shared__ __align__(128) unsigned char sg_smem_t[];
  const int lane = threadIdx.x % L;
  const int wi = threadIdx.x / L;
  const uint32_t w = blockIdx.x * WPB + wi;
  if (w >= p.numChunks) return;
  const unsigned wmask = (L == 32) ? 0xffffffffu
                                   : (((1u << L) - 1u) << (((threadIdx.x & 31) / L) * L));
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
        if (epi) epi_store<4>(acc[ch], dst + ch * L, curT - curS, epi);
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
  const uint32_t strideB = (uint32_t)p.ldIn * 16u;
  const uint32_t rowB = p.Q * 16u;
  // MODE 2: the source ids never sit in front of the issue.  Lane j of the worker loads, once and up front, the
  // ids of units j, j + L, ... of the worker's edge range (a worker has at most 127 edges = 32 units) and
  // issues those units itself when their ring slot frees (on MODE 0 the id load of the stage about to be issued
  // is a large share of the stalls).
  constexpr int NU = (MODE == 2) ? (32 / L) : 1;
  uint4 ids[NU];
  if (MODE == 2 && nE) {
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
    if (MODE == 2) {
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
    if (k < nStages && lane == 0) {
      const uint32_t off = k * G;
      const uint32_t* cp = col + eb + off;
      const uint32_t bar = bars + slot * 8;
      const uint32_t dst = ring + slot * STAGEB;
      const uint32_t nv = min((uint32_t)G, nE - off);
      if (MODE == 0) {
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
      } else {
        mbar_expect_tx_a(bar, nv * rowB);
#pragma unroll
        for (int u = 0; u < G; u++) {
          if ((uint32_t)u < nv) {
            const uint32_t src = __ldg(cp + u);
            bulk_row(dst + u * SLOTB, inB + (size_t)src * strideB, rowB, bar);
          }
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
    const uint32_t sa = ring + slot * STAGEB + lane * 16;
    if (segEnd - e0 >= (uint32_t)G) {
      // the whole stage lies inside the current row segment
#pragma unroll
      for (int u = 0; u < G; u++)
#pragma unroll
        for (int ch = 0; ch < NCH; ch++) {
          const float4 v = lds128(sa + u * SLOTB + ch * L * 16);
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
              const float4 v = lds128(sa + u * SLOTB + ch * L * 16);
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

// ------------------------------------------------- main kernel, variant R ---
// Producer / consumer ring.  The gather of an R-MAT row mix (most row fetches hit L2) is latency-bound:
// the register-held gather of variant A is limited by the requests the register file can back, while a
// shared-memory ring filled by the TMA unit keeps more bytes in flight when (a) the ring is large, (b) the
// index loads never sit on the issue path and (c) several warps per SM issue copies.
// So: a CTA is ONE producer warp and TWO worker warps that share a two-slot ring; six CTAs per SM for rows
// of up to 256 bytes.  A slot holds one 64-edge chunk of gathered rows (64 x SLOTB bytes) and completes on
// one `full` mbarrier.  The CTA walks a contiguous range of chunk pairs; worker h owns the chunks of parity
// h and slot h holds them.  The producer's lane j (of half-warp h) holds the four source ids of unit #j
// of its chunk in registers — one coalesced LDG.128 per lane, loaded one pair ahead — and issues it as soon
// as the slot's `empty` barrier says both readers are done.
// Readers of a slot: the chunk's own worker, and the worker of the PREVIOUS chunk, whose last rows may run
// up to 63 edges into it (rows of degree <= 64 are finished by their owner).  Each of the two arrives on
// `empty` (count 2) after it has waited on `full` for that use, so every waiter sees every phase of the
// barriers it uses (a parity wait can only be one phase ahead).
// A worker is a whole warp: lane l owns VW consecutive floats of the row (float2 for rows of up to 64
// floats, so all 32 lanes work and an edge costs LDS.64 + 2 FADD), there is no second worker in the warp to
// diverge from, and the row ends of the chunk sit in a register batch (one coalesced load, read by shuffle)
// instead of being fetched one dependent load per row.  The per-row summation order is the chunk plan's, as
// in A / C / T: the results are bit-identical.
template <int VW> struct RV;
template <> struct RV<2> {
  typedef float2 T;
  static __device__ __forceinline__ T lds(uint32_t a) {
    T v; asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory"); return v;
  }
  static __device__ __forceinline__ T zero() { return make_float2(0.f, 0.f); }
  static __device__ __forceinline__ void add(T& a, const T& b) { a.x += b.x; a.y += b.y; }
  static __device__ __forceinline__ void store(T* dst, T v, uint32_t deg, int epi) {
    if (epi & ROC_SG_EPI_NORM) {
      const RowDiv rd = rowdiv_make(sqrtf((float)deg));
      float t[4] = {v.x, v.y, 0.f, 0.f};
      rowdiv4(t, rd, 2);
      v = make_float2(t[0], t[1]);
    }
    if (epi & ROC_SG_EPI_RELU) v = make_float2(relu_nanprop(v.x), relu_nanprop(v.y));
    *dst = v;
  }
};
template <> struct RV<4> {
  typedef float4 T;
  static __device__ __forceinline__ T lds(uint32_t a) { return lds128(a); }
  static __device__ __forceinline__ T zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
  static __device__ __forceinline__ void add(T& a, const T& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
  static __device__ __forceinline__ void store(T* dst, T v, uint32_t deg, int epi) {
    if (epi) epi_store<4>(v, dst, deg, epi); else *dst = v;
  }
};

template <int VW, int NCH, int NPW, int MINB>
__global__ void __launch_bounds__(32 * (NPW + 2), MINB)
sg_ring_kernel(const SgParams p, uint32_t pairsPerCta) {
  typedef typename RV<VW>::T T;
  constexpr uint32_t CH = SG_CH;
  constexpr uint32_t LANEB = VW * 4;                // bytes per lane per column block
  constexpr uint32_t SLOTB = NCH * 32 * LANEB;      // shared-memory bytes per gathered row
  constexpr uint32_t G4B = 4 * SLOTB;
  constexpr uint32_t CHUNKB = CH * SLOTB;           // one slot
  extern __shared__ __align__(128) unsigned char sg_smem_r[];
  const uint32_t ring = (uint32_t)__cvta_generic_to_shared(sg_smem_r);
  const uint32_t fullB = ring + 2 * CHUNKB, emptyB = fullB + 16;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t numPairs = (p.numChunks + 1u) >> 1;
  const uint32_t p0 = blockIdx.x * pairsPerCta;
  if (p0 >= numPairs) return;
  const uint32_t p1 = min(numPairs, p0 + pairsPerCta);
  const uint32_t nIt = p1 - p0;
  const uint32_t c0 = 2u * p0;
  const uint32_t nLoaded = (p.E + CH - 1u) / CH;           // chunks that hold at least one edge
  if (threadIdx.x == 0) {
    mbar_init_a(fullB, 1); mbar_init_a(fullB + 8, 1);
    mbar_init_a(emptyB, 2); mbar_init_a(emptyB + 8, 2);
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp < NPW) {
    // ----------------------------------------------------------- producers ---
    // NPW warps share the 32 units of a chunk pair: 32 / NPW lanes of each are active, lanes of one warp
    // always serve the same slot (so the warp sees every phase of that slot's `empty` barrier).
    constexpr int PERW = 32 / NPW;                        // units per producer warp and pair
    const int g = warp * PERW + lane;                     // unit index within the pair: 0..15 slot 0, 16..31 slot 1
    const int h = g >> 4, j = g & 15;
    const bool mine = lane < PERW;
    const uint32_t* __restrict__ col = p.col;
    const char* inB = reinterpret_cast<const char*>(p.in);
    const uint32_t strideB = (uint32_t)p.ldIn * 16u, rowB = p.Q * 16u;
    auto load_ids = [&](uint32_t c, uint4& v) {           // the four sources of unit #j of chunk c
      const uint32_t e = c * CH + 4u * (uint32_t)j;
      if (e + 4u <= p.E) {
        v = __ldg(reinterpret_cast<const uint4*>(col + e));
      } else if (e < p.E) {                                // the partial tail repeats the last edge's source
        const uint32_t last = p.E - 1u;
        v.x = __ldg(col + e); v.y = __ldg(col + min(e + 1u, last)); v.z = __ldg(col + min(e + 2u, last)); v.w = __ldg(col + min(e + 3u, last));
      } else {
        v = make_uint4(0u, 0u, 0u, 0u);
      }
    };
    if (!mine) return;
    uint4 nxt;
    load_ids(c0 + (uint32_t)h, nxt);
    // uses of slot h: it = 0 .. nIt-1, plus (h == 0 only) the chunk after the range, read by worker 1's tail
    const uint32_t uses = nIt + (h == 0 ? 1u : 0u);
#pragma unroll 1
    for (uint32_t it = 0; it < uses; it++) {
      const uint32_t c = c0 + 2u * it + (uint32_t)h;
      const uint4 ids = nxt;
      if (it + 1u < uses) load_ids(c + 2u, nxt);
      if (c < nLoaded) {
        const uint32_t nv = min(CH, p.E - c * CH);
        const uint32_t n4 = (nv + 3u) >> 2;
        mbar_wait_a(emptyB + 8u * h, (it & 1u) ^ 1u);
        if (j == 0) mbar_expect_tx_a(fullB + 8u * h, n4 * 4u * rowB);
        if ((uint32_t)j < n4)
          bulk_rows4(ring + (uint32_t)h * CHUNKB + (uint32_t)j * G4B, inB, strideB, rowB, SLOTB, ids.x, ids.y, ids.z, ids.w,
                     fullB + 8u * h);
      }
    }
    return;
  }

  // ---------------------------------------------------------------- workers ---
  const int h = warp - NPW;                                 // worker 0 / 1
  const uint32_t* __restrict__ rs = p.rs;
  const uint32_t validLanes = (p.Q * 16u + LANEB - 1u) / LANEB;      // lanes (per column block) that hold row data
  bool act[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) act[ch] = (uint32_t)(lane + ch * 32) < validLanes;
  if (h == 1) {
    // Worker 1 first reads slot 0 at its SECOND use; it has to see the first one complete before it may wait
    // for that (parity waits).  Its arrive stands in for the previous range's last worker, which reads its
    // tail from its own CTA's copy of chunk c0.
    if (c0 < nLoaded) mbar_wait_a(fullB, 0u);
    if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(emptyB) : "memory");
  }
  const uint4* __restrict__ descs = reinterpret_cast<const uint4*>(p.desc);
  uint4 d0, d1;
  {
    const uint32_t c = c0 + (uint32_t)h;
    if (c < p.numChunks) { d0 = __ldg(descs + 2 * (size_t)c); d1 = __ldg(descs + 2 * (size_t)c + 1); }
    else { d0 = make_uint4(0, 0, 0, 0); d1 = make_uint4(0, 0, 2u, 0); }
  }
  const uint32_t sa = ring + (uint32_t)lane * LANEB;
  const size_t ldOutT = p.ldOut * 4 / VW, ldCT = p.ldC * 4 / VW;     // SgParams counts rows in float4 units

#pragma unroll 1
  for (uint32_t it = 0; it < nIt; it++) {
    const uint32_t c = c0 + 2u * it + (uint32_t)h;
    // this chunk's start state; the next one's record is requested now and used next iteration
    const uint32_t eb = d0.x, ee = d0.y, r1 = d1.y, flags = d1.z, carrySlot = d1.w;
    uint32_t cur = d0.z, curS = d0.w, curT = d1.x;
    {
      const uint32_t cn = c + 2u;
      if (it + 1u < nIt && cn < p.numChunks) { d0 = __ldg(descs + 2 * (size_t)cn); d1 = __ldg(descs + 2 * (size_t)cn + 1); }
      else { d0 = make_uint4(0, 0, 0, 0); d1 = make_uint4(0, 0, 2u, 0); }
    }
    const bool idle = (flags & 2u) != 0u || c >= p.numChunks;
    const uint32_t ce = min(c * CH + CH, p.E);
    int kind = (flags & 1u) ? 0 : ((curT - curS > CH) ? 2 : 1);
    uint32_t segEnd = (kind == 1) ? curT : min(curT, ce);
    const uint32_t boundary = (c + 1u) * CH;
    // row ends of the rows after `cur`: lane i holds rs[rsBase + i] (clamped to the partition's last entry)
    uint32_t rsBase = cur + 2u;
    uint32_t rsReg = idle ? 0u : __ldg(rs + min(rsBase + (uint32_t)lane, p.nloc));

    T acc[NCH];
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) acc[ch] = RV<VW>::zero();
    auto flush = [&]() {
      T* dst = (kind == 0) ? reinterpret_cast<T*>(p.carry) + (size_t)carrySlot * ldCT
                           : reinterpret_cast<T*>(p.out) + (size_t)cur * ldOutT;
      dst += lane;
      const int epi = (kind == 1) ? p.epi : 0;
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        if (act[ch]) RV<VW>::store(dst + ch * 32, acc[ch], curT - curS, epi);
        acc[ch] = RV<VW>::zero();
      }
    };
    auto advance = [&]() {
      cur += 1; curS = curT;
      const uint32_t k = cur + 1u - rsBase;                // rs[cur + 1] is entry k of the batch
      if (k >= 32u) { rsBase = cur + 1u; rsReg = __ldg(rs + min(rsBase + (uint32_t)lane, p.nloc)); }
      curT = __shfl_sync(0xffffffffu, rsReg, (int)((cur + 1u - rsBase) & 31u));
      const bool heavy = curT - curS > CH;
      segEnd = heavy ? min(curT, ce) : curT;
      kind = heavy ? 2 : 1;
    };

    // phase 0: the worker's own chunk (slot h, use `it`); phase 1: its tail in the next chunk
    // (slot h^1; for worker 1 that is slot 0's NEXT use)
#pragma unroll 1
    for (int ph = 0; ph < 2; ph++) {
      const uint32_t s = (uint32_t)(h ^ ph);
      const uint32_t use = it + (uint32_t)(h & ph);
      const uint32_t cc = c + (uint32_t)ph;
      const bool loaded = cc < nLoaded;
      if (loaded) mbar_wait_a(fullB + 8u * s, use & 1u);
      const uint32_t eFrom = ph == 0 ? eb : max(eb, boundary);
      const uint32_t eTo = ph == 0 ? min(ee, boundary) : ee;
      if (!idle && eFrom < eTo) {
#pragma unroll 1
        for (uint32_t e0 = eFrom & ~3u; e0 < eTo; e0 += 4u) {
          const uint32_t lo = max(eFrom, e0) - e0;
          const uint32_t hi = min(eTo, e0 + 4u) - e0;
          const uint32_t a = sa + (e0 & 127u) * SLOTB;
          if (lo == 0u && hi == 4u && segEnd - e0 >= 4u) {
            T v[4][NCH];
#pragma unroll
            for (int u = 0; u < 4; u++)
#pragma unroll
              for (int ch = 0; ch < NCH; ch++) v[u][ch] = RV<VW>::lds(a + u * SLOTB + ch * 32 * LANEB);
#pragma unroll
            for (int u = 0; u < 4; u++)
#pragma unroll
              for (int ch = 0; ch < NCH; ch++) RV<VW>::add(acc[ch], v[u][ch]);
          } else {
            uint32_t pos = lo;
            for (;;) {
              const uint32_t lim = min(hi, segEnd - e0);
#pragma unroll
              for (int u = 0; u < 4; u++) {
                if ((uint32_t)u >= pos && (uint32_t)u < lim) {
#pragma unroll
                  for (int ch = 0; ch < NCH; ch++) RV<VW>::add(acc[ch], RV<VW>::lds(a + u * SLOTB + ch * 32 * LANEB));
                }
              }
              pos = max(pos, lim);
              if (pos >= hi) break;
              flush();
              advance();
            }
          }
        }
      }
      if (loaded) {
        __syncwarp();
        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(emptyB + 8u * s) : "memory");
      }
    }
    if (!idle) {
      flush();
      while (cur + 1 < r1) { advance(); flush(); }
    }
  }
}

// ----------------------------------------------------------- fix-up kernel ---
// One worker per heavy row: out[R] = epilogue(out[R] + sum_k carry[slot0 + k]), k ascending.
template <int VEC, int L, int NCH, int U>
__global__ void __launch_bounds__(SG_THREADS)
sg_fixup_kernel(const SgParams p) {
  typedef typename V<VEC>::T T;
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
  bool act[NCH];
  T acc[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) {
    act[ch] = (uint32_t)(lane + ch * L) < p.Q;
    acc[ch] = act[ch] ? V<VEC>::ld_plain(dst + lane + ch * L) : V<VEC>::zero();
  }
  for (uint32_t k = 0; k < n; k += U) {
    T v[U][NCH];
#pragma unroll
    for (int u = 0; u < U; u++)
#pragma unroll
      for (int ch = 0; ch < NCH; ch++)
        v[u][ch] = (k + u < n && act[ch]) ? V<VEC>::ld_plain(cbase + (size_t)(k + u) * p.ldC + lane + ch * L)
                                          : V<VEC>::zero();
#pragma unroll
    for (int u = 0; u < U; u++)
      if (k + u < n)
#pragma unroll
        for (int ch = 0; ch < NCH; ch++) V<VEC>::add(acc[ch], v[u][ch]);
  }
#pragma unroll
  for (int ch = 0; ch < NCH; ch++)
    if (act[ch]) epi_store<VEC>(acc[ch], dst + lane + ch * L, t - s, p.epi);
}

// Rows with more than SG_BIG carries (hubs: R-MAT-22's largest row spans 1 524 chunks) get a
// whole CTA: each of the 256/L lane groups sums a contiguous block of the carries, the blocks
// are combined in order through shared memory.  With one worker per row the hubs' serial
// chains set the kernel's duration.
constexpr uint32_t SG_BIG = 32;

template <int VEC, int L, int NCH, int U>
__global__ void __launch_bounds__(SG_THREADS)
sg_fixup_big_kernel(const SgParams p) {
  typedef typename V<VEC>::T T;
  constexpr int WPB = SG_THREADS / L;
  constexpr uint32_t CH = SG_CH;
  __shared__ __align__(16) float part[WPB * NCH * L * VEC];
  const int lane = threadIdx.x % L;
  const int g = threadIdx.x / L;
  const uint32_t R = p.bigRows[blockIdx.x];
  const uint32_t s = p.rs[R], t = p.rs[R + 1];
  const uint32_t c0 = s / CH, cLast = (t - 1) / CH;
  const uint32_t n = cLast - c0;
  const uint32_t slot0 = p.carryIdx[c0 + 1];
  const T* cbase = reinterpret_cast<const T*>(p.carry) + (size_t)slot0 * p.ldC;
  const uint32_t per = (n + WPB - 1) / WPB;
  const uint32_t k0 = min(n, (uint32_t)g * per), k1 = min(n, k0 + per);
  bool act[NCH];
  T acc[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) { act[ch] = (uint32_t)(lane + ch * L) < p.Q; acc[ch] = V<VEC>::zero(); }
  for (uint32_t k = k0; k < k1; k += U) {
    T v[U][NCH];
#pragma unroll
    for (int u = 0; u < U; u++)
#pragma unroll
      for (int ch = 0; ch < NCH; ch++)
        v[u][ch] = (k + u < k1 && act[ch]) ? V<VEC>::ld_plain(cbase + (size_t)(k + u) * p.ldC + lane + ch * L)
                                           : V<VEC>::zero();
#pragma unroll
    for (int u = 0; u < U; u++)
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) V<VEC>::add(acc[ch], v[u][ch]);
  }
  T* sp = reinterpret_cast<T*>(part);
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) sp[(g * NCH + ch) * L + lane] = acc[ch];
  __syncthreads();
  if (g == 0) {
    T* dst = reinterpret_cast<T*>(p.out) + (size_t)R * p.ldOut;
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) {
      if (act[ch]) {
        T a = V<VEC>::ld_plain(dst + lane + ch * L);      // the owner chunk's raw partial
        for (int gg = 0; gg < WPB; gg++) V<VEC>::add(a, sp[(gg * NCH + ch) * L + lane]);
        epi_store<VEC>(a, dst + lane + ch * L, t - s, p.epi);
      }
    }
  }
}

// Min / max: one worker per heavy row takes the owner's partial (out[R], arg[R]), then the carries, k ascending,
// with the same ordering rule.
template <int VEC, int L, int NCH, int U, int RED>
__global__ void __launch_bounds__(SG_THREADS)
sg_fixup_minmax_kernel(const SgParams p) {
  typedef typename V<VEC>::T T;
  typedef typename V<VEC>::I I;
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
  bool act[NCH];
  T acc[NCH];
  I* adst = reinterpret_cast<I*>(p.arg) + (size_t)R * p.ldArg;
  const I* abase = reinterpret_cast<const I*>(p.carryArg) + (size_t)slot0 * p.ldC;
  I ai[NCH];
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) {
    act[ch] = (uint32_t)(lane + ch * L) < p.Q;
    acc[ch] = act[ch] ? V<VEC>::ld_plain(dst + lane + ch * L) : V<VEC>::zero();
    ai[ch] = act[ch] ? adst[lane + ch * L] : mm_noarg((I*)nullptr);
  }
  for (uint32_t k = 0; k < n; k += U) {
    T v[U][NCH];
    I vi[U][NCH];
#pragma unroll
    for (int u = 0; u < U; u++)
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        const bool ok = k + u < n && act[ch];
        v[u][ch] = ok ? V<VEC>::ld_plain(cbase + (size_t)(k + u) * p.ldC + lane + ch * L) : V<VEC>::zero();
        vi[u][ch] = ok ? abase[(size_t)(k + u) * p.ldC + lane + ch * L] : mm_noarg((I*)nullptr);
      }
#pragma unroll
    for (int u = 0; u < U; u++)
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) mm_combine<RED>(acc[ch], ai[ch], v[u][ch], vi[u][ch]);
  }
#pragma unroll
  for (int ch = 0; ch < NCH; ch++)
    if (act[ch]) { V<VEC>::st(dst + lane + ch * L, acc[ch]); adst[lane + ch * L] = ai[ch]; }
}

// Min / max rows with more than SG_BIG carries: each lane group reduces its block of carries in order, then group 0
// takes the owner's partial and the groups' results in group order — chunk order again.
template <int VEC, int L, int NCH, int U, int RED>
__global__ void __launch_bounds__(SG_THREADS)
sg_fixup_big_minmax_kernel(const SgParams p) {
  typedef typename V<VEC>::T T;
  typedef typename V<VEC>::I I;
  constexpr int WPB = SG_THREADS / L;
  constexpr uint32_t CH = SG_CH;
  __shared__ __align__(16) float part[WPB * NCH * L * VEC];
  __shared__ __align__(16) uint32_t parti[WPB * NCH * L * VEC];
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
    act[ch] = (uint32_t)(lane + ch * L) < p.Q; acc[ch] = V<VEC>::zero(); ai[ch] = mm_noarg((I*)nullptr);
  }
  for (uint32_t k = k0; k < k1; k += U) {
    T v[U][NCH];
    I vi[U][NCH];
#pragma unroll
    for (int u = 0; u < U; u++)
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) {
        const bool ok = k + u < k1 && act[ch];
        v[u][ch] = ok ? V<VEC>::ld_plain(cbase + (size_t)(k + u) * p.ldC + lane + ch * L) : V<VEC>::zero();
        vi[u][ch] = ok ? abase[(size_t)(k + u) * p.ldC + lane + ch * L] : mm_noarg((I*)nullptr);
      }
#pragma unroll
    for (int u = 0; u < U; u++)
#pragma unroll
      for (int ch = 0; ch < NCH; ch++) mm_combine<RED>(acc[ch], ai[ch], v[u][ch], vi[u][ch]);
  }
  T* sp = reinterpret_cast<T*>(part);
  I* spi = reinterpret_cast<I*>(parti);
#pragma unroll
  for (int ch = 0; ch < NCH; ch++) { sp[(g * NCH + ch) * L + lane] = acc[ch]; spi[(g * NCH + ch) * L + lane] = ai[ch]; }
  __syncthreads();
  if (g == 0) {
    T* dst = reinterpret_cast<T*>(p.out) + (size_t)R * p.ldOut;
    I* adst = reinterpret_cast<I*>(p.arg) + (size_t)R * p.ldArg;
#pragma unroll
    for (int ch = 0; ch < NCH; ch++) {
      if (act[ch]) {
        T a = V<VEC>::ld_plain(dst + lane + ch * L);      // the owner chunk's partial
        I ia = adst[lane + ch * L];
        for (int gg = 0; gg < WPB; gg++) mm_combine<RED>(a, ia, sp[(gg * NCH + ch) * L + lane], spi[(gg * NCH + ch) * L + lane]);
        V<VEC>::st(dst + lane + ch * L, a);
        adst[lane + ch * L] = ia;
      }
    }
  }
}

// Variant A keeps the gathers in registers, variant C stages them in shared memory with
// cp.async; C wins once a row needs two or more float4 per lane at L = 32 (H > 128).
// ROC_SG_VARIANT=a|c forces one (experiments / cross-checks).
static int sg_variant_env() {   // -1 default, 0 = A, 2 = C, 3 = T (bulk-copy ring), 4 = T with per-stage ids and one copy per row, 5 = R (ring)
  const char* e = getenv("ROC_SG_VARIANT");   // re-read per call: the kernel bench switches it in-process
  if (!e) return -1;
  switch (e[0]) { case 'a': return 0; case 'c': return 2; case 't': return 3; case 'b': return 4; case 'r': return 5; case 'u': return 6; default: return -1; }
}
static int sg_deep_env() {   // ROC_SG_DEEP=1: variant C with a 2x deeper ring (experiments)
  const char* e = getenv("ROC_SG_DEEP");
  return (e && e[0] == '1') ? 1 : 0;
}
static int sg_tcfg_env() {   // ROC_SG_TCFG=<n>: ring shape of variant T (experiments; see launch_t_cfg)
  const char* e = getenv("ROC_SG_TCFG");
  return e ? atoi(e) : -1;
}

template <int L, int NCH, int GROUP, int P>
static cudaError_t launch_c(const SgParams& p, unsigned grid, cudaStream_t st) {
  constexpr int WPB = SG_THREADS / L;
  constexpr size_t smem = (size_t)WPB * GROUP * P * NCH * L * sizeof(float4);
  static std::atomic<uint64_t> configured{0};      // one bit per device: the attribute is per device
  cudaError_t e = once_per_device(configured, [] {
    return cudaFuncSetAttribute(sg_chunk_kernel_c2<L, NCH, GROUP, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  });
  if (e != cudaSuccess) return e;
  sg_chunk_kernel_c2<L, NCH, GROUP, P><<<grid, SG_THREADS, smem, st>>>(p);
  return cudaGetLastError();
}

// ---- variant T launchers: ring = P stages x S four-row units per worker, NT threads per CTA
template <int L, int NCH, int S, int P, int NT, int MINB, int MODE>
static cudaError_t launch_t(const SgParams& p, cudaStream_t st) {
  constexpr int WPB = NT / L;
  constexpr size_t smem = (size_t)WPB * P * S * 4 * NCH * L * 16 + (size_t)WPB * P * 8;
  static_assert(smem <= 227 * 1024, "ring too large");
  static std::atomic<uint64_t> configured{0};
  cudaError_t e = once_per_device(configured, [] {
    return cudaFuncSetAttribute(sg_chunk_kernel_t<L, NCH, S, P, NT, MINB, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  });
  if (e != cudaSuccess) return e;
  const unsigned grid = (p.numChunks + WPB - 1) / WPB;
  sg_chunk_kernel_t<L, NCH, S, P, NT, MINB, MODE><<<grid, NT, smem, st>>>(p);
  return cudaGetLastError();
}

// ---- variant R launcher: NPW producer warps + two worker warps per CTA, MINB CTAs per SM
template <int VW, int NCH, int NPW, int MINB>
static cudaError_t launch_r(const SgParams& p, cudaStream_t st) {
  constexpr size_t smem = (size_t)2 * SG_CH * NCH * 32 * VW * 4 + 64;
  static_assert(smem * MINB <= 227 * 1024, "ring too large");
  static std::atomic<uint64_t> configured{0};
  cudaError_t e = once_per_device(configured, [] {
    return cudaFuncSetAttribute(sg_ring_kernel<VW, NCH, NPW, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  });
  if (e != cudaSuccess) return e;
  const uint32_t numPairs = (p.numChunks + 1u) >> 1;
  uint32_t grid = (uint32_t)sm_count() * MINB * 2u;        // two CTA ranges per resident slot
  if (grid > numPairs) grid = numPairs;
  const uint32_t per = (numPairs + grid - 1) / grid;
  grid = (numPairs + per - 1) / per;
  sg_ring_kernel<VW, NCH, NPW, MINB><<<grid, 32 * (NPW + 2), smem, st>>>(p, per);
  return cudaGetLastError();
}
// rows of up to 256 / 512 / 1024 bytes: 32 / 64 / 128 KB of ring per CTA.  cfg = producer warps (experiments)
static cudaError_t launch_r_cfg(const SgParams& p, int cfg, cudaStream_t st) {
  if (p.Q <= 16) {
    switch (cfg) {
      case 1: return launch_r<2, 1, 1, 6>(p, st);
      case 4: return launch_r<2, 1, 4, 6>(p, st);
      default: return launch_r<2, 1, 2, 6>(p, st);
    }
  }
  if (p.Q <= 32) {
    switch (cfg) {
      case 1: return launch_r<4, 1, 1, 3>(p, st);
      case 4: return launch_r<4, 1, 4, 3>(p, st);
      default: return launch_r<4, 1, 2, 3>(p, st);
    }
  }
  switch (cfg) {
    case 1: return launch_r<4, 2, 1, 1>(p, st);
    case 4: return launch_r<4, 2, 4, 1>(p, st);
    default: return launch_r<4, 2, 2, 1>(p, st);
  }
}

// Ring shapes.  cfg < 0: the default for this width (chosen by measurement, DESIGN.md §3.1).
template <int L, int NCH, int MODE>
static cudaError_t launch_t_cfg(const SgParams& p, int cfg, cudaStream_t st) {
  // bytes per row slot = NCH*L*16; per worker ring = P*S*4 slots
  if constexpr (NCH * L <= 16) {          // rows <= 256 B: 2+ workers per warp
    switch (cfg) {
      case 1: return launch_t<L, NCH, 2, 2, 128, 4, MODE>(p, st);
      case 2: return launch_t<L, NCH, 1, 8, 128, 3, MODE>(p, st);
      case 3: return launch_t<L, NCH, 2, 4, 128, 3, MODE>(p, st);
      case 4: return launch_t<L, NCH, 1, 4, 256, 3, MODE>(p, st);
      case 5: return launch_t<L, NCH, 1, 3, 128, 8, MODE>(p, st);
      case 6: return launch_t<L, NCH, 1, 6, 128, 4, MODE>(p, st);
      default: return launch_t<L, NCH, 1, 4, 128, 6, MODE>(p, st);
    }
  } else if constexpr (NCH == 1) {        // 512 B rows, one worker per warp
    if (cfg < 0 && MODE == 2) cfg = 1;     // ids held by the lanes: two 8-edge stages
    switch (cfg) {
      case 1: return launch_t<L, NCH, 2, 2, 128, 4, MODE>(p, st);
      case 2: return launch_t<L, NCH, 1, 8, 128, 3, MODE>(p, st);
      case 3: return launch_t<L, NCH, 1, 3, 128, 8, MODE>(p, st);
      default: return launch_t<L, NCH, 1, 4, 128, 6, MODE>(p, st);
    }
  } else {                                 // 1 KB rows: two 4 KB stages per warp, 6 CTAs
    switch (cfg) {
      case 1: return launch_t<L, NCH, 1, 4, 128, 3, MODE>(p, st);
      case 2: return launch_t<L, NCH, 1, 6, 128, 2, MODE>(p, st);
      case 3: return launch_t<L, NCH, 1, 3, 128, 4, MODE>(p, st);
      default: return launch_t<L, NCH, 1, 2, 128, 6, MODE>(p, st);
    }
  }
}

// variant C rings: DEPTH = GROUP * P row slots per worker, 64 KB per CTA (128 KB with ROC_SG_DEEP=1)
template <int L, int NCH>
static cudaError_t launch_c_cfg(const SgParams& p, unsigned grid, cudaStream_t st) {
  const bool deep = sg_deep_env() == 1;
  if constexpr (NCH == 1) return deep ? launch_c<L, NCH, 4, 8>(p, grid, st) : launch_c<L, NCH, 4, 4>(p, grid, st);
  else if constexpr (NCH == 2) return deep ? launch_c<L, NCH, 2, 8>(p, grid, st) : launch_c<L, NCH, 2, 4>(p, grid, st);
  else if constexpr (NCH == 4) return deep ? launch_c<L, NCH, 1, 8>(p, grid, st) : launch_c<L, NCH, 1, 4>(p, grid, st);
  else return deep ? launch_c<L, NCH, 1, 4>(p, grid, st) : launch_c<L, NCH, 1, 2>(p, grid, st);
}

struct SgLaunch {
  int variant;               // 0 = A, 2 = C, 3 = T (bulk-copy ring), 4 = T (one copy per row)
  int tcfg;                  // ring shape of variant T (-1 = default)
};

// Min / max forward (MAX, MIN) and its backward (MASK): kernel A and its fix-ups only.  The backward's partials are
// sums, so it uses the sum fix-ups.
template <int VEC, int L, int NCH, int U, int MINB, int RED>
static int launch_red(const SgParams& p, cudaStream_t st) {
  constexpr int WPB = SG_THREADS / L;
  if (p.numChunks) {
    sg_chunk_kernel<VEC, L, NCH, U, MINB, RED><<<(p.numChunks + WPB - 1) / WPB, SG_THREADS, 0, st>>>(p);
    ROC_LAUNCH_CHECK();
  }
  if (p.numHeavy) {
    if constexpr (RED == SG_RED_MASK) sg_fixup_kernel<VEC, L, NCH, U><<<(p.numHeavy + WPB - 1) / WPB, SG_THREADS, 0, st>>>(p);
    else sg_fixup_minmax_kernel<VEC, L, NCH, U, RED><<<(p.numHeavy + WPB - 1) / WPB, SG_THREADS, 0, st>>>(p);
    ROC_LAUNCH_CHECK();
  }
  if (p.numBig) {
    if constexpr (RED == SG_RED_MASK) sg_fixup_big_kernel<VEC, L, NCH, U><<<p.numBig, SG_THREADS, 0, st>>>(p);
    else sg_fixup_big_minmax_kernel<VEC, L, NCH, U, RED><<<p.numBig, SG_THREADS, 0, st>>>(p);
    ROC_LAUNCH_CHECK();
  }
  return ROC_OK;
}

// Column blocks of the min / max entry points: 128 T-columns vectorised (512 floats: the big-row fix-up keeps values
// and indices of every lane group in static shared memory), 256 scalar.  Gathers in flight (U) are lowered where the
// index per float (forward) or the second gathered row (backward) would otherwise spill under kernel A's occupancy.
template <int VEC, int RED>
static int dispatch_red(const SgParams& p, cudaStream_t st) {
  constexpr bool B = RED == SG_RED_MASK;
  const uint32_t Q = p.Q;
  if (Q <= 4) return launch_red<VEC, 4, 1, 4, 4, RED>(p, st);
  if (Q <= 8) return launch_red<VEC, 8, 1, 4, 4, RED>(p, st);
  if (Q <= 16) return launch_red<VEC, 16, 1, 4, 4, RED>(p, st);
  if (Q <= 32) return launch_red<VEC, 32, 1, 4, 4, RED>(p, st);
  if (Q <= 64) return launch_red<VEC, 32, 2, B ? 2 : 4, 3, RED>(p, st);
  if (Q <= 128) return launch_red<VEC, 32, 4, 1, 3, RED>(p, st);
  if constexpr (VEC == 1) {
    if (Q <= 256) return launch_red<VEC, 32, 8, 1, 2, RED>(p, st);
  }
  return ROC_ERR_UNSUPPORTED;
}

template <int VEC, int L, int NCH, int U, int MINB>
static int launch_cfg(const SgParams& p, const SgLaunch& how, cudaStream_t st) {
  constexpr int WPB = SG_THREADS / L;
  if (p.numChunks) {
    unsigned grid = (p.numChunks + WPB - 1) / WPB;
    int variant = how.variant;
    bool done = false;
    if constexpr (VEC == 4 && NCH <= 2 && L >= 16) {
      if (variant == 5) {
        cudaError_t e = launch_r_cfg(p, how.tcfg, st);
        if (e != cudaSuccess) return (int)e;
        count_launch();
        done = true;
      }
    }
    if constexpr (VEC == 4 && NCH <= 2 && L >= 16) {
      if (variant == 6) {
        cudaError_t e = launch_t_cfg<L, NCH, 2>(p, how.tcfg, st);
        if (e != cudaSuccess) return (int)e;
        count_launch();
        done = true;
      }
    }
    if constexpr (VEC == 4 && NCH <= 2) {
      if (variant == 3 || variant == 4) {
        cudaError_t e = (variant == 3) ? launch_t_cfg<L, NCH, 0>(p, how.tcfg, st)
                                       : launch_t_cfg<L, NCH, 1>(p, how.tcfg, st);
        if (e != cudaSuccess) return (int)e;
        count_launch();
        done = true;
      }
    }
    if constexpr (VEC == 4) {
      if (!done && variant == 2) {
        cudaError_t e = launch_c_cfg<L, NCH>(p, grid, st);
        if (e != cudaSuccess) return (int)e;
        count_launch();
        done = true;
      }
    }
    if (!done) {
      sg_chunk_kernel<VEC, L, NCH, U, MINB><<<grid, SG_THREADS, 0, st>>>(p);
      ROC_LAUNCH_CHECK();
    }
  }
  if (p.numHeavy) {
    unsigned grid = (p.numHeavy + WPB - 1) / WPB;
    sg_fixup_kernel<VEC, L, NCH, U><<<grid, SG_THREADS, 0, st>>>(p);
    ROC_LAUNCH_CHECK();
  }
  if (p.numBig) {
    sg_fixup_big_kernel<VEC, L, NCH, U><<<p.numBig, SG_THREADS, 0, st>>>(p);
    ROC_LAUNCH_CHECK();
  }
  return ROC_OK;
}

template <int VEC>
static int dispatch(const SgParams& p, const SgLaunch& how, cudaStream_t st) {
  const uint32_t Q = p.Q;
  if (Q <= 4) return launch_cfg<VEC, 4, 1, 4, 4>(p, how, st);
  if (Q <= 8) return launch_cfg<VEC, 8, 1, 8, 4>(p, how, st);
  if (Q <= 16) return launch_cfg<VEC, 16, 1, 8, 4>(p, how, st);
  if (Q <= 32) return launch_cfg<VEC, 32, 1, 8, 4>(p, how, st);
  if (Q <= 64) return launch_cfg<VEC, 32, 2, 4, 3>(p, how, st);
  if (Q <= 128) return launch_cfg<VEC, 32, 4, 2, 3>(p, how, st);
  if (Q <= 256) return launch_cfg<VEC, 32, 8, 1, 2>(p, how, st);
  return ROC_ERR_UNSUPPORTED;
}

// The variant for a vectorised launch of Q float4 columns.  Default: chosen by measurement per width
// (DESIGN.md §3.1); ROC_SG_VARIANT=a|c|t|b forces one (experiments / cross-checks).
static int pick_variant(uint32_t Q, bool vec) {
  int v = sg_variant_env();
  if (!vec) return 0;
  // measured on R-MAT-22 (H100, ms at H = 41 / 64 / 128 / 256): A 3.23 / 3.56 / 8.26 / 19.04, C 3.94 / 3.89 / 8.27 /
  // 19.03, T 4.14 / 4.09 / 8.28 / 19.07, T with lane-held ids (U) 3.88 / 3.78 / 8.23 / 18.95, R 4.03 / 4.02 / 8.59 / 24.0
  // -> registers up to 64 floats; beyond, every kernel but R is within 1 %: the ring with lane-held ids for 65..128,
  // with per-stage ids for 129..256
  if (v < 0) v = (Q > 64) ? 2 : (Q > 32 ? 3 : (Q > 16 ? 6 : 0));
  if ((v == 3 || v == 4 || v == 5 || v == 6) && Q > 64) v = 2;     // the ring kernels take rows of at most 256 floats
  if ((v == 5 || v == 6) && Q <= 8) v = 0;                // these want rows of 9+ float4
  return v;
}

// Carry slots for rows cut at chunk boundaries.  roc_sg_plan_reserve sizes them up front (plain cudaMalloc, an
// init-time call).  A launch that still finds them too small grows them on its own stream with stream-ordered
// allocation: the old buffer is returned in stream order, after the launches that used it — no device
// synchronisation in the middle of a step.
static int ensure_carry(roc_sg_plan* plan, size_t ldFloats, cudaStream_t st, bool inStream) {
  if (plan->numCarries == 0 || ldFloats <= plan->carryLd) return ROC_OK;
  if (plan->carry) {
    if (inStream) ROC_CUDA(cudaFreeAsync(plan->carry, st));
    else { ROC_CUDA(cudaDeviceSynchronize()); ROC_CUDA(cudaFree(plan->carry)); }
    plan->carry = nullptr; plan->carryLd = 0;
  }
  const size_t bytes = (size_t)plan->numCarries * ldFloats * sizeof(float);
  cudaError_t e = inStream ? cudaMallocAsync((void**)&plan->carry, bytes, st) : cudaMalloc((void**)&plan->carry, bytes);
  if (e != cudaSuccess) { plan->carry = nullptr; plan->carryLd = 0; return (int)e; }
  plan->carryLd = ldFloats;
  return ROC_OK;
}

// The index carries of the min / max forward: u32 [numCarries][carryLd], the shape of the float carries (the kernels
// address both with one leading dimension), grown the same way.
static int ensure_carry_arg(roc_sg_plan* plan, cudaStream_t st) {
  if (plan->numCarries == 0 || plan->carryArgLd == plan->carryLd) return ROC_OK;
  if (plan->carryArg) {
    ROC_CUDA(cudaFreeAsync(plan->carryArg, st));
    plan->carryArg = nullptr; plan->carryArgLd = 0;
  }
  const size_t bytes = (size_t)plan->numCarries * plan->carryLd * sizeof(uint32_t);
  cudaError_t e = cudaMallocAsync((void**)&plan->carryArg, bytes, st);
  if (e != cudaSuccess) { plan->carryArg = nullptr; plan->carryArgLd = 0; return (int)e; }
  plan->carryArgLd = plan->carryLd;
  return ROC_OK;
}

}  // namespace roc

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
  cudaFree(pl->carryArg);
  delete pl;
}

extern "C" int roc_sg_plan_reserve(roc_sg_plan* pl, int maxH) {
  if (!pl || maxH <= 0) return ROC_ERR_INVALID;
  return ensure_carry(pl, ((size_t)maxH + 3) / 4 * 4, nullptr, false);
}

extern "C" int roc_sg_plan_info(const roc_sg_plan* pl, uint64_t* numChunks, uint64_t* numCarries,
                                uint64_t* numHeavyRows) {
  if (!pl) return ROC_ERR_INVALID;
  if (numChunks) *numChunks = pl->numChunks;
  if (numCarries) *numCarries = pl->numCarries;
  if (numHeavyRows) *numHeavyRows = (uint64_t)pl->numHeavy + pl->numBig;
  return ROC_OK;
}

extern "C" int roc_sg_forward_planned(const roc_sg_plan* plc, int H, const float* in, int64_t ldIn,
                                      float* out, int64_t ldOut, int epilogue, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  if (!pl || H <= 0 || !in || !out || ldIn < H || ldOut < H) return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  const bool vec = (ldIn % 4 == 0) && (ldOut % 4 == 0) && aligned16(in) && aligned16(out);
  // column blocks: the widest kernel covers 256 T-columns (1024 floats vectorised, 256 scalar);
  // the ring variants take 64 T-columns (they are instantiated for rows of at most 256 floats)
  int variant = pick_variant(vec ? ((uint32_t)H + 3) / 4 : (uint32_t)H, vec);
  if ((variant == 3 || variant == 4 || variant == 5 || variant == 6) && H > 256 && sg_variant_env() < 0) variant = 2;
  const int blockCols = !vec ? 256 : ((variant == 3 || variant == 4 || variant == 5 || variant == 6) ? 256 : 1024);
  {
    int need = H < blockCols ? H : blockCols;
    int rc = ensure_carry(pl, ((size_t)need + 3) / 4 * 4, st, true);
    if (rc != ROC_OK) return rc;
  }
  for (int c0 = 0; c0 < H; c0 += blockCols) {
    int hb = (H - c0 < blockCols) ? H - c0 : blockCols;
    SgParams p;
    p.rs = pl->rs; p.firstRow = pl->firstRow; p.carryIdx = pl->carryIdx; p.heavyRows = pl->heavyRows; p.bigRows = pl->bigRows;
    p.col = pl->col; p.in = in + c0; p.out = out + c0; p.carry = pl->carry;
    p.E = pl->E; p.numChunks = pl->numChunks; p.numHeavy = pl->numHeavy; p.numBig = pl->numBig; p.epi = epilogue;
    p.dense = (pl->nloc > 0 && pl->E / pl->nloc >= (uint32_t)SG_CH) ? 1 : 0;
    p.desc = pl->desc; p.nloc = pl->nloc;
    SgLaunch how;
    how.variant = variant; how.tcfg = sg_tcfg_env();
    int rc;
    if (vec) {
      p.ldIn = (size_t)ldIn / 4; p.ldOut = (size_t)ldOut / 4; p.ldC = pl->carryLd / 4;
      p.Q = ((uint32_t)hb + 3) / 4;
      if (variant == 5 && (!aligned16(pl->col) || p.Q <= 8)) how.variant = 0;   // producer reads col as uint4
      rc = dispatch<4>(p, how, st);
    } else {
      p.ldIn = (size_t)ldIn; p.ldOut = (size_t)ldOut; p.ldC = pl->carryLd;
      p.Q = (uint32_t)hb;
      rc = dispatch<1>(p, how, st);
    }
    if (rc != ROC_OK) return rc;
  }
  return ROC_OK;
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

// The plan parameters shared by every launch of column block c0 (units of T applied by the caller).
static SgParams plan_params(const roc_sg_plan* pl) {
  SgParams p;
  memset(&p, 0, sizeof(p));
  p.rs = pl->rs; p.firstRow = pl->firstRow; p.carryIdx = pl->carryIdx; p.heavyRows = pl->heavyRows; p.bigRows = pl->bigRows;
  p.col = pl->col; p.carry = pl->carry; p.carryArg = pl->carryArg;
  p.E = pl->E; p.numChunks = pl->numChunks; p.numHeavy = pl->numHeavy; p.numBig = pl->numBig; p.epi = 0;
  p.desc = pl->desc; p.nloc = pl->nloc;
  return p;
}

extern "C" int roc_sg_minmax_forward_planned(const roc_sg_plan* plc, int aggr, int H, const float* in, int64_t ldIn,
                                             float* out, int64_t ldOut, roc_vid_t* arg, int64_t ldArg,
                                             roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  if (!pl || (aggr != ROC_SG_AGGR_MAX && aggr != ROC_SG_AGGR_MIN) || H <= 0 || !in || !out || !arg || ldIn < H ||
      ldOut < H || ldArg < H)
    return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  const bool vec = (ldIn % 4 == 0) && (ldOut % 4 == 0) && (ldArg % 4 == 0) && aligned16(in) && aligned16(out) &&
                   aligned16(arg);
  const int blockCols = vec ? 512 : 256;
  {
    int need = H < blockCols ? H : blockCols;
    int rc = ensure_carry(pl, ((size_t)need + 3) / 4 * 4, st, true);
    if (rc != ROC_OK) return rc;
    rc = ensure_carry_arg(pl, st);
    if (rc != ROC_OK) return rc;
  }
  for (int c0 = 0; c0 < H; c0 += blockCols) {
    const int hb = (H - c0 < blockCols) ? H - c0 : blockCols;
    SgParams p = plan_params(pl);
    p.in = in + c0; p.out = out + c0; p.arg = arg + c0;
    int rc;
    if (vec) {
      p.ldIn = (size_t)ldIn / 4; p.ldOut = (size_t)ldOut / 4; p.ldArg = (size_t)ldArg / 4; p.ldC = pl->carryLd / 4;
      p.Q = ((uint32_t)hb + 3) / 4;
      rc = aggr == ROC_SG_AGGR_MAX ? dispatch_red<4, SG_RED_MAX>(p, st) : dispatch_red<4, SG_RED_MIN>(p, st);
    } else {
      p.ldIn = (size_t)ldIn; p.ldOut = (size_t)ldOut; p.ldArg = (size_t)ldArg; p.ldC = pl->carryLd;
      p.Q = (uint32_t)hb;
      rc = aggr == ROC_SG_AGGR_MAX ? dispatch_red<1, SG_RED_MAX>(p, st) : dispatch_red<1, SG_RED_MIN>(p, st);
    }
    if (rc != ROC_OK) return rc;
  }
  return ROC_OK;
}

extern "C" int roc_sg_minmax_backward_planned(const roc_sg_plan* plc, int H, roc_vid_t selfBase, const float* outGrad,
                                              int64_t ldG, const roc_vid_t* arg, int64_t ldArg, float* inGrad,
                                              int64_t ldIn, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  if (!pl || H <= 0 || !outGrad || !arg || !inGrad || ldG < H || ldArg < H || ldIn < H) return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  const bool vec = (ldG % 4 == 0) && (ldArg % 4 == 0) && (ldIn % 4 == 0) && aligned16(outGrad) && aligned16(arg) &&
                   aligned16(inGrad);
  const int blockCols = vec ? 512 : 256;
  {
    int need = H < blockCols ? H : blockCols;
    int rc = ensure_carry(pl, ((size_t)need + 3) / 4 * 4, st, true);
    if (rc != ROC_OK) return rc;
  }
  for (int c0 = 0; c0 < H; c0 += blockCols) {
    const int hb = (H - c0 < blockCols) ? H - c0 : blockCols;
    SgParams p = plan_params(pl);
    p.in = outGrad + c0; p.out = inGrad + c0; p.arg = const_cast<roc_vid_t*>(arg) + c0; p.selfBase = selfBase;
    int rc;
    if (vec) {
      p.ldIn = (size_t)ldG / 4; p.ldOut = (size_t)ldIn / 4; p.ldArg = (size_t)ldArg / 4; p.ldC = pl->carryLd / 4;
      p.Q = ((uint32_t)hb + 3) / 4;
      rc = dispatch_red<4, SG_RED_MASK>(p, st);
    } else {
      p.ldIn = (size_t)ldG; p.ldOut = (size_t)ldIn; p.ldArg = (size_t)ldArg; p.ldC = pl->carryLd;
      p.Q = (uint32_t)hb;
      rc = dispatch_red<1, SG_RED_MASK>(p, st);
    }
    if (rc != ROC_OK) return rc;
  }
  return ROC_OK;
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
