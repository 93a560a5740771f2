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
//  * the main kernel, sg_chunk_kernel, gathers the neighbour rows in registers.  A row is Q T-columns (float4
//    when the rows are 16-byte aligned, else float); a worker is L = 4, 8, 16 or 32 lanes, the fewest that cover
//    Q, and each lane loads its NCH = ceil(Q / L) columns of U rows per group.  A launch covers up to 256
//    T-columns (1024 floats vectorised, 256 scalar); wider rows are split into column blocks.
//  * vectorised rows of 65..256 floats run on sg_chunk_kernel_t instead, which fetches them with cp.async.bulk
//    copies into a shared-memory ring: it was faster there on a products-shaped graph (DESIGN.md §3.1).  It
//    shares the plan and the per-row summation order, so its results are bit-identical to sg_chunk_kernel's.
//  * min / max aggregation (roc_sg_minmax_*) runs the same kernel and fix-ups templated on the reduction; its
//    backward is the sum schedule with a second gathered row and a predicated add, finished by the sum's fix-ups.
//    The three planned entry points check their arguments and share one column-block driver (run_planned).
//
// Algorithmic bytes per launch (DESIGN.md): E*(4H+4) + Nloc*(4H+8); min / max forward E*(4H+4) + Nloc*(8H+8),
// backward E*(8H+4) + Nloc*(4H+8).
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
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
  const uint32_t* desc; // [numChunks][8] chunk start records (k_chunk_desc)
  // min / max aggregation
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
// the lanes that issue them.
// A row slot is L*NCH*16 bytes (the worker's whole lane span), so the shared-memory row pitch is a
// compile-time constant and the adds are unpredicated; lanes past the row's end add stale slot
// contents they never store.
__device__ __forceinline__ float4 lds128(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr) : "memory");
  return v;
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

// ---------------------------------------------------------- fix-up kernels ---
// A row cut at chunk boundaries is finished from its owner's partial (out[R]; arg[R] for MAX / MIN) and its carries,
// taken in chunk order: added for the sum (whose partials include the min / max backward's), combined by the
// ordering rule for MAX / MIN.  Only the sum has an epilogue.
// U carries are loaded per batch.  The carries are taken in chunk order whatever U is, so U never changes a result;
// MAX / MIN take fewer per batch where their index carries would otherwise spill.
__host__ __device__ constexpr int sg_fixup_u(int L, int NCH, int RED) {
  return RED == SG_RED_SUM ? (NCH == 1 ? (L == 4 ? 4 : 8) : 8 / NCH) : (NCH <= 2 ? 4 : 1);
}

// One worker per heavy row.
template <int VEC, int L, int NCH, int RED>
__global__ void __launch_bounds__(SG_THREADS)
sg_fixup_kernel(const SgParams p) {
  typedef typename V<VEC>::T T;
  typedef typename V<VEC>::I I;
  constexpr bool MM = RED != SG_RED_SUM;
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
      else epi_store<VEC>(acc[ch], dst + lane + ch * L, t - s, p.epi);
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
  constexpr bool MM = RED != SG_RED_SUM;
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
        epi_store<VEC>(a, dst + lane + ch * L, t - s, p.epi);
      }
    }
  }
}

// sg_chunk_kernel_t's two shapes, the measured defaults (DESIGN.md §3.1), four workers per CTA: rows of 65..128 floats
// (one float4 per lane) with lane-held ids and two stages of two four-row units per worker; rows of 129..256 floats
// with the ids loaded per stage and two stages of one unit.
template <int NCH>
static int launch_ring(const SgParams& p, cudaStream_t st) {
  constexpr int L = 32, P = 2, NT = 128;
  constexpr int S = NCH == 1 ? 2 : 1, MINB = NCH == 1 ? 4 : 6, MODE = NCH == 1 ? 2 : 0;
  constexpr int WPB = NT / L;
  constexpr size_t smem = (size_t)WPB * P * S * 4 * NCH * L * 16 + (size_t)WPB * P * 8;
  static std::atomic<uint64_t> configured{0};
  ROC_CUDA(once_per_device(configured, [] {
    return cudaFuncSetAttribute(sg_chunk_kernel_t<L, NCH, S, P, NT, MINB, MODE>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }));
  sg_chunk_kernel_t<L, NCH, S, P, NT, MINB, MODE><<<(p.numChunks + WPB - 1) / WPB, NT, smem, st>>>(p);
  ROC_LAUNCH_CHECK();
  return ROC_OK;
}

// One ScatterGather launch: the main kernel (RING: sg_chunk_kernel_t), then the fix-ups of the rows it cut.  The
// partials of the min / max backward (MASK) are sums, so it runs the sum's fix-ups.
template <int VEC, int L, int NCH, int U, int MINB, int RED, bool RING = false>
static int launch(const SgParams& p, cudaStream_t st) {
  constexpr int FIX = RED == SG_RED_MASK ? SG_RED_SUM : RED;
  constexpr int WPB = SG_THREADS / L;
  if (p.numChunks) {
    if constexpr (RING) {
      const int rc = launch_ring<NCH>(p, st);
      if (rc != ROC_OK) return rc;
    } else {
      sg_chunk_kernel<VEC, L, NCH, U, MINB, RED><<<(p.numChunks + WPB - 1) / WPB, SG_THREADS, 0, st>>>(p);
      ROC_LAUNCH_CHECK();
    }
  }
  if (p.numHeavy) {
    sg_fixup_kernel<VEC, L, NCH, FIX><<<(p.numHeavy + WPB - 1) / WPB, SG_THREADS, 0, st>>>(p);
    ROC_LAUNCH_CHECK();
  }
  if (p.numBig) {
    sg_fixup_big_kernel<VEC, L, NCH, FIX><<<p.numBig, SG_THREADS, 0, st>>>(p);
    ROC_LAUNCH_CHECK();
  }
  return ROC_OK;
}

// Kernel shape for Q T-columns.  The sum takes up to 256 T-columns (1024 floats vectorised, 256 scalar); min / max
// take 128 vectorised (512 floats: the big-row fix-up keeps values and indices of every lane group in static shared
// memory).  Gathers in flight (U) are lowered for min / max where the index per float (forward) or the second
// gathered row (backward) would otherwise spill under the kernel's occupancy.  The vectorised sum of 65..256 floats
// runs on sg_chunk_kernel_t, which is faster there on a products-shaped graph (DESIGN.md §3.1).
template <int VEC, int RED>
static int dispatch(const SgParams& p, cudaStream_t st) {
  constexpr bool S = RED == SG_RED_SUM;
  constexpr bool B = RED == SG_RED_MASK;
  const uint32_t Q = p.Q;
  if (Q <= 4) return launch<VEC, 4, 1, 4, 4, RED>(p, st);
  if (Q <= 8) return launch<VEC, 8, 1, S ? 8 : 4, 4, RED>(p, st);
  if (Q <= 16) return launch<VEC, 16, 1, S ? 8 : 4, 4, RED>(p, st);
  if (Q <= 32) {
    if constexpr (VEC == 4 && S) return launch<VEC, 32, 1, 8, 4, RED, true>(p, st);
    else return launch<VEC, 32, 1, S ? 8 : 4, 4, RED>(p, st);
  }
  if (Q <= 64) {
    if constexpr (VEC == 4 && S) return launch<VEC, 32, 2, 4, 3, RED, true>(p, st);
    else return launch<VEC, 32, 2, B ? 2 : 4, 3, RED>(p, st);
  }
  if (Q <= 128) return launch<VEC, 32, 4, S ? 2 : 1, 3, RED>(p, st);
  if constexpr (S || VEC == 1) {
    if (Q <= 256) return launch<VEC, 32, 8, 1, 2, RED>(p, st);
  }
  return ROC_ERR_UNSUPPORTED;
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

// The plan parameters shared by every launch of column block c0 (units of T applied by the caller).
static SgParams plan_params(const roc_sg_plan* pl) {
  SgParams p;
  memset(&p, 0, sizeof(p));
  p.rs = pl->rs; p.firstRow = pl->firstRow; p.carryIdx = pl->carryIdx; p.heavyRows = pl->heavyRows; p.bigRows = pl->bigRows;
  p.col = pl->col; p.carry = pl->carry; p.carryArg = pl->carryArg;
  p.E = pl->E; p.numChunks = pl->numChunks; p.numHeavy = pl->numHeavy; p.numBig = pl->numBig; p.epi = 0;
  p.desc = pl->desc;
  return p;
}

// Reduction RED over the columns [0, H) of every row, in column blocks: 1,024 floats for the sum and 512 for min /
// max when every leading dimension and pointer allows float4 rows, else 256.  `arg` holds the min / max indices
// (written by the forward, gathered by the backward); the sum passes none.
template <int RED>
static int run_planned(roc_sg_plan* pl, int H, const float* in, int64_t ldIn, float* out, int64_t ldOut,
                       const roc_vid_t* arg, int64_t ldArg, int epilogue, roc_vid_t selfBase, cudaStream_t st) {
  const bool vec = (ldIn % 4 == 0) && (ldOut % 4 == 0) && (ldArg % 4 == 0) && aligned16(in) && aligned16(out) &&
                   aligned16(arg);
  const int vw = vec ? 4 : 1;                 // floats per T-column
  const int blockCols = !vec ? 256 : RED == SG_RED_SUM ? 1024 : 512;
  {
    int need = H < blockCols ? H : blockCols;
    int rc = ensure_carry(pl, ((size_t)need + 3) / 4 * 4, st, true);
    if (rc != ROC_OK) return rc;
    if constexpr (RED == SG_RED_MAX || RED == SG_RED_MIN) {
      rc = ensure_carry_arg(pl, st);
      if (rc != ROC_OK) return rc;
    }
  }
  for (int c0 = 0; c0 < H; c0 += blockCols) {
    const int hb = (H - c0 < blockCols) ? H - c0 : blockCols;
    SgParams p = plan_params(pl);
    p.in = in + c0; p.out = out + c0; p.epi = epilogue; p.selfBase = selfBase;
    if (arg) p.arg = const_cast<roc_vid_t*>(arg) + c0;
    p.ldIn = (size_t)ldIn / vw; p.ldOut = (size_t)ldOut / vw; p.ldArg = (size_t)ldArg / vw; p.ldC = pl->carryLd / vw;
    p.Q = ((uint32_t)hb + vw - 1) / vw;
    const int rc = vec ? dispatch<4, RED>(p, st) : dispatch<1, RED>(p, st);
    if (rc != ROC_OK) return rc;
  }
  return ROC_OK;
}

extern "C" int roc_sg_forward_planned(const roc_sg_plan* plc, int H, const float* in, int64_t ldIn,
                                      float* out, int64_t ldOut, int epilogue, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  if (!pl || H <= 0 || !in || !out || ldIn < H || ldOut < H) return ROC_ERR_INVALID;
  return run_planned<SG_RED_SUM>(pl, H, in, ldIn, out, ldOut, nullptr, 0, epilogue, 0, as_stream(stream));
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

extern "C" int roc_sg_minmax_forward_planned(const roc_sg_plan* plc, int aggr, int H, const float* in, int64_t ldIn,
                                             float* out, int64_t ldOut, roc_vid_t* arg, int64_t ldArg,
                                             roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  if (!pl || (aggr != ROC_SG_AGGR_MAX && aggr != ROC_SG_AGGR_MIN) || H <= 0 || !in || !out || !arg || ldIn < H ||
      ldOut < H || ldArg < H)
    return ROC_ERR_INVALID;
  cudaStream_t st = as_stream(stream);
  return aggr == ROC_SG_AGGR_MAX ? run_planned<SG_RED_MAX>(pl, H, in, ldIn, out, ldOut, arg, ldArg, 0, 0, st)
                                 : run_planned<SG_RED_MIN>(pl, H, in, ldIn, out, ldOut, arg, ldArg, 0, 0, st);
}

extern "C" int roc_sg_minmax_backward_planned(const roc_sg_plan* plc, int H, roc_vid_t selfBase, const float* outGrad,
                                              int64_t ldG, const roc_vid_t* arg, int64_t ldArg, float* inGrad,
                                              int64_t ldIn, roc_stream_t stream) {
  roc_sg_plan* pl = const_cast<roc_sg_plan*>(plc);
  if (!pl || H <= 0 || !outGrad || !arg || !inGrad || ldG < H || ldArg < H || ldIn < H) return ROC_ERR_INVALID;
  return run_planned<SG_RED_MASK>(pl, H, outGrad, ldG, inGrad, ldIn, arg, ldArg, 0, selfBase, as_stream(stream));
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
