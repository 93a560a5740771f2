/*
 * minmax_oracle.c — CPU definition of ScatterGather with max / min aggregation.
 *
 * TEST INFRASTRUCTURE, NOT THE PRODUCT: loaded only by tests/ (through
 * tests/minmax_oracle.py, which compiles it).  The product never links it.
 *
 * Conventions as in oracle/roc_oracle.c: V_ID = uint32, E_ID = uint64,
 * rowEnd[v - rowLeft] = global END offset of v's in-edge list, the first local
 * row starts at colLeft, colSrc[e - colLeft] = source vertex, node tensors are
 * row-major [numNodes][H] fp32.  Plain C11 + OpenMP.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

typedef uint32_t V_ID;
typedef uint64_t E_ID;

/* ------------------------------------------------------------------------- *
 * ScatterGather with max / min aggregation.  NOT a restatement: the reference
 * declares AGGR_MAX / AGGR_MIN (gnn.h:75-80) but its ScatterGather only sums.
 * These routines DEFINE the semantics the product's roc_sg_minmax_* follow
 * (include/roc_b200.h).  aggr: 1 = max, 2 = min.  For row v, edges in CSR order:
 *   the row starts with its first edge's value and source id; a later value
 *   replaces them only if it is strictly greater (smaller for min), or it is NaN
 *   and the current value is not.  out = that value, arg = that source id.
 *   A row of degree 0: out = 0, arg = 0xFFFFFFFF.
 * ------------------------------------------------------------------------- */
#define MINMAX_NOARG 0xFFFFFFFFu

void minmax_oracle_forward(V_ID rowLeft, V_ID rowRight, E_ID colLeft, int H,
                           const E_ID* rowEnd, const V_ID* colSrc, const float* in,
                           int aggr, float* out, V_ID* arg) {
  int64_t nloc = (int64_t)rowRight - (int64_t)rowLeft + 1;
#pragma omp parallel for schedule(dynamic, 64)
  for (int64_t n = 0; n < nloc; n++) {
    E_ID s = (n == 0) ? colLeft : rowEnd[n - 1];
    E_ID e = rowEnd[n];
    float* o = out + (size_t)n * H;
    V_ID* a = arg + (size_t)n * H;
    for (int h = 0; h < H; h++) { o[h] = 0.0f; a[h] = MINMAX_NOARG; }
    for (E_ID k = s; k < e; k++) {
      V_ID src = colSrc[k - colLeft];
      const float* r = in + (size_t)src * H;
      for (int h = 0; h < H; h++) {
        float v = r[h], cur = o[h];
        int take;
        if (a[h] == MINMAX_NOARG) take = 1;
        else if (isnan(v)) take = !isnan(cur);
        else take = (aggr == 1) ? (v > cur) : (v < cur);
        if (take) { o[h] = v; a[h] = src; }
      }
    }
  }
}

/* Its backward, a gather over the same CSR like the sum's (quirk Q1):
 *   inGrad[u][h] = sum_{e in row u, v = colSrc[e]} (arg[v][h] == selfBase + u ? outGrad[v][h] : 0)
 * outGrad / arg are indexed by source id (whole [N][H] matrices); selfBase + u is
 * local row u's id.  The true adjoint of the forward only on a symmetric graph
 * without duplicate edges.  acc64 != 0: fp64 accumulation; 0: fp32 in edge order. */
void minmax_oracle_backward(V_ID rowLeft, V_ID rowRight, E_ID colLeft, int H,
                            const E_ID* rowEnd, const V_ID* colSrc,
                            const float* outGrad, const V_ID* arg, V_ID selfBase,
                            float* inGrad, int acc64) {
  int64_t nloc = (int64_t)rowRight - (int64_t)rowLeft + 1;
#pragma omp parallel
  {
    double* acc = (double*)malloc(sizeof(double) * (size_t)(H > 0 ? H : 1));
#pragma omp for schedule(dynamic, 64)
    for (int64_t n = 0; n < nloc; n++) {
      E_ID s = (n == 0) ? colLeft : rowEnd[n - 1];
      E_ID e = rowEnd[n];
      V_ID me = selfBase + (V_ID)n;
      float* o = inGrad + (size_t)n * H;
      for (int h = 0; h < H; h++) { acc[h] = 0.0; o[h] = 0.0f; }
      for (E_ID k = s; k < e; k++) {
        V_ID v = colSrc[k - colLeft];
        const float* g = outGrad + (size_t)v * H;
        const V_ID* a = arg + (size_t)v * H;
        for (int h = 0; h < H; h++) {
          float t = (a[h] == me) ? g[h] : 0.0f;
          if (acc64) acc[h] += (double)t;
          else o[h] += t;
        }
      }
      if (acc64)
        for (int h = 0; h < H; h++) o[h] = (float)acc[h];
    }
    free(acc);
  }
}

