/*
 * roc_oracle.c — CPU restatement of jiazhihao/ROC's GCN-training path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT THE PRODUCT.  Only tests/, the smoke check in
 * __graft_entry__.py and bench.py's cpu_baseline / --impl reference legs may
 * load it.  The product (roc_b200/) never links, imports or calls anything here.
 *
 * Every function states the reference file:line it follows (paths relative to
 * the reference checkout, jiazhihao/ROC @ 1f58108).  The reference ships no CPU
 * kernels and no tests; this restatement is pinned against the reference's own
 * CUDA kernels (compiled from /root/reference by oracle/Makefile into
 * oracle/_ref/ and run on the GPU; outputs committed under tests/golden/).
 *
 * Conventions (types.h:5-15, load_task.cu:283-292):
 *   V_ID = uint32, E_ID = uint64, DATATYPE = float.
 *   rowEnd[v - rowLeft] = global END offset of v's in-edge list (NodeStruct.index)
 *   first local row starts at colLeft (scattergather_kernel.cu:46-50).
 *   colSrc[e - colLeft] = source vertex (EdgeStruct.src); dst is implicit.
 *   node tensors are row-major [numNodes][H] fp32 (gnn.cc:480-486).
 *
 * Plain C11 + OpenMP; `acc64 != 0` selects fp64 accumulation (the parity
 * oracle), `acc64 == 0` sums in fp32 in edge order (the timed CPU baseline).
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef uint32_t V_ID;
typedef uint64_t E_ID;

int roc_oracle_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

void roc_oracle_set_num_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}

/* ------------------------------------------------------------------------- *
 * Partitioner — gnn.cc:806-829 (vertex ranges) and gnn.cc:852-870 (edge ranges)
 * Returns the number of ranges the greedy scan produced (the reference asserts
 * it equals numParts, gnn.cc:829).  vb[2c], vb[2c+1] = [left,right] inclusive;
 * eb[2c], eb[2c+1] = [lo,hi] inclusive edge range (hi may be lo-1 if empty).
 * At most max_ranges ranges are written.
 * ------------------------------------------------------------------------- */
int roc_oracle_partition(V_ID numNodes, E_ID numEdges, int numParts,
                         const E_ID* raw_rows, V_ID* vb, E_ID* eb,
                         int max_ranges) {
  V_ID left_bound = 0;
  E_ID edge_cnt = 0;
  E_ID edge_cap = (numEdges + (E_ID)numParts - 1) / (E_ID)numParts;
  int n = 0;
  for (V_ID v = 0; v < numNodes; v++) {
    if (v == 0)
      edge_cnt += raw_rows[v];
    else
      edge_cnt += raw_rows[v] - raw_rows[v - 1];
    if (edge_cnt > edge_cap) { /* strict '>' : gnn.cc:816 */
      if (n < max_ranges) { vb[2 * n] = left_bound; vb[2 * n + 1] = v; }
      n++;
      edge_cnt = 0;
      left_bound = v + 1;
    }
  }
  if (edge_cnt > 0) { /* gnn.cc:823-826 */
    if (n < max_ranges) { vb[2 * n] = left_bound; vb[2 * n + 1] = numNodes - 1; }
    n++;
  }
  E_ID index = 0; /* gnn.cc:855-866 */
  for (int c = 0; c < n && c < max_ranges; c++) {
    eb[2 * c] = index;
    eb[2 * c + 1] = raw_rows[vb[2 * c + 1]] - 1;
    index = raw_rows[vb[2 * c + 1]];
  }
  return n;
}

/* ------------------------------------------------------------------------- *
 * Device CSR build — init_graph_kernel, load_task.cu:271-294.
 * rawRows[n] = global END offset of local row n; rawCols[e - colLeft] = src.
 * rowPtrs[n] (NodeStruct.index) = rawRows[n];
 * colIdxs[2*(e-colLeft)] = src, colIdxs[2*(e-colLeft)+1] = dst = n + rowLeft.
 * ------------------------------------------------------------------------- */
void roc_oracle_build_csr(V_ID rowLeft, V_ID rowRight, E_ID colLeft,
                          const E_ID* rawRows, const V_ID* rawCols,
                          E_ID* rowPtrs, V_ID* colIdxs /* [Eloc][2] */) {
  V_ID nloc = rowRight - rowLeft + 1;
  for (V_ID n = 0; n < nloc; n++) {
    E_ID startColIdx, endColIdx = rawRows[n];
    if (n == 0)
      startColIdx = colLeft;
    else
      startColIdx = rawRows[n - 1];
    rowPtrs[n] = endColIdx;
    for (E_ID e = startColIdx; e < endColIdx; e++) {
      colIdxs[2 * (e - colLeft)] = rawCols[e - colLeft];
      colIdxs[2 * (e - colLeft) + 1] = n + rowLeft;
    }
  }
}

/* ------------------------------------------------------------------------- *
 * ScatterGather (sum aggregation) — aggre_coop_kernel,
 * scattergather_kernel.cu:20-76; backward_task :160-170 runs the identical
 * computation on gradients (A, not A^T).
 *   out[v - rowLeft][h] = sum_{e in [start(v), rowEnd[v])} in[src[e]][h]
 * `in` is the WHOLE [numNodes][H] matrix indexed by global src ids
 * (scattergather.cc:69-73); `out` is the partition's [Nloc][H] slab.
 * The reference's sum order is nondeterministic (smem atomics, :66).
 * ------------------------------------------------------------------------- */
void roc_oracle_scatter_gather(V_ID rowLeft, V_ID rowRight, E_ID colLeft, int H,
                               const E_ID* rowEnd, const V_ID* colSrc,
                               const float* in, float* out, int acc64) {
  int64_t nloc = (int64_t)rowRight - (int64_t)rowLeft + 1;
#pragma omp parallel
  {
    double* acc = (double*)malloc(sizeof(double) * (size_t)(H > 0 ? H : 1));
#pragma omp for schedule(dynamic, 64)
    for (int64_t n = 0; n < nloc; n++) {
      E_ID s = (n == 0) ? colLeft : rowEnd[n - 1];
      E_ID e = rowEnd[n];
      float* o = out + (size_t)n * H;
      if (acc64) {
        for (int h = 0; h < H; h++) acc[h] = 0.0;
        for (E_ID k = s; k < e; k++) {
          const float* r = in + (size_t)colSrc[k - colLeft] * H;
          for (int h = 0; h < H; h++) acc[h] += (double)r[h];
        }
        for (int h = 0; h < H; h++) o[h] = (float)acc[h];
      } else {
        for (int h = 0; h < H; h++) o[h] = 0.0f;
        for (E_ID k = s; k < e; k++) {
          const float* r = in + (size_t)colSrc[k - colLeft] * H;
          for (int h = 0; h < H; h++) o[h] += r[h];
        }
      }
    }
    free(acc);
  }
}

/* ------------------------------------------------------------------------- *
 * InDegreeNorm — norm_coop_kernel, graphnorm_kernel.cu:19-57 (bwd :126-136 is
 * the same kernel).  y = x / sqrt((float)deg), deg cast from a V_ID (u32);
 * IEEE fp32 sqrt and divide.  in/out are the partition's own rows.
 * ------------------------------------------------------------------------- */
void roc_oracle_indegree_norm(V_ID rowLeft, V_ID rowRight, E_ID colLeft, int H,
                              const E_ID* rowEnd, const float* in, float* out) {
  int64_t nloc = (int64_t)rowRight - (int64_t)rowLeft + 1;
#pragma omp parallel for schedule(static)
  for (int64_t n = 0; n < nloc; n++) {
    E_ID s = (n == 0) ? colLeft : rowEnd[n - 1];
    V_ID deg = (V_ID)(rowEnd[n] - s);
    float d = sqrtf((float)deg);
    for (int h = 0; h < H; h++)
      out[(size_t)n * H + h] = in[(size_t)n * H + h] / d;
  }
}

/* ------------------------------------------------------------------------- *
 * Linear forward — linear_kernel.cu:76-80: cublasSgemm(OP_T, OP_N, m=outDim,
 * n=Nloc, k=inDim, W ld=inDim, X ld=inDim, Y ld=outDim), beta=0; optional
 * in-place ReLU (:83-104).   Y[v][o] = sum_i X[v][i] * W[o*inDim + i].
 * ------------------------------------------------------------------------- */
void roc_oracle_linear_fwd(int64_t nloc, int inDim, int outDim, const float* X,
                           const float* W, float* Y, int relu, int acc64) {
#pragma omp parallel for schedule(static)
  for (int64_t v = 0; v < nloc; v++) {
    const float* x = X + (size_t)v * inDim;
    float* y = Y + (size_t)v * outDim;
    for (int o = 0; o < outDim; o++) {
      const float* w = W + (size_t)o * inDim;
      float r;
      if (acc64) {
        double a = 0.0;
        for (int i = 0; i < inDim; i++) a += (double)x[i] * (double)w[i];
        r = (float)a;
      } else {
        float a = 0.0f;
        for (int i = 0; i < inDim; i++) a += x[i] * w[i];
        r = a;
      }
      if (relu) r = (r > 0.0f) ? r : 0.0f; /* NaN propagates like cuDNN */
      y[o] = r;
    }
  }
}

/* ------------------------------------------------------------------------- *
 * Linear backward — linear_kernel.cu:129-245.
 *  (1) if activation==RELU: dY = (Y > 0) ? dY : 0 in place  (reluBackward :120-127,
 *      launched :206-207)
 *  (2) dW[o*inDim+i] += sum_v X[v][i]*dY[v][o]   (sgemm OP_N,OP_T beta=1 :220-224)
 *  (3) dX[v][i] (+)= sum_o W[o*inDim+i]*dY[v][o] (sgemm OP_N,OP_N beta=1 :227-231;
 *      the buffer is zero-filled when resetInputGrads, types.cu:75-82, so
 *      accumulate_dx==0 means overwrite).  dX may be NULL (leaf input, Q8).
 * ------------------------------------------------------------------------- */
void roc_oracle_linear_bwd(int64_t nloc, int inDim, int outDim, const float* X,
                           const float* W, const float* Y, float* dY,
                           float* dW, float* dX, int relu, int accumulate_dx,
                           int acc64) {
  if (relu) {
#pragma omp parallel for schedule(static)
    for (int64_t k = 0; k < nloc * (int64_t)outDim; k++)
      dY[k] = (Y[k] > 0.0f) ? dY[k] : 0.0f;
  }
  /* dW: parallel over (o,i) pairs so each output element has one writer */
  int64_t nw = (int64_t)inDim * outDim;
  if (acc64) {
#pragma omp parallel for schedule(static)
    for (int64_t k = 0; k < nw; k++) {
      int o = (int)(k / inDim), i = (int)(k % inDim);
      double a = 0.0;
      for (int64_t v = 0; v < nloc; v++)
        a += (double)X[(size_t)v * inDim + i] * (double)dY[(size_t)v * outDim + o];
      dW[k] = (float)((double)dW[k] + a);
    }
  } else {
    /* blocked fp32: each thread owns a private dW replica, summed in order */
    int nt = roc_oracle_num_threads();
    float* rep = (float*)calloc((size_t)nt * (size_t)nw, sizeof(float));
#pragma omp parallel
    {
      int t = 0;
#ifdef _OPENMP
      t = omp_get_thread_num();
#endif
      float* r = rep + (size_t)t * nw;
#pragma omp for schedule(static)
      for (int64_t v = 0; v < nloc; v++) {
        const float* x = X + (size_t)v * inDim;
        const float* g = dY + (size_t)v * outDim;
        for (int o = 0; o < outDim; o++) {
          float go = g[o];
          float* ro = r + (size_t)o * inDim;
          for (int i = 0; i < inDim; i++) ro[i] += x[i] * go;
        }
      }
    }
    for (int t = 0; t < nt; t++)
      for (int64_t k = 0; k < nw; k++) dW[k] += rep[(size_t)t * nw + k];
    free(rep);
  }
  if (dX) {
#pragma omp parallel for schedule(static)
    for (int64_t v = 0; v < nloc; v++) {
      const float* g = dY + (size_t)v * outDim;
      float* dx = dX + (size_t)v * inDim;
      for (int i = 0; i < inDim; i++) {
        float r;
        if (acc64) {
          double a = 0.0;
          for (int o = 0; o < outDim; o++)
            a += (double)W[(size_t)o * inDim + i] * (double)g[o];
          r = (float)a;
        } else {
          float a = 0.0f;
          for (int o = 0; o < outDim; o++) a += W[(size_t)o * inDim + i] * g[o];
          r = a;
        }
        dx[i] = accumulate_dx ? dx[i] + r : r;
      }
    }
  }
}

/* ------------------------------------------------------------------------- *
 * Activation — activation_kernel.cu:50-66 (fwd), :114-132 (bwd, beta = 1 so
 * it accumulates into dX unless the buffer was reset).  mode 1 = ReLU,
 * 2 = sigmoid (ActiMode, gnn.h:82-86).  cuDNN bwd: relu dx = dy*(y>0)
 * (cuDNN tests x>0, identical for relu since y>0 <=> x>0); sigmoid dx = dy*y*(1-y).
 * ------------------------------------------------------------------------- */
void roc_oracle_activation_fwd(int64_t n, int mode, const float* x, float* y) {
#pragma omp parallel for schedule(static)
  for (int64_t k = 0; k < n; k++) {
    if (mode == 1)
      y[k] = (x[k] > 0.0f) ? x[k] : ((x[k] != x[k]) ? x[k] : 0.0f);
    else
      y[k] = 1.0f / (1.0f + expf(-x[k]));
  }
}

void roc_oracle_activation_bwd(int64_t n, int mode, const float* y,
                               const float* dy, float* dx, int accumulate) {
#pragma omp parallel for schedule(static)
  for (int64_t k = 0; k < n; k++) {
    float g = (mode == 1) ? ((y[k] > 0.0f) ? dy[k] : 0.0f)
                          : dy[k] * y[k] * (1.0f - y[k]);
    dx[k] = accumulate ? dx[k] + g : g;
  }
}

/* ------------------------------------------------------------------------- *
 * Element add — op_kernel, element_kernel.cu:19-39 (fwd); bwd :93-101:
 * dA (+)= dOut, dB (+)= dOut via add_kernel (cuda_helper.cu:29-36).
 * ------------------------------------------------------------------------- */
void roc_oracle_add_fwd(int64_t n, const float* a, const float* b, float* y) {
#pragma omp parallel for schedule(static)
  for (int64_t k = 0; k < n; k++) y[k] = a[k] + b[k];
}

void roc_oracle_add_bwd(int64_t n, const float* dy, float* da, int acc_a,
                        float* db, int acc_b) {
#pragma omp parallel for schedule(static)
  for (int64_t k = 0; k < n; k++) {
    da[k] = acc_a ? da[k] + dy[k] : dy[k];
    db[k] = acc_b ? db[k] + dy[k] : dy[k];
  }
}

/* ------------------------------------------------------------------------- *
 * Dropout — dropout_kernel.cu:98-99 (fwd), :149-150 (bwd), :159-180 (infer =
 * copy).  y = x * keep / (1 - rate).  cuDNN's RNG stream cannot be reproduced
 * (SURVEY §8c), so the keep mask is an INPUT here: either injected by the test
 * or produced by roc_oracle_dropout_mask below, which restates the product's
 * documented counter-based generator (Philox4x32-10, Salmon et al. SC'11) so
 * the two sides can be compared bit for bit.
 * ------------------------------------------------------------------------- */
static inline void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; r++) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c[0];
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c[2];
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k0;
    uint32_t n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k1;
    uint32_t n3 = (uint32_t)p0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}

/* the raw generator, exposed so the tests can pin it to Random123's known-answer vectors */
void roc_oracle_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
  uint32_t c[4] = {ctr[0], ctr[1], ctr[2], ctr[3]};
  philox4x32_10(c, key[0], key[1]);
  out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
}

/* keep[(r - firstRow) * H + c] for rows firstRow .. firstRow+rows-1 of a width-H tensor:
 * element (global row r, column c) keeps iff 16-bit lane (c & 7) of Philox counter
 * (r lo, r hi, c >> 3, step) under key (seed lo, seed hi) is >= round(rate * 65536);
 * lanes are numbered low half of word 0, high half of word 0, low half of word 1, ...
 * (include/roc_b200.h, roc_dropout_fwd). */
void roc_oracle_dropout_mask(int64_t firstRow, int64_t rows, int H, float rate,
                             uint64_t seed, uint32_t step, uint8_t* keep) {
  double t = (double)rate * 65536.0 + 0.5;
  uint32_t thresh = (t >= 65535.0) ? 65535u : (uint32_t)t;
#pragma omp parallel for schedule(static)
  for (int64_t j = 0; j < rows; j++) {
    uint64_t r = (uint64_t)(firstRow + j);
    for (int g = 0; g * 8 < H; g++) {
      uint32_t c[4] = {(uint32_t)r, (uint32_t)(r >> 32), (uint32_t)g, step};
      philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
      for (int l = 0; l < 8 && g * 8 + l < H; l++) {
        uint32_t u16 = (c[l >> 1] >> (16 * (l & 1))) & 0xFFFFu;
        keep[(size_t)j * H + g * 8 + l] = (u16 >= thresh) ? 1 : 0;
      }
    }
  }
}

void roc_oracle_dropout_apply(int64_t n, float rate, const uint8_t* keep,
                              const float* x, float* y) {
  float scale = 1.0f / (1.0f - rate);
#pragma omp parallel for schedule(static)
  for (int64_t k = 0; k < n; k++) y[k] = keep[k] ? x[k] * scale : 0.0f;
}

/* ------------------------------------------------------------------------- *
 * SoftmaxCrossEntropy backward (+ metrics) — softmax_kernel.cu:81-171.
 *  P = softmax over each row (cudnnSoftmaxForward ACCURATE, :124-126:
 *      subtract row max, exp, normalise);
 *  metrics on P (calc_loss :41-79): argmax starts from maxVal=0.0f/label=-1,
 *      strict '>' so the first max wins; trueLabel = index with label > 0.5;
 *      trainLoss += 1 - P[true] for MASK_TRAIN rows; per-class counts;
 *  grad = (P - labels) if mask==MASK_TRAIN else 0 (softmax_backward :19-33).
 * perf[7] = {trainLoss(float bits as float), trainAll, testAll, valAll,
 *            trainCorrect, testCorrect, valCorrect}  (PerfMetrics :35-39).
 * ------------------------------------------------------------------------- */
typedef struct {
  float trainLoss;
  int trainAll, testAll, valAll, trainCorrect, testCorrect, valCorrect;
} roc_oracle_perf;

void roc_oracle_softmax_xent_bwd(int64_t nloc, int C, const float* logits,
                                 const float* labels, const int* mask,
                                 float* grad, roc_oracle_perf* perf) {
  double loss = 0.0;
  long tA = 0, teA = 0, vA = 0, tC = 0, teC = 0, vC = 0;
#pragma omp parallel for schedule(static) reduction(+ : loss, tA, teA, vA, tC, teC, vC)
  for (int64_t v = 0; v < nloc; v++) {
    const float* z = logits + (size_t)v * C;
    float* p = grad + (size_t)v * C;
    float m = z[0];
    for (int i = 1; i < C; i++) m = (z[i] > m) ? z[i] : m;
    float sum = 0.0f;
    for (int i = 0; i < C; i++) { p[i] = expf(z[i] - m); sum += p[i]; }
    for (int i = 0; i < C; i++) p[i] = p[i] / sum;
    float maxVal = 0.0f;
    int trueLabel = -1, myLabel = -1;
    for (int i = 0; i < C; i++) {
      if (p[i] > maxVal) { maxVal = p[i]; myLabel = i; }
      if (labels[(size_t)v * C + i] > 0.5f) trueLabel = i;
    }
    int mk = mask[v];
    if (mk == 0) {
      loss += (double)(1.0f - p[trueLabel]);
      tA++; if (trueLabel == myLabel) tC++;
    } else if (mk == 1) {
      vA++; if (trueLabel == myLabel) vC++;
    } else if (mk == 2) {
      teA++; if (trueLabel == myLabel) teC++;
    }
    for (int i = 0; i < C; i++)
      p[i] = (mk == 0) ? p[i] - labels[(size_t)v * C + i] : 0.0f;
  }
  if (perf) {
    perf->trainLoss = (float)loss;
    perf->trainAll = (int)tA; perf->testAll = (int)teA; perf->valAll = (int)vA;
    perf->trainCorrect = (int)tC; perf->testCorrect = (int)teC;
    perf->valCorrect = (int)vC;
  }
}

/* ------------------------------------------------------------------------- *
 * Adam — optimizer.cc:79-85 (next: running beta powers and alpha_t in double)
 * and adam_update, optimizer_kernel.cu:43-63 (float, coupled L2, eps outside
 * the sqrt).  WGrad is the replica sum g0 += g_i in order (:88-94).
 * ------------------------------------------------------------------------- */
void roc_oracle_adam_next(double alpha, double beta1, double beta2,
                          double* beta1_t, double* beta2_t, double* alpha_t) {
  *beta1_t *= beta1;
  *beta2_t *= beta2;
  *alpha_t = alpha * sqrt(1 - *beta2_t) / (1 - *beta1_t);
}

void roc_oracle_adam_update(int64_t count, float alpha_t, float beta1,
                            float beta2, float weight_decay, float epsilon,
                            const float* WGrad, float* M, float* V, float* W) {
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < count; i++) {
    float gt = WGrad[i] + weight_decay * W[i];
    float mt = beta1 * M[i] + (1 - beta1) * gt;
    float vt = beta2 * V[i] + (1 - beta2) * gt * gt;
    M[i] = mt;
    V[i] = vt;
    W[i] -= alpha_t * mt / (sqrtf(vt) + epsilon);
  }
}

/* replica sum: optimizer_kernel.cu:88-94 — g0 += g_i for i = 1..P-1 in order */
void roc_oracle_replica_sum(int64_t count, int numReplicas, float* WGrad) {
  for (int r = 1; r < numReplicas; r++) {
    const float* src = WGrad + (size_t)r * count;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < count; i++) WGrad[i] += src[i] * 1.0f;
  }
}

/* Glorot scaling — initializer_kernel.cu:38-48 + scale_kernel cuda_helper.cu:2-9:
 * scale = sqrt(6.0/(in+out)) (double -> float); W = (b - a)*u + a with a=-scale,
 * b=scale, u = cuRAND uniform in (0,1] (the caller supplies u). */
void roc_oracle_glorot_scale(int64_t count, int inDim, int outDim, float* w) {
  float scale = (float)sqrt(6.0 / (inDim + outDim));
  float a = -scale, b = scale;
  for (int64_t i = 0; i < count; i++) w[i] = (b - a) * w[i] + a;
}

/* ------------------------------------------------------------------------- *
 * .lux reader — gnn.cc:756-801 (header + row ends) and load_task.cu:223-244
 * (per-partition slices).  Returns 0 on success.
 * ------------------------------------------------------------------------- */
int roc_oracle_lux_header(const char* path, V_ID* numNodes, E_ID* numEdges) {
  FILE* fd = fopen(path, "rb");
  if (!fd) return -1;
  int ok = fread(numNodes, sizeof(V_ID), 1, fd) == 1 &&
           fread(numEdges, sizeof(E_ID), 1, fd) == 1;
  fclose(fd);
  return ok ? 0 : -2;
}

int roc_oracle_lux_read(const char* path, V_ID rowLeft, V_ID rowRight,
                        E_ID colLeft, E_ID colRight, E_ID* raw_rows,
                        V_ID* raw_cols) {
  FILE* fd = fopen(path, "rb");
  if (!fd) return -1;
  V_ID nv; E_ID ne;
  if (fread(&nv, sizeof(V_ID), 1, fd) != 1 || fread(&ne, sizeof(E_ID), 1, fd) != 1) {
    fclose(fd); return -2;
  }
  const size_t hdr = sizeof(E_ID) + sizeof(V_ID); /* FILE_HEADER_SIZE gnn.h:33 */
  size_t nr = (size_t)(rowRight - rowLeft + 1);
  if (fseeko(fd, (off_t)(hdr + sizeof(E_ID) * (size_t)rowLeft), SEEK_SET) != 0 ||
      fread(raw_rows, sizeof(E_ID), nr, fd) != nr) { fclose(fd); return -3; }
  size_t nc = (colRight + 1 >= colLeft) ? (size_t)(colRight + 1 - colLeft) : 0;
  if (nc) {
    if (fseeko(fd, (off_t)(hdr + sizeof(E_ID) * (size_t)nv + sizeof(V_ID) * (size_t)colLeft), SEEK_SET) != 0 ||
        fread(raw_cols, sizeof(V_ID), nc, fd) != nc) { fclose(fd); return -4; }
  }
  fclose(fd);
  return 0;
}
