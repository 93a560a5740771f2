/*
 * roc_b200.h — C ABI of the H100-native kernel layer for ROC's GCN-training path.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  The reference has no FFI: its
 * device code is reached through Legion task variants
 *   static void X::forward_task(const Task*, const std::vector<PhysicalRegion>&, Context, Runtime*)
 * (gnn.h:224-349, registered gnn.cc:241-426).  Every entry point below replaces
 * the CUDA work one of those tasks did; the comment on each cites the task /
 * kernel / library call it stands in for.  INTEGRATION.md shows the stub a ROC
 * maintainer adds inside each *_task to call it.
 *
 * Conventions
 *  - plain C, no torch / Legion types; all data pointers are DEVICE pointers
 *    unless a name says `host`; caller owns every buffer;
 *  - `roc_stream_t` is a `cudaStream_t`; calls enqueue work and return (no
 *    device sync) unless documented otherwise;
 *  - return value: 0 = ROC_OK; > 0 = a cudaError_t; < 0 = ROC_ERR_*;
 *  - node tensors are row-major [rows][ld] fp32 with `ld >= H` floats between
 *    rows (the reference's layout is ld == H, gnn.cc:480-486).  The vectorised
 *    paths need ld % 4 == 0 and 16-byte aligned bases; other shapes take a
 *    scalar path.  Pad columns H..ld-1 may be read and rewritten by the
 *    vectorised paths (whole float4s) but never influence columns < H; the host
 *    keeps them zero;
 *  - graph ids follow types.h:5-15: V_ID = uint32, E_ID = uint64;
 *    rowEnd[v-rowLeft] is the GLOBAL END offset of v's in-edge list
 *    (NodeStruct.index, load_task.cu:283-288), the first local row starts at
 *    colLeft (scattergather_kernel.cu:46-50); colSrc[e-colLeft] is the source
 *    vertex of edge e (EdgeStruct.src; the redundant .dst is dropped).
 */
#ifndef ROC_B200_H_
#define ROC_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint32_t roc_vid_t;   /* V_ID,  types.h:5 */
typedef uint64_t roc_eid_t;   /* E_ID,  types.h:6 */
typedef void*    roc_stream_t; /* cudaStream_t */

#define ROC_OK               0
#define ROC_ERR_INVALID     (-1)  /* bad argument (NULL pointer, negative size ...) */
#define ROC_ERR_UNSUPPORTED (-2)  /* shape outside what the kernels handle */
#define ROC_ERR_NOMEM       (-3)
#define ROC_ERR_NO_DEVICE   (-4)  /* no CUDA device: the product has no CPU fallback */
#define ROC_ERR_IO          (-5)

/* ActiMode, gnn.h:82-86 */
#define ROC_AC_MODE_NONE    0
#define ROC_AC_MODE_RELU    1
#define ROC_AC_MODE_SIGMOID 2
#define ROC_AC_MODE_ELU     3   /* not in the reference: ELU with alpha = 1 (roc_activation_* only) */

/* MaskType, gnn.h:98-103 */
#define ROC_MASK_TRAIN 0
#define ROC_MASK_VAL   1
#define ROC_MASK_TEST  2
#define ROC_MASK_NONE  3

/* epilogue fused into the ScatterGather store (what the model applies right
 * after it, gnn.cc:83-85): NORM = the following indegree_norm, RELU = the relu
 * after that.  Applied in that order. */
#define ROC_SG_EPI_NONE 0
#define ROC_SG_EPI_NORM 1
#define ROC_SG_EPI_RELU 2
/* roc_sg_forward_teleport_planned only: the indegree_norm after the teleport (the next hop's) */
#define ROC_SG_EPI_NORM_OUT 4

/* aggregation of roc_sg_minmax_forward_planned (the values of AGGR_MAX / AGGR_MIN, gnn.h:75-80) */
#define ROC_SG_AGGR_MAX 1
#define ROC_SG_AGGR_MIN 2

/* PerfMetrics, softmax_kernel.cu:35-39 (same field order) */
typedef struct {
  float trainLoss;
  int trainAll, testAll, valAll, trainCorrect, testCorrect, valCorrect;
} roc_perf_metrics;

/* Metrics of the multi-label sigmoid cross-entropy (roc_sigmoid_xent_bwd), each field indexed by split:
 * [0] train, [1] val, [2] test (the ROC_MASK_* value of the row).  loss: the sum of the per-element loss over the
 * split's rows and classes; rows: the split's rows; exact: rows whose C predictions all equal their labels;
 * tp / fp / fn: true positives, false positives, false negatives over the split's rows and classes. */
typedef struct {
  double loss[3];
  uint64_t rows[3], exact[3], tp[3], fp[3], fn[3];
} roc_multilabel_metrics;

const char* roc_version(void);
/* Number of usable CUDA devices (0 if none); never fails. */
int roc_device_count(void);
/* Total kernels this library has launched in this process (for bench's gpu_launches). */
uint64_t roc_launch_count(void);
/* Persistent / grid-stride kernels launched by the CALLING THREAD from now on size their grids for
 * (SMs - numSMs), leaving SMs to work running beside them on another stream (the peer-write halo exchange:
 * a tensor-core GEMM CTA holds a whole SM, nothing co-resides with it).  0 restores full-chip grids.  Returns the
 * previous reserve. */
int roc_set_sm_reserve(int numSMs);

/* ---------------------------------------------------------------- graph --- */

/* Replaces Graph::Graph's partition loop, gnn.cc:806-829 + 852-870 (HOST code,
 * host pointers).  Greedy edge-balanced contiguous vertex ranges; a range is
 * closed when its in-edge count exceeds ceil(E/P) (strict).  vbounds[2c..2c+1] =
 * [left,right] inclusive, ebounds[2c..2c+1] = [lo,hi] inclusive.  Returns the
 * number of ranges produced in *numRanges; the reference asserts it equals
 * numParts (gnn.cc:829) — here that case returns ROC_ERR_UNSUPPORTED after
 * filling what fits. */
int roc_partition(roc_vid_t numNodes, roc_eid_t numEdges, int numParts,
                  const roc_eid_t* host_rowEnd, roc_vid_t* host_vbounds,
                  roc_eid_t* host_ebounds, int* numRanges);

/* Replaces init_graph_kernel, load_task.cu:271-294.  From the partition's raw
 * slices (rawRows = global END offsets of local rows, rawCols = sources) writes
 *   rowPtrs[n]  = rawRows[n]                          (NodeStruct, u64)     if non-NULL
 *   edgeStructs = {src = rawCols[e], dst = n+rowLeft} (EdgeStruct, 2 x u32) if non-NULL
 *   colSrc[e]   = rawCols[e]                          (lean u32 layout)     if non-NULL */
int roc_build_csr(roc_vid_t rowLeft, roc_vid_t rowRight, roc_eid_t colLeft,
                  const roc_eid_t* rawRows, const roc_vid_t* rawCols,
                  roc_eid_t* rowPtrs, roc_vid_t* edgeStructs, roc_vid_t* colSrc,
                  roc_stream_t stream);

/* -------------------------------------------------------- ScatterGather --- */

/* A plan holds the edge-balanced schedule for one partition's CSR: 64-edge
 * chunks, a start record per chunk, carry slots for rows longer than a
 * chunk.  It is a private, derived structure; rowEnd/colSrc stay the canonical
 * CSR and must outlive the plan.  Creation synchronises the stream. */
typedef struct roc_sg_plan roc_sg_plan;

int roc_sg_plan_create(roc_vid_t rowLeft, roc_vid_t rowRight, roc_eid_t colLeft,
                       const roc_eid_t* rowEnd, const roc_vid_t* colSrc,
                       roc_stream_t stream, roc_sg_plan** plan);
/* Pre-size the carry workspace for feature widths up to maxH (otherwise it is grown on the stream of the first
 * call that needs it, with stream-ordered allocation: no device synchronisation, but the plan must then be used
 * from that one stream). */
int roc_sg_plan_reserve(roc_sg_plan* plan, int maxH);
void roc_sg_plan_destroy(roc_sg_plan* plan);
/* Introspection for tests / DESIGN.md numbers. */
int roc_sg_plan_info(const roc_sg_plan* plan, uint64_t* numChunks,
                     uint64_t* numCarries, uint64_t* numHeavyRows);
/* *sorted = 1 if every row's sources are strictly increasing (so no row has a duplicate edge), else 0.  One device
 * pass; synchronises the stream. */
int roc_sg_plan_rows_sorted(const roc_sg_plan* plan, int* sorted, roc_stream_t stream);

/* Replaces aggre_coop_kernel + ScatterGather::forward_task,
 * scattergather_kernel.cu:20-76, 78-158:
 *   out[v-rowLeft][h] = sum_{e in in(v)} in[colSrc[e]][h],  h < H
 * `in` is indexed by whatever ids colSrc holds (global ids over the whole
 * [N][ldIn] matrix as in scattergather.cc:69-73, or local+halo ids).
 * Deterministic: the per-row summation order is fixed by the plan and no atomics are used, so the same call on
 * the same inputs gives the same bits every time. */
int roc_sg_forward_planned(const roc_sg_plan* plan, int H, const float* in,
                           int64_t ldIn, float* out, int64_t ldOut, int epilogue,
                           roc_stream_t stream);
/* roc_sg_forward_planned over bf16 rows (raw bits, see roc_f32_to_bf16): half the bytes per gathered row, each value
 * widened exactly in registers and accumulated in fp32, with the same epilogues and the same fp32 output.  `in` is
 * 16-byte aligned and ldIn (in elements) is a multiple of 8, else ROC_ERR_INVALID.  The result is bit-identical to
 * roc_sg_forward_planned on roc_bf16_to_f32(in) written to a 16-byte aligned buffer with a leading dimension that is a
 * multiple of 4: the plan, the row shapes, the column blocks, the per-float add order, the carries and the fix-ups are
 * that call's.  Its launches report reduction 12 (the sum over bf16 rows) in roc_sg_last_call_info. */
int roc_sg_forward_planned_bf16(const roc_sg_plan* plan, int H, const uint16_t* in, int64_t ldIn, float* out,
                                int64_t ldOut, int epilogue, roc_stream_t stream);
/* The sum with a teleport (initial residual) fused into its store, the hop of APPNP and GCNII:
 *   out[v][h] = post( fmaf(alpha, pre( sum_{e in in(v)} in[colSrc[e]][h] ), beta * t[v][h]) ),  h < H
 * with beta * t rounded to fp32 first, pre the divide by sqrtf(in-degree) of ROC_SG_EPI_NORM and post the same divide
 * of ROC_SG_EPI_NORM_OUT (the next hop's indegree_norm).  t has one row per plan row (like out), any pitch ldT >= H.
 * The bytes of out[v][0..H) are those of roc_sg_forward_planned(epilogue & ROC_SG_EPI_NORM) into a buffer laid out like
 * out, then roc_scaled_add_fwd(alpha, that, beta, t), then (NORM_OUT) roc_indegree_norm, also on rows of degree 0 and
 * NaN where that chain gives NaN: the same plan, row shapes, column blocks, add order and fix-ups as the sum.  The pad
 * floats of a float4 row of `out` (past H, up to the next multiple of 4) are written with unspecified values: the
 * teleport of the sum's pad with t = 0.  Every width runs on the
 * register kernel (no ring form).  ROC_ERR_INVALID: a NULL pointer, out == t, a leading dimension < H, non-finite
 * alpha or beta, or an epilogue with any bit but NORM and NORM_OUT (RELU included).  Its launches report reduction 13
 * in roc_sg_last_call_info. */
int roc_sg_forward_teleport_planned(const roc_sg_plan* plan, int H, const float* in, int64_t ldIn, float alpha,
                                    const float* t, int64_t ldT, float beta, float* out, int64_t ldOut, int epilogue,
                                    roc_stream_t stream);

/* Max / min aggregation (GraphSAGE-pool).  The reference declares AGGR_MAX / AGGR_MIN but never implements them;
 * these semantics are this library's own.  For a row v with in-edges e in CSR order:
 *   out[v-rowLeft][h] = max (aggr = ROC_SG_AGGR_MAX) or min (ROC_SG_AGGR_MIN) of in[colSrc[e]][h]
 *   arg[v-rowLeft][h] = colSrc[e] of the FIRST edge in CSR order that holds that value
 * A row starts with its first edge's value and id; a later value replaces them only if it is strictly greater
 * (smaller) or it is NaN and the current value is not, so NaN propagates as in torch.amax.  A row of degree 0 gets
 * out = 0 and arg = 0xFFFFFFFF.  Exact (no rounding) and independent of how the plan cuts rows into chunks.
 * `in` is indexed like roc_sg_forward_planned's.
 * ROC_ERR_INVALID for an aggr other than MAX / MIN, a NULL pointer or a leading dimension < H. */
int roc_sg_minmax_forward_planned(const roc_sg_plan* plan, int aggr, int H, const float* in, int64_t ldIn,
                                  float* out, int64_t ldOut, roc_vid_t* arg, int64_t ldArg, roc_stream_t stream);
/* roc_sg_minmax_forward_planned over bf16 rows (raw bits, see roc_f32_to_bf16), each value widened exactly in
 * registers: the same fp32 out and the same arg. `in` is 16-byte aligned and ldIn (in elements) is a multiple of 8,
 * else ROC_ERR_INVALID. The result is bit-identical to roc_sg_minmax_forward_planned on roc_bf16_to_f32(in) written
 * to a 16-byte aligned buffer with a leading dimension that is a multiple of 4: the plan, the row shapes, the column
 * blocks, the per-float order, the carries and the fix-ups are that call's. Its main launches report reduction 17
 * (max) or 18 (min) in roc_sg_last_call_info. */
int roc_sg_minmax_forward_planned_bf16(const roc_sg_plan* plan, int aggr, int H, const uint16_t* in, int64_t ldIn,
                                       float* out, int64_t ldOut, roc_vid_t* arg, int64_t ldArg, roc_stream_t stream);
/* Its backward, as a gather over the same CSR (like the sum's, quirk Q1), in the plan's fixed order, no atomics:
 *   inGrad[u][h] = sum_{e in row u, v = colSrc[e]} (arg[v][h] == selfBase + u ? outGrad[v][h] : 0)
 * outGrad and arg are indexed by colSrc's ids; selfBase + u is local row u's id in that space (0 for a whole graph,
 * rowLeft for a slice with global ids).  This is the true adjoint only when the graph is symmetric and has no
 * duplicate edges. */
int roc_sg_minmax_backward_planned(const roc_sg_plan* plan, int H, roc_vid_t selfBase,
                                   const float* outGrad, int64_t ldG, const roc_vid_t* arg, int64_t ldArg,
                                   float* inGrad, int64_t ldIn, roc_stream_t stream);

/* Attention aggregation (GAT, Velickovic et al. 2018).  `heads` heads over features of width H = heads * F; `score`
 * has 2 * heads columns: column k is the destination score s_dst[.][k] of head k, column heads + k the source score
 * s_src[.][k].  For plan row r with id i = selfBase + r and in-edges e in CSR order, sources j = colSrc[e]:
 *   y(i,j,k)     = LeakyReLU_slope(s_dst[i][k] + s_src[j][k])          (z > 0 ? z : slope * z)
 *   m[i][k]      = max_e y(i,j,k);   Z[i][k] = sum_e exp(y(i,j,k) - m[i][k])
 *   a(i<-j,k)    = exp(y(i,j,k) - m[i][k]) / Z[i][k]
 *   out[r][kF+f] = sum_e a(i<-j,k) * in[j][kF+f]
 *   stats[r][k]  = m[i][k],   stats[r][heads+k] = 1 / Z[i][k]
 * A row of degree 0 gets out = 0, m = 0 and 1/Z = 0, so its a is 0 wherever the backward recomputes it.  `in`,
 * `score` and every per-node input of the backward are indexed by colSrc's ids (a whole graph, or a slice with global
 * ids and selfBase = rowLeft).
 * Backward, as gathers over the same CSR (quirk Q1: the true adjoint of the source-score and feature parts only on a
 * symmetric graph; the destination-score part is exact on any graph).  G = outGrad, O = out, X = in, score and stats
 * all indexed by colSrc's ids.  With D[i][k] = sum_f G[i][kF+f] O[i][kF+f], l = (s_dst[i][k] + s_src[j][k] > 0) ? 1 :
 * slope and dz(i<-j,k) = a(i<-j,k) (sum_f G[i][kF+f] X[j][kF+f] - D[i][k]) l  (a recomputed from stats[i]):
 *   scoreGrad[r][k]       = sum_{e in row r, j = col[e]} dz(i<-j,k)                 (d s_dst)
 *   scoreGrad[r][heads+k] = sum_{e in row r, j = col[e]} dz(j<-i,k)                 (d s_src)
 *   inGrad[r][kF+f]       = sum_{e in row r, j = col[e]} a(j<-i,k) G[j][kF+f]
 * Shapes: heads in {1, 2, 4, 8}, H % heads == 0; for heads > 1, F is a power of two >= 4.  H <= 512 when every
 * feature leading dimension is a multiple of 4 and every feature pointer 16-byte aligned, else H <= 256.  slope is
 * finite and >= 0.  IEEE expf and divides; no atomics, so the same call on the same inputs returns the same bits.
 * Both calls overwrite their outputs.  ROC_ERR_INVALID: a NULL pointer, a leading dimension too small (< H, or
 * < 2 * heads for score / stats / scoreGrad), heads <= 0, H <= 0, a bad slope.  ROC_ERR_UNSUPPORTED: any other
 * head layout or width.  The backward keeps a per-node record {s_dst, m, 1/Z, D} (16 bytes per head) in the plan;
 * its first call finds the largest id in colSrc (one synchronisation of the stream). */
int roc_sg_attn_forward_planned(const roc_sg_plan* plan, int heads, int H, float slope, roc_vid_t selfBase,
                                const float* in, int64_t ldIn, const float* score, int64_t ldS,
                                float* out, int64_t ldOut, float* stats, int64_t ldStats, roc_stream_t stream);
int roc_sg_attn_backward_planned(const roc_sg_plan* plan, int heads, int H, float slope, roc_vid_t selfBase,
                                 const float* in, int64_t ldIn, const float* score, int64_t ldS, const float* out,
                                 int64_t ldOut, const float* stats, int64_t ldStats, const float* outGrad,
                                 int64_t ldG, float* inGrad, int64_t ldInG, float* scoreGrad, int64_t ldSG,
                                 roc_stream_t stream);
/* The attention forward and its backward over bf16 feature rows X = in (raw bits, see roc_f32_to_bf16), each value
 * widened exactly in registers; score, stats, out, outGrad and every output stay fp32. The forward gathers X[j] at
 * half width (its stats pass reads only the scores); the backward gathers X[j] in its d s_dst pass and reads X[i],
 * the row's own row, in its input-gradient pass. `in` is 16-byte aligned and ldIn (in elements) is a multiple of 8,
 * else ROC_ERR_INVALID. The result is bit-identical to the fp32 call on roc_bf16_to_f32(in) written to a 16-byte
 * aligned buffer with a leading dimension that is a multiple of 4: the plan, the row shapes, the column blocks, the
 * per-float order, the carries and the fix-ups are that call's. Their main launches report reduction 21 (the
 * forward's weighted sum), 22 (d s_dst) and 23 (the input gradient) in roc_sg_last_call_info; the stats pass, the
 * record and the fix-ups are the fp32 call's and report as there. */
int roc_sg_attn_forward_planned_bf16(const roc_sg_plan* plan, int heads, int H, float slope, roc_vid_t selfBase,
                                     const uint16_t* in, int64_t ldIn, const float* score, int64_t ldS, float* out,
                                     int64_t ldOut, float* stats, int64_t ldStats, roc_stream_t stream);
int roc_sg_attn_backward_planned_bf16(const roc_sg_plan* plan, int heads, int H, float slope, roc_vid_t selfBase,
                                      const uint16_t* in, int64_t ldIn, const float* score, int64_t ldS,
                                      const float* out, int64_t ldOut, const float* stats, int64_t ldStats,
                                      const float* outGrad, int64_t ldG, float* inGrad, int64_t ldInG,
                                      float* scoreGrad, int64_t ldSG, roc_stream_t stream);

/* Attention dropout (the paper's dropout of the normalised attention coefficients; PyG GATConv(dropout=), DGL
 * GATConv(attn_drop=)).  y, m, Z, a and stats are as above: m and Z come from the undropped softmax.  For plan row r
 * with id i = selfBase + r and each in-edge's source j = colSrc[e], with T16 = round(rate * 65536) as in
 * roc_dropout_fwd:
 *   keep(i<-j,k) = 16-bit lane k of Philox4x32-10(counter = {i, j, 0, step}, key = {seed lo, seed hi}) >= T16
 * with the lanes numbered as in roc_dropout_fwd: one Philox block decides all heads of one (destination, source) pair.
 * The mask is keyed by the pair, not by the edge's position, so any edge order computes it, and the duplicate edges of
 * a multigraph share it.  With s = 1.0f / (1.0f - rate) (fp32, roc_dropout_fwd's scale) and M = keep ? s : 0:
 *   a'(i<-j,k)   = keep(i<-j,k) ? a(i<-j,k) * s : 0
 *   out[r][kF+f] = sum_e a'(i<-j,k) * in[j][kF+f]
 * Backward, with D[i][k] = sum_f G[i][kF+f] O[i][kF+f] over the dropped output O:
 *   dz(i<-j,k)   = a(i<-j,k) (M(i<-j,k) sum_f G[i][kF+f] X[j][kF+f] - D[i][k]) l
 *   inGrad gathers a'(i<-j,k) G[i] where the calls above gather a(i<-j,k) G[i]; d s_dst and d s_src are the sums of
 *   dz as there.
 * The passes read the mask as one keep byte per edge (bit k = head k), made by roc_sg_attn_keep_mask:
 *   keep     the forward plan's edge order, pairs (i <- j) with the row the destination        (the forward and B1)
 *   keepRev  the same plan's order with the row the source: edge e of row r holds keep(j <- i)  (the planned B2)
 *   keepT    the transposed plan's order (roc_sg_transpose_info's planT, selfBase 0), the row the source (exact B2)
 * rate = 0, or NULL masks: the calls above, byte for byte.  ROC_ERR_INVALID also for a rate outside [0, 1) and, in a
 * backward, for one NULL mask of two.  Everything else (shapes, errors, determinism, the launches but the main
 * kernels' reduction numbers) is the call without dropout's. */
int roc_sg_attn_forward_dropout_planned(const roc_sg_plan* plan, int heads, int H, float slope, roc_vid_t selfBase,
                                        const float* in, int64_t ldIn, const float* score, int64_t ldS, float* out,
                                        int64_t ldOut, float* stats, int64_t ldStats, const uint8_t* keep, float rate,
                                        roc_stream_t stream);
int roc_sg_attn_forward_dropout_planned_bf16(const roc_sg_plan* plan, int heads, int H, float slope,
                                             roc_vid_t selfBase, const uint16_t* in, int64_t ldIn, const float* score,
                                             int64_t ldS, float* out, int64_t ldOut, float* stats, int64_t ldStats,
                                             const uint8_t* keep, float rate, roc_stream_t stream);
int roc_sg_attn_backward_dropout_planned(const roc_sg_plan* plan, int heads, int H, float slope, roc_vid_t selfBase,
                                         const float* in, int64_t ldIn, const float* score, int64_t ldS,
                                         const float* out, int64_t ldOut, const float* stats, int64_t ldStats,
                                         const float* outGrad, int64_t ldG, float* inGrad, int64_t ldInG,
                                         float* scoreGrad, int64_t ldSG, const uint8_t* keep, const uint8_t* keepRev,
                                         float rate, roc_stream_t stream);
int roc_sg_attn_backward_dropout_planned_bf16(const roc_sg_plan* plan, int heads, int H, float slope,
                                              roc_vid_t selfBase, const uint16_t* in, int64_t ldIn, const float* score,
                                              int64_t ldS, const float* out, int64_t ldOut, const float* stats,
                                              int64_t ldStats, const float* outGrad, int64_t ldG, float* inGrad,
                                              int64_t ldInG, float* scoreGrad, int64_t ldSG, const uint8_t* keep,
                                              const uint8_t* keepRev, float rate, roc_stream_t stream);
/* The keep bytes of every edge of `plan` in its edge order: keep[e - colLeft] bit k = keep(i<-j,k) for all 8 lanes,
 * with, for edge e of plan row r and c = colSrc[e], (i, j) = (selfBase + r, c) when rowIsSource == 0 (the forward
 * order) and (c, selfBase + r) when rowIsSource == 1 (keepRev over the forward plan, keepT over the transposed plan
 * with selfBase 0).  One Philox block per edge, E bytes written.  ROC_ERR_INVALID: a NULL plan, a NULL keep with
 * edges, rowIsSource not 0 or 1, a rate outside [0, 1).  Launch: ROC_SG_LAUNCH_KEEP_MASK. */
int roc_sg_attn_keep_mask(const roc_sg_plan* plan, roc_vid_t selfBase, int rowIsSource, float rate, uint64_t seed,
                          uint32_t step, uint8_t* keep, roc_stream_t stream);

/* Dynamic attention (GATv2: Brody et al., "How Attentive are Graph Attention Networks?", PyG GATv2Conv without bias,
 * edge features or head averaging).  xl holds the source (value) rows and xr the target rows, H = heads * F columns,
 * 1 <= H <= 256, heads <= 8; `a` holds the attention vector of each head, a[k][f] at a[f * heads + k] (F x heads
 * floats: the memory of a Model parameter of parameter_shape (heads, F)).  The plan covers a whole graph: every id in
 * colSrc is one of its rows, which index xl, xr and every other row operand.  For row v, each in-edge e from u =
 * colSrc[e] (self loops are in the graph, duplicate edges count once each), head k and l(z) = LeakyReLU(z) (z > 0 ? z :
 * slope * z; l'(z) = z > 0 ? 1 : slope, as torch):
 *   z[v,u][c]  = xl[u][c] + xr[v][c]
 *   e[v,u,k]   = sum_f a[k][f] * l(z[v,u][kF+f])
 *   m[v][k]    = max_u e,  Z[v][k] = sum_u exp(e - m),  p[v,u,k] = exp(e - m) / Z
 *   out[v][kF+f] = sum_u p[v,u,k] * xl[u][kF+f]           (accumulated as fmaf(p, xl, acc) from +0 in CSR order)
 * stats[v] = m | 1/Z per head, as roc_sg_attn_forward_planned's (0 | 0 for a row of degree 0, whose out is 0).
 * e is computed by one device function whose summation order depends on (H, heads) only: lane l of a warp holds
 * columns l + 32 j; a head's terms are added in column order within each lane, then across the warp by an xor
 * butterfly.  The forward and both backward passes therefore see the same bits for every e.
 * Backward, from outGrad = gy and the forward's out and stats, with c[v][k] = gy[v]_k . out[v]_k (the record pass) and
 * d[v,u,k] = p (gy[v]_k . xl[u]_k - c[v][k]):
 *   dxr[v][c] = sum_u d[v,u,k] * a[k][f] * l'(z)          (the destination pass, over the plan)
 *   R[v][c]   = sum_u d[v,u,k] * l(z)                     (the same pass; N x H floats of workspace of the call)
 *   dxl[u][c] = sum over u's out-edges (v <- u) of p gy[v][c] + d a[k][f] l'(z)   (the source pass)
 *   da[k][f]  = sum_v R[v][kF+f], in a's layout: fp64 sums over blocks of 512 rows, then the blocks in order
 * roc_sg_attn_v2_backward_planned runs the source pass over the same CSR, reading row u's in-edges as its out-edges:
 * exact on a symmetric graph, as roc_sg_attn_backward_planned.  roc_sg_attn_v2_backward_exact runs it over the
 * transposed plan: exact on any graph, multigraphs included.  When xl and xr are one tensor, its gradient is dxl + dxr.
 * No per-edge buffer: every pass recomputes e from the rows.  No atomics: every output is the same bits run to run and
 * whatever the grid or the SMs available.  Every call overwrites its outputs; dxl and dxr are distinct buffers.
 * ROC_ERR_INVALID: a NULL pointer, heads <= 0, H <= 0, a leading dimension < H (stats < 2 * heads), a bad slope, dxl ==
 * dxr, and for the exact call a transpose of another graph.  ROC_ERR_UNSUPPORTED: H % heads != 0, H > 256, heads > 8,
 * or a plan whose colSrc names an id outside its rows.  The first call on a plan finds its largest id (one
 * synchronisation of the stream).  Launches (roc_sg_last_call_info): the main kernel reports reduction 64 (stats), 65
 * (weighted sum), 66 (destination pass) and 67 (source pass), with lanes 32 and nch = ceil(H / 32); the stats fix-up
 * and the sum's fix-ups of cut rows follow their pass (the destination pass: dxr's, then R's); the backward starts with
 * a ROC_SG_LAUNCH_RECORD and ends with two ROC_SG_LAUNCH_COLSUM launches (da). */
int roc_sg_attn_v2_forward_planned(const roc_sg_plan* plan, int heads, int H, float slope, const float* xl,
                                   int64_t ldXl, const float* xr, int64_t ldXr, const float* a, float* out,
                                   int64_t ldOut, float* stats, int64_t ldStats, roc_stream_t stream);
int roc_sg_attn_v2_backward_planned(const roc_sg_plan* plan, int heads, int H, float slope, const float* xl,
                                    int64_t ldXl, const float* xr, int64_t ldXr, const float* a, const float* out,
                                    int64_t ldOut, const float* stats, int64_t ldStats, const float* outGrad,
                                    int64_t ldG, float* dxl, int64_t ldDxl, float* dxr, int64_t ldDxr, float* da,
                                    roc_stream_t stream);
int roc_sg_attn_v2_backward_exact(const roc_sg_plan* plan, struct roc_sg_transpose* tr, int heads, int H, float slope,
                                  const float* xl, int64_t ldXl, const float* xr, int64_t ldXr, const float* a,
                                  const float* out, int64_t ldOut, const float* stats, int64_t ldStats,
                                  const float* outGrad, int64_t ldG, float* dxl, int64_t ldDxl, float* dxr,
                                  int64_t ldDxr, float* da, roc_stream_t stream);

/* Softmax aggregation with one temperature t (PyG SoftmaxAggregation(t, learn=True), GENConv's default aggregator;
 * DeeperGCN, Li et al. 2020).  For row v, column f and the in-edges u = colSrc[e] of v (duplicates counted):
 *   z_u = t * x[u][f],  m = max_u z_u,  Z = sum_u exp(z_u - m),  p_u = exp(z_u - m) / Z,  y[v][f] = sum_u p_u x[u][f]
 * (y = 0 for a row with no in-edge).  Every column is its own softmax; t = 0 gives the mean, a large t approaches the
 * max and a negative t leans towards the min.  t is one float in device memory (so that a learned t never needs a
 * host synchronisation).  The plan covers a whole graph: every id in colSrc is one of its rows, which index x, y,
 * stats and every gradient.  Any H >= 1; rows wider than 256 columns run in column blocks of 256.
 * Forward: one pass with an online softmax per column (running m, s = sum exp(z - m), w = sum exp(z - m) x, added as
 * s = fmaf(s, c, 1), w = fmaf(w, c, x) when z raises m, else s += e, w = fmaf(e, x, w)); a row cut at chunk
 * boundaries is merged in chunk order by rescale-and-add, y = w / s.  stats (may be NULL, e.g. in inference): when
 * given, [Nloc][ldStats >= 2H] rows of m | 1/Z per column (0 | 0 for a row with no in-edge), which the backward reads.
 * Backward, with g = gy[v] and e = exp(t x[u] - m_v), never split into exp(t x) exp(-m):
 *   dx[u][f] = sum over v with u in N(v) of g p_vu (1 + t (x[u][f] - y[v][f]))
 *   dt       = sum_v sum_f g sum_u p_vu (x[u][f] - y[v][f])^2
 * A record pass packs {m | g / Z | y} per destination (3 min(H, 256) floats per node); a source pass per row u gathers
 * each in-edge's record, accumulates dx and, when dt is wanted, R[u][f] = sum_v (g / Z) e (x - y)^2 (N x H floats).
 * Both live in a workspace of the plan, grown on demand and kept (freed with the plan); an inference forward on a plan
 * with cut rows keeps their (m, s) there (2 min(H, 256) floats per node).  dt is R's sum in fp64 over blocks of 512 rows, added in block order, written (not added) as one
 * fp32.  dt NULL: R and dt are skipped.  roc_sg_softmax_backward_planned runs the source pass over the same CSR,
 * reading row u's in-edges as its out-edges: exact on a symmetric graph.  roc_sg_softmax_backward_exact runs it over
 * the transposed plan: exact on any graph, multigraphs included.  No per-edge buffer and no atomics: every output is
 * the same bits run to run and whatever the grid or the SMs available.  expf throughout, in a fixed order.
 * ROC_ERR_INVALID: a NULL pointer (dt and the forward's stats may be NULL), H <= 0, a leading dimension < H (stats
 * < 2H), y == x, dx aliasing x, y, stats, gy or t, dt == t, and for the exact call a transpose of another graph.
 * ROC_ERR_UNSUPPORTED: a plan whose colSrc names an id outside its rows.  The first call on a plan finds its largest id
 * (one synchronisation of the stream).  Launches (roc_sg_last_call_info), per column block: the forward's main kernel
 * reports reduction 72, then its own fix-ups of cut rows (ROC_SG_LAUNCH_FIXUP, ROC_SG_LAUNCH_BIG_FIXUP, reduction 72);
 * the backward's ROC_SG_LAUNCH_RECORD, then the source pass, reduction 73 (without dt) or 74 (with dt), then the
 * sum's fix-ups of dx and, with dt, of R; with dt the backward ends with two ROC_SG_LAUNCH_COLSUM launches.  Every
 * pass runs lanes 32 and nch = ceil(Hb / 32) for the block's Hb columns. */
int roc_sg_softmax_forward_planned(const roc_sg_plan* plan, int H, const float* t, const float* x, int64_t ldX,
                                   float* y, int64_t ldY, float* stats, int64_t ldStats, roc_stream_t stream);
int roc_sg_softmax_backward_planned(const roc_sg_plan* plan, int H, const float* t, const float* x, int64_t ldX,
                                    const float* y, int64_t ldY, const float* stats, int64_t ldStats, const float* gy,
                                    int64_t ldG, float* dx, int64_t ldDx, float* dt, roc_stream_t stream);
int roc_sg_softmax_backward_exact(const roc_sg_plan* plan, struct roc_sg_transpose* tr, int H, const float* t,
                                  const float* x, int64_t ldX, const float* y, int64_t ldY, const float* stats,
                                  int64_t ldStats, const float* gy, int64_t ldG, float* dx, int64_t ldDx, float* dt,
                                  roc_stream_t stream);

/* Edge dropout of the sum (the APPNP paper's dropout of the propagation matrix, PyG APPNP(dropout=); DropEdge, Rong et
 * al. 2020, applied to GCN).  keep(i<-j) is bit 0 of the byte roc_sg_attn_keep_mask writes for the pair (i <- j): lane 0
 * of Philox4x32-10 with counter {i, j, 0, step} and key {seed lo, seed hi}, against T16 = round(rate * 65536), the same
 * generator as attention dropout, so duplicate edges of a multigraph share one decision.  With s = 1.0f / (1.0f - rate)
 * (fp32, roc_dropout_fwd's scale):
 *   out[v][h] = epilogue( sum over the kept in-edges e of v, in the sum's per-row order, acc = fmaf(s, in[j][h], acc) )
 * accumulated from +0; a dropped edge contributes nothing and its source row is not loaded, and a row whose edges are
 * all dropped gets epilogue(0).  The degrees the epilogues divide by stay the full graph's: this is dropout on the
 * normalised adjacency entries (PyG APPNP's form), not DropEdge's renormalisation on the sampled graph.  On finite
 * inputs the bytes equal roc_sg_weighted_forward_planned with w[e] = keep ? s : 0 (the sum's column blocks and order)
 * followed by the unfused kernels the epilogue replaces (roc_indegree_norm for NORM, then relu for RELU).  keep holds
 * one byte per edge of the plan, in its edge order (roc_sg_attn_keep_mask with rowIsSource 0 over the forward plan).
 * rate = 0 or keep = NULL: roc_sg_forward_planned itself, byte for byte and launch for launch.  ROC_ERR_INVALID: as
 * roc_sg_forward_planned, and a rate outside [0, 1).  Every width runs on the register kernel (no ring form); its main
 * launches report reduction 32 in roc_sg_last_call_info, its fix-ups as the sum's. */
int roc_sg_forward_dropout_planned(const roc_sg_plan* plan, int H, const float* in, int64_t ldIn, float* out,
                                   int64_t ldOut, int epilogue, const uint8_t* keep, float rate, roc_stream_t stream);
/* roc_sg_forward_teleport_planned over the dropped sum: post(fmaf(alpha, pre(dropped sum), beta * t)), bytes equal to
 * roc_sg_forward_dropout_planned (epilogue & NORM) followed by the chain roc_sg_forward_teleport_planned documents.
 * rate = 0 or keep = NULL: roc_sg_forward_teleport_planned itself.  ROC_ERR_INVALID: as that call, and a rate outside
 * [0, 1).  Main launches report reduction 45, the fix-ups 13. */
int roc_sg_forward_teleport_dropout_planned(const roc_sg_plan* plan, int H, const float* in, int64_t ldIn, float alpha,
                                            const float* t, int64_t ldT, float beta, float* out, int64_t ldOut,
                                            int epilogue, const uint8_t* keep, float rate, roc_stream_t stream);

/* Edge-weighted aggregation (GCN with edge weights, weighted graphs, edge saliency).  The reference declares edge
 * tensors (gnn.h:178) but never reads them; these semantics are this library's own.  For plan row r with id
 * i = selfBase + r and in-edges e in CSR order with sources j = colSrc[e], the edge's weight is w[e - colLeft]: a flat
 * fp32 array in the plan's edge order.
 *   out[r][h] = sum_e w[e] * in[j][h]
 * accumulated as fmaf(w, in, acc) from +0 in the plan's fixed per-row order, with no atomics.  A row of degree 0 gets
 * 0.  With every weight 1.0 the result is bit-identical to roc_sg_forward_planned with ROC_SG_EPI_NONE: both take the
 * same column blocks (1,024 floats on float4 rows, else 256) and the same row shapes.  `in` is
 * indexed like roc_sg_forward_planned's.  ROC_ERR_INVALID: a NULL pointer or a leading dimension < H. */
int roc_sg_weighted_forward_planned(const roc_sg_plan* plan, int H, const float* in, int64_t ldIn, const float* w,
                                    float* out, int64_t ldOut, roc_stream_t stream);
/* roc_sg_weighted_forward_planned over bf16 rows (raw bits, see roc_f32_to_bf16), each value widened exactly in
 * registers and accumulated in fp32. `in` is 16-byte aligned and ldIn (in elements) is a multiple of 8, else
 * ROC_ERR_INVALID. The result is bit-identical to roc_sg_weighted_forward_planned on roc_bf16_to_f32(in) written to a
 * 16-byte aligned buffer with a leading dimension that is a multiple of 4: the plan, the row shapes, the column
 * blocks, the per-float order, the carries and the fix-ups are that call's. Its main launches report reduction 24 in
 * roc_sg_last_call_info. */
int roc_sg_weighted_forward_planned_bf16(const roc_sg_plan* plan, int H, const uint16_t* in, int64_t ldIn,
                                         const float* w, float* out, int64_t ldOut, roc_stream_t stream);
/* The gradient of the edge weights (an SDDMM): for every edge e of the plan, with G = outGrad indexed by plan row
 * and X = in indexed like the forward's input,
 *   dw[e - colLeft] = sum_h G[r][h] * X[j][h]          (accumulate != 0: added to the value dw holds)
 * in a fixed reduction order (columns in blocks of 512 floats on float4 rows, 256 otherwise, added in block order),
 * so the same call gives the same bits.  ROC_ERR_INVALID: a NULL pointer or a leading dimension < H. */
int roc_sg_edge_dot_planned(const roc_sg_plan* plan, int H, const float* outGrad, int64_t ldG, const float* in,
                            int64_t ldIn, float* dw, int accumulate, roc_stream_t stream);
/* roc_sg_edge_dot_planned with X = in in bf16 (raw bits, see roc_f32_to_bf16), each value widened exactly in
 * registers; G and dw stay fp32. `in` is 16-byte aligned and ldIn (in elements) is a multiple of 8, else
 * ROC_ERR_INVALID. The result is bit-identical to roc_sg_edge_dot_planned on roc_bf16_to_f32(in) written to a 16-byte
 * aligned buffer with a leading dimension that is a multiple of 4: the plan, the row shapes, the column blocks, the
 * per-float order, the carries and the fix-ups are that call's. Its launches report reduction 25 in
 * roc_sg_last_call_info. */
int roc_sg_edge_dot_planned_bf16(const roc_sg_plan* plan, int H, const float* outGrad, int64_t ldG,
                                 const uint16_t* in, int64_t ldIn, float* dw, int accumulate, roc_stream_t stream);
/* The transpose of a whole graph's CSR (rows 0..numNodes-1, edges 0..rowEnd[numNodes-1], every id < numNodes), for
 * the exact input gradient of the weighted aggregation on any graph (directed, asymmetric weights, duplicate edges):
 *   rowEndT  u64[numNodes]  END offsets of node v's out-edges
 *   colT     u32[E]         their destinations
 *   perm     u32[E]         the original edge of each transposed edge
 * built by a stable radix sort of (colSrc, edge index), so destinations increase within a transposed row; on a
 * symmetric graph whose rows have strictly increasing sources (rowEndT, colT) equals (rowEnd, colSrc).  It holds a plan
 * over (rowEndT, colT) and a buffer for the permuted weights.  rowEnd / colSrc must outlive it only during creation.
 * Creation synchronises the stream three times: to read E, to check the ids after the sort, and in the plan build
 * (roc_sg_plan_create).  ROC_ERR_INVALID: a NULL pointer or numNodes == 0; ROC_ERR_UNSUPPORTED: an id >= numNodes
 * (as a slice with global ids has), or E > 2^31 - 1.  roc_sg_transpose_info returns its device arrays and plan (tests). */
typedef struct roc_sg_transpose roc_sg_transpose;
int roc_sg_transpose_create(roc_vid_t numNodes, const roc_eid_t* rowEnd, const roc_vid_t* colSrc,
                            roc_stream_t stream, roc_sg_transpose** transpose);
int roc_sg_transpose_info(const roc_sg_transpose* transpose, const roc_eid_t** rowEndT, const roc_vid_t** colT,
                          const uint32_t** perm, const roc_sg_plan** planT);
void roc_sg_transpose_destroy(roc_sg_transpose* transpose);
/* The weighted aggregation's input gradient, exact on any graph:
 *   inGrad[j][h] = sum_{e : colSrc[e] = j} w[e] * outGrad[dst(e)][h]
 * computed as wT[t] = w[perm[t]] (one small kernel per call, into a buffer the transpose grows on the stream like a
 * plan's carries, so that changed weights are always seen) and roc_sg_weighted_forward_planned over the transposed
 * plan with wT.  outGrad and inGrad have numNodes rows.  ROC_ERR_INVALID: a NULL pointer or a leading dimension < H. */
int roc_sg_weighted_backward_planned(roc_sg_transpose* transpose, int H, const float* outGrad, int64_t ldG,
                                     const float* w, float* inGrad, int64_t ldIn, roc_stream_t stream);

/* Exact backwards of the sum, max / min and attention aggregations on any whole graph (directed, with duplicate edges
 * or nodes without in- or out-edges), over the transpose.  The gathers over the same CSR above (quirk Q1) stay the
 * default; these are the opt-in alternative (Model::set_exact_backward).  dst(e) is the row that owns edge e, and
 * transposed row j lists j's out-edges in the transpose's stable order.  outGrad, arg, inGrad and every per-node input
 * have numNodes rows.  On a symmetric graph whose rows have strictly increasing sources the transposed CSR is the CSR,
 * and each call returns exactly the bits of its counterpart named below.  They take the same row shapes and column
 * blocks as those, run in the plan's fixed order with no atomics (the same call gives the same bits), and report their
 * launches through roc_sg_last_call_info.  ROC_ERR_INVALID: a NULL pointer or a leading dimension < H.
 *
 * Sum (counterpart roc_sg_forward_planned with the same epilogue):
 *   inGrad[j][h] = epi( sum_{e : colSrc[e] = j} outGrad[dst(e)][h] )
 * NORM divides by sqrtf of j's IN-degree in the original graph, read from its rowEnd (required with NORM, else
 * ROC_ERR_INVALID), in the form that gives roc_indegree_norm's bits; RELU as in the forward. */
int roc_sg_transpose_sum_backward(roc_sg_transpose* transpose, int H, const float* outGrad, int64_t ldG, float* inGrad,
                                  int64_t ldIn, int epilogue, const roc_eid_t* rowEnd, roc_stream_t stream);
/* The exact backward of roc_sg_forward_dropout_planned: roc_sg_transpose_sum_backward over the kept edges only,
 *   inGrad[j][h] = epi( sum over the kept edges e with colSrc[e] = j: acc = fmaf(s, outGrad[dst(e)][h], acc) )
 * keep in the transposed plan's edge order (roc_sg_attn_keep_mask over roc_sg_transpose_info's planT, selfBase 0,
 * rowIsSource 1), so transposed edge j -> i carries keep(i <- j).  NORM divides by the original graph's in-degree, as
 * there.  Bytes equal roc_sg_weighted_backward_planned with w[e] = keep ? s : 0 followed by the unfused epilogue.
 * rate = 0 or keep = NULL: roc_sg_transpose_sum_backward itself.  ROC_ERR_INVALID: as that call, and a rate outside
 * [0, 1).  Main launches report reduction 42 with NORM (fix-ups 10), else 32 (fix-ups 0).  The backward over the same
 * CSR (quirk Q1) is roc_sg_forward_dropout_planned over the output gradient with the reverse-pair bytes (rowIsSource 1
 * over the forward plan), so that row u's edge to w carries keep(w <- u): exact on a symmetric graph. */
int roc_sg_transpose_sum_backward_dropout(roc_sg_transpose* transpose, int H, const float* outGrad, int64_t ldG,
                                          float* inGrad, int64_t ldIn, int epilogue, const roc_eid_t* rowEnd,
                                          const uint8_t* keep, float rate, roc_stream_t stream);
/* Max / min (counterpart roc_sg_minmax_backward_planned with selfBase 0), for arg from roc_sg_minmax_forward_planned:
 *   inGrad[j][h] = sum over the DISTINCT destinations i of j's out-edges of (arg[i][h] == j ? outGrad[i][h] : 0)
 * A duplicate edge j -> i lies next to its twin in transposed row j; an entry whose destination equals the previous
 * entry's in the same row adds nothing, so the result is the true adjoint on multigraphs too. */
int roc_sg_transpose_minmax_backward(roc_sg_transpose* transpose, int H, const float* outGrad, int64_t ldG,
                                     const roc_vid_t* arg, int64_t ldArg, float* inGrad, int64_t ldIn,
                                     roc_stream_t stream);
/* Attention (counterpart roc_sg_attn_backward_planned with selfBase 0), `plan` the whole graph's forward plan:
 *   scoreGrad[i][k]       = sum_{e : dst(e) = i, j = colSrc[e]} dz(i<-j,k)              (d s_dst, over `plan`)
 *   scoreGrad[j][heads+k] = sum_{e : colSrc[e] = j, i = dst(e)} dz(i<-j,k)              (d s_src)
 *   inGrad[j][kF+f]       = sum_{e : colSrc[e] = j, i = dst(e)} a(i<-j,k) G[i][kF+f]
 * with a, dz and the per-node record as in roc_sg_attn_backward_planned; a duplicate edge counts once per edge, as in
 * the forward.  The records cover ids [0, numNodes): no id scan, no synchronisation.  Head layouts and widths are
 * refused exactly as there; ROC_ERR_INVALID also when `plan` does not have the transpose's rows and edges. */
int roc_sg_attn_backward_exact(const roc_sg_plan* plan, roc_sg_transpose* transpose, int heads, int H, float slope,
                               const float* in, int64_t ldIn, const float* score, int64_t ldS, const float* out,
                               int64_t ldOut, const float* stats, int64_t ldStats, const float* outGrad, int64_t ldG,
                               float* inGrad, int64_t ldInG, float* scoreGrad, int64_t ldSG, roc_stream_t stream);
/* roc_sg_attn_backward_exact over bf16 feature rows X = in, as roc_sg_attn_backward_planned_bf16 is to
 * roc_sg_attn_backward_planned: bit-identical to roc_sg_attn_backward_exact on the widened rows, under the same input
 * rules, with its main launches reporting 22 and 23. */
int roc_sg_attn_backward_exact_bf16(const roc_sg_plan* plan, roc_sg_transpose* transpose, int heads, int H,
                                    float slope, const uint16_t* in, int64_t ldIn, const float* score, int64_t ldS,
                                    const float* out, int64_t ldOut, const float* stats, int64_t ldStats,
                                    const float* outGrad, int64_t ldG, float* inGrad, int64_t ldInG, float* scoreGrad,
                                    int64_t ldSG, roc_stream_t stream);
/* roc_sg_attn_backward_exact and its bf16 form with attention dropout (see roc_sg_attn_forward_dropout_planned): keep
 * in the forward plan's edge order, keepT in the transposed plan's (roc_sg_attn_keep_mask over planT, selfBase 0,
 * rowIsSource 1). */
int roc_sg_attn_backward_dropout_exact(const roc_sg_plan* plan, roc_sg_transpose* transpose, int heads, int H,
                                       float slope, const float* in, int64_t ldIn, const float* score, int64_t ldS,
                                       const float* out, int64_t ldOut, const float* stats, int64_t ldStats,
                                       const float* outGrad, int64_t ldG, float* inGrad, int64_t ldInG,
                                       float* scoreGrad, int64_t ldSG, const uint8_t* keep, const uint8_t* keepT,
                                       float rate, roc_stream_t stream);
int roc_sg_attn_backward_dropout_exact_bf16(const roc_sg_plan* plan, roc_sg_transpose* transpose, int heads, int H,
                                            float slope, const uint16_t* in, int64_t ldIn, const float* score,
                                            int64_t ldS, const float* out, int64_t ldOut, const float* stats,
                                            int64_t ldStats, const float* outGrad, int64_t ldG, float* inGrad,
                                            int64_t ldInG, float* scoreGrad, int64_t ldSG, const uint8_t* keep,
                                            const uint8_t* keepT, float rate, roc_stream_t stream);

/* Plan-less form with exactly the reference kernel's argument list
 * (scattergather_kernel.cu:21-28, EdgeStruct.dst dropped), dense ld == H.
 * Builds and frees a plan internally (synchronises); use the planned form in
 * loops. */
int roc_sg_forward(roc_vid_t rowLeft, roc_vid_t rowRight, roc_eid_t colLeft, int H,
                   const roc_eid_t* rowEnd, const roc_vid_t* colSrc,
                   const float* in, float* out, roc_stream_t stream);
/* Replaces ScatterGather::backward_task, scattergather_kernel.cu:160-170: the
 * identical computation on gradients (A, not A^T — quirk Q1). */
int roc_sg_backward(roc_vid_t rowLeft, roc_vid_t rowRight, roc_eid_t colLeft, int H,
                    const roc_eid_t* rowEnd, const roc_vid_t* colSrc,
                    const float* outGrad, float* inGrad, roc_stream_t stream);

/* Test hook: the kernel launches of the calling thread's last planned ScatterGather call (the roc_sg_*_planned entry
 * points, and the plan-less forms through them), in launch order, so that a test can assert which instantiation of
 * the row-shape table served a width and which fix-ups ran.  Column blocks and the passes of an attention call append
 * to one list.  Each entry:
 *   kind   ROC_SG_LAUNCH_*: the main kernel, its cp.async.bulk ring form (float4 sums of 17..64 T-columns), the
 *          fix-up of rows with at most 32 carries (one worker each), of rows with more (one CTA each), the attention
 *          stats fix-up, the attention backward's per-node record, the fix-ups of its heads-wide partials, the
 *          weighted backward's weight permutation (first in its list), the keep mask, and the dynamic attention
 *          backward's column sums of da (and the softmax backward's sums of dt)
 *   red    the reduction the kernel is instantiated for: 0 sum, 1 max, 2 min, 3 the min / max backward, 4 attention
 *          stats, 5 the attention forward, 6 its d s_dst gather, 7 its input-gradient gather, 8 the weighted sum
 *          (forward and backward), 9 the edge-weight gradient, 10 the exact sum backward with NORM (the sum whose
 *          epilogue divides by the original graph's in-degree; its main kernel, ring and fix-ups), 11 the exact max /
 *          min backward, 12 the sum over bf16 rows (its main kernel and ring), 13 the teleport sum
 *          (roc_sg_forward_teleport_planned: its main kernel and fix-ups); 16 + r for the main kernel of
 *          reduction r over bf16 feature rows (17 max, 18 min, 21 attention forward, 22 d s_dst, 23 input gradient,
 *          24 weighted sum, 25 edge-weight gradient: the roc_sg_*_bf16 calls), whose fix-ups are reduction r's and
 *          report as there; 32 + r for the main kernel of attention pass r (5, 6, 7, or 21, 22, 23 on bf16 feature
 *          rows) with dropout (the roc_sg_attn_*_dropout_* calls at rate > 0: 37, 38, 39, 53, 54, 55), whose other
 *          launches report as without dropout; likewise 32, 42 and 45 for the sum, the exact sum backward with NORM
 *          and the teleport sum with edge dropout (roc_sg_forward_dropout_planned,
 *          roc_sg_transpose_sum_backward_dropout, roc_sg_forward_teleport_dropout_planned at rate > 0); 64, 65, 66 and 67 for
 *          the dynamic attention passes (roc_sg_attn_v2_*); 72, 73 and 74 for the softmax aggregation's forward and
 *          source passes (roc_sg_softmax_*: its forward fix-ups report 72); -1 for the records, the permutation, the keep mask and
 *          the column sums, which have none.  A sum fix-up finishing another
 *          reduction's partials reports 0.
 *   vec    4 for float4 rows, else 1;  lanes, nch: the row shape (L lanes, chunks per lane);  grid: CTAs launched
 * count is the number of launches; the first ROC_SG_MAX_LAUNCHES are stored.  Every planned call clears the list first,
 * also one that fails before it launches anything.  ROC_ERR_INVALID for a NULL info. */
#define ROC_SG_LAUNCH_MAIN 0
#define ROC_SG_LAUNCH_RING 1
#define ROC_SG_LAUNCH_FIXUP 2
#define ROC_SG_LAUNCH_BIG_FIXUP 3
#define ROC_SG_LAUNCH_STAT_FIXUP 4
#define ROC_SG_LAUNCH_RECORD 5
#define ROC_SG_LAUNCH_HEADS_FIXUP 6
#define ROC_SG_LAUNCH_HEADS_BIG_FIXUP 7
#define ROC_SG_LAUNCH_PERMUTE 8
#define ROC_SG_LAUNCH_KEEP_MASK 9     /* roc_sg_attn_keep_mask (red -1) */
#define ROC_SG_LAUNCH_COLSUM 10       /* roc_sg_attn_v2_backward_*: da's fp64 column sums; roc_sg_softmax_backward_*:
                                         dt's fp64 sums (red -1) */
#define ROC_SG_MAX_LAUNCHES 32
typedef struct {
  int kind, red, vec, lanes, nch;
  int64_t grid;
} roc_sg_launch;
typedef struct {
  int count;
  roc_sg_launch launch[ROC_SG_MAX_LAUNCHES];
} roc_sg_call_info;
int roc_sg_last_call_info(roc_sg_call_info* info);

/* ----------------------------------------------------------------- halo --- */

/* Boundary-node structures of one partition (multi-GPU).  The reference hands every
 * partition the WHOLE input region before ScatterGather (scattergather.cc:69-73); here a
 * partition receives only the distinct remote rows its edges read.  From the partition's
 * sources (global ids, device) builds
 *   ids[nHalo]      sorted distinct sources outside [rowLeft, rowRight] (grouped by owner,
 *                   since partitions are contiguous id ranges)
 *   colLocal[nEdges] = src - rowLeft (own rows) | Nloc + rank in ids (halo rows)
 * — a private, derived copy; colSrc stays the canonical CSR.  Synchronises the stream. */
typedef struct roc_halo roc_halo;
int roc_halo_create(roc_vid_t rowLeft, roc_vid_t rowRight, uint64_t nEdges, const roc_vid_t* colSrc,
                    roc_stream_t stream, roc_halo** out);
void roc_halo_destroy(roc_halo* h);
uint32_t roc_halo_size(const roc_halo* h);
const roc_vid_t* roc_halo_ids(const roc_halo* h);         /* device */
const roc_vid_t* roc_halo_col_local(const roc_halo* h);   /* device */
/* Host-side bookkeeping of the exchange (HOST pointers, no device work).  recv: the sorted halo ids are
 * grouped by owner (partitions are contiguous id ranges, host_vbounds as in roc_partition):
 * recvOffs[q] / recvCounts[q] = first halo row owned by partition q / how many; ROC_ERR_INVALID if the
 * list is not strictly increasing, leaves every range, or names one of this partition's own rows.
 * send: host_allCounts[q * P + r] = rows partition q requests from owner r (every rank's recvCounts,
 * all-gathered); this rank packs the rows q asked of it for q = 0..P-1 in order. */
int roc_halo_recv_layout(uint32_t nHalo, const roc_vid_t* host_ids, int numParts, int myPart,
                         const roc_vid_t* host_vbounds, uint64_t* recvCounts, uint64_t* recvOffs);
int roc_halo_send_layout(int numParts, int myPart, const int32_t* host_allCounts, uint64_t* sendCounts,
                         uint64_t* sendOffs, uint64_t* numSendRows);
/* roc_pack_rows for a subset: dst[sel[t]] = src[rows[sel[t]]] for t < nSel — the send-list entries of one row
 * block, written to their places in the send buffer, so that the block can travel (copy engines, peer slabs) while
 * the producer computes the next one.  Writes the float4 pad columns [H, round_up(H, 4)) as roc_pack_rows does. */
int roc_pack_rows_at(int64_t nSel, int H, const roc_vid_t* sel, const roc_vid_t* rows, const float* src,
                     int64_t ldSrc, float* dst, int64_t ldDst, roc_stream_t stream);
/* Fused pack + exchange over peer memory: row srcRows[j] of `src` is stored to
 * host_peerBase[peer[j]] + dstRow[j] * ldDst — the halo slab of the partition that reads it, in ANOTHER GPU's
 * memory (device pointers the caller mapped with cudaIpcOpenMemHandle; the stores travel over NVLink).  Replaces
 * roc_pack_rows + the NCCL all-to-all-v of the staged rows (themselves the replacement of the reference's
 * whole-region request, scattergather.cc:69-73).  srcRows / peer / dstRow are device arrays of nRows entries;
 * host_peerBase is a HOST array of numPeers <= ROC_MAX_PEERS device pointers (entries never named by peer[] may be
 * NULL).  smLimit > 0 sizes the grid for that many SMs (the ones a producer running beside it left free, see
 * roc_set_sm_reserve); 0 = whole chip.  The caller orders the consumer after every producer (a barrier across
 * the partitions).  With ldSrc, ldDst, src and every non-NULL peer base 16-byte aligned, each row is stored as whole
 * float4s: columns [H, round_up(H, 4)) of the destination row receive the source row's pad columns; columns from
 * round_up(H, 4) on are never written.  Otherwise exactly columns [0, H) are. */
#define ROC_MAX_PEERS 16
int roc_push_rows(int64_t nRows, int H, const roc_vid_t* srcRows, const uint8_t* peer, const roc_vid_t* dstRow,
                  const float* src, int64_t ldSrc, float* const* host_peerBase, int numPeers, int64_t ldDst,
                  int smLimit, roc_stream_t stream);
/* dst[j][0:H] = src[rows[j]][0:H]: packs the rows another partition asked for into a send buffer.
 * Pad columns: when ldSrc and ldDst are multiples of 4 and both bases are 16-byte aligned, the rows travel as whole
 * float4s, so dst[j][H:round_up(H, 4)] also receives src[rows[j]][H:round_up(H, 4)]; columns from round_up(H, 4) on
 * are never written.  Otherwise exactly dst[j][0:H] is written.  The same holds for roc_pack_rows_at and, with every
 * peer base aligned, for roc_push_rows: callers pass whole padded rows. */
int roc_pack_rows(int64_t nRows, int H, const roc_vid_t* rows, const float* src, int64_t ldSrc,
                  float* dst, int64_t ldDst, roc_stream_t stream);

/* ---------------------------------------------------------- elementwise --- */

/* Replaces norm_coop_kernel, graphnorm_kernel.cu:19-57 (fwd and bwd :126-136):
 * out[n][h] = in[n][h] / sqrtf((float)deg(n)); in/out are the partition's rows.
 * If `also_relu_mask_of` is non-NULL (fused backward of relu∘norm, gnn.cc:84-85):
 * out = (also_relu_mask_of > 0 ? in : 0) / sqrtf(deg); it has `in`'s shape and
 * leading dimension (it is the relu output whose gradient `in` is).
 * Pad columns: when ldIn and ldOut are multiples of 4 and in, out and the mask are 16-byte
 * aligned, rows are processed as whole float4s, whatever H is: columns [H, round_up(H, 4))
 * of each output row receive that row's input pad columns, masked and divided the same
 * way (a NaN pad gives NaN, a zero pad 0, or NaN in a row of degree 0).  Columns from
 * round_up(H, 4) on are never written.  Otherwise exactly columns [0, H) are. */
int roc_indegree_norm(roc_vid_t rowLeft, roc_vid_t rowRight, roc_eid_t colLeft, int H,
                      const roc_eid_t* rowEnd, const float* in, int64_t ldIn,
                      float* out, int64_t ldOut, const float* also_relu_mask_of,
                      roc_stream_t stream);

/* Replaces cudnnActivationForward/Backward, activation_kernel.cu:64-66, 128-132.
 * bwd: dX (+)= dY * f'(.) evaluated from the OUTPUT y; accumulate != 0 adds
 * into dX (the reference's beta = 1 on a loaded buffer, gnn.cc:704-713).
 * ROC_AC_MODE_ELU: y = x > 0 ? x : expm1f(x) (NaN propagates), and dX (+)= dY * (y > 0 ? 1 : y + 1), which is the
 * derivative because y > 0 exactly when x > 0 (torch's elu_backward with is_result). */
int roc_activation_fwd(int64_t rows, int H, int mode, const float* x, int64_t ldX,
                       float* y, int64_t ldY, roc_stream_t stream);
int roc_activation_bwd(int64_t rows, int H, int mode, const float* y, int64_t ldY,
                       const float* dY, int64_t ldDY, float* dX, int64_t ldDX,
                       int accumulate, roc_stream_t stream);
/* ROC_AC_MODE_RELU with a bf16 output (raw bits, see roc_f32_to_bf16): fwd stores exactly roc_f32_to_bf16 of what
 * roc_activation_fwd stores, in columns [0, H) (the rest of each row is never written); bwd is roc_activation_bwd on
 * the widened y, so its mask is the stored bf16 value's.  That mask differs from the fp32 value's in one case only: a
 * positive fp32 value no larger than 2^-134 (half of bf16's smallest subnormal) rounds to +0 and masks its gradient.
 * Any other mode is ROC_ERR_UNSUPPORTED. */
int roc_activation_fwd_y_bf16(int64_t rows, int H, int mode, const float* x, int64_t ldX, uint16_t* y, int64_t ldY,
                              roc_stream_t stream);
int roc_activation_bwd_y_bf16(int64_t rows, int H, int mode, const uint16_t* y, int64_t ldY, const float* dY,
                              int64_t ldDY, float* dX, int64_t ldDX, int accumulate, roc_stream_t stream);

/* Replaces op_kernel (EW_TYPE_ADD), element_kernel.cu:19-39, and its backward
 * add_kernel pair, :93-101. */
int roc_add_fwd(int64_t rows, int H, const float* a, int64_t ldA, const float* b,
                int64_t ldB, float* y, int64_t ldY, roc_stream_t stream);
int roc_add_bwd(int64_t rows, int H, const float* dY, int64_t ldDY, float* dA,
                int64_t ldDA, int accA, float* dB, int64_t ldDB, int accB,
                roc_stream_t stream);
/* Scaled add (APPNP / GCNII's initial residual; not in the reference): y = fmaf(alpha, a, beta * b), the product
 * beta * b rounded to fp32 first.  At alpha = beta = 1 it gives roc_add_fwd's bits.  Backward: dA = alpha * dY, or
 * fmaf(alpha, dY, dA) with accA; dB likewise with beta; a NULL dA or dB is skipped.  16-byte streaming accesses when H,
 * the leading dimensions and the pointers allow.  ROC_ERR_INVALID: a NULL a, b, y or dY, a leading dimension < H,
 * non-finite alpha or beta, or dA == dB. */
int roc_scaled_add_fwd(int64_t rows, int H, float alpha, const float* a, int64_t ldA, float beta, const float* b,
                       int64_t ldB, float* y, int64_t ldY, roc_stream_t stream);
int roc_scaled_add_bwd(int64_t rows, int H, const float* dY, int64_t ldDY, float alpha, float* dA, int64_t ldDA,
                       int accA, float beta, float* dB, int64_t ldDB, int accB, roc_stream_t stream);

/* Replaces cudnnDropoutForward/Backward, dropout_kernel.cu:98-99, 149-150.
 * y = keep ? x / (1 - rate) : 0.  cuDNN's generator is not reproducible, so the
 * mask is defined here instead: element (globalRow r, column c) keeps iff 16-bit
 * lane (c & 7) of Philox4x32-10(counter = {r lo, r hi, c >> 3, step},
 * key = {seed lo, seed hi}) >= round(rate * 65536); lanes are numbered low half
 * of word 0, high half of word 0, low half of word 1, ...  One Philox block
 * decides 8 consecutive columns of one row; the mask does not depend on the
 * tensor's width or on how rows are split across GPUs.  It is recomputed in bwd
 * (no reserve space).  `firstRow` = global index of the slab's first row (rowLeft). */
int roc_dropout_fwd(int64_t rows, int H, int64_t firstRow, float rate, uint64_t seed,
                    uint32_t step, const float* x, int64_t ldX, float* y, int64_t ldY,
                    roc_stream_t stream);
int roc_dropout_bwd(int64_t rows, int H, int64_t firstRow, float rate, uint64_t seed,
                    uint32_t step, const float* dY, int64_t ldDY, float* dX,
                    int64_t ldDX, roc_stream_t stream);
/* roc_dropout_fwd on a bf16 x (raw bits, see roc_f32_to_bf16), writing fp32 y.  Each element
 * widens to fp32 exactly, so y is bit-identical to roc_dropout_fwd on the widened x (same
 * mask, same scale).  rate == 0 is the widening copy. */
int roc_dropout_fwd_bf16(int64_t rows, int H, int64_t firstRow, float rate, uint64_t seed,
                         uint32_t step, const uint16_t* x, int64_t ldX, float* y, int64_t ldY,
                         roc_stream_t stream);

/* The same mask, packed one bit per element: bit (h & 31) of
 * mask[row * ldMask + (h >> 5)] = keep(firstRow + row, h).  ldMask (32-bit words per
 * row) must be a multiple of 4 and >= ceil(H/32); words / bits beyond H are written 0.
 * Feeds roc_linear_fwd_dropout / roc_linear_bwd_dropout, which apply dropout to the
 * Linear's input while loading it, so the dropped copy of X (dropout_kernel.cu:98's
 * output tensor) is never written to or re-read from HBM. */
int roc_dropout_mask(int64_t rows, int H, int64_t firstRow, float rate, uint64_t seed,
                     uint32_t step, uint32_t* mask, int64_t ldMask, roc_stream_t stream);

/* Replaces SoftmaxCrossEntropy::backward_task, softmax_kernel.cu:81-171:
 * cudnnSoftmaxForward(ACCURATE) -> calc_loss (:41-79) -> softmax_backward
 * (:19-33) in ONE kernel.  `labels` is the one-hot fp32 [rows][ldL] tensor the
 * reference loads (load_task.cu:118-123); `mask` is int32 per row.
 * `perf` (device, may be NULL) is ACCUMULATED into (zero it first). */
int roc_softmax_xent_bwd(int64_t rows, int C, const float* logits, int64_t ldZ,
                         const float* labels, int64_t ldL, const int32_t* mask,
                         float* grad, int64_t ldG, roc_perf_metrics* perf,
                         roc_stream_t stream);

/* Same computation with compact labels: labelIdx[v] = class index (what
 * load_task.cu:118-123 expands to one-hot); 4 B/row instead of 4C B/row. */
int roc_softmax_xent_bwd_idx(int64_t rows, int C, const float* logits, int64_t ldZ,
                             const int32_t* labelIdx, const int32_t* mask, float* grad,
                             int64_t ldG, roc_perf_metrics* perf, roc_stream_t stream);

/* roc_softmax_xent_bwd(_idx) with the backward of the InDegreeNorm that produced the logits
 * (gnn.cc:85 / graphnorm_kernel.cu:133) folded in: grad[v] = ((P - labels) or 0) / sqrtf(deg(v)).
 * Exactly one of `labels` (one-hot fp32) / `labelIdx` (class index per row) is non-NULL;
 * rowEnd is rowLeft-relative as everywhere.  Bit-identical to roc_softmax_xent_bwd followed
 * by roc_indegree_norm on the gradient. */
int roc_softmax_xent_bwd_norm(int64_t rows, int C, const float* logits, int64_t ldZ,
                              const float* labels, int64_t ldL, const int32_t* labelIdx,
                              const int32_t* mask, float* grad, int64_t ldG,
                              const roc_eid_t* rowEnd, roc_eid_t colLeft,
                              roc_perf_metrics* perf, roc_stream_t stream);

/* Multi-label sigmoid cross-entropy: loss, gradient and metrics in one pass over logits Z[rows][C] (row pitch ldZ)
 * with hard labels Y[rows][C] in {0, 1} and the row mask (ROC_MASK_*).
 *  - Labels are bit-packed: each row holds W = ceil(C / 32) words, bit (c % 32) of word c / 32 is label c, and the
 *    row pitch is ldB words.
 *  - Per element the loss is  l = max(z, 0) - z*y + log1p(exp(-|z|))  (torch's binary_cross_entropy_with_logits in its
 *    stable form), computed in fp32.
 *  - grad[r][c] = sigmoid(z) - y on rows whose mask is ROC_MASK_TRAIN and 0 on every other row (no averaging, the
 *    softmax head's convention).  Exactly columns [0, C) of every row are written.
 *  - A class is predicted positive iff z > 0 (so z = 0 and NaN are negative).
 *  - With a non-NULL rowEnd the gradient is divided by sqrtf(in-degree) as roc_softmax_xent_bwd_norm does (the
 *    backward of the InDegreeNorm that produced the logits; rowEnd is rowLeft-relative): bit-identical to the call
 *    with rowEnd = NULL followed by roc_indegree_norm on the gradient.
 *  - `metrics` (device, may be NULL) is ACCUMULATED into: zero it first.  Rows with mask ROC_MASK_NONE (or any value
 *    outside 0..2) count nowhere.  The loss is summed in fp32 over each run of up to 4 consecutive elements of a row,
 *    then in fp64 into per-block partials that one block adds in block order, so the same call on the same device
 *    with the same SM budget gives the same bits; the counts are exact.  The loss's bits may differ between SM
 *    counts: each thread sums the rows it visits, and which rows those are depends on the grid, which is sized from
 *    the SMs the calling thread may use (roc_set_sm_reserve).  The gradient's bits never depend on it.  Calls that
 *    pass `metrics` share one per-device scratch for the partials: do not run two of them at once on different
 *    streams of one device.
 * ROC_ERR_INVALID: a NULL logits / labelBits / mask / grad, rows < 0, C < 1, ldZ or ldG < C, ldB < W. */
int roc_sigmoid_xent_bwd(int64_t rows, int C, const float* logits, int64_t ldZ, const uint32_t* labelBits,
                         int64_t ldB, const int32_t* mask, float* grad, int64_t ldG,
                         const roc_eid_t* rowEnd /* NULL: no norm */, roc_eid_t colLeft,
                         roc_multilabel_metrics* metrics /* may be NULL */, roc_stream_t stream);

/* ------------------------------------------------------- batch normalisation --- */

/* Batch normalisation over the rows of X[rows][H] (torch.nn.BatchNorm1d over every row), one forward and one
 * backward entry.  X, Y, dY and dX rows are read and written as 16-byte groups: their pitches must be multiples of 4
 * and their bases 16-byte aligned (ROC_ERR_INVALID otherwise).  Columns [H, ld) of a row may be loaded but are never
 * written, and their values reach no result.
 *  - Statistics: per column, the mean and the biased variance (divide by rows) from one pass that sums (x - K) and
 *    (x - K)^2 in fp64 with K = X[0][c], so the variance stays accurate when |mean| >> std.  Rows are summed in fixed
 *    blocks whose size depends on (rows, H) only, each block's fp64 partial is added in block order, so the same call
 *    gives the same bits on any device.
 *  - training != 0: a = gamma * invstd and b = beta - mean * a, invstd = 1 / sqrt(var + eps), computed in fp64 and
 *    stored in fp32 in saveA / saveB; saveMean / saveInvStd (fp64) keep mean and invstd for the backward.  The running
 *    statistics (fp32, may both be NULL) become  runMean = (1 - momentum) runMean + momentum mean  and
 *    runVar = (1 - momentum) runVar + momentum var rows / (rows - 1), computed in fp64.  Needs rows >= 2.
 *  - training == 0: a and b from runMean / runVar instead (both required), into the workspace; nothing else is
 *    written but Y.
 *  - Y = fma(X, a, b) per column, then relu (x > 0 ? x : 0, NaN kept) when relu != 0.
 * The workspace holds the coefficients and the fp64 partials: roc_batchnorm_workspace_bytes(rows, H), 16-byte aligned.
 * ROC_ERR_INVALID: a NULL x / gamma / beta / y / workspace, rows < 0, H <= 0, ldX or ldY < H, eps < 0, momentum
 * outside [0, 1], only one running statistic, a missing save pointer or rows < 2 in training, no running statistics in
 * inference, a short workspace. */
size_t roc_batchnorm_workspace_bytes(int64_t rows, int H);
int roc_batchnorm_fwd(int64_t rows, int H, const float* x, int64_t ldX, const float* gamma, const float* beta,
                      double eps, double momentum, float* runMean, float* runVar, int training, int relu,
                      float* y, int64_t ldY, float* saveA, float* saveB, double* saveMean, double* saveInvStd,
                      void* workspace, size_t workspaceBytes, roc_stream_t stream);
/* The backward of a training roc_batchnorm_fwd on the same x, gamma and saved values.  With g' = dY, or with relu != 0
 * dY masked by fma(x, saveA, saveB) > 0 (the forward's own relu test, so no Y is read):
 *   dBeta = sum_rows g',  dGamma = invstd * sum_rows g' (x - mean)        (fp64 sums as the forward's, stored fp32)
 *   dX (+)= A g' + B x + C  with  A = gamma invstd,  B = -A invstd dGamma / rows,  C = -A dBeta / rows - B mean
 * (fp64 coefficients stored in fp32, two fp32 FMAs per element), which is gamma invstd (g' - dBeta / rows -
 * xhat dGamma / rows).  accumulate selects += over =; dX == NULL computes dGamma and dBeta only.  dGamma and dBeta are
 * overwritten.  ROC_ERR_INVALID as for the forward, and for rows < 2, a NULL dY / gamma / saved statistics / dGamma /
 * dBeta, or relu without saveA / saveB. */
int roc_batchnorm_bwd(int64_t rows, int H, const float* x, int64_t ldX, const float* dY, int64_t ldDY, int relu,
                      const float* gamma, const float* saveA, const float* saveB, const double* saveMean,
                      const double* saveInvStd, float* dGamma, float* dBeta, float* dX, int64_t ldDX, int accumulate,
                      void* workspace, size_t workspaceBytes, roc_stream_t stream);

/* ------------------------------------------------------- layer normalisation --- */

/* Layer normalisation over the columns of each row of X[rows][H] (torch.nn.LayerNorm(H, eps) with its affine gamma,
 * beta), one forward and one backward entry.  Per row, in fp32:
 *   mu = mean_c x[c],  var = mean_c (x[c] - mu)^2  (the biased variance about the mean, never E[x^2] - E[x]^2),
 *   rstd = 1 / sqrt(var + eps),  xhat = (x - mu) rstd,  y = xhat gamma[c] + beta[c]  (one fma),
 * then relu (x > 0 ? x : 0, NaN kept) when relu != 0.  The sums are fp32 in a fixed order (each row's own elements in
 * column order within a lane, then an xor butterfly across the lanes of the row) and the divisions and the square
 * root are correctly rounded, so a row's results depend on that row alone and are the same bits on any device and at
 * any SM budget.  The same forward serves training and inference: nothing is kept per row and there are no running
 * statistics.  An H = 1 row gives y = beta.  X, Y, dY and dX rows are read and written as 16-byte groups: their
 * pitches must be multiples of 4 and their bases 16-byte aligned (ROC_ERR_INVALID otherwise).  Columns [H, ld) may be
 * loaded but are never written, and their values reach no result.  rows = 0 writes nothing.
 * ROC_ERR_INVALID: a NULL x / gamma / beta / y, rows < 0, H <= 0, ldX or ldY < H, a misaligned base or pitch, eps
 * negative or not finite. */
int roc_layernorm_fwd(int64_t rows, int H, const float* x, int64_t ldX, const float* gamma, const float* beta,
                      float eps, int relu, float* y, int64_t ldY, roc_stream_t stream);
/* The fp64 gamma / beta partials of roc_layernorm_bwd: double2 [ceil(rows / 1024)][H] (at least one block). */
size_t roc_layernorm_workspace_bytes(int64_t rows, int H);
/* The backward of roc_layernorm_fwd on the same x, gamma, beta and eps.  It recomputes each row's mu, rstd and xhat
 * from x, bit for bit the forward's.  With g' = dY, or with relu != 0 dY masked by the forward's own pre-relu value
 * xhat gamma + beta > 0 (so no Y is read):
 *   gh = g' gamma,  dX (+)= rstd (gh - mean_c gh - xhat mean_c(gh xhat))       (fp32; accumulate selects += over =)
 *   dGamma = sum_rows g' xhat,  dBeta = sum_rows g'
 * The column sums are fp64 over fixed blocks of 1024 rows, the blocks added in block order and rounded once to fp32,
 * so they are the same bits on any device.  dGamma and dBeta are overwritten; rows = 0 writes zeros there.  dX == NULL
 * computes dGamma and dBeta only.  An H = 1 row gives dX = 0.  A NaN in a row reaches that row's y and dx, and dGamma
 * through its xhat; dBeta only through dY.  One pass over x and dY (and dX when accumulating), no atomics.
 * ROC_ERR_INVALID: as for the forward, and for a NULL dY / dGamma / dBeta / workspace, ldDY or ldDX < H, a
 * misaligned dY / dX / workspace, or workspaceBytes < roc_layernorm_workspace_bytes(rows, H). */
int roc_layernorm_bwd(int64_t rows, int H, const float* x, int64_t ldX, const float* dY, int64_t ldDY, int relu,
                      const float* gamma, const float* beta, float eps, float* dGamma, float* dBeta, float* dX,
                      int64_t ldDX, int accumulate, void* workspace, size_t workspaceBytes, roc_stream_t stream);

/* ------------------------------------------------------- attention scores --- */

/* The per-head GAT attention scores (Velickovic et al., 2018; PyG's GATConv): X is [rows][H] with H = heads * F, and
 * column c belongs to head c / F.  A is [2 * heads][F], dense: row k is a_dst of head k and row heads + k its a_src.
 * S is [rows][2 * heads] in the layout roc_sg_attn_* read:
 *   S[v][k] = sum_f A[k][f] X[v][kF + f],   S[v][heads + k] = sum_f A[heads + k][f] X[v][kF + f]
 * each summed in fp32 with one fma per product, f = 0 .. F - 1 in order.  Only columns [0, 2 * heads) of S and
 * [0, H) of dX are written; columns [H, ldX) of X may be loaded but reach no result.
 * bwd:
 *   dX[v][kF + f] (+)= fma(dS[v][heads + k], A[heads + k][f], dS[v][k] * A[k][f])   (accumulate != 0: +=)
 *   dA[k][f] = sum_v dS[v][k] X[v][kF + f],  dA[heads + k][f] = sum_v dS[v][heads + k] X[v][kF + f]
 * dA is overwritten; its sums are taken in fp64 over row blocks whose size depends on (rows, H) only, the blocks'
 * partials added in block order, then rounded once to fp32, so the same call gives the same bits every time.
 * dX == NULL computes dA only.  The workspace holds the partials: roc_attn_scores_workspace_bytes(rows, H, heads),
 * 16-byte aligned.  X rows are read as 16-byte vectors (bf16: 8-byte) when ldX is a multiple of 4 and X is so
 * aligned, else element by element, with the same results.
 * ROC_ERR_INVALID: a NULL X / A / S / dS / dA / workspace, rows < 0, H <= 0, heads <= 0, ldX < H, ldS or
 * ldDS < 2 * heads, ldDX < H with a dX, a short or misaligned workspace.  ROC_ERR_UNSUPPORTED: H % heads != 0 or
 * H > 1024.  The _bf16 forms take X as raw bf16 bits (see roc_f32_to_bf16) and give the bytes of the fp32 call on the
 * widened rows. */
size_t roc_attn_scores_workspace_bytes(int64_t rows, int H, int heads);
int roc_attn_scores_fwd(int64_t rows, int H, int heads, const float* X, int64_t ldX, const float* A, float* S,
                        int64_t ldS, roc_stream_t stream);
int roc_attn_scores_bwd(int64_t rows, int H, int heads, const float* X, int64_t ldX, const float* A, const float* dS,
                        int64_t ldDS, float* dX, int64_t ldDX, int accumulate, float* dA, void* workspace,
                        size_t workspaceBytes, roc_stream_t stream);
int roc_attn_scores_fwd_bf16(int64_t rows, int H, int heads, const uint16_t* X, int64_t ldX, const float* A, float* S,
                             int64_t ldS, roc_stream_t stream);
int roc_attn_scores_bwd_bf16(int64_t rows, int H, int heads, const uint16_t* X, int64_t ldX, const float* A,
                             const float* dS, int64_t ldDS, float* dX, int64_t ldDX, int accumulate, float* dA,
                             void* workspace, size_t workspaceBytes, roc_stream_t stream);

/* --------------------------------------------------------------- Linear --- */

/* Replaces cublasSgemm in Linear::forward_task, linear_kernel.cu:76-80 (+ the
 * optional in-place ReLU :83-104):  Y[v][o] = sum_i X[v][i] * W[o*inDim + i].
 * W is the reference's column-major [inDim][outDim] weight (ld = inDim, Q6).
 * flags: ROC_LINEAR_NORM_EPILOGUE divides row v by sqrtf(deg(v)) (fuses the
 * indegree_norm that follows linear in the model, gnn.cc:81-82); then needs
 * rowLeft-relative rowEnd/colLeft (else pass NULL/0). */
#define ROC_LINEAR_NORM_EPILOGUE 1
/* ROC_LINEAR_Y_BF16 (roc_linear_fwd, roc_linear_fwd_dropout, roc_linear_fwd_bf16): Y holds bf16 bits (pass a
 * uint16_t buffer cast to float*), ldY is in elements and a multiple of 8, else ROC_ERR_INVALID.  Each stored value is
 * exactly roc_f32_to_bf16 of what the same call stores without the flag, and the columns [outDim, ldY) are never
 * written.  The wgmma kernel stores a tile of at most 64 columns through a bf16 staging tile by TMA, wider ones and
 * the last outDim % 8 columns directly; the SIMT kernel narrows as it stores. */
#define ROC_LINEAR_Y_BF16 2
int roc_linear_fwd(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX,
                   const float* W, float* Y, int64_t ldY, int activation, int flags,
                   const roc_eid_t* rowEnd, roc_eid_t colLeft, roc_stream_t stream);

/* Replaces Linear::backward_task, linear_kernel.cu:129-245:
 *   if activation == RELU: dY = (Y > 0) ? dY : 0 in place (reluBackward :120-127)
 *   dW[o*inDim+i] += sum_v X[v][i] * dY[v][o]        (sgemm beta = 1, :220-224)
 *   dX[v][i] (+)= sum_o W[o*inDim+i] * dY[v][o]       (:227-231) — skipped when
 *   dX == NULL (leaf input, quirk Q8); accumulate_dX selects += vs =.
 * `workspace` holds split-K partials of dW; size from roc_linear_bwd_workspace_bytes. */
/* roc_linear_fwd on dropout(X): Y = (keep ? X / (1 - rate) : 0) W^T with `mask` from
 * roc_dropout_mask (same rate).  Bit-identical to roc_dropout_fwd followed by
 * roc_linear_fwd.  rate == 0 ignores the mask (infer mode: dropout is a copy,
 * dropout_kernel.cu:159-180). */
int roc_linear_fwd_dropout(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX,
                           const float* W, float* Y, int64_t ldY, int activation, int flags,
                           const roc_eid_t* rowEnd, roc_eid_t colLeft, const uint32_t* mask,
                           int64_t ldMask, float rate, roc_stream_t stream);

/* ---- bf16 input features.  A leaf node tensor (the raw features X) may be stored in bf16:
 * raw bits as uint16_t, round-to-nearest-even from fp32 (roc_f32_to_bf16), rows of
 * ld >= inDim elements.  The tensor-core kernels read it by TMA and take ld a multiple of 8
 * (16-byte rows) and a 16-byte aligned base; other layouts, and the shapes they refuse, run on
 * the SIMT kernels as the fp32 entry points do (roc_last_gemm_info tells which).  A bf16 value
 * has 8 significant bits, so it widens to fp32 exactly and its TF32 split has a zero low part:
 * each kernel widens X as it reads it and then computes what it computes in fp32.
 *
 * roc_linear_fwd_dropout with a bf16 X: mask == NULL and rate == 0 means no dropout.  Y is
 * bit-identical to roc_linear_fwd_dropout on the widened X (on the same path, tensor cores or
 * SIMT). */
int roc_linear_fwd_bf16(int64_t rows, int inDim, int outDim, const uint16_t* X, int64_t ldX,
                        const float* W, float* Y, int64_t ldY, int activation, int flags,
                        const roc_eid_t* rowEnd, roc_eid_t colLeft, const uint32_t* mask,
                        int64_t ldMask, float rate, roc_stream_t stream);
/* dW of a Linear whose input is a bf16 X (a leaf: there is no dX):
 *   if activation == RELU: dY = (Y > 0) ? dY : 0 in place
 *   dW[o*inDim+i] += sum_v dropout(X)[v][i] * dY[v][o]
 * with the dropout as in roc_linear_fwd_bf16 and `workspace` sized by
 * roc_linear_bwd_workspace_bytes.  dY and dW are bit-identical to roc_linear_bwd_dropout with
 * dX == NULL on the widened X (on the same path and dW kernel). */
int roc_linear_dw_bf16(int64_t rows, int inDim, int outDim, const uint16_t* X, int64_t ldX,
                       const float* Y, int64_t ldY, float* dY, int64_t ldDY, float* dW,
                       int activation, void* workspace, size_t workspaceBytes,
                       const uint32_t* mask, int64_t ldMask, float rate, roc_stream_t stream);

size_t roc_linear_bwd_workspace_bytes(int64_t rows, int inDim, int outDim);
int roc_linear_bwd(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX,
                   const float* W, const float* Y, int64_t ldY, float* dY,
                   int64_t ldDY, float* dW, float* dX, int64_t ldDX,
                   int activation, int accumulate_dX, void* workspace,
                   size_t workspaceBytes, roc_stream_t stream);

/* roc_linear_bwd where the forward input was dropout(X) (X = the tensor BEFORE dropout):
 * dW uses the masked, scaled X; dX (if non-NULL) is the gradient of the dropout's INPUT,
 * i.e. cudnnDropoutBackward (dropout_kernel.cu:149-150) applied to the Linear's dX in
 * the same kernel.  Bit-identical to roc_linear_bwd followed by roc_dropout_bwd. */
int roc_linear_bwd_dropout(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX,
                           const float* W, const float* Y, int64_t ldY, float* dY,
                           int64_t ldDY, float* dW, float* dX, int64_t ldDX, int activation,
                           int accumulate_dX, void* workspace, size_t workspaceBytes,
                           const uint32_t* mask, int64_t ldMask, float rate,
                           roc_stream_t stream);

/* roc_linear_bwd with the backward of the ops upstream of X folded into the dX epilogue,
 * so dX is written once, already as the gradient the next ScatterGather backward reads.
 * In model order (gnn.cc:81-88)  ... -> indegree_norm -> relu -> dropout -> linear:
 *   dX = dY W                                           (linear_kernel.cu:227-231)
 *   dX = keep ? dX / (1 - dropRate) : 0   if dropMask    (dropout_kernel.cu:149-150)
 *   dX = dxReluOf > 0 ? dX : 0            if dxReluOf    (Activation backward, cudnnActivationBackward
 *                                                         on the stored relu output, activation_kernel.cu)
 *   dX = dX / sqrtf(deg(row))             if dxNormRowEnd (InDegreeNorm backward, graphnorm_kernel.cu:133)
 * Zero / NULL fields switch the stage off; with all off this is roc_linear_bwd.  Each stage is
 * bit-identical to the separate kernel it replaces. */
typedef struct roc_linear_bwd_args {
  int64_t rows; int inDim, outDim;
  const float* X; int64_t ldX;
  const float* W;
  const float* Y; int64_t ldY;
  float* dY; int64_t ldDY;
  float* dW;
  float* dX; int64_t ldDX;
  int activation, accumulate_dX;
  void* workspace; size_t workspaceBytes;
  const uint32_t* dropMask; int64_t ldMask; float dropRate;
  const float* dxReluOf; int64_t ldReluOf;
  const roc_eid_t* dxNormRowEnd; roc_eid_t colLeft;
  int parts;   /* 0 = dW and dX (if non-NULL); ROC_LINEAR_BWD_ONLY_DX / _ONLY_DW compute one of them — the host
                * computes dX in row blocks (each pushed to the partitions that read it while the next is computed)
                * and dW, which nothing waits for, last.  Only with activation == NONE (no in-place relu backward). */
} roc_linear_bwd_args;
#define ROC_LINEAR_BWD_ONLY_DX 1
#define ROC_LINEAR_BWD_ONLY_DW 2
int roc_linear_bwd_fused(const roc_linear_bwd_args* args, roc_stream_t stream);

/* Test hook: which kernel family served the calling thread's last Linear GEMM — which = 0 forward, 1 dW, 2 dX;
 * returns ROC_GEMM_PATH_TCGEN05, ROC_GEMM_PATH_SIMT (the exact-fp32 fallback for shapes / alignments the tensor-core
 * kernels do not take) or 0 (none yet). */
#define ROC_GEMM_PATH_TCGEN05 1
#define ROC_GEMM_PATH_SIMT 2
int roc_last_gemm_path(int which);

/* Test hook: how the calling thread's last Linear GEMM of kind `which` (as above) ran, so that a test can assert that
 * a shape reached the kernel instantiation and pipeline regime it was chosen for.  On the SIMT path only `path` is
 * set, and for dW also `splits` / `v_per_split` (the rest is 0).  Tensor cores:
 *   nc        wgmma chunks of 32 columns per N tile (1, 2, 4; dW 1, 2, 4, 8)
 *   epi       forward / dX epilogue instantiation: its EPI bit mask, or -1 for the generic kernel;  dW: the kernel,
 *             1 the warp-specialised one (outDim <= 128), 0 the CTA-synchronised one (outDim > 128, ROC_B200_DW=sync)
 *   grid_x/y  forward / dX: persistent CTAs along the rows x N tiles;  dW: splits x 128-column M tiles
 *   stages    depth of the TMA ring (dW: 32-vertex slots)
 *   splits, v_per_split   dW only: split-K ranges and the rows each holds (the partials are added in range order)
 *   w_resident  forward / dX: 1 when the CTA's W_hi / W_lo slice is loaded into shared memory once (the ring carries
 *             only the streaming operand), 0 when W streams through the ring with it
 *   epi_bufs  forward / dX: shared-memory buffers of the epilogue operands (relu-mask source, output-mask words) the
 *             producer loads ahead of each tile: 0 when the epilogue has none, else 1 or 2
 * Returns ROC_ERR_INVALID for a bad `which` or a NULL `info`. */
typedef struct {
  int path, nc, epi, grid_x, grid_y, stages, splits;
  int64_t v_per_split;
  int w_resident, epi_bufs;
} roc_gemm_info;
int roc_last_gemm_info(int which, roc_gemm_info* info);

/* ------------------------------------------------------------ optimizer --- */

/* Replaces adam_update, optimizer_kernel.cu:43-63 (launch :98-101).  alpha_t is
 * the bias-corrected step computed on the host in double (optimizer.cc:79-85).
 * The reference first sums per-GPU replicas g0 += g_i (:88-94); here WGrad is
 * already the all-reduced gradient. */
int roc_adam_update(int64_t count, float alpha_t, float beta1, float beta2,
                    float weight_decay, float epsilon, const float* WGrad, float* M,
                    float* V, float* W, roc_stream_t stream);

/* Replaces GlorotUniform::init_task's scale_kernel, initializer_kernel.cu:46-47 +
 * cuda_helper.cu:2-9: W = (b - a) * u + a over `count` uniforms already in W. */
int roc_scale(int64_t count, float a, float b, float* W, roc_stream_t stream);
/* Replaces assign_kernel, cuda_helper.cu:11-18 (zero_grad_task_impl,
 * ZerosInitializer): 2-D fill of the [rows][H] window of a [rows][ld] tensor. */
int roc_fill(int64_t rows, int H, float value, float* x, int64_t ld, roc_stream_t stream);
/* Test hook: the fused indegree_norm epilogues divide by a row-uniform sqrtf(deg) with a shared
 * reciprocal + FMA correction instead of one div.rn per element.  Counts, over the `count` fp32 bit
 * patterns starting at firstBits, how many results differ from `x / d` (must be 0; NaN == NaN).
 * *d_mismatches (device u64) is accumulated into. */
int roc_selftest_rowdiv(float d, uint64_t firstBits, uint64_t count, uint64_t* d_mismatches,
                        roc_stream_t stream);
/* Replaces copy_kernel, cuda_helper.cu:20-27 (dropout's infer path, staging): 2-D copy of
 * the [rows][H] window between tensors of different leading dimensions. */
int roc_copy2d(int64_t rows, int H, const float* src, int64_t ldSrc, float* dst, int64_t ldDst,
               roc_stream_t stream);
/* fp32 -> bf16 (raw bits) of the [rows][H] window, round to nearest even, as torch's
 * Tensor.to(torch.bfloat16): a finite value past the largest bf16 rounds to +-inf, and a NaN
 * becomes the quiet NaN 0x7FC0 (sign and payload are not kept).  Writes whole destination rows: columns [H, ldDst) get zero.  Uploads
 * convert staged fp32 chunks with it, so no full-size fp32 copy is ever on the device. */
int roc_f32_to_bf16(int64_t rows, int H, const float* src, int64_t ldSrc, uint16_t* dst,
                    int64_t ldDst, roc_stream_t stream);
/* bf16 -> fp32 of the [rows][H] window: exact. */
int roc_bf16_to_f32(int64_t rows, int H, const uint16_t* src, int64_t ldSrc, float* dst,
                    int64_t ldDst, roc_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* ROC_B200_H_ */
