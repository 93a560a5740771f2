/*
 * roc_host.h — C ABI over the C++ host (roc_gnn.h) so non-C++ callers (the
 * Python mirror in roc_b200/, bench.py, tests) can build and train a model.
 * One roc_host per process / GPU.  Mirrors the public surface of Model
 * (gnn.h:162-203): same op-builder calls, same train-loop calls.  Tensors are
 * referred to by small integer handles.  Unless stated, return 0 on success;
 * host-side precondition failures abort the process like the reference's
 * asserts do (cuda_helper.h:6-12).
 */
#ifndef ROC_HOST_H_
#define ROC_HOST_H_
#include <stdint.h>
#include "roc_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct roc_host roc_host;

/* device: CUDA ordinal; myPart/numParts: this process's vertex-range partition. */
roc_host* roc_host_create(int device, int myPart, int numParts);
void roc_host_destroy(roc_host* h);
int roc_host_nccl_unique_id(unsigned char id[128]);
int roc_host_nccl_init(roc_host* h, const unsigned char id[128]);
int roc_host_synchronize(roc_host* h);
/* the host's CUDA stream (a cudaStream_t), so callers can record events on it */
void* roc_host_stream(roc_host* h);

/* Graph (gnn.cc:751-872): from <prefix>.add_self_edge.lux, or from host arrays. */
int roc_host_graph_from_lux(roc_host* h, const char* prefix);
int roc_host_graph_from_arrays(roc_host* h, uint32_t numNodes, uint64_t numEdges,
                               const uint64_t* host_rowEnd, const uint32_t* host_colSrc);
/* out[0..5] = numNodes, numEdges(lo), rowLeft, rowRight, colLeft, colRight as u64 */
int roc_host_graph_info(roc_host* h, uint64_t out[6]);
const roc_sg_plan* roc_host_graph_plan(roc_host* h);

/* Model builder — returns a tensor handle (>= 0). */
int roc_host_create_node_tensor(roc_host* h, int hidden, int is_int);
/* a leaf feature tensor stored in bf16 (Model::create_node_tensor<__nv_bfloat16>): only linear and dropout may read
 * it; set_tensor / get_tensor move fp32 rows (rounded / widened), the _bf16 calls below its raw bits */
int roc_host_create_node_tensor_bf16(roc_host* h, int hidden);
int roc_host_dropout(roc_host* h, int t, float rate, int seed);
int roc_host_linear(roc_host* h, int t, int outDim, int activation);
int roc_host_indegree_norm(roc_host* h, int t);
int roc_host_scatter_gather(roc_host* h, int t);
/* Model::scatter_gather(t, aggr); aggr = AggrType (0 AVG, 1 MAX, 2 MIN, 3 SUM) */
int roc_host_scatter_gather_aggr(roc_host* h, int t, int aggr);
/* Model::scatter_gather(t, AGGR_SUM, rate, seed): the sum with edge dropout at `rate` in train mode */
int roc_host_scatter_gather_dropout(roc_host* h, int t, float rate, int seed);
/* Model::attention_gather(t, scores, heads, slope); scores has 2 * heads columns */
int roc_host_attention_gather(roc_host* h, int t, int scores, int heads, float slope);
/* Model::attention_gather(t, scores, heads, slope, rate, seed): with attention dropout at `rate` in train mode */
int roc_host_attention_gather_dropout(roc_host* h, int t, int scores, int heads, float slope, float rate, int seed);
/* Model::dynamic_attention_gather(xl, xr, heads, slope): GATv2's attention; xl and xr may be one tensor */
int roc_host_dynamic_attention_gather(roc_host* h, int xl, int xr, int heads, float slope);
/* Model::softmax_gather(t, temperature, learnTemperature): softmax aggregation with one temperature */
int roc_host_softmax_gather(roc_host* h, int t, float temperature, int learnTemperature);
/* Model::dot_attention_gather(q, k, v, heads, scale): dot-product attention; q, k and v may be one tensor */
int roc_host_dot_attention_gather(roc_host* h, int q, int k, int v, int heads, float scale);
/* Model::create_edge_tensor<float>(hidden): rows = this partition's edge count */
int roc_host_create_edge_tensor(roc_host* h, int hidden);
/* Model::scatter_gather(t, edges): edge-weighted aggregation */
int roc_host_scatter_gather_weighted(roc_host* h, int t, int edges);
/* Model::set_edge_grad(edges, on) */
int roc_host_set_edge_grad(roc_host* h, int edges, int on);
int roc_host_relu(roc_host* h, int t);
int roc_host_sigmoid(roc_host* h, int t);
/* Model::elu(t) */
int roc_host_elu(roc_host* h, int t);
/* Model::attention_scores(t, heads): appends one parameter (A, 2 * heads rows of F).  One partition only. */
int roc_host_attention_scores(roc_host* h, int t, int heads);
int roc_host_add(roc_host* h, int a, int b);
/* Model::scaled_add(a, b, alpha, beta): fmaf(alpha, a, beta * b) */
int roc_host_scaled_add(roc_host* h, int a, int b, float alpha, float beta);
/* Model::batch_norm(t, momentum, eps): appends two parameters (gamma, beta).  One partition only. */
int roc_host_batch_norm(roc_host* h, int t, float momentum, float eps);
/* the running mean and variance (H floats each) of the batch_norm whose output is t (Model::get / set_batch_norm_stats) */
int roc_host_get_batch_norm_stats(roc_host* h, int t, float* mean, float* var);
int roc_host_set_batch_norm_stats(roc_host* h, int t, const float* mean, const float* var);
/* Model::layer_norm(t, eps): appends two parameters (gamma, beta).  One partition only.  op_info reports it as
 * ROC_HOST_OP_BATCH_NORM. */
int roc_host_layer_norm(roc_host* h, int t, float eps);
int roc_host_softmax_cross_entropy(roc_host* h, int logits, int labels, int mask);
/* Model::sigmoid_cross_entropy: the multi-label loss of roc_sigmoid_xent_bwd; labels set by roc_host_set_multilabels.
 * One partition only. */
int roc_host_sigmoid_cross_entropy(roc_host* h, int logits, int labels, int mask);
/* AdamOptimizer(&model, lr) + set_weight_decay; call after all linear() calls. */
int roc_host_adam(roc_host* h, double lr, double weight_decay);
int roc_host_set_lr(roc_host* h, double lr);
double roc_host_get_lr(roc_host* h);
void roc_host_srand(unsigned seed);               /* std::srand(config.seed), gnn.cc:56 */
int roc_host_set_fusion(roc_host* h, int on);
/* Model::set_exact_backward(on); before roc_host_init */
int roc_host_set_exact_backward(roc_host* h, int on);
/* Model::set_bf16_aggregation(on); before roc_host_init */
int roc_host_set_bf16_aggregation(roc_host* h, int on);
int roc_host_init(roc_host* h);

/* data: dense host buffers of this partition's rows ([rows][hidden]) */
int roc_host_load_features(roc_host* h, int t, const char* prefix);
int roc_host_load_labels(roc_host* h, int t, const char* prefix);
int roc_host_load_train_mask(roc_host* h, int t, const char* prefix);
int roc_host_set_tensor(roc_host* h, int t, const void* host, int grad);
int roc_host_get_tensor(roc_host* h, int t, void* host, int grad);
int roc_host_set_tensor_bf16(roc_host* h, int t, const uint16_t* host);   /* raw bf16 bits, rows x hidden */
int roc_host_get_tensor_bf16(roc_host* h, int t, uint16_t* host);
int roc_host_set_labels(roc_host* h, int t, const int32_t* host_class_idx);
/* multi-labels of a [rows][C] label tensor, bit-packed as roc_sigmoid_xent_bwd takes them: ceil(C / 32) words per
 * row, dense (Model::set_multilabels) */
int roc_host_set_multilabels(roc_host* h, int t, const uint32_t* host_packed_bits);
/* the source ids a max / min scatter_gather output t was taken from, [rows][hidden] u32 (Model::get_aggr_index) */
int roc_host_get_aggr_index(roc_host* h, int t, uint32_t* host);
int roc_host_tensor_shape(roc_host* h, int t, int64_t out[3]);   /* rows, hidden, ld */
void* roc_host_tensor_ptr(roc_host* h, int t, int grad);          /* device pointer (a bf16 tensor: its bits) */
/* how the tensor's data is stored: ROC_HOST_DTYPE_*.  After roc_host_init it shows which tensors
 * set_bf16_aggregation made bf16 (their gradients stay fp32). */
#define ROC_HOST_DTYPE_FLOAT32 0
#define ROC_HOST_DTYPE_BFLOAT16 1
#define ROC_HOST_DTYPE_INT32 2
int roc_host_tensor_dtype(roc_host* h, int t);
int roc_host_num_parameters(roc_host* h);
int roc_host_parameter_shape(roc_host* h, int p, int64_t out[2]); /* inDim, outDim */
int roc_host_get_parameter(roc_host* h, int p, float* host, int which); /* 0 W, 1 dW, 2 m, 3 v */
int roc_host_set_parameter(roc_host* h, int p, const float* host);

/* What Model::init decided for each layer (read-only; call after roc_host_init).  Layers are numbered in creation
 * order (AGGR_AVG appends three).  Every tensor field is a tensor handle, -1 for none, or -2 for a tensor the
 * caller holds no handle for (the inner tensors of AGGR_AVG).  Returns ROC_ERR_INVALID for a bad layer or NULL out. */
#define ROC_HOST_OP_LINEAR 0
#define ROC_HOST_OP_INDEGREE_NORM 1
#define ROC_HOST_OP_SCATTER_GATHER 2          /* the sum */
#define ROC_HOST_OP_SCATTER_GATHER_MAX 3
#define ROC_HOST_OP_SCATTER_GATHER_MIN 4
#define ROC_HOST_OP_SCATTER_GATHER_WEIGHTED 5
#define ROC_HOST_OP_ATTENTION_GATHER 6
#define ROC_HOST_OP_RELU 7
#define ROC_HOST_OP_SIGMOID 8
#define ROC_HOST_OP_ADD 9
#define ROC_HOST_OP_DROPOUT 10
#define ROC_HOST_OP_SOFTMAX_CROSS_ENTROPY 11
#define ROC_HOST_OP_SIGMOID_CROSS_ENTROPY 12
#define ROC_HOST_OP_BATCH_NORM 13            /* the normalisations: batch_norm and layer_norm */
#define ROC_HOST_OP_ELU 14
#define ROC_HOST_OP_ATTENTION_SCORES 15
#define ROC_HOST_OP_SCALED_ADD 16
struct roc_host_op_info {   /* a struct tag only: roc_host_op_info is also the function's name */
  int kind;          /* ROC_HOST_OP_* */
  int fusedInto;     /* >= 0: the layer whose kernel does this op's forward */
  int bwdFused;      /* norm: its backward is done by a Linear's dX epilogue or by the loss */
  int epilogue;      /* sum ScatterGather: ROC_SG_EPI_* of the forward store (with a scaled_add fused into it: NORM and
                        NORM_OUT of roc_sg_forward_teleport_planned) */
  int bwdEpilogue;   /*   ... and of the backward store */
  int fwdOut;        /*   the tensor the forward writes (-1: its own output); also a Linear's and a batch_norm's or a
                        layer_norm's (the output of the relu fused into it) */
  int bwdOut;        /*   the tensor whose gradient the backward writes (-1: its input's) */
  int flags;         /* Linear: ROC_LINEAR_* of the forward */
  int dropOp;        /*   >= 0: the Dropout layer applied while X is loaded */
  int dxOut;         /*   the tensor whose gradient dX goes to (-1: its input's) */
  int dxReluOf;      /*   the tensor whose relu mask the dX epilogue applies (-1: none) */
  int dxNorm;        /*   the dX epilogue divides by sqrt(in-degree) */
  int gradOut;       /* softmax or sigmoid cross-entropy: the tensor whose gradient it writes, divided by
                        sqrt(in-degree) (-1: the logits') */
};
int roc_host_num_ops(roc_host* h);
int roc_host_op_info(roc_host* h, int layer, struct roc_host_op_info* out);

/* train loop (gnn.cc:99-111) */
int roc_host_train_mode(roc_host* h);
int roc_host_infer_mode(roc_host* h);
int roc_host_zero_gradients(roc_host* h);
int roc_host_forward(roc_host* h);
int roc_host_backward(roc_host* h);
int roc_host_update(roc_host* h);
/* one full training epoch: zero_gradients; forward; backward; update */
int roc_host_train_epoch(roc_host* h);
/* PerfMetrics of the last loss pass.  After a sigmoid cross-entropy: trainLoss = (float)loss[0], *All = rows,
 * *Correct = exact (subset accuracy) of its roc_multilabel_metrics. */
int roc_host_metrics(roc_host* h, roc_perf_metrics* out);
/* The roc_multilabel_metrics of the last sigmoid cross-entropy pass; ROC_ERR_INVALID before that loss has run. */
int roc_host_multilabel_metrics(roc_host* h, roc_multilabel_metrics* out);
/* Per-launch device time of the ScatterGather kernels (CUDA events on the host's
 * stream around each roc_sg_forward_planned): enable, run steps, read {H, ms}. */
int roc_host_profile_sg(roc_host* h, int on);
int roc_host_profile_sg_read(roc_host* h, int maxEntries, int* H, float* ms);

#ifdef __cplusplus
}
#endif
#endif
