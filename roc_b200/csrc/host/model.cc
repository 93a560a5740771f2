// model.cc — Model, the op classes, AdamOptimizer, initializers, dataset loaders.
// Mirrors gnn.cc:433-749 and the per-op .cc files of the reference; each op's
// forward/backward enqueues C-ABI kernels (roc_b200.h) on the Runtime's stream
// instead of launching a Legion index task.
#include <cuda_bf16.h>
#include <curand.h>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <fstream>
#include <set>
#include <sstream>

#include "host_internal.h"

using namespace roc::host;

// roc_softmax_xent_bwd_idx is declared in roc_b200.h

// ------------------------------------------------------------------ GnnOp ---
// gnn.cc:433-465
GnnOp::GnnOp(const Tensor& _input) : numInputs(1), numOutputs(0), fusedInto(-1) {
  inputs[0] = _input;
  trainableInputs[0] = true;
  resetInputGrads[0] = true;
}
GnnOp::GnnOp(const Tensor& _input1, const Tensor& _input2) : numInputs(2), numOutputs(0), fusedInto(-1) {
  inputs[0] = _input1; inputs[1] = _input2;
  for (int i = 0; i < 2; i++) { trainableInputs[i] = true; resetInputGrads[i] = true; }
}
GnnOp::GnnOp(const Tensor& _input1, const Tensor& _input2, const Tensor& _input3)
    : numInputs(3), numOutputs(0), fusedInto(-1) {
  inputs[0] = _input1; inputs[1] = _input2; inputs[2] = _input3;
  for (int i = 0; i < 3; i++) { trainableInputs[i] = true; resetInputGrads[i] = true; }
}

// ------------------------------------------------------------------ Model ---
Model::Model(const Graph& _graph, Context _ctx, Runtime* _runtime)
    : mode(MD_MODE_TRAIN), myGraph(_graph), ctx(_ctx), runtime(_runtime), optimizer(NULL), epoch_num(0),
      fuse(true), printMetrics(true), exactBackward(false), bf16Aggregation(false) {}

// gnn.cc:475-532: node tensor = [numNodes][H]; this process holds its vertex range.
template <>
Tensor Model::create_node_tensor<DATATYPE>(int _numHidden) const {
  Tensor t(Tensor::NODE_TENSOR);
  t.numDim = 2;
  t.dims[0] = _numHidden;
  t.dims[1] = myGraph.numNodes;
  t.region = ctx->new_tensor(local_rows(), _numHidden, round_up4(_numHidden), false, false);
  return t;
}
template <>
Tensor Model::create_node_tensor<__nv_bfloat16>(int _numHidden) const {
  Tensor t(Tensor::NODE_TENSOR);
  t.numDim = 2;
  t.dims[0] = _numHidden;
  t.dims[1] = myGraph.numNodes;
  t.region = ctx->new_tensor(local_rows(), _numHidden, round_up8(_numHidden), false, false);
  ctx->t(t.region).isBf16 = true;
  return t;
}
template <>
Tensor Model::create_node_tensor<int>(int _numHidden) const {
  Tensor t(Tensor::NODE_TENSOR);
  t.numDim = 2;
  t.dims[0] = _numHidden;
  t.dims[1] = myGraph.numNodes;
  t.region = ctx->new_tensor(local_rows(), _numHidden, _numHidden, true, false);
  return t;
}

// gnn.cc:534-560: edge tensor = [numEdges][numHidden]; this process holds its partition's edges, in CSR order.
template <>
Tensor Model::create_edge_tensor<DATATYPE>(int numHidden) const {
  if (numHidden != 1) ROC_FATAL("create_edge_tensor: only numHidden == 1 (one weight per edge) is supported");
  Tensor t(Tensor::EDGE_TENSOR);
  t.numDim = 2;
  t.dims[0] = numHidden;
  t.dims[1] = myGraph.numEdges;
  t.region = ctx->new_tensor((int64_t)(myGraph.colRight - myGraph.colLeft + 1), numHidden, numHidden, false, false);
  return t;
}

// gnn.cc:591-623: weight [inDim][outDim] (dim0 = inDim fastest => W_mem[o*inDim + i]).
// The reference keeps one dW replica per GPU inside one region; here each process
// owns its replica and replicas are summed by one NCCL all-reduce (Model::update).
Tensor Model::create_weight_tensor(int _inDim, int _outDim, Initializer* initializer) const {
  Tensor w(Tensor::WEIGHT_TENSOR);
  w.numDim = 2;
  w.dims[0] = _inDim;
  w.dims[1] = _outDim;
  w.region = ctx->new_tensor(_outDim, _inDim, _inDim, false, true);
  ctx->t(w.region).requiresGrad = true;
  if (initializer == NULL) {
    GlorotUniform glorot;   // default initializer, gnn.cc:614-618
    glorot.init(this, &w);
  } else {
    initializer->init(this, &w);
  }
  return w;
}

Tensor Model::add(const Tensor& a, const Tensor& b) {
  GnnOp* op = new Element(*this, a, b, EW_TYPE_ADD);
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::scaled_add(const Tensor& a, const Tensor& b, float alpha, float beta) {
  if (!std::isfinite(alpha) || !std::isfinite(beta)) ROC_FATAL("scaled_add: alpha and beta must be finite");
  if (a.region == b.region) ROC_FATAL("scaled_add: a and b must be different tensors");
  if (a.numDim != b.numDim) ROC_FATAL("scaled_add: a and b must have the same shape");
  for (int i = 0; i < a.numDim; i++)
    if (a.dims[i] != b.dims[i]) ROC_FATAL("scaled_add: a and b must have the same shape");
  GnnOp* op = new ScaledAdd(*this, a, b, alpha, beta);
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::dropout(const Tensor& _input, float rate, int seed) {
  Dropout* op = new Dropout(*this, _input, rate, seed);
  op->opIndex = (int)layers.size();
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::scatter_gather(const Tensor& _input) {
  GnnOp* op = new ScatterGather(*this, _input);
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::scatter_gather(const Tensor& _input, AggrType aggr) {
  switch (aggr) {
    case AGGR_SUM: return scatter_gather(_input);
    case AGGR_AVG: return indegree_norm(indegree_norm(scatter_gather(_input)));   // the fusions of init() apply
    case AGGR_MAX:
    case AGGR_MIN: {
      if (ctx->numParts > 1)
        ROC_FATAL("scatter_gather: max / min aggregation runs on one partition only (numParts > 1 is not supported)");
      GnnOp* op = new ScatterGather(*this, _input, aggr);
      layers.push_back(op);
      return op->outputs[0];
    }
  }
  ROC_FATAL("scatter_gather: unknown AggrType");
  return Tensor();
}
Tensor Model::scatter_gather(const Tensor& _input, AggrType aggr, float dropout, int seed) {
  if (!(dropout >= 0.0f && dropout < 1.0f)) ROC_FATAL("scatter_gather: the edge dropout rate must be in [0, 1)");
  if (dropout == 0.0f) return scatter_gather(_input, aggr);
  if (aggr != AGGR_SUM) ROC_FATAL("scatter_gather: edge dropout goes with the sum aggregation only");
  if (ctx->numParts > 1)
    ROC_FATAL("scatter_gather: edge dropout runs on one partition only (numParts > 1 is not supported)");
  ScatterGather* op = new ScatterGather(*this, _input);
  op->dropRate = dropout;
  op->seed = seed;
  op->opIndex = (int)layers.size();
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::attention_gather(const Tensor& input, const Tensor& scores, int heads, float negativeSlope, float dropout,
                               int seed) {
  if (ctx->numParts > 1)
    ROC_FATAL("attention_gather: runs on one partition only (numParts > 1 is not supported)");
  AttentionGather* op = new AttentionGather(*this, input, scores, heads, negativeSlope, dropout, seed);
  op->opIndex = (int)layers.size();
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::dynamic_attention_gather(const Tensor& xl, const Tensor& xr, int heads, float negativeSlope) {
  if (ctx->numParts > 1)
    ROC_FATAL("dynamic_attention_gather: runs on one partition only (numParts > 1 is not supported)");
  AttentionGather* op = new AttentionGather(*this, xl, xr, heads, negativeSlope);
  op->opIndex = (int)layers.size();
  layers.push_back(op);
  parameters.push_back(op->a);
  return op->outputs[0];
}
Tensor Model::softmax_gather(const Tensor& x, float temperature, bool learnTemperature) {
  if (ctx->numParts > 1)
    ROC_FATAL("softmax_gather: runs on one partition only (numParts > 1 is not supported)");
  AttentionGather* op = new AttentionGather(*this, x, temperature, learnTemperature);
  op->opIndex = (int)layers.size();
  layers.push_back(op);
  if (learnTemperature) parameters.push_back(op->temperature);
  return op->outputs[0];
}
Tensor Model::dot_attention_gather(const Tensor& q, const Tensor& k, const Tensor& v, int heads, float scale) {
  if (ctx->numParts > 1)
    ROC_FATAL("dot_attention_gather: runs on one partition only (numParts > 1 is not supported)");
  AttentionGather* op = new AttentionGather(*this, q, k, v, heads, scale);
  op->opIndex = (int)layers.size();
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::attention_scores(const Tensor& input, int heads) {
  if (ctx->numParts > 1)
    ROC_FATAL("attention_scores: runs on one partition only (numParts > 1 is not supported)");
  AttentionScores* op = new AttentionScores(*this, input, heads);
  layers.push_back(op);
  parameters.push_back(op->a);
  return op->outputs[0];
}
Tensor Model::scatter_gather(const Tensor& input, const Tensor& edgeWeights) {
  if (ctx->numParts > 1)
    ROC_FATAL("scatter_gather: edge-weighted aggregation runs on one partition only (numParts > 1 is not supported)");
  GnnOp* op = new WeightedScatterGather(*this, input, edgeWeights);
  layers.push_back(op);
  return op->outputs[0];
}
void Model::set_edge_grad(const Tensor& edges, bool on) {
  if (edges.type != Tensor::EDGE_TENSOR) ROC_FATAL("set_edge_grad: not an edge tensor");
  ctx->t(edges.region).requiresGrad = on;
}
void Model::set_exact_backward(bool on) {
  if (on && ctx->numParts > 1)
    ROC_FATAL("set_exact_backward: the exact backward runs on one partition only (numParts > 1 is not supported)");
  if (ctx->flatGrad) ROC_FATAL("set_exact_backward: call it before init()");
  exactBackward = on;
}
void Model::set_bf16_aggregation(bool on) {
  if (ctx->flatGrad) ROC_FATAL("set_bf16_aggregation: call it before init()");
  bf16Aggregation = on;
}
void Model::get_aggr_index(const Tensor& out, uint32_t* host) const {
  for (GnnOp* op : layers) {
    ScatterGather* sg = dynamic_cast<ScatterGather*>(op);
    if (!sg || sg->outputs[0].region != out.region) continue;
    if (sg->aggr != AGGR_MAX && sg->aggr != AGGR_MIN) ROC_FATAL("get_aggr_index: not a max / min scatter_gather");
    if (!sg->arg) ROC_FATAL("get_aggr_index: run forward() first");
    const int64_t H = (int64_t)sg->outputs[0].dims[0];
    ROC_CHECK(cudaMemcpy2DAsync(host, (size_t)H * sizeof(uint32_t), sg->arg, (size_t)sg->argLd * sizeof(uint32_t),
                                (size_t)H * sizeof(uint32_t), (size_t)local_rows(), cudaMemcpyDeviceToHost, ctx->stream));
    ROC_CHECK(cudaStreamSynchronize(ctx->stream));
    return;
  }
  ROC_FATAL("get_aggr_index: no scatter_gather produces this tensor");
}
static BatchNorm* batch_norm_of(const std::vector<GnnOp*>& layers, const Tensor& out, const char* what) {
  for (GnnOp* op : layers) {
    BatchNorm* bn = dynamic_cast<BatchNorm*>(op);
    if (bn && bn->outputs[0].region == out.region) return bn;
  }
  ROC_FATAL((std::string(what) + ": no batch_norm produces this tensor").c_str());
}
void Model::get_batch_norm_stats(const Tensor& out, float* mean, float* var) const {
  const BatchNorm* bn = batch_norm_of(layers, out, "get_batch_norm_stats");
  const size_t bytes = (size_t)bn->outputs[0].dims[0] * sizeof(float);
  ROC_CHECK(cudaMemcpyAsync(mean, bn->runMean, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  ROC_CHECK(cudaMemcpyAsync(var, bn->runVar, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  ROC_CHECK(cudaStreamSynchronize(ctx->stream));
}
void Model::set_batch_norm_stats(const Tensor& out, const float* mean, const float* var) {
  BatchNorm* bn = batch_norm_of(layers, out, "set_batch_norm_stats");
  const size_t bytes = (size_t)bn->outputs[0].dims[0] * sizeof(float);
  ROC_CHECK(cudaMemcpyAsync(bn->runMean, mean, bytes, cudaMemcpyHostToDevice, ctx->stream));
  ROC_CHECK(cudaMemcpyAsync(bn->runVar, var, bytes, cudaMemcpyHostToDevice, ctx->stream));
  ROC_CHECK(cudaStreamSynchronize(ctx->stream));
}
void Model::softmax_cross_entropy(const Tensor& logits, const Tensor& labels, const Tensor& mask) {
  layers.push_back(new SoftmaxCrossEntropy(*this, logits, labels, mask));
}
void Model::sigmoid_cross_entropy(const Tensor& logits, const Tensor& labels, const Tensor& mask) {
  if (ctx->numParts > 1)
    ROC_FATAL("sigmoid_cross_entropy: runs on one partition only (numParts > 1 is not supported)");
  layers.push_back(new SigmoidCrossEntropy(*this, logits, labels, mask));
}
Tensor Model::indegree_norm(const Tensor& _input) {
  GnnOp* op = new InDegreeNorm(*this, _input);
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::linear(const Tensor& _input, int outDim, ActiMode activation, Initializer* initializer) {
  if (activation == AC_MODE_ELU) ROC_FATAL("linear: a Linear cannot apply AC_MODE_ELU; call elu() on its output");
  Linear* op = new Linear(*this, _input, outDim, activation, initializer);
  layers.push_back(op);
  parameters.push_back(op->weight);   // linear.cc:30
  return op->outputs[0];
}
Tensor Model::relu(const Tensor& _input) {
  GnnOp* op = new Activation(*this, _input, AC_MODE_RELU);
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::sigmoid(const Tensor& _input) {
  GnnOp* op = new Activation(*this, _input, AC_MODE_SIGMOID);
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::elu(const Tensor& _input) {
  GnnOp* op = new Activation(*this, _input, AC_MODE_ELU);
  layers.push_back(op);
  return op->outputs[0];
}
Tensor Model::batch_norm(const Tensor& input, float momentum, float eps) {
  if (ctx->numParts > 1)
    ROC_FATAL("batch_norm: runs on one partition only (numParts > 1 is not supported)");
  BatchNorm* op = new BatchNorm(*this, input, momentum, eps);
  layers.push_back(op);
  parameters.push_back(op->gamma);
  parameters.push_back(op->beta);
  return op->outputs[0];
}
Tensor Model::layer_norm(const Tensor& input, float eps) {
  if (ctx->numParts > 1)
    ROC_FATAL("layer_norm: runs on one partition only (numParts > 1 is not supported)");
  LayerNorm* op = new LayerNorm(*this, input, eps);
  layers.push_back(op);
  parameters.push_back(op->gamma);
  parameters.push_back(op->beta);
  return op->outputs[0];
}

void Model::train_mode(void) { mode = MD_MODE_TRAIN; }
void Model::infer_mode(void) { mode = MD_MODE_INFER; }

const char* const roc::host::opKindNames[ROC_HOST_OP_SCALED_ADD + 1] = {
    "linear", "indegree_norm", "scatter_gather", "scatter_gather(max)", "scatter_gather(min)",
    "scatter_gather(weighted)", "attention_gather", "relu", "sigmoid", "add", "dropout", "softmax_cross_entropy",
    "sigmoid_cross_entropy", "batch_norm", "elu", "attention_scores", "scaled_add"};
int roc::host::op_kind(const GnnOp* op) {
  if (const ScatterGather* sg = dynamic_cast<const ScatterGather*>(op))
    return sg->aggr == AGGR_MAX   ? ROC_HOST_OP_SCATTER_GATHER_MAX
           : sg->aggr == AGGR_MIN ? ROC_HOST_OP_SCATTER_GATHER_MIN
                                  : ROC_HOST_OP_SCATTER_GATHER;
  if (const Activation* a = dynamic_cast<const Activation*>(op))
    return a->actiMode == AC_MODE_RELU ? ROC_HOST_OP_RELU
           : a->actiMode == AC_MODE_ELU ? ROC_HOST_OP_ELU
                                        : ROC_HOST_OP_SIGMOID;
  return dynamic_cast<const Linear*>(op)                  ? ROC_HOST_OP_LINEAR
         : dynamic_cast<const InDegreeNorm*>(op)          ? ROC_HOST_OP_INDEGREE_NORM
         : dynamic_cast<const WeightedScatterGather*>(op) ? ROC_HOST_OP_SCATTER_GATHER_WEIGHTED
         : dynamic_cast<const AttentionGather*>(op)       ? ROC_HOST_OP_ATTENTION_GATHER
         : dynamic_cast<const Dropout*>(op)               ? ROC_HOST_OP_DROPOUT
         : dynamic_cast<const SoftmaxCrossEntropy*>(op)   ? ROC_HOST_OP_SOFTMAX_CROSS_ENTROPY
         : dynamic_cast<const SigmoidCrossEntropy*>(op)   ? ROC_HOST_OP_SIGMOID_CROSS_ENTROPY
         : dynamic_cast<const BatchNorm*>(op)             ? ROC_HOST_OP_BATCH_NORM
         : dynamic_cast<const LayerNorm*>(op)             ? ROC_HOST_OP_BATCH_NORM   // the normalisation kind
         : dynamic_cast<const AttentionScores*>(op)       ? ROC_HOST_OP_ATTENTION_SCORES
         : dynamic_cast<const ScaledAdd*>(op)             ? ROC_HOST_OP_SCALED_ADD
                                                          : ROC_HOST_OP_ADD;
}

namespace {
struct Wiring {
  std::map<int, int> producer;    // region -> layer index
  std::map<int, int> consumers;   // region -> number of consuming op inputs
  std::map<int, int> consumerOp;  // region -> a consuming layer index
};
Wiring wire(const std::vector<GnnOp*>& layers) {
  Wiring w;
  for (size_t l = 0; l < layers.size(); l++) {
    for (int j = 0; j < layers[l]->numOutputs; j++) w.producer[layers[l]->outputs[j].region] = (int)l;
    for (int j = 0; j < layers[l]->numInputs; j++) {
      int r = layers[l]->inputs[j].region;
      if (r < 0) continue;
      w.consumers[r] += 1;
      w.consumerOp[r] = (int)l;
    }
  }
  return w;
}
template <typename T>
T* as(GnnOp* op) { return dynamic_cast<T*>(op); }
// a ScatterGather that sums: the only kind the epilogue fusions apply to (a max / min op keeps its own output)
ScatterGather* as_sum_sg(GnnOp* op) {
  ScatterGather* sg = dynamic_cast<ScatterGather*>(op);
  return (sg && sg->aggr == AGGR_SUM) ? sg : nullptr;
}
}  // namespace

// ---- the passes of Model::init, in the order it runs them

// a bf16 tensor is read by linear (its X) and dropout only; any other op would need an fp32 view of it
static void check_bf16_readers(const Model& m) {
  RuntimeImpl* rt = m.ctx;
  if (m.bf16Aggregation && rt->numParts > 1)
    ROC_FATAL("set_bf16_aggregation: bf16 aggregation inputs run on one partition only (numParts > 1 is not supported)");
  for (GnnOp* op : m.layers) {
    const bool takesBf16 = as<Linear>(op) || as<Dropout>(op);
    for (int j = 0; j < op->numInputs; j++) {
      const int r = op->inputs[j].region;
      if (r < 0 || !rt->t(r).isBf16 || (takesBf16 && j == 0)) continue;
      ROC_FATAL((std::string(opKindNames[op_kind(op)]) +
                 " cannot read a bf16 tensor: only linear and dropout take bf16 input").c_str());
    }
  }
}

// which tensors carry gradients: anything downstream of a parameter
static void mark_gradients(const Model& m) {
  RuntimeImpl* rt = m.ctx;
  for (GnnOp* op : m.layers) {
    bool any = false;
    for (int j = 0; j < op->numInputs; j++)
      if (op->inputs[j].region >= 0) any = any || rt->t(op->inputs[j].region).requiresGrad;
    const AttentionGather* ag = as<AttentionGather>(op);
    if (as<Linear>(op) || as<BatchNorm>(op) || as<LayerNorm>(op) || as<AttentionScores>(op) ||
        (ag && (ag->dynamic || ag->learnTemperature)))
      any = true;   // their own parameters
    for (int j = 0; j < op->numOutputs; j++) {
      rt->t(op->outputs[j].region).requiresGrad = any;
      rt->t(op->outputs[j].region).produced = true;
    }
  }
}

// flat dW buffer (one all-reduce per step instead of the reference's serial
// replica sum, optimizer_kernel.cu:88-94)
static void lay_out_flat_dw(RuntimeImpl* rt, const std::vector<Tensor>& parameters) {
  size_t total = 0;
  for (size_t p = 0; p < parameters.size(); p++) total += (size_t)parameters[p].dims[0] * parameters[p].dims[1];
  rt->flatGradCount = total;
  rt->flatGrad = (float*)rt->dmalloc((total ? total : 4) * sizeof(float));
  ROC_CHECK(cudaMemsetAsync(rt->flatGrad, 0, (total ? total : 4) * sizeof(float), rt->stream));
  size_t off = 0;
  for (size_t p = 0; p < parameters.size(); p++) {
    rt->t(parameters[p].region).grad = rt->flatGrad + off;
    off += (size_t)parameters[p].dims[0] * parameters[p].dims[1];
  }
}

// scratch: Linear split-K workspace, SG carry slots, the gathered feature matrix.  Returns the widest ScatterGather
// input, the width the graph's plan reserves its carries for (set_up_halo).
static int size_scratch_and_plans(Model& m) {
  RuntimeImpl* rt = m.ctx;
  Graph& g = m.myGraph;
  g.maxHidden = 0;
  size_t ws = 0;
  int maxSg = 0;
  bool minmax = false;
  for (GnnOp* op : m.layers) {
    for (int j = 0; j < op->numOutputs; j++) g.maxHidden = std::max(g.maxHidden, (int)op->outputs[j].dims[0]);
    for (int j = 0; j < op->numInputs; j++)
      if (op->inputs[j].numDim == 2) g.maxHidden = std::max(g.maxHidden, (int)op->inputs[j].dims[0]);
    if (Linear* lin = as<Linear>(op))
      ws = std::max(ws, roc_linear_bwd_workspace_bytes(m.local_rows(), (int)lin->weight.dims[0], (int)lin->weight.dims[1]));
    if (ScatterGather* sg = as<ScatterGather>(op)) {
      maxSg = std::max(maxSg, (int)sg->inputs[0].dims[0]);
      minmax = minmax || sg->aggr == AGGR_MAX || sg->aggr == AGGR_MIN;
    }
  }
  rt->ensure_lin_ws(ws);
  // max / min aggregation sends each gradient to one source per (row, feature): a duplicate edge would receive it
  // twice.  Strictly increasing sources per row rule duplicates out.  The exact backward takes each distinct edge once
  // and needs no such rule.
  if (minmax && !m.exactBackward) {
    int sorted = 0;
    ROC_CHECK(roc_sg_plan_rows_sorted(g.plan, &sorted, rt->stream));
    if (!sorted) ROC_FATAL("scatter_gather(max / min): every row's sources must be strictly increasing (no duplicate edges)");
  }
  return maxSg;
}

// the graph's transpose, built once and shared by the exact backward and the weighted ops, its plan's carries reserved
// for the widest aggregation the exact backward serves, as the forward plan's are
static void build_transpose(const Model& m) {
  RuntimeImpl* rt = m.ctx;
  const Graph& g = m.myGraph;
  int maxT = 0;
  bool weighted = false;
  for (GnnOp* op : m.layers) {
    if (m.exactBackward && (as<ScatterGather>(op) || as<AttentionGather>(op)))
      maxT = std::max(maxT, (int)op->inputs[0].dims[0]);
    weighted = weighted || as<WeightedScatterGather>(op);
  }
  if (maxT == 0 && !weighted) return;
  if (!rt->sgTranspose)
    ROC_CHECK(roc_sg_transpose_create(g.numNodes, g.d_rowEnd, g.d_colSrc, rt->stream, &rt->sgTranspose));
  if (maxT > 0) {
    const roc_sg_plan* planT = nullptr;
    ROC_CHECK(roc_sg_transpose_info(rt->sgTranspose, nullptr, nullptr, nullptr, &planT));
    ROC_CHECK(roc_sg_plan_reserve(const_cast<roc_sg_plan*>(planT), maxT));
  }
}

// the plan's carries for the widest ScatterGather; with more than one partition, the gathered matrix, or the halo
// slabs behind the tensors a ScatterGather reads and the way they are exchanged
static void set_up_halo(RuntimeImpl* rt, const Graph& myGraph, const std::vector<GnnOp*>& layers, int maxSg) {
  if (maxSg > 0) {
    ROC_CHECK(roc_sg_plan_reserve(myGraph.plan, maxSg));
    if (rt->numParts > 1 && !myGraph.halo) rt->ensure_gather((size_t)myGraph.numNodes * (size_t)round_up4(maxSg));
    if (myGraph.halo) {
      // the tensors a ScatterGather reads get the halo slab appended to their own rows
      rt->ensure_sendbuf((myGraph.numSendRows ? myGraph.numSendRows : 1) * (size_t)round_up4(maxSg));
      for (size_t l = 0; l < layers.size(); l++) {
        if (!as<ScatterGather>(layers[l])) continue;
        TensorImpl& xin = rt->t(layers[l]->inputs[0].region);
        TensorImpl& xout = rt->t(layers[l]->outputs[0].region);
        // Usually neither buffer exists yet (lazy allocation).  A tensor the script already filled — e.g. an
        // SGC-style scatter_gather(input) after load_features / set_tensor, which the reference's script order
        // (gnn.cc:72-74) allows — is re-homed with the halo rows behind its own.
        rt->grow_halo(xin, /*grad=*/false, myGraph.numHalo);
        rt->grow_halo(xout, /*grad=*/true, myGraph.numHalo);
      }
      // Exchange by peer writes (roc_push_rows): the slabs exist now and every partition maps the others' copies.
      // ROC_B200_HALO=nccl keeps the staged-rows + NCCL all-to-all-v exchange (cross-check; also the fallback when
      // CUDA IPC is not available between the devices).
      const char* he = getenv("ROC_B200_HALO");
      rt->p2p = !(he && he[0] == 'n') && rt->numParts <= ROC_MAX_PEERS;
      // Two ways to fill the peers' slabs: pack + one DMA copy per peer at 2 GPUs (the copy engines do not keep
      // many peer copies busy), the SM kernel roc_push_rows beyond.  ROC_B200_HALO=push | ce forces one.
      rt->p2pCopyEngines = (he && he[0] == 'c') ? true : (he && he[0] == 'p') ? false : rt->numParts == 2;
      for (size_t l = 0; l < layers.size() && rt->p2p; l++) {
        if (!as<ScatterGather>(layers[l])) continue;
        const int rin = layers[l]->inputs[0].region, rout = layers[l]->outputs[0].region;
        rt->data(rin);
        if (!rt->open_peers(rt->t(rin), false)) { rt->p2p = false; break; }
        if (rt->t(rin).requiresGrad) {
          rt->grad(rout);
          if (!rt->open_peers(rt->t(rout), true)) { rt->p2p = false; break; }
        }
      }
      if (rt->myPart == 0)
        fprintf(stderr, "[roc_b200] halo exchange: %s\n",
                !rt->p2p ? "staged rows + NCCL all-to-all-v"
                : rt->p2pCopyEngines ? "pack + copy-engine writes into the peers' slabs (CUDA IPC over NVLink), pipelined with the producer"
                                     : "roc_push_rows peer writes (CUDA IPC over NVLink), pipelined with the producer");
    }
  }
}

// ---- fusion of  linear -> indegree_norm -> scatter_gather -> indegree_norm -> relu  (gnn.cc:81-85)
static void fuse_gcn_block(const std::vector<GnnOp*>& layers, Wiring& w) {
  for (size_t l = 0; l < layers.size(); l++) {
    ScatterGather* sg = as_sum_sg(layers[l]);
    if (!sg) continue;
    // upstream: Linear(NONE) -> InDegreeNorm -> SG, each feeding only the next
    int rin = sg->inputs[0].region;
    if (w.producer.count(rin) && w.consumers[rin] == 1) {
      InDegreeNorm* n1 = as<InDegreeNorm>(layers[w.producer[rin]]);
      if (n1 && n1->fusedInto < 0) {
        int rl = n1->inputs[0].region;
        if (w.producer.count(rl) && w.consumers[rl] == 1) {
          Linear* lin = as<Linear>(layers[w.producer[rl]]);
          if (lin && lin->activation == AC_MODE_NONE && lin->fwdOut < 0) {
            lin->flags |= ROC_LINEAR_NORM_EPILOGUE;
            lin->fwdOut = n1->outputs[0].region;       // linear writes the normalised rows
            n1->fusedInto = w.producer[rl];
            sg->bwdEpilogue = ROC_SG_EPI_NORM;          // SG backward writes d(linear out)
            sg->bwdOut = lin->outputs[0].region;
          }
        }
      }
    }
    // downstream: SG -> InDegreeNorm -> [relu]
    int rout = sg->outputs[0].region;
    if (w.consumers[rout] == 1) {
      InDegreeNorm* n2 = as<InDegreeNorm>(layers[w.consumerOp[rout]]);
      if (n2 && n2->fusedInto < 0) {
        sg->epilogue = ROC_SG_EPI_NORM;
        sg->fwdOut = n2->outputs[0].region;
        n2->fusedInto = (int)l;   // forward only; its backward kernel still runs
        int rn = n2->outputs[0].region;
        if (w.consumers[rn] == 1) {
          Activation* act = as<Activation>(layers[w.consumerOp[rn]]);
          if (act && act->actiMode == AC_MODE_RELU && act->fusedInto < 0) {
            sg->epilogue |= ROC_SG_EPI_RELU;
            sg->fwdOut = act->outputs[0].region;
            act->fusedInto = (int)l;
            n2->reluOut = act->outputs[0].region;   // backward: relu mask + norm in one pass
          }
        }
      }
    }
  }
}

// which indegree_norm and dropout ops read a tensor a scaled_add also reads: their backward adds to an input gradient
// another op already wrote, where any other wiring is refused (quirk Q7)
static void mark_scaled_add_readers(const std::vector<GnnOp*>& layers) {
  std::set<int> read;
  for (GnnOp* op : layers)
    if (as<ScaledAdd>(op))
      for (int j = 0; j < op->numInputs; j++) read.insert(op->inputs[j].region);
  for (GnnOp* op : layers) {
    if (InDegreeNorm* n = as<InDegreeNorm>(op)) n->sharesWithScaledAdd = read.count(n->inputs[0].region) > 0;
    if (Dropout* d = as<Dropout>(op)) d->sharesWithScaledAdd = read.count(d->inputs[0].region) > 0;
  }
}

// ---- fusion of  sum scatter_gather -> indegree_norm -> scaled_add(., t) [-> indegree_norm]  (APPNP / GCNII's hop):
//      on a scatter_gather whose store fuse_gcn_block fused with its indegree_norm (no relu), that norm's output feeding
//      only a scaled_add as its first input.  The scatter_gather's store applies the teleport
//      (roc_sg_forward_teleport_planned), reading t = the scaled_add's second input, and writes the scaled_add's output;
//      when that output feeds only an unfused indegree_norm (the next hop's), the store also divides by sqrt(deg)
//      (ROC_SG_EPI_NORM_OUT) and writes that norm's output.  Forward only: the scaled_add's and both norms' backward
//      kernels still run.  t must exist when the scatter_gather runs: produced before it, or a leaf.  It runs after
//      choose_bf16_aggregation (which none of its decisions changes): a scatter_gather whose input that pass made bf16
//      has no teleport kernel, and is left unfused.
static void fuse_teleport(const Model& m, Wiring& w) {
  const std::vector<GnnOp*>& layers = m.layers;
  for (size_t l = 0; l < layers.size(); l++) {
    ScatterGather* sg = as_sum_sg(layers[l]);
    if (!sg || sg->epilogue != ROC_SG_EPI_NORM || sg->fwdOut < 0 || sg->teleT >= 0) continue;
    if (m.ctx->t(sg->inputs[0].region).isBf16) continue;
    const int rn = sg->fwdOut;
    if (w.consumers[rn] != 1) continue;
    ScaledAdd* sa = as<ScaledAdd>(layers[w.consumerOp[rn]]);
    if (!sa || sa->fusedInto >= 0 || sa->inputs[0].region != rn) continue;
    const int rt = sa->inputs[1].region;
    if (w.producer.count(rt) && w.producer[rt] >= (int)l) continue;
    sg->teleT = rt;
    sg->teleAlpha = sa->alpha;
    sg->teleBeta = sa->beta;
    sg->fwdOut = sa->outputs[0].region;
    sa->fusedInto = (int)l;
    const int ry = sa->outputs[0].region;
    if (w.consumers[ry] != 1) continue;
    InDegreeNorm* n = as<InDegreeNorm>(layers[w.consumerOp[ry]]);
    if (!n || n->fusedInto >= 0) continue;
    sg->epilogue |= ROC_SG_EPI_NORM_OUT;
    sg->fwdOut = n->outputs[0].region;
    n->fusedInto = (int)l;   // forward only; its backward kernel still runs
  }
}

// ---- fusion of  batch_norm -> relu  and  layer_norm -> relu: the norm's output feeds only the relu.  The norm's
//      forward writes the relu's output, and its backward reads that output's gradient and masks it by the forward's
//      own pre-relu test (batch norm: fma(x, a, b) > 0 from its saved affine map; layer norm: xhat gamma + beta > 0,
//      recomputed from x).  The other peepholes never cross a norm.  In GCN, SG -> indegree_norm still fuses, and the
//      relu after the norm is this pass's.  The backward fusion (b) needs an indegree_norm under the relu, so it does
//      not match here.
static void fuse_batch_norm_relu(const std::vector<GnnOp*>& layers, Wiring& w) {
  for (size_t l = 0; l < layers.size(); l++) {
    int* fwdOut = nullptr;
    if (BatchNorm* bn = as<BatchNorm>(layers[l])) fwdOut = &bn->fwdOut;
    else if (LayerNorm* ln = as<LayerNorm>(layers[l])) fwdOut = &ln->fwdOut;
    if (!fwdOut || *fwdOut >= 0) continue;
    const int ro = layers[l]->outputs[0].region;
    if (w.consumers[ro] != 1) continue;
    Activation* act = as<Activation>(layers[w.consumerOp[ro]]);
    if (!act || act->actiMode != AC_MODE_RELU || act->fusedInto >= 0) continue;
    *fwdOut = act->outputs[0].region;
    act->fusedInto = (int)l;
  }
}

// ---- fusion of  dropout -> linear  (gnn.cc:79-81, 86-88): the dropout output feeds only the linear.  Not when a
//      scaled_add also reads the dropout's input: the Linear's dX epilogue overwrites that gradient, where the dropout
//      alone adds its part to what the scaled_add wrote.
static void fuse_dropout_into_linear(const std::vector<GnnOp*>& layers, Wiring& w) {
  for (size_t l = 0; l < layers.size(); l++) {
    Dropout* d = as<Dropout>(layers[l]);
    if (!d || d->fusedInto >= 0 || d->sharesWithScaledAdd) continue;
    const int ro = d->outputs[0].region;
    if (w.consumers[ro] != 1) continue;
    Linear* lin = as<Linear>(layers[w.consumerOp[ro]]);
    if (!lin || lin->dropOp >= 0 || lin->inputs[0].region != ro) continue;
    lin->dropOp = (int)l;
    d->fusedInto = w.consumerOp[ro];
  }
}

// ---- backward-only fusions into epilogues
static void fuse_backward_epilogues(RuntimeImpl* rt, const std::vector<GnnOp*>& layers, Wiring& w) {
  for (size_t l = 0; l < layers.size(); l++) {
    // (a) ... -> indegree_norm -> softmax_cross_entropy or sigmoid_cross_entropy: the loss kernel divides the
    //     logits' gradient by sqrt(deg) and writes it where the norm's input gradient lives (not when a scaled_add
    //     also reads that input: the norm's own backward adds to it instead)
    int* lossGradOut = nullptr;
    if (SoftmaxCrossEntropy* sce = as<SoftmaxCrossEntropy>(layers[l])) lossGradOut = &sce->gradOut;
    else if (SigmoidCrossEntropy* bce = as<SigmoidCrossEntropy>(layers[l])) lossGradOut = &bce->gradOut;
    if (lossGradOut) {
      const int rz = layers[l]->inputs[0].region;
      if (!w.producer.count(rz) || w.consumers[rz] != 1) continue;
      InDegreeNorm* n = as<InDegreeNorm>(layers[w.producer[rz]]);
      if (!n || n->bwdFused || n->reluOut >= 0 || n->sharesWithScaledAdd) continue;
      if (n->fusedInto >= 0 && as<Linear>(layers[(size_t)n->fusedInto])) continue;   // handled by the SG epilogue
      if (!rt->t(n->inputs[0].region).requiresGrad) continue;
      *lossGradOut = n->inputs[0].region;
      n->bwdFused = true;
      continue;
    }
    // (b) indegree_norm -> relu -> [dropout ->] linear: the linear's dX epilogue applies the dropout
    //     backward, the relu mask and the norm, and writes the norm's input gradient directly
    Linear* lin = as<Linear>(layers[l]);
    if (!lin || lin->dxOut >= 0) continue;
    const int rin = lin->dropOp >= 0 ? layers[(size_t)lin->dropOp]->inputs[0].region : lin->inputs[0].region;
    if (!rt->t(rin).requiresGrad || !w.producer.count(rin) || w.consumers[rin] != 1) continue;
    Activation* act = as<Activation>(layers[w.producer[rin]]);
    if (!act || act->actiMode != AC_MODE_RELU || act->fusedInto < 0) continue;
    const int rn = act->inputs[0].region;
    if (!w.producer.count(rn)) continue;
    InDegreeNorm* n = as<InDegreeNorm>(layers[w.producer[rn]]);
    if (!n || n->bwdFused || n->reluOut != rin) continue;
    lin->dxReluOf = rin;
    lin->dxNorm = true;
    lin->dxOut = n->inputs[0].region;
    n->bwdFused = true;
  }
}

// ---- bf16 aggregation inputs: what a Linear(NONE) writes (its output, or the fused norm's) and one sum
//      scatter_gather alone reads is stored in bf16, rows of round_up(H, 8) elements; its gradient twin keeps that ld
static void make_bf16(RuntimeImpl* rt, int r) {
  TensorImpl& x = rt->t(r);
  if (x.data || x.grad) ROC_FATAL("set_bf16_aggregation: a tensor that becomes bf16 was already allocated");
  x.isBf16 = true;
  x.ld = round_up8(x.H);
}
static void choose_bf16_aggregation(RuntimeImpl* rt, const std::vector<GnnOp*>& layers, Wiring& w) {
  for (size_t l = 0; l < layers.size(); l++) {
    Linear* lin = as<Linear>(layers[l]);
    if (!lin || lin->activation != AC_MODE_NONE) continue;
    const int r = lin->fwdOut >= 0 ? lin->fwdOut : lin->outputs[0].region;
    // a sum with edge dropout has no bf16 form: it reads fp32
    ScatterGather* sg = w.consumers[r] == 1 ? as_sum_sg(layers[w.consumerOp[r]]) : nullptr;
    if (!sg || sg->dropRate > 0.0f) continue;
    make_bf16(rt, r);
  }
  // ... and what a Linear(NONE) or an unfused relu writes when a max / min, weighted or attention aggregation reads it
  // as its feature input, and every other reader is one of those, a Linear reading it as X (no fused dropout) or an
  // attention_scores
  for (size_t l = 0; l < layers.size(); l++) {
    int r = -1;
    if (Linear* lin = as<Linear>(layers[l]))
      r = lin->activation == AC_MODE_NONE ? (lin->fwdOut >= 0 ? lin->fwdOut : lin->outputs[0].region) : -1;
    else if (Activation* act = as<Activation>(layers[l]))
      r = (act->actiMode == AC_MODE_RELU && act->fusedInto < 0) ? act->outputs[0].region : -1;
    if (r < 0 || rt->t(r).isBf16) continue;
    bool aggregated = false, others = true;
    for (GnnOp* op : layers)
      for (int j = 0; j < op->numInputs; j++) {
        if (op->inputs[j].region != r) continue;
        ScatterGather* sg = as<ScatterGather>(op);
        Linear* lin = as<Linear>(op);
        AttentionGather* ag = as<AttentionGather>(op);   // dynamic, softmax and dot ones have no bf16 form: they read fp32
        if (j == 0 && ((sg && sg->aggr != AGGR_SUM) || as<WeightedScatterGather>(op) ||
                       (ag && !ag->dynamic && !ag->softmax && !ag->dot)))
          aggregated = true;
        else if (!(j == 0 && ((lin && lin->dropOp < 0) || as<AttentionScores>(op))))
          others = false;
      }
    if (aggregated && others) make_bf16(rt, r);
  }
}

// gnn.cc:625-673.  No graph loading / ResourceManager creation left to do here
// (Graph's constructor already built the device CSR); what remains are the passes
// above, in an order each later one relies on (a fusion sees the earlier ones'
// decisions, op_info reports them all).
bool Model::init(const Config&) {
  check_bf16_readers(*this);
  mark_gradients(*this);
  lay_out_flat_dw(ctx, parameters);
  const int maxSg = size_scratch_and_plans(*this);
  build_transpose(*this);
  set_up_halo(ctx, myGraph, layers, maxSg);
  Wiring w = wire(layers);   // the passes below change no op's inputs or outputs
  mark_scaled_add_readers(layers);
  if (fuse) {
    fuse_gcn_block(layers, w);
    fuse_batch_norm_relu(layers, w);
    fuse_dropout_into_linear(layers, w);
    fuse_backward_epilogues(ctx, layers, w);
  }
  if (bf16Aggregation) choose_bf16_aggregation(ctx, layers, w);
  if (fuse && ctx->numParts == 1) fuse_teleport(*this, w);   // after the bf16 choice, which it reads
  for (size_t l = 0; l < layers.size(); l++) layers[l]->init(*this);
  ctx->opNames.clear();
  for (size_t l = 0; l < layers.size(); l++)
    ctx->opNames.push_back(std::string(opKindNames[op_kind(layers[l])]) + (layers[l]->fusedInto >= 0 ? " (fused)" : ""));
  ROC_CHECK(cudaStreamSynchronize(ctx->stream));
  return true;
}

// gnn.cc:696-700
void Model::forward(void) {
  if (mode == MD_MODE_TRAIN) ctx->trainStep += 1;
  for (size_t l = 0; l < layers.size(); l++) {
    ctx->op_begin((int)l, 0);
    layers[l]->forward(*this);
    ctx->op_end();
  }
}

// gnn.cc:702-716
void Model::backward(void) {
  std::set<int> resetedInputGrads;
  for (int l = (int)layers.size() - 1; l >= 0; l--) {
    for (int i = 0; i < layers[l]->numInputs; i++) {
      int r = layers[l]->inputs[i].region;
      if (resetedInputGrads.find(r) == resetedInputGrads.end()) {
        resetedInputGrads.insert(r);
        layers[l]->resetInputGrads[i] = true;
      } else {
        // This input's gradients has been reseted by other layers
        layers[l]->resetInputGrads[i] = false;
      }
    }
    ctx->op_begin(l, 1);
    layers[l]->backward(*this);
    ctx->op_end();
  }
}

// gnn.cc:718-724 (+ the replica sum of optimizer_kernel.cu:88-94 as one all-reduce)
void Model::update(void) {
  RuntimeImpl* rt = ctx;
  rt->op_begin(-1, 2);
  optimizer->next();
  if (rt->numParts > 1 && rt->flatGradCount) {
    ROC_ASSERT(rt->commReady);
    ROC_CHECK(rt->comm.allreduce_sum(rt->flatGrad, rt->flatGradCount, rt->stream));
  }
  for (int p = (int)parameters.size() - 1; p >= 0; p--) optimizer->update(&parameters[p]);
  rt->op_end();
}

// gnn.cc:726-739
void Model::zero_gradients(void) {
  RuntimeImpl* rt = ctx;
  if (rt->flatGradCount)
    ROC_CHECK(cudaMemsetAsync(rt->flatGrad, 0, rt->flatGradCount * sizeof(float), rt->stream));
}

// Dense fp32 host rows <-> x's rows through the staging buffer, ~256 MB of floats at a time, so no full-size fp32 copy
// is ever resident.  Each chunk of rows [r0, r0 + nr) goes from `in` into staging before convert(r0, nr), or from
// staging to `out` after it (waited for: the next chunk reuses the buffer); one of `in` / `out` is null.
template <typename Convert>
static void staged_rows(RuntimeImpl* rt, const TensorImpl& x, const float* in, float* out, Convert convert) {
  const int64_t chunkRows = std::max<int64_t>(1, (int64_t)(64u << 20) / x.H);
  rt->ensure_staging((size_t)std::min<int64_t>(chunkRows, x.rows) * x.H * sizeof(float));
  for (int64_t r0 = 0; r0 < x.rows; r0 += chunkRows) {
    const int64_t nr = std::min<int64_t>(chunkRows, x.rows - r0);
    if (in) ROC_CHECK(cudaMemcpyAsync(rt->staging, in + r0 * x.H, (size_t)nr * x.H * 4, cudaMemcpyHostToDevice, rt->stream));
    convert(r0, nr);
    if (out) {
      ROC_CHECK(cudaMemcpyAsync(out + r0 * x.H, rt->staging, (size_t)nr * x.H * 4, cudaMemcpyDeviceToHost, rt->stream));
      ROC_CHECK(cudaStreamSynchronize(rt->stream));
    }
  }
}

void Model::set_tensor(const Tensor& t, const void* host, bool grad) {
  RuntimeImpl* rt = ctx;
  TensorImpl& x = rt->t(t.region);
  if (x.isBf16 && !(grad && x.produced)) {
    // fp32 host rows, rounded on the device chunk by chunk
    if (grad) ROC_FATAL("set_tensor(grad=true): a bf16 leaf tensor has no gradient");
    uint16_t* dst = rt->data_bf16(t.region);
    staged_rows(rt, x, static_cast<const float*>(host), nullptr, [&](int64_t r0, int64_t nr) {
      ROC_CHECK(roc_f32_to_bf16(nr, x.H, (const float*)rt->staging, x.H, dst + r0 * x.ld, x.ld, rt->stream));
    });
    ROC_CHECK(cudaStreamSynchronize(rt->stream));
    return;
  }
  float* dst = grad ? rt->grad(t.region) : rt->data(t.region);
  if (x.ld == x.H || x.isInt) {
    ROC_CHECK(cudaMemcpyAsync(dst, host, (size_t)x.rows * x.H * 4, cudaMemcpyHostToDevice, rt->stream));
  } else {
    // Dense host rows -> padded device rows.  A strided cudaMemcpy2D of 2.4 KB rows runs at
    // ~17 GB/s; contiguous chunks into a staging buffer run at PCIe speed and the re-pitch
    // is a device copy at HBM speed.
    staged_rows(rt, x, static_cast<const float*>(host), nullptr, [&](int64_t r0, int64_t nr) {
      ROC_CHECK(roc_copy2d(nr, x.H, (const float*)rt->staging, x.H, dst + r0 * x.ld, x.ld, rt->stream));
    });
  }
  ROC_CHECK(cudaStreamSynchronize(rt->stream));
}

void Model::get_tensor(const Tensor& t, void* host, bool grad) const {
  RuntimeImpl* rt = ctx;
  TensorImpl& x = rt->t(t.region);
  if (x.isBf16 && !(grad && x.produced)) {
    // widened exactly on the device into staging, chunk by chunk
    if (grad) ROC_FATAL("get_tensor(grad=true): a bf16 leaf tensor has no gradient");
    const uint16_t* src = rt->data_bf16(t.region);
    staged_rows(rt, x, nullptr, static_cast<float*>(host), [&](int64_t r0, int64_t nr) {
      ROC_CHECK(roc_bf16_to_f32(nr, x.H, src + r0 * x.ld, x.ld, (float*)rt->staging, x.H, rt->stream));
    });
    return;
  }
  const float* src = grad ? rt->grad(t.region) : rt->data(t.region);
  ROC_CHECK(cudaMemcpy2DAsync(host, (size_t)x.H * 4, src, (size_t)x.ld * 4, (size_t)x.H * 4, (size_t)x.rows,
                              cudaMemcpyDeviceToHost, rt->stream));
  ROC_CHECK(cudaStreamSynchronize(rt->stream));
}

void Model::set_tensor_bf16(const Tensor& t, const uint16_t* host) {
  RuntimeImpl* rt = ctx;
  TensorImpl& x = rt->t(t.region);
  if (!x.isBf16) ROC_FATAL("set_tensor_bf16: not a bf16 tensor");
  ROC_CHECK(cudaMemcpy2DAsync(rt->data_bf16(t.region), (size_t)x.ld * 2, host, (size_t)x.H * 2, (size_t)x.H * 2,
                              (size_t)x.rows, cudaMemcpyHostToDevice, rt->stream));
  ROC_CHECK(cudaStreamSynchronize(rt->stream));
}

void Model::get_tensor_bf16(const Tensor& t, uint16_t* host) const {
  RuntimeImpl* rt = ctx;
  TensorImpl& x = rt->t(t.region);
  if (!x.isBf16) ROC_FATAL("get_tensor_bf16: not a bf16 tensor");
  ROC_CHECK(cudaMemcpy2DAsync(host, (size_t)x.H * 2, rt->data_bf16(t.region), (size_t)x.ld * 2, (size_t)x.H * 2,
                              (size_t)x.rows, cudaMemcpyDeviceToHost, rt->stream));
  ROC_CHECK(cudaStreamSynchronize(rt->stream));
}

void Model::set_labels(const Tensor& label, const int* host_class_idx) {
  RuntimeImpl* rt = ctx;
  TensorImpl& x = rt->t(label.region);
  if (!x.labelIdx) x.labelIdx = (int32_t*)rt->dmalloc((size_t)x.rows * sizeof(int32_t));
  for (int64_t v = 0; v < x.rows; v++) ROC_ASSERT(host_class_idx[v] >= 0 && host_class_idx[v] < x.H);  // load_task.cu:120
  ROC_CHECK(cudaMemcpyAsync(x.labelIdx, host_class_idx, (size_t)x.rows * sizeof(int32_t), cudaMemcpyHostToDevice, rt->stream));
  ROC_CHECK(cudaStreamSynchronize(rt->stream));
}

void Model::set_multilabels(const Tensor& label, const uint32_t* host_packed_bits) {
  RuntimeImpl* rt = ctx;
  TensorImpl& x = rt->t(label.region);
  const size_t words = (size_t)x.rows * (size_t)((x.H + 31) / 32);
  if (!x.labelBits) x.labelBits = (uint32_t*)rt->dmalloc((words ? words : 1) * sizeof(uint32_t));
  ROC_CHECK(cudaMemcpyAsync(x.labelBits, host_packed_bits, words * sizeof(uint32_t), cudaMemcpyHostToDevice, rt->stream));
  ROC_CHECK(cudaStreamSynchronize(rt->stream));
}

roc_perf_metrics Model::last_metrics(void) const {
  RuntimeImpl* rt = ctx;
  roc_multilabel_metrics ml;
  if (rt->lossKind == ROC_HOST_OP_SIGMOID_CROSS_ENTROPY && last_multilabel_metrics(&ml)) {
    // the multi-label head's PerfMetrics: its train loss, its rows, and its exact matches (subset accuracy)
    rt->h_perf.trainLoss = (float)ml.loss[0];
    rt->h_perf.trainAll = (int)ml.rows[ROC_MASK_TRAIN];
    rt->h_perf.valAll = (int)ml.rows[ROC_MASK_VAL];
    rt->h_perf.testAll = (int)ml.rows[ROC_MASK_TEST];
    rt->h_perf.trainCorrect = (int)ml.exact[ROC_MASK_TRAIN];
    rt->h_perf.valCorrect = (int)ml.exact[ROC_MASK_VAL];
    rt->h_perf.testCorrect = (int)ml.exact[ROC_MASK_TEST];
    return rt->h_perf;
  }
  ROC_CHECK(cudaMemcpyAsync(&rt->h_perf, rt->d_perf, sizeof(roc_perf_metrics), cudaMemcpyDeviceToHost, rt->stream));
  ROC_CHECK(cudaStreamSynchronize(rt->stream));
  return rt->h_perf;
}

bool Model::last_multilabel_metrics(roc_multilabel_metrics* out) const {
  RuntimeImpl* rt = ctx;
  if (!rt->multilabelRan) return false;
  ROC_CHECK(cudaMemcpyAsync(out, rt->d_multilabel, sizeof(roc_multilabel_metrics), cudaMemcpyDeviceToHost, rt->stream));
  ROC_CHECK(cudaStreamSynchronize(rt->stream));
  return true;
}

// ---- dataset loaders: load_task.cu:25-199 (formats in SURVEY Appendix C) ----
void Model::load_features(const Tensor& input, const std::string& prefix) {
  RuntimeImpl* rt = ctx;
  TensorImpl& x = rt->t(input.region);
  const int inDim = x.H;
  const size_t nloc = (size_t)x.rows;
  std::vector<float> buf(nloc * (size_t)inDim);
  std::string binFile = prefix + ".feats.bin", csvFile = prefix + ".feats.csv";
  FILE* binFin = fopen(binFile.c_str(), "rb");
  if (binFin == NULL) {
    // CSV: one line per vertex, inDim comma-separated values (load_task.cu:42-62); the
    // whole file is parsed so the .feats.bin cache can be written (load_task.cu:63-65)
    fprintf(stderr, "[roc_b200] Load features from CSV: %s\n", csvFile.c_str());
    std::ifstream csvFin(csvFile.c_str());
    if (!csvFin.good()) ROC_FATAL(("cannot open " + binFile + " or " + csvFile).c_str());
    std::vector<float> all((size_t)myGraph.numNodes * inDim);
    std::string line, word;
    for (V_ID v = 0; v < myGraph.numNodes; v++) {
      std::getline(csvFin, line);
      std::stringstream ss(line);
      int feat_cnt = 0;
      while (std::getline(ss, word, ',')) {
        ROC_ASSERT(feat_cnt < inDim);
        all[(size_t)v * inDim + feat_cnt] = std::stof(word);
        feat_cnt++;
      }
      ROC_ASSERT(feat_cnt == inDim);
    }
    if (rt->myPart == 0) {
      // the cache appears atomically (tmp + rename): another rank or job that finds <prefix>.feats.bin can read it whole
      const std::string tmpFile = binFile + ".tmp";
      FILE* binFout = fopen(tmpFile.c_str(), "wb");
      if (binFout) {
        const bool ok = fwrite(all.data(), sizeof(float), all.size(), binFout) == all.size();
        if (fclose(binFout) == 0 && ok) rename(tmpFile.c_str(), binFile.c_str());
        else remove(tmpFile.c_str());
      }
    }
    memcpy(buf.data(), all.data() + (size_t)myGraph.rowLeft * inDim, buf.size() * sizeof(float));
  } else {
    ROC_ASSERT(fseeko(binFin, (off_t)((size_t)myGraph.rowLeft * inDim * sizeof(float)), SEEK_SET) == 0);
    size_t ret = fread(buf.data(), sizeof(float), buf.size(), binFin);
    ROC_ASSERT(ret == buf.size());
    fclose(binFin);
  }
  set_tensor(input, buf.data());
}

void Model::load_labels(const Tensor& label, const std::string& prefix) {
  RuntimeImpl* rt = ctx;
  TensorImpl& x = rt->t(label.region);
  std::string filename = prefix + ".label";
  FILE* file = fopen(filename.c_str(), "r");
  if (!file) ROC_FATAL(("cannot open " + filename).c_str());
  int idx;
  for (V_ID v = 0; v < myGraph.rowLeft; v++) ROC_ASSERT(fscanf(file, "%d", &idx) == 1);
  std::vector<int> cls((size_t)x.rows);
  for (int64_t v = 0; v < x.rows; v++) {
    ROC_ASSERT(fscanf(file, "%d", &idx) == 1);
    cls[(size_t)v] = idx;
  }
  fclose(file);
  set_labels(label, cls.data());
}

void Model::load_train_mask(const Tensor& mask, const std::string& prefix) {
  RuntimeImpl* rt = ctx;
  TensorImpl& x = rt->t(mask.region);
  std::string filename = prefix + ".mask";
  std::ifstream fin(filename.c_str());
  if (!fin.good()) ROC_FATAL(("cannot open " + filename).c_str());
  std::string line;
  for (V_ID v = 0; v < myGraph.rowLeft; v++) std::getline(fin, line);
  std::vector<int> m((size_t)x.rows);
  for (int64_t v = 0; v < x.rows; v++) {
    std::getline(fin, line);
    if (line == "Train") m[(size_t)v] = MASK_TRAIN;
    else if (line == "Val") m[(size_t)v] = MASK_VAL;
    else if (line == "Test") m[(size_t)v] = MASK_TEST;
    else if (line == "None") m[(size_t)v] = MASK_NONE;
    else { printf("Unrecognized mask: %s\n", line.c_str()); ROC_ASSERT(false); }
  }
  set_tensor(mask, m.data());
}

namespace {
// Entries [selA, selB) of the block-ordered selection (or the whole requester-grouped list when blockK < 0) go to
// the peers: packed into the send buffer on commStream, then one DMA copy per peer on that peer's stream.
void exchange_rows(RuntimeImpl* rt, const Graph& g, float* local, int64_t ld, int H, std::vector<float*>& peers,
                   int blockK, bool last, int smLimit) {
  const size_t nb = g.pushBlockRow.size() - 1;
  const int P = rt->numParts, me = rt->myPart;
  ROC_CHECK(cudaEventRecord(rt->evProduced, rt->stream));
  ROC_CHECK(cudaStreamWaitEvent(rt->commStream, rt->evProduced, 0));
  if (!rt->p2pCopyEngines) {
    const size_t a = blockK < 0 ? 0 : g.pushBlockOff[(size_t)blockK], b = blockK < 0 ? g.numSendRows : g.pushBlockOff[(size_t)blockK + 1];
    if (b > a)
      ROC_CHECK(roc_push_rows((int64_t)(b - a), H, g.d_pushRows + a, g.d_pushPeer + a, g.d_pushDst + a, local, ld,
                              peers.data(), P, ld, smLimit, rt->commStream));
    if (last) ROC_CHECK(cudaEventRecord(rt->evPushed, rt->commStream));
    return;
  }
  const size_t uld = (size_t)ld;
  rt->ensure_sendbuf((g.numSendRows ? g.numSendRows : 1) * uld);
  if ((blockK <= 0) && rt->exchInFlight) {
    // the previous exchange's copies read the send buffer: the first pack of this one waits for them
    for (int q = 0; q < P; q++) if (q != me) ROC_CHECK(cudaStreamWaitEvent(rt->commStream, rt->peerDone[(size_t)q], 0));
  }
  if (blockK < 0) ROC_CHECK(roc_pack_rows((int64_t)g.numSendRows, H, g.d_sendRows, local, ld, rt->sendBuf, ld, rt->commStream));
  else ROC_CHECK(roc_pack_rows_at((int64_t)(g.packBlockOff[(size_t)blockK + 1] - g.packBlockOff[(size_t)blockK]), H,
                                  g.d_packSel + g.packBlockOff[(size_t)blockK], g.d_sendRows, local, ld, rt->sendBuf, ld,
                                  rt->commStream));
  ROC_CHECK(cudaEventRecord(rt->evPacked, rt->commStream));
  for (int q = 0; q < P; q++) {
    if (q == me) continue;
    const size_t j0 = blockK < 0 ? g.sendOffs[(size_t)q] : g.packPeerOff[(size_t)q * (nb + 1) + (size_t)blockK];
    const size_t j1 = blockK < 0 ? g.sendOffs[(size_t)q] + g.sendCounts[(size_t)q] : g.packPeerOff[(size_t)q * (nb + 1) + (size_t)blockK + 1];
    cudaStream_t ps = rt->peerStreams[(size_t)q];
    if (j1 > j0) {
      ROC_CHECK(cudaStreamWaitEvent(ps, rt->evPacked, 0));
      float* dst = peers[(size_t)q] + ((size_t)g.peerSlab0[(size_t)q] + (j0 - g.sendOffs[(size_t)q])) * uld;
      ROC_CHECK(cudaMemcpyAsync(dst, rt->sendBuf + j0 * uld, (j1 - j0) * uld * sizeof(float), cudaMemcpyDeviceToDevice, ps));
    }
    if (last) ROC_CHECK(cudaEventRecord(rt->peerDone[(size_t)q], ps));
  }
  if (last) rt->exchInFlight = true;
}
// the compute stream waits for this partition's outgoing rows, then crosses the barrier behind which every
// partition's rows have landed here
void exchange_wait(RuntimeImpl* rt) {
  if (!rt->p2pCopyEngines) ROC_CHECK(cudaStreamWaitEvent(rt->stream, rt->evPushed, 0));
  else
    for (int q = 0; q < rt->numParts; q++) if (q != rt->myPart) ROC_CHECK(cudaStreamWaitEvent(rt->stream, rt->peerDone[(size_t)q], 0));
  ROC_CHECK(rt->comm.barrier(rt->d_barrier, rt->stream));
}
}  // namespace

// ---- pipelined peer-write exchange: a producer computes its rows block by block and pushes block k's boundary
// rows (commStream) while it computes block k + 1 (compute stream, on SMs - pushSMs)
namespace {
struct PushPipe {
  RuntimeImpl* rt; const Graph* g; TensorImpl* x; bool isGrad; bool on; int prevReserve;
  // the tensor `region` (data or grad) is read by a ScatterGather through peer-mapped halo slabs?
  PushPipe(const Model& model, int region, bool grad) : rt(model.ctx), g(&model.myGraph), x(nullptr), isGrad(grad), on(false), prevReserve(0) {
    if (region < 0 || !rt->p2p || rt->numParts == 1) return;
    x = &rt->t(region);
    const std::vector<float*>& peers = grad ? x->peerGrad : x->peerData;
    on = !peers.empty() && g->pushBlockRow.size() >= 2;
    if (on && !rt->p2pCopyEngines) prevReserve = roc_set_sm_reserve(rt->pushSMs);   // the push KERNEL needs free SMs; DMA copies do not
  }
  size_t blocks() const { return on ? g->pushBlockRow.size() - 1 : 1; }
  int64_t row0(size_t k) const { return on ? (int64_t)g->pushBlockRow[k] : 0; }
  int64_t rows(size_t k, int64_t all) const { return on ? (int64_t)g->pushBlockRow[k + 1] - (int64_t)g->pushBlockRow[k] : all; }
  E_ID colLeft(size_t k) const { return on ? g->pushBlockColLeft[k] : g->colLeft; }
  // block k of `local` has been enqueued on the compute stream
  void pushed(size_t k, float* local, int64_t ld, int H) {
    if (!on) return;
    std::vector<float*>& peers = isGrad ? x->peerGrad : x->peerData;
    const bool last = k + 1 == blocks();
    exchange_rows(rt, *g, local, ld, H, peers, (int)k, last, rt->pushGridSMs >= 0 ? rt->pushGridSMs : rt->pushSMs);
    if (last) (isGrad ? x->freshGrad : x->freshData) = true;
  }
  // kernels enqueued after this may use the whole chip again
  void done() { if (on) { if (!rt->p2pCopyEngines) roc_set_sm_reserve(prevReserve); on = false; } }
  ~PushPipe() { done(); }
};
}  // namespace

// -------------------------------------------------------- ScatterGather -----
ScatterGather::ScatterGather(const Model& model, const Tensor& _input, AggrType _aggr)
    : GnnOp(_input), aggr(_aggr), arg(nullptr), argLd(0), epilogue(0), bwdEpilogue(0), fwdOut(-1), bwdOut(-1), teleT(-1),
      teleAlpha(1.0f), teleBeta(1.0f), dropRate(0.0f), seed(0), opIndex(0) {
  // scattergather.cc:33-37
  ROC_ASSERT(inputs[0].type == Tensor::NODE_TENSOR);
  ROC_ASSERT(inputs[0].numDim == 2);
  ROC_ASSERT(inputs[0].dims[1] == model.myGraph.numNodes);
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)inputs[0].dims[0]);
}
void ScatterGather::init(const Model&) {}

namespace {
// The exchange step of ScatterGather (scattergather.cc:69-73 asks Legion for the
// WHOLE input region): all-gather every partition's slab into [numNodes][ld] so
// the kernel can index rows by global source id.  numParts == 1: no copy at all.
// Default for numParts > 1: the halo exchange — each partition packs the rows the others read
// (roc_pack_rows), one grouped NCCL send/recv moves them, and they land right behind the
// partition's own rows ([Nloc | halo] is what the remapped col indexes).  ROC_B200_HALO=0 keeps
// the whole-matrix all-gather (the reference's semantics) for comparison.
const float* gathered(const Model& model, float* local, int64_t ld, int H, TensorImpl* x, bool isGrad) {
  RuntimeImpl* rt = model.ctx;
  if (rt->numParts == 1) return local;
  ROC_ASSERT(rt->commReady);
  const Graph& g = model.myGraph;
  if (g.halo && rt->p2p) {
    // Peer writes: unless the producer already pushed its rows block by block (fresh), push them all now; then wait
    // for the pushes and cross the barrier after which every partition's rows are in this partition's slab.
    std::vector<float*>& peers = isGrad ? x->peerGrad : x->peerData;
    bool& fresh = isGrad ? x->freshGrad : x->freshData;
    ROC_ASSERT(!peers.empty());
    if (!fresh) exchange_rows(rt, g, local, ld, H, peers, /*blockK=*/-1, /*last=*/true, /*smLimit=*/0);
    fresh = false;
    exchange_wait(rt);
    return local;
  }
  if (g.halo) {
    const size_t uld = (size_t)ld;
    rt->ensure_sendbuf((g.numSendRows ? g.numSendRows : 1) * uld);
    ROC_CHECK(roc_pack_rows((int64_t)g.numSendRows, H, g.d_sendRows, local, ld, rt->sendBuf, ld, rt->stream));
    std::vector<size_t> sc(g.sendCounts), so(g.sendOffs), rc(g.recvCounts), ro(g.recvOffs);
    for (size_t q = 0; q < sc.size(); q++) { sc[q] *= uld; so[q] *= uld; rc[q] *= uld; ro[q] *= uld; }
    float* haloBase = local + (size_t)model.local_rows() * uld;
    ROC_CHECK(rt->comm.alltoallv(rt->sendBuf, sc, so, haloBase, rc, ro, /*isFloat=*/true, rt->stream));
    return local;
  }
  rt->ensure_gather((size_t)g.numNodes * (size_t)ld);
  std::vector<size_t> counts((size_t)rt->numParts), offs((size_t)rt->numParts);
  for (int r = 0; r < rt->numParts; r++) {
    counts[(size_t)r] = ((size_t)g.vbounds[2 * r + 1] - g.vbounds[2 * r] + 1) * (size_t)ld;
    offs[(size_t)r] = (size_t)g.vbounds[2 * r] * (size_t)ld;
  }
  ROC_CHECK(rt->comm.allgatherv(local, rt->gatherBuf, counts, offs, rt->stream));
  return rt->gatherBuf;
}
}  // namespace

void ScatterGather::forward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int H = (int)inputs[0].dims[0];
  const int64_t ldIn = rt->t(inputs[0].region).ld;
  if (aggr == AGGR_MAX || aggr == AGGR_MIN) {   // one partition (Model::scatter_gather): no exchange, no fusion
    const int64_t ldOut = rt->t(outputs[0].region).ld;
    if (!arg) {
      argLd = ldOut;
      arg = (uint32_t*)rt->dmalloc((size_t)model.local_rows() * (size_t)argLd * sizeof(uint32_t));
    }
    const int how = aggr == AGGR_MAX ? ROC_SG_AGGR_MAX : ROC_SG_AGGR_MIN;
    rt->sg_begin(H);
    if (rt->t(inputs[0].region).isBf16)
      ROC_CHECK(roc_sg_minmax_forward_planned_bf16(model.myGraph.plan, how, H, rt->data_bf16(inputs[0].region), ldIn,
                                                   rt->data(outputs[0].region), ldOut, arg, argLd, rt->stream));
    else
      ROC_CHECK(roc_sg_minmax_forward_planned(model.myGraph.plan, how, H, rt->data(inputs[0].region), ldIn,
                                              rt->data(outputs[0].region), ldOut, arg, argLd, rt->stream));
    rt->sg_end();
    return;
  }
  const int outRegion = fwdOut >= 0 ? fwdOut : outputs[0].region;
  const bool xBf16 = rt->t(inputs[0].region).isBf16;   // set_bf16_aggregation: one partition, nothing to exchange
  rt->sg_begin(-H);          // negative width = the exposed part of the halo exchange (profile mode only)
  const float* src =
      xBf16 ? nullptr : gathered(model, rt->data(inputs[0].region), ldIn, H, &rt->t(inputs[0].region), false);
  rt->sg_end();
  float* dst = rt->data(outRegion);
  const float rate = drop_rate(model);
  const uint8_t* keep = rate > 0.0f ? keep_mask(model, model.myGraph.plan, model.myGraph.rowLeft, 0) : nullptr;
  rt->sg_begin(H);
  if (teleT >= 0)   // a fused scaled_add (fuse_teleport: one partition, fp32 input)
    ROC_CHECK(roc_sg_forward_teleport_dropout_planned(model.myGraph.plan, H, src, ldIn, teleAlpha, rt->data(teleT),
                                                      rt->t(teleT).ld, teleBeta, dst, rt->t(outRegion).ld, epilogue,
                                                      keep, rate, rt->stream));
  else if (rate > 0.0f)   // edge dropout: one partition, fp32 input
    ROC_CHECK(roc_sg_forward_dropout_planned(model.myGraph.plan, H, src, ldIn, dst, rt->t(outRegion).ld, epilogue, keep,
                                             rate, rt->stream));
  else if (xBf16)
    ROC_CHECK(roc_sg_forward_planned_bf16(model.myGraph.plan, H, rt->data_bf16(inputs[0].region), ldIn, dst,
                                          rt->t(outRegion).ld, epilogue, rt->stream));
  else
    ROC_CHECK(roc_sg_forward_planned(model.myGraph.plan, H, src, ldIn, dst, rt->t(outRegion).ld, epilogue, rt->stream));
  rt->sg_end();
}

void ScatterGather::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  ROC_ASSERT(resetInputGrads[0]);   // scattergather_kernel.cu:167
  if (!rt->t(inputs[0].region).requiresGrad) return;
  const int H = (int)inputs[0].dims[0];
  const int64_t ld = rt->t(outputs[0].region).ld;
  if (aggr == AGGR_MAX || aggr == AGGR_MIN) {
    // each output gradient goes to the source its forward chose; a gather over the same CSR (no atomics), or over the
    // transpose with the exact backward
    const int src = inputs[0].region;
    rt->sg_begin(H);
    if (model.exactBackward)
      ROC_CHECK(roc_sg_transpose_minmax_backward(rt->sgTranspose, H, rt->grad(outputs[0].region), ld, arg, argLd,
                                                 rt->grad(src), rt->t(src).ld, rt->stream));
    else
      ROC_CHECK(roc_sg_minmax_backward_planned(model.myGraph.plan, H, model.myGraph.rowLeft, rt->grad(outputs[0].region),
                                               ld, arg, argLd, rt->grad(src), rt->t(src).ld, rt->stream));
    rt->sg_end();
    return;
  }
  const int dstRegion = bwdOut >= 0 ? bwdOut : inputs[0].region;
  // Forward and backward do exactly the same thing, on gradients (scattergather_kernel.cu:168-169); the exact backward
  // sums over the transpose instead, its fused NORM dividing by the in-degree of the graph's rowEnd
  rt->sg_begin(-H);
  const float* src = gathered(model, rt->grad(outputs[0].region), ld, H, &rt->t(outputs[0].region), true);
  rt->sg_end();
  float* dst = rt->grad(dstRegion);
  // edge dropout: the keep bytes of the pairs this pass weighs, (w <- u) for row u's edge to w, in the order of the
  // plan it runs over (the same CSR's reverse pairs, or the transposed plan's)
  const float rate = drop_rate(model);
  const uint8_t* keep = nullptr;
  if (rate > 0.0f) {
    const roc_sg_plan* planT = nullptr;
    if (model.exactBackward) ROC_CHECK(roc_sg_transpose_info(rt->sgTranspose, nullptr, nullptr, nullptr, &planT));
    keep = keep_mask(model, model.exactBackward ? planT : model.myGraph.plan,
                     model.exactBackward ? 0 : model.myGraph.rowLeft, 1);
  }
  rt->sg_begin(H);
  if (model.exactBackward)
    ROC_CHECK(roc_sg_transpose_sum_backward_dropout(rt->sgTranspose, H, src, ld, dst, rt->t(dstRegion).ld, bwdEpilogue,
                                                    model.myGraph.d_rowEnd, keep, rate, rt->stream));
  else
    ROC_CHECK(roc_sg_forward_dropout_planned(model.myGraph.plan, H, src, ld, dst, rt->t(dstRegion).ld, bwdEpilogue, keep,
                                             rate, rt->stream));
  rt->sg_end();
}

// edge dropout's rate in the current mode (infer: none)
float ScatterGather::drop_rate(const Model& model) const { return model.mode == MD_MODE_TRAIN ? dropRate : 0.0f; }

// The keep bytes of every edge of `plan` for this op's key and the current step, in the runtime's one E-byte buffer
// (allocated on first use): each dropped sum fills it right before the kernel that reads it, so the ops and the
// forward / backward passes share it.
const uint8_t* ScatterGather::keep_mask(const Model& model, const roc_sg_plan* plan, roc_vid_t selfBase,
                                        int rowIsSource) const {
  RuntimeImpl* rt = model.ctx;
  if (!rt->sgKeep) rt->sgKeep = (uint8_t*)rt->dmalloc(std::max<size_t>((size_t)model.myGraph.numEdges, 16));
  const uint64_t key = ((uint64_t)(uint32_t)seed << 32) | (uint32_t)opIndex;
  ROC_CHECK(roc_sg_attn_keep_mask(plan, selfBase, rowIsSource, dropRate, key, rt->trainStep, rt->sgKeep, rt->stream));
  return rt->sgKeep;
}

// An op whose kernel overwrites an input gradient writes it into the gradient itself when `direct`, else into
// `scratch` (allocated on first use), which add_scratch then adds to the gradient another op already wrote.
static float* grad_or_scratch(const Model& model, int region, bool direct, float*& scratch) {
  RuntimeImpl* rt = model.ctx;
  if (direct) return rt->grad(region);
  if (!scratch)
    scratch = (float*)rt->dmalloc((size_t)std::max<int64_t>(model.local_rows(), 1) * (size_t)rt->t(region).ld * sizeof(float));
  return scratch;
}
static void add_scratch(const Model& model, int region, const float* scratch) {
  RuntimeImpl* rt = model.ctx;
  const TensorImpl& x = rt->t(region);
  float* g = rt->grad(region);
  ROC_CHECK(roc_add_fwd(model.local_rows(), x.H, g, x.ld, scratch, x.ld, g, x.ld, rt->stream));
}

// ------------------------------------------------------- AttentionGather -----
AttentionGather::AttentionGather(const Model& model, const Tensor& _input, const Tensor& _scores, int _heads, float _slope,
                                 float _dropRate, int _seed)
    : GnnOp(_input, _scores), heads(_heads), slope(_slope), dropRate(_dropRate), seed(_seed), opIndex(0),
      keep(nullptr), keep2(nullptr), stats(nullptr), statsLd(0), dynamic(false), softmax(false),
      learnTemperature(false), tConst(nullptr), dot(false), scale(0.0f) {
  scratch[0] = scratch[1] = scratch[2] = nullptr;
  ROC_ASSERT(_input.type == Tensor::NODE_TENSOR && _scores.type == Tensor::NODE_TENSOR);
  ROC_ASSERT(_input.numDim == 2 && _scores.numDim == 2);
  ROC_ASSERT(_input.dims[1] == model.myGraph.numNodes && _scores.dims[1] == model.myGraph.numNodes);
  if (_heads <= 0 || _scores.dims[0] != 2 * (E_ID)_heads)
    ROC_FATAL("attention_gather: the scores need 2 * heads columns ([s_dst | s_src] per head)");
  if (!(_slope >= 0.0f) || !std::isfinite(_slope)) ROC_FATAL("attention_gather: the negative slope must be finite and >= 0");
  if (!(_dropRate >= 0.0f && _dropRate < 1.0f)) ROC_FATAL("attention_gather: the dropout rate must be in [0, 1)");
  // the layouts roc_sg_attn_* take on node tensors (rows padded to float4: the vector path)
  const int64_t H = (int64_t)_input.dims[0], F = H / _heads;
  if (_heads != 1 && _heads != 2 && _heads != 4 && _heads != 8)
    ROC_FATAL("attention_gather: heads must be 1, 2, 4 or 8");
  if (H % _heads || (_heads > 1 && (F < 4 || (F & (F - 1)))))
    ROC_FATAL("attention_gather: with heads > 1, the input width must be heads * F with F a power of two >= 4");
  if (H > 512) ROC_FATAL("attention_gather: the input width must be at most 512");
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)_input.dims[0]);
}
// The dynamic mode: xl and xr are the op's two inputs, one region twice when they are one tensor (the second then adds
// its gradient through scratch, as any input another op already wrote).
AttentionGather::AttentionGather(const Model& model, const Tensor& xl, const Tensor& xr, int _heads, float _slope)
    : GnnOp(xl, xr), heads(_heads), slope(_slope), dropRate(0.0f), seed(0), opIndex(0), keep(nullptr), keep2(nullptr),
      stats(nullptr), statsLd(0), dynamic(true), softmax(false), learnTemperature(false), tConst(nullptr),
      dot(false), scale(0.0f) {
  scratch[0] = scratch[1] = scratch[2] = nullptr;
  ROC_ASSERT(xl.type == Tensor::NODE_TENSOR && xr.type == Tensor::NODE_TENSOR);
  ROC_ASSERT(xl.numDim == 2 && xr.numDim == 2);
  ROC_ASSERT(xl.dims[1] == model.myGraph.numNodes && xr.dims[1] == model.myGraph.numNodes);
  const int64_t H = (int64_t)xl.dims[0];
  if (xr.dims[0] != xl.dims[0]) ROC_FATAL("dynamic_attention_gather: xl and xr must have the same width");
  if (_heads <= 0 || _heads > 8 || H % _heads)
    ROC_FATAL("dynamic_attention_gather: the width must be heads * F with 1 <= heads <= 8");
  if (H > 256) ROC_FATAL("dynamic_attention_gather: the width must be at most 256");
  if (!(_slope >= 0.0f) || !std::isfinite(_slope))
    ROC_FATAL("dynamic_attention_gather: the negative slope must be finite and >= 0");
  if (model.ctx->t(xl.region).isBf16 || model.ctx->t(xr.region).isBf16)
    ROC_FATAL("dynamic_attention_gather: xl and xr must be fp32 (there is no bf16 form)");
  a = model.create_weight_tensor(_heads, (int)(H / _heads), NULL);   // GlorotUniform: +-sqrt(6 / (heads + F))
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)H);
}
// The softmax aggregation mode: one input x, and t as a (1, 1) parameter or a constant device float, both filled
// without a random draw.
AttentionGather::AttentionGather(const Model& model, const Tensor& x, float _temperature, bool _learn)
    : GnnOp(x), heads(1), slope(0.0f), dropRate(0.0f), seed(0), opIndex(0), keep(nullptr), keep2(nullptr),
      stats(nullptr), statsLd(0), dynamic(false), softmax(true), learnTemperature(_learn), tConst(nullptr),
      dot(false), scale(0.0f) {
  scratch[0] = scratch[1] = scratch[2] = nullptr;
  ROC_ASSERT(x.type == Tensor::NODE_TENSOR && x.numDim == 2 && x.dims[1] == model.myGraph.numNodes);
  if (!std::isfinite(_temperature)) ROC_FATAL("softmax_gather: the temperature must be finite");
  if (model.ctx->t(x.region).isBf16) ROC_FATAL("softmax_gather: x must be fp32 (there is no bf16 form)");
  RuntimeImpl* rt = model.ctx;
  float* t;
  if (_learn) {
    ZerosInitializer zeros;
    temperature = model.create_weight_tensor(1, 1, &zeros);
    t = rt->data(temperature.region);
  } else {
    t = tConst = (float*)rt->dmalloc(sizeof(float));
  }
  ROC_CHECK(roc_fill(1, 1, _temperature, t, 1, rt->stream));
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)x.dims[0]);
}
// The dot-product mode: q, k and v are the op's three inputs, one region more than once when they are one tensor (a
// later one then adds its gradient through scratch, as any input another op already wrote).  No parameter.
AttentionGather::AttentionGather(const Model& model, const Tensor& q, const Tensor& k, const Tensor& v, int _heads,
                                 float _scale)
    : GnnOp(q, k, v), heads(_heads), slope(0.0f), dropRate(0.0f), seed(0), opIndex(0), keep(nullptr), keep2(nullptr),
      stats(nullptr), statsLd(0), dynamic(false), softmax(false), learnTemperature(false), tConst(nullptr), dot(true),
      scale(_scale) {
  scratch[0] = scratch[1] = scratch[2] = nullptr;
  for (const Tensor* t : {&q, &k, &v}) {
    ROC_ASSERT(t->type == Tensor::NODE_TENSOR && t->numDim == 2 && t->dims[1] == model.myGraph.numNodes);
    if (model.ctx->t(t->region).isBf16)
      ROC_FATAL("dot_attention_gather: q, k and v must be fp32 (there is no bf16 form)");
  }
  const int64_t H = (int64_t)q.dims[0];
  if (k.dims[0] != q.dims[0] || v.dims[0] != q.dims[0])
    ROC_FATAL("dot_attention_gather: q, k and v must have the same width");
  if (_heads <= 0 || _heads > 8 || H % _heads)
    ROC_FATAL("dot_attention_gather: the width must be heads * F with 1 <= heads <= 8");
  if (H > 256) ROC_FATAL("dot_attention_gather: the width must be at most 256");
  if (_scale == 0.0f || !std::isfinite(_scale)) ROC_FATAL("dot_attention_gather: the scale must be finite and not 0");
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)H);
}
void AttentionGather::init(const Model& model) {
  if (dynamic && (model.ctx->t(inputs[0].region).isBf16 || model.ctx->t(inputs[1].region).isBf16))
    ROC_FATAL("dynamic_attention_gather: xl and xr must be fp32 (there is no bf16 form)");
  if (softmax && model.ctx->t(inputs[0].region).isBf16)
    ROC_FATAL("softmax_gather: x must be fp32 (there is no bf16 form)");
  if (dot)
    for (int i = 0; i < 3; i++)
      if (model.ctx->t(inputs[i].region).isBf16)
        ROC_FATAL("dot_attention_gather: q, k and v must be fp32 (there is no bf16 form)");
}

// the attention dropout rate in the current mode (infer: none) and its Philox key
float AttentionGather::drop_rate(const Model& model) const { return model.mode == MD_MODE_TRAIN ? dropRate : 0.0f; }
uint64_t AttentionGather::drop_key() const { return ((uint64_t)(uint32_t)seed << 32) | (uint32_t)opIndex; }

// one keep byte per edge of `plan`, in buffer `buf` (allocated on first use)
void AttentionGather::keep_mask(const Model& model, const roc_sg_plan* plan, roc_vid_t selfBase, int rowIsSource,
                                uint8_t*& buf) {
  RuntimeImpl* rt = model.ctx;
  if (!buf) buf = (uint8_t*)rt->dmalloc(std::max<size_t>((size_t)model.myGraph.numEdges, 16));
  ROC_CHECK(roc_sg_attn_keep_mask(plan, selfBase, rowIsSource, dropRate, drop_key(), rt->trainStep, buf, rt->stream));
}

void AttentionGather::forward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int H = (int)inputs[0].dims[0];
  if (softmax) {
    // a training forward keeps m | 1/Z per column for the backward; an inference forward writes none
    const bool train = model.mode == MD_MODE_TRAIN;
    if (train && !stats) {
      statsLd = round_up4(2 * H);
      stats = (float*)rt->dmalloc((size_t)std::max<int64_t>(model.local_rows(), 1) * (size_t)statsLd * sizeof(float));
    }
    const int x = inputs[0].region, y = outputs[0].region;
    const float* t = learnTemperature ? rt->data(temperature.region) : tConst;
    rt->sg_begin(H);
    ROC_CHECK(roc_sg_softmax_forward_planned(model.myGraph.plan, H, t, rt->data(x), rt->t(x).ld, rt->data(y),
                                             rt->t(y).ld, train ? stats : nullptr, statsLd, rt->stream));
    rt->sg_end();
    return;
  }
  if (dot) {
    // a training forward keeps m | 1/Z per head for the backward; an inference forward writes none
    const bool train = model.mode == MD_MODE_TRAIN;
    if (train && !stats) {
      statsLd = round_up4(2 * heads);
      stats = (float*)rt->dmalloc((size_t)std::max<int64_t>(model.local_rows(), 1) * (size_t)statsLd * sizeof(float));
    }
    const int q = inputs[0].region, k = inputs[1].region, v = inputs[2].region, y = outputs[0].region;
    rt->sg_begin(H);
    ROC_CHECK(roc_sg_attn_dot_forward_planned(model.myGraph.plan, heads, H, scale, rt->data(q), rt->t(q).ld,
                                              rt->data(k), rt->t(k).ld, rt->data(v), rt->t(v).ld, rt->data(y),
                                              rt->t(y).ld, train ? stats : nullptr, statsLd, rt->stream));
    rt->sg_end();
    return;
  }
  if (!stats) {
    statsLd = round_up4(2 * heads);
    stats = (float*)rt->dmalloc((size_t)std::max<int64_t>(model.local_rows(), 1) * (size_t)statsLd * sizeof(float));
  }
  if (dynamic) {
    const int xl = inputs[0].region, xr = inputs[1].region, y = outputs[0].region;
    rt->sg_begin(H);
    ROC_CHECK(roc_sg_attn_v2_forward_planned(model.myGraph.plan, heads, H, slope, rt->data(xl), rt->t(xl).ld,
                                             rt->data(xr), rt->t(xr).ld, rt->data(a.region), rt->data(y), rt->t(y).ld,
                                             stats, statsLd, rt->stream));
    rt->sg_end();
    return;
  }
  const int x = inputs[0].region, sc = inputs[1].region, y = outputs[0].region;
  const roc_sg_plan* plan = model.myGraph.plan;
  const roc_vid_t self = model.myGraph.rowLeft;
  const float rate = drop_rate(model);
  if (rate > 0.0f) keep_mask(model, plan, self, 0, keep);
  const uint8_t* k = rate > 0.0f ? keep : nullptr;
  rt->sg_begin(H);
  if (rt->t(x).isBf16)
    ROC_CHECK(roc_sg_attn_forward_dropout_planned_bf16(plan, heads, H, slope, self, rt->data_bf16(x), rt->t(x).ld,
                                                       rt->data(sc), rt->t(sc).ld, rt->data(y), rt->t(y).ld, stats,
                                                       statsLd, k, rate, rt->stream));
  else
    ROC_CHECK(roc_sg_attn_forward_dropout_planned(plan, heads, H, slope, self, rt->data(x), rt->t(x).ld, rt->data(sc),
                                                  rt->t(sc).ld, rt->data(y), rt->t(y).ld, stats, statsLd, k, rate,
                                                  rt->stream));
  rt->sg_end();
}

void AttentionGather::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  if (dynamic) {
    dynamic_backward(model);
    return;
  }
  if (softmax) {
    softmax_backward(model);
    return;
  }
  if (dot) {
    dot_backward(model);
    return;
  }
  if (!rt->t(inputs[0].region).requiresGrad && !rt->t(inputs[1].region).requiresGrad) return;
  const int H = (int)inputs[0].dims[0];
  // The kernel overwrites both gradients.  An input whose gradient another op already wrote (the features feed the
  // score Linear too) gets its part in scratch, added afterwards; so does one that needs no gradient.
  float* dst[2];
  for (int i = 0; i < 2; i++)
    dst[i] = grad_or_scratch(model, inputs[i].region, rt->t(inputs[i].region).requiresGrad && resetInputGrads[i], scratch[i]);
  const int ox = outputs[0].region, x = inputs[0].region, sc = inputs[1].region;
  const int64_t ldX = rt->t(x).ld, ldS = rt->t(sc).ld, ldO = rt->t(ox).ld;
  const bool xBf16 = rt->t(x).isBf16;
  const roc_sg_plan* plan = model.myGraph.plan;
  // the forward's mask, and the input-gradient pass's: the reverse pairs over the same plan, or the transposed plan's
  const float rate = drop_rate(model);
  if (rate > 0.0f) {
    const roc_sg_plan* planT = nullptr;
    if (model.exactBackward) ROC_CHECK(roc_sg_transpose_info(rt->sgTranspose, nullptr, nullptr, nullptr, &planT));
    keep_mask(model, model.exactBackward ? planT : plan, model.exactBackward ? 0 : model.myGraph.rowLeft, 1, keep2);
  }
  const uint8_t* k1 = rate > 0.0f ? keep : nullptr;
  const uint8_t* k2 = rate > 0.0f ? keep2 : nullptr;
  rt->sg_begin(H);
  if (model.exactBackward && xBf16)
    ROC_CHECK(roc_sg_attn_backward_dropout_exact_bf16(plan, rt->sgTranspose, heads, H, slope, rt->data_bf16(x), ldX,
                                                      rt->data(sc), ldS, rt->data(ox), ldO, stats, statsLd,
                                                      rt->grad(ox), ldO, dst[0], ldX, dst[1], ldS, k1, k2, rate,
                                                      rt->stream));
  else if (model.exactBackward)
    ROC_CHECK(roc_sg_attn_backward_dropout_exact(plan, rt->sgTranspose, heads, H, slope, rt->data(x), ldX,
                                                 rt->data(sc), ldS, rt->data(ox), ldO, stats, statsLd, rt->grad(ox),
                                                 ldO, dst[0], ldX, dst[1], ldS, k1, k2, rate, rt->stream));
  else if (xBf16)
    ROC_CHECK(roc_sg_attn_backward_dropout_planned_bf16(plan, heads, H, slope, model.myGraph.rowLeft,
                                                        rt->data_bf16(x), ldX, rt->data(sc), ldS, rt->data(ox), ldO,
                                                        stats, statsLd, rt->grad(ox), ldO, dst[0], ldX, dst[1], ldS,
                                                        k1, k2, rate, rt->stream));
  else
    ROC_CHECK(roc_sg_attn_backward_dropout_planned(plan, heads, H, slope, model.myGraph.rowLeft, rt->data(x), ldX,
                                                   rt->data(sc), ldS, rt->data(ox), ldO, stats, statsLd, rt->grad(ox),
                                                   ldO, dst[0], ldX, dst[1], ldS, k1, k2, rate, rt->stream));
  rt->sg_end();
  for (int i = 0; i < 2; i++)
    if (rt->t(inputs[i].region).requiresGrad && !resetInputGrads[i]) add_scratch(model, inputs[i].region, scratch[i]);
}

// dxl, dxr and da (overwritten) from the same CSR, or over the transpose with the exact backward.  The kernels overwrite
// both input gradients; an input whose gradient another op already wrote (or xr when it is xl) takes its part through
// scratch, added afterwards.
void AttentionGather::dynamic_backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int H = (int)inputs[0].dims[0];
  const int xl = inputs[0].region, xr = inputs[1].region, y = outputs[0].region;
  float* dst[2];
  for (int i = 0; i < 2; i++)
    dst[i] = grad_or_scratch(model, inputs[i].region, rt->t(inputs[i].region).requiresGrad && resetInputGrads[i], scratch[i]);
  const int64_t ld0 = rt->t(xl).ld, ld1 = rt->t(xr).ld, ldY = rt->t(y).ld;
  rt->sg_begin(H);
  if (model.exactBackward)
    ROC_CHECK(roc_sg_attn_v2_backward_exact(model.myGraph.plan, rt->sgTranspose, heads, H, slope, rt->data(xl), ld0,
                                            rt->data(xr), ld1, rt->data(a.region), rt->data(y), ldY, stats, statsLd,
                                            rt->grad(y), ldY, dst[0], ld0, dst[1], ld1, rt->grad(a.region), rt->stream));
  else
    ROC_CHECK(roc_sg_attn_v2_backward_planned(model.myGraph.plan, heads, H, slope, rt->data(xl), ld0, rt->data(xr), ld1,
                                              rt->data(a.region), rt->data(y), ldY, stats, statsLd, rt->grad(y), ldY,
                                              dst[0], ld0, dst[1], ld1, rt->grad(a.region), rt->stream));
  rt->sg_end();
  for (int i = 0; i < 2; i++)
    if (rt->t(inputs[i].region).requiresGrad && !resetInputGrads[i]) add_scratch(model, inputs[i].region, scratch[i]);
}

// dx (and, with a learned t, dt into t's gradient) from the same CSR, or over the transpose with the exact backward.  The
// kernels overwrite dx: when another op wrote x's gradient first (or x needs none) it goes through scratch, added
// afterwards only in the first case.
void AttentionGather::softmax_backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int x = inputs[0].region, y = outputs[0].region;
  const bool wantDx = rt->t(x).requiresGrad;
  if (!wantDx && !learnTemperature) return;
  const int H = (int)inputs[0].dims[0];
  float* dx = grad_or_scratch(model, x, wantDx && resetInputGrads[0], scratch[0]);
  const float* t = learnTemperature ? rt->data(temperature.region) : tConst;
  float* dt = learnTemperature ? rt->grad(temperature.region) : nullptr;
  const int64_t ldX = rt->t(x).ld, ldY = rt->t(y).ld;
  rt->sg_begin(H);
  if (model.exactBackward)
    ROC_CHECK(roc_sg_softmax_backward_exact(model.myGraph.plan, rt->sgTranspose, H, t, rt->data(x), ldX, rt->data(y),
                                            ldY, stats, statsLd, rt->grad(y), ldY, dx, ldX, dt, rt->stream));
  else
    ROC_CHECK(roc_sg_softmax_backward_planned(model.myGraph.plan, H, t, rt->data(x), ldX, rt->data(y), ldY, stats,
                                              statsLd, rt->grad(y), ldY, dx, ldX, dt, rt->stream));
  rt->sg_end();
  if (wantDx && !resetInputGrads[0]) add_scratch(model, x, scratch[0]);
}

// dq, dk and dv from the same CSR, or over the transpose with the exact backward.  The kernels overwrite all three: an
// input whose gradient another op already wrote (or a repeat of an earlier input) takes its part through scratch,
// added afterwards; so does one that needs no gradient.
void AttentionGather::dot_backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  bool any = false;
  for (int i = 0; i < 3; i++) any = any || rt->t(inputs[i].region).requiresGrad;
  if (!any) return;
  const int H = (int)inputs[0].dims[0];
  const int q = inputs[0].region, k = inputs[1].region, v = inputs[2].region, y = outputs[0].region;
  float* dst[3];
  for (int i = 0; i < 3; i++)
    dst[i] = grad_or_scratch(model, inputs[i].region, rt->t(inputs[i].region).requiresGrad && resetInputGrads[i], scratch[i]);
  const int64_t ldQ = rt->t(q).ld, ldK = rt->t(k).ld, ldV = rt->t(v).ld, ldY = rt->t(y).ld;
  rt->sg_begin(H);
  if (model.exactBackward)
    ROC_CHECK(roc_sg_attn_dot_backward_exact(model.myGraph.plan, rt->sgTranspose, heads, H, scale, rt->data(q), ldQ,
                                             rt->data(k), ldK, rt->data(v), ldV, rt->data(y), ldY, stats, statsLd,
                                             rt->grad(y), ldY, dst[0], ldQ, dst[1], ldK, dst[2], ldV, rt->stream));
  else
    ROC_CHECK(roc_sg_attn_dot_backward_planned(model.myGraph.plan, heads, H, scale, rt->data(q), ldQ, rt->data(k), ldK,
                                               rt->data(v), ldV, rt->data(y), ldY, stats, statsLd, rt->grad(y), ldY,
                                               dst[0], ldQ, dst[1], ldK, dst[2], ldV, rt->stream));
  rt->sg_end();
  for (int i = 0; i < 3; i++)
    if (rt->t(inputs[i].region).requiresGrad && !resetInputGrads[i]) add_scratch(model, inputs[i].region, scratch[i]);
}

// ------------------------------------------------------- AttentionScores -----
AttentionScores::AttentionScores(const Model& model, const Tensor& _input, int _heads)
    : GnnOp(_input), heads(_heads), workspace(nullptr), workspaceBytes(0) {
  ROC_ASSERT(_input.type == Tensor::NODE_TENSOR && _input.numDim == 2 && _input.dims[1] == model.myGraph.numNodes);
  const int64_t H = (int64_t)_input.dims[0];
  if (_heads <= 0 || H % _heads) ROC_FATAL("attention_scores: the input width must be heads * F with heads >= 1");
  if (H > 1024) ROC_FATAL("attention_scores: the input width must be at most 1024");
  a = model.create_weight_tensor((int)(H / _heads), 2 * _heads, NULL);   // a Linear F -> 2 * heads's GlorotUniform
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>(2 * _heads);
}
void AttentionScores::init(const Model& model) {
  workspaceBytes = roc_attn_scores_workspace_bytes(model.local_rows(), (int)inputs[0].dims[0], heads);
  workspace = model.ctx->dmalloc(std::max<size_t>(workspaceBytes, 16));
}
void AttentionScores::forward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int x = inputs[0].region, s = outputs[0].region, H = (int)inputs[0].dims[0];
  if (rt->t(x).isBf16)   // set_bf16_aggregation: GAT's wh
    ROC_CHECK(roc_attn_scores_fwd_bf16(model.local_rows(), H, heads, rt->data_bf16(x), rt->t(x).ld, rt->data(a.region),
                                       rt->data(s), rt->t(s).ld, rt->stream));
  else
    ROC_CHECK(roc_attn_scores_fwd(model.local_rows(), H, heads, rt->data(x), rt->t(x).ld, rt->data(a.region),
                                  rt->data(s), rt->t(s).ld, rt->stream));
}
// dA is overwritten; dX is written by the first op to run backward on the input (resetInputGrads) and added to in the
// others (in GAT the attention_gather has written it)
void AttentionScores::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int x = inputs[0].region, s = outputs[0].region, H = (int)inputs[0].dims[0];
  float* dX = rt->t(x).requiresGrad ? rt->grad(x) : nullptr;
  const int acc = resetInputGrads[0] ? 0 : 1;
  if (rt->t(x).isBf16)
    ROC_CHECK(roc_attn_scores_bwd_bf16(model.local_rows(), H, heads, rt->data_bf16(x), rt->t(x).ld, rt->data(a.region),
                                       rt->grad(s), rt->t(s).ld, dX, rt->t(x).ld, acc, rt->grad(a.region), workspace,
                                       workspaceBytes, rt->stream));
  else
    ROC_CHECK(roc_attn_scores_bwd(model.local_rows(), H, heads, rt->data(x), rt->t(x).ld, rt->data(a.region),
                                  rt->grad(s), rt->t(s).ld, dX, rt->t(x).ld, acc, rt->grad(a.region), workspace,
                                  workspaceBytes, rt->stream));
}

// ------------------------------------------------- WeightedScatterGather -----
WeightedScatterGather::WeightedScatterGather(const Model& model, const Tensor& _input, const Tensor& _edges)
    : GnnOp(_input, _edges), scratch(nullptr) {
  ROC_ASSERT(_input.type == Tensor::NODE_TENSOR && _input.numDim == 2 && _input.dims[1] == model.myGraph.numNodes);
  if (_edges.type != Tensor::EDGE_TENSOR || _edges.dims[0] != 1)
    ROC_FATAL("scatter_gather: the weights must be an edge tensor with one value per edge");
  trainableInputs[1] = false;
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)_input.dims[0]);
}
void WeightedScatterGather::init(const Model&) {}

void WeightedScatterGather::forward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int H = (int)inputs[0].dims[0];
  const int x = inputs[0].region, y = outputs[0].region;
  rt->sg_begin(H);
  if (rt->t(x).isBf16)
    ROC_CHECK(roc_sg_weighted_forward_planned_bf16(model.myGraph.plan, H, rt->data_bf16(x), rt->t(x).ld,
                                                   rt->data(inputs[1].region), rt->data(y), rt->t(y).ld, rt->stream));
  else
    ROC_CHECK(roc_sg_weighted_forward_planned(model.myGraph.plan, H, rt->data(x), rt->t(x).ld,
                                              rt->data(inputs[1].region), rt->data(y), rt->t(y).ld, rt->stream));
  rt->sg_end();
}

// dX by the weighted sum over the transpose, then (opt-in) the edge gradient.  Both overwrite in the first op to run
// backward on their input (resetInputGrads) and add in the others.
void WeightedScatterGather::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int H = (int)inputs[0].dims[0];
  const int x = inputs[0].region, e = inputs[1].region, y = outputs[0].region;
  const bool wantX = rt->t(x).requiresGrad, wantE = rt->t(e).requiresGrad;
  if (!rt->t(y).requiresGrad) {
    if (wantE) ROC_FATAL("set_edge_grad: call it before init() when the weighted scatter_gather's input has no gradient");
    return;
  }
  const int64_t ldY = rt->t(y).ld, ldX = rt->t(x).ld;
  rt->sg_begin(H);
  if (wantX) {
    float* dst = grad_or_scratch(model, x, resetInputGrads[0], scratch);
    ROC_CHECK(roc_sg_weighted_backward_planned(rt->sgTranspose, H, rt->grad(y), ldY, rt->data(e), dst, ldX, rt->stream));
    if (!resetInputGrads[0]) add_scratch(model, x, scratch);
  }
  if (wantE && rt->t(x).isBf16)
    ROC_CHECK(roc_sg_edge_dot_planned_bf16(model.myGraph.plan, H, rt->grad(y), ldY, rt->data_bf16(x), ldX, rt->grad(e),
                                           resetInputGrads[1] ? 0 : 1, rt->stream));
  else if (wantE)
    ROC_CHECK(roc_sg_edge_dot_planned(model.myGraph.plan, H, rt->grad(y), ldY, rt->data(x), ldX, rt->grad(e),
                                      resetInputGrads[1] ? 0 : 1, rt->stream));
  rt->sg_end();
}

// --------------------------------------------------------- InDegreeNorm -----
InDegreeNorm::InDegreeNorm(const Model& model, const Tensor& _input)
    : GnnOp(_input), reluOut(-1), bwdFused(false), sharesWithScaledAdd(false), scratch(nullptr) {
  ROC_ASSERT(inputs[0].type == Tensor::NODE_TENSOR);   // graphnorm.cc:33-35
  ROC_ASSERT(inputs[0].numDim == 2);
  ROC_ASSERT(inputs[0].dims[1] == model.myGraph.numNodes);
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)inputs[0].dims[0]);
}
void InDegreeNorm::init(const Model&) {}

void InDegreeNorm::forward(const Model& model) {
  if (fusedInto >= 0) return;   // done in the producer's epilogue
  RuntimeImpl* rt = model.ctx;
  const Graph& g = model.myGraph;
  ROC_CHECK(roc_indegree_norm(g.rowLeft, g.rowRight, g.colLeft, (int)inputs[0].dims[0], g.d_rowEnd,
                              rt->data(inputs[0].region), rt->t(inputs[0].region).ld, rt->data(outputs[0].region),
                              rt->t(outputs[0].region).ld, NULL, rt->stream));
}

// The kernel overwrites the input gradient, so an input whose gradient another op's backward already wrote is refused
// (graphnorm_kernel.cu:133, quirk Q7), unless a scaled_add also reads it (sharesWithScaledAdd: APPNP's MLP output,
// which every hop's scaled_add reads): that one gets its part in scratch, added afterwards.
void InDegreeNorm::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  ROC_ASSERT(resetInputGrads[0] || sharesWithScaledAdd);   // graphnorm_kernel.cu:133
  if (!rt->t(inputs[0].region).requiresGrad) return;
  // fused into the linear's epilogue forward => the SG backward epilogue already
  // produced d(linear out); nothing to do here
  if (fusedInto >= 0 && dynamic_cast<Linear*>(model.layers[(size_t)fusedInto])) { ROC_ASSERT(resetInputGrads[0]); return; }
  if (bwdFused) { ROC_ASSERT(resetInputGrads[0]); return; }   // a Linear's dX epilogue / the softmax already wrote this gradient
  const Graph& g = model.myGraph;
  const int src = reluOut >= 0 ? reluOut : outputs[0].region, in = inputs[0].region;
  float* dst = grad_or_scratch(model, in, resetInputGrads[0], scratch);
  ROC_CHECK(roc_indegree_norm(g.rowLeft, g.rowRight, g.colLeft, (int)inputs[0].dims[0], g.d_rowEnd, rt->grad(src),
                              rt->t(src).ld, dst, rt->t(in).ld, reluOut >= 0 ? rt->data(reluOut) : NULL, rt->stream));
  if (!resetInputGrads[0]) add_scratch(model, in, scratch);
}

// ----------------------------------------------------------------- Linear ---
Linear::Linear(const Model& model, const Tensor& _input, int outDim, ActiMode _activation, Initializer* initializer)
    : GnnOp(_input), activation(_activation), flags(0), fwdOut(-1), dropOp(-1), dropMask(nullptr), dropLd(0),
      dxReluOf(-1), dxNorm(false), dxOut(-1) {
  ROC_ASSERT(_input.numDim == 2);   // linear.cc:41-42
  ROC_ASSERT(_input.dims[1] == model.myGraph.numNodes);
  weight = model.create_weight_tensor((int)_input.dims[0], outDim, initializer);
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>(outDim);
}
void Linear::init(const Model& model) {
  if (dropOp < 0) return;
  RuntimeImpl* rt = model.ctx;
  dropLd = (((int64_t)weight.dims[0] + 31) / 32 + 3) / 4 * 4;
  dropMask = (uint32_t*)rt->dmalloc((size_t)std::max<int64_t>(model.local_rows(), 1) * (size_t)dropLd * sizeof(uint32_t));
}

namespace {
// a Dropout's rate in the current mode (infer: dropout is a copy, dropout_kernel.cu:159-180) and its Philox key
struct DropDraw { float rate; uint64_t key; };
DropDraw drop_draw(const Model& model, const Dropout& d) {
  return {model.mode == MD_MODE_TRAIN ? d.rate : 0.0f, ((uint64_t)(uint32_t)d.seed << 32) | (uint32_t)d.opIndex};
}
}  // namespace

void Linear::forward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const Graph& g = model.myGraph;
  const int outRegion = fwdOut >= 0 ? fwdOut : outputs[0].region;
  // If a ScatterGather on other GPUs reads this output (peer-mapped halo slabs), the rows are computed in blocks
  // and block k's boundary rows travel while block k + 1 is computed; otherwise one block = all rows.
  PushPipe pipe(model, outRegion, /*grad=*/false);
  const int inDim = (int)weight.dims[0], outDim = (int)weight.dims[1];
  const int64_t ldY = rt->t(outRegion).ld;
  // a bf16 Y (set_bf16_aggregation) holds bits: rows of ldY elements, stored by the kernels under ROC_LINEAR_Y_BF16
  const bool yBf16 = rt->t(outRegion).isBf16;
  float* Y = yBf16 ? reinterpret_cast<float*>(rt->data_bf16(outRegion)) : rt->data(outRegion);
  auto yRow = [&](int64_t r0) {
    return yBf16 ? reinterpret_cast<float*>(rt->data_bf16(outRegion) + r0 * ldY) : Y + r0 * ldY;
  };
  const int flags = this->flags | (yBf16 ? ROC_LINEAR_Y_BF16 : 0);
  int xRegion = inputs[0].region;
  float rate = 0.0f;
  if (dropOp >= 0) {
    // dropout -> linear: the mask is generated packed (1 bit / element) and applied while the GEMM
    // loads X, so the dropped copy of X is never materialised
    const Dropout* d = static_cast<const Dropout*>(model.layers[(size_t)dropOp]);
    const DropDraw f = drop_draw(model, *d);
    if (f.rate > 0.0f)
      ROC_CHECK(roc_dropout_mask(model.local_rows(), inDim, g.rowLeft, f.rate, f.key, rt->trainStep,
                                 dropMask, dropLd, rt->stream));
    xRegion = d->inputs[0].region;
    rate = f.rate;
  }
  const int64_t ldX = rt->t(xRegion).ld;
  // a bf16 X (a leaf) is read directly by the GEMM
  const bool xBf16 = rt->t(xRegion).isBf16;
  for (size_t k = 0; k < pipe.blocks(); k++) {
    const int64_t r0 = pipe.row0(k), nr = pipe.rows(k, model.local_rows());
    const uint32_t* mask = rate > 0.0f ? dropMask + r0 * dropLd : NULL;
    if (xBf16)
      ROC_CHECK(roc_linear_fwd_bf16(nr, inDim, outDim, rt->data_bf16(xRegion) + r0 * ldX, ldX, rt->data(weight.region),
                                    yRow(r0), ldY, (int)activation, flags, g.d_rowEnd + r0, pipe.colLeft(k), mask,
                                    dropLd, rate, rt->stream));
    else
      ROC_CHECK(roc_linear_fwd_dropout(nr, inDim, outDim, rt->data(xRegion) + r0 * ldX, ldX, rt->data(weight.region),
                                       yRow(r0), ldY, (int)activation, flags, g.d_rowEnd + r0, pipe.colLeft(k), mask,
                                       dropLd, rate, rt->stream));
    pipe.pushed(k, Y, ldY, outDim);
  }
}

void Linear::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const Graph& g = model.myGraph;
  roc_linear_bwd_args a;
  memset(&a, 0, sizeof(a));
  int xRegion = inputs[0].region;
  a.accumulate_dX = resetInputGrads[0] ? 0 : 1;
  if (dropOp >= 0) {
    // dW from the masked X; dX lands directly in the gradient of the dropout's input (the dropout
    // backward, dropout_kernel.cu:149-150, runs in the dX epilogue; it always overwrites, :119)
    const Dropout* d = static_cast<const Dropout*>(model.layers[(size_t)dropOp]);
    ROC_ASSERT(resetInputGrads[0]);
    xRegion = d->inputs[0].region;
    a.accumulate_dX = 0;
    a.dropMask = dropMask; a.ldMask = dropLd; a.dropRate = drop_draw(model, *d).rate;
  }
  // a bf16 X: dW by the bf16 kernel (with the relu backward of dY when activation is RELU), the same bits as the fp32
  // path on the widened X; only one an op produced (set_bf16_aggregation) has a gradient
  const bool xBf16 = rt->t(xRegion).isBf16;
  const int dxRegion = dxOut >= 0 ? dxOut : xRegion;
  a.rows = model.local_rows(); a.inDim = (int)weight.dims[0]; a.outDim = (int)weight.dims[1];
  a.X = xBf16 ? NULL : rt->data(xRegion); a.ldX = rt->t(xRegion).ld;
  a.W = rt->data(weight.region);
  a.Y = (activation != AC_MODE_NONE) ? rt->data(outputs[0].region) : NULL; a.ldY = rt->t(outputs[0].region).ld;
  a.dY = rt->grad(outputs[0].region); a.ldDY = rt->t(outputs[0].region).ld;
  a.dW = rt->grad(weight.region);
  a.dX = rt->t(xRegion).requiresGrad ? rt->grad(dxRegion) : NULL;   // Q8: leaf grads skipped
  a.ldDX = rt->t(dxRegion).ld;
  a.activation = (int)activation;
  a.workspace = rt->linWs; a.workspaceBytes = rt->linWsBytes;
  if (xBf16) {
    ROC_CHECK(roc_linear_dw_bf16(a.rows, a.inDim, a.outDim, rt->data_bf16(xRegion), a.ldX, a.Y, a.ldY, a.dY, a.ldDY,
                                 a.dW, a.activation, a.workspace, a.workspaceBytes, a.dropMask, a.ldMask, a.dropRate,
                                 rt->stream));
    if (!a.dX) return;
  }
  if (a.dX && dxReluOf >= 0) { a.dxReluOf = rt->data(dxReluOf); a.ldReluOf = rt->t(dxReluOf).ld; }
  if (a.dX && dxNorm) { a.dxNormRowEnd = g.d_rowEnd; a.colLeft = g.colLeft; }
  if (xBf16) {
    // dX by the fp32 kernel, which never reads X (the bf16 rows stand in for it in the argument check) and takes dY
    // as the dW call left it, relu-masked in place; one partition, so no pipelined row blocks
    a.parts = ROC_LINEAR_BWD_ONLY_DX;
    a.activation = AC_MODE_NONE;
    a.X = reinterpret_cast<const float*>(rt->data_bf16(xRegion));
    ROC_CHECK(roc_linear_bwd_fused(&a, rt->stream));
    return;
  }
  // dX feeds a ScatterGather backward on other GPUs (peer-mapped slabs): dX in row blocks, each pushed while the
  // next is computed, then dW — which nothing downstream waits for — while the last rows travel.
  PushPipe pipe(model, (a.dX && activation == AC_MODE_NONE) ? dxRegion : -1, /*grad=*/true);
  if (pipe.on) {
    for (size_t k = 0; k < pipe.blocks(); k++) {
      const int64_t r0 = pipe.row0(k), nr = pipe.rows(k, model.local_rows());
      roc_linear_bwd_args b = a;
      b.parts = ROC_LINEAR_BWD_ONLY_DX;
      b.rows = nr;
      b.X = a.X + r0 * a.ldX;
      b.dY = a.dY + r0 * a.ldDY;
      b.dX = a.dX + r0 * a.ldDX;
      if (a.dropMask) b.dropMask = a.dropMask + r0 * a.ldMask;
      if (a.dxReluOf) b.dxReluOf = a.dxReluOf + r0 * a.ldReluOf;
      if (a.dxNormRowEnd) { b.dxNormRowEnd = a.dxNormRowEnd + r0; b.colLeft = pipe.colLeft(k); }
      ROC_CHECK(roc_linear_bwd_fused(&b, rt->stream));
      pipe.pushed(k, a.dX, a.ldDX, a.inDim);
    }
    a.parts = ROC_LINEAR_BWD_ONLY_DW;
  }
  ROC_CHECK(roc_linear_bwd_fused(&a, rt->stream));
}

// ------------------------------------------------------------- Activation ---
Activation::Activation(const Model& model, const Tensor& _input, ActiMode _actiMode)
    : GnnOp(_input), actiMode(_actiMode) {
  ROC_ASSERT(_input.numDim == 2);
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)_input.dims[0]);
}
void Activation::init(const Model&) {}
void Activation::forward(const Model& model) {
  if (fusedInto >= 0) return;
  RuntimeImpl* rt = model.ctx;
  const int x = inputs[0].region, y = outputs[0].region;
  if (rt->t(y).isBf16)   // set_bf16_aggregation: a relu output that an aggregation reads
    ROC_CHECK(roc_activation_fwd_y_bf16(model.local_rows(), (int)inputs[0].dims[0], (int)actiMode, rt->data(x),
                                        rt->t(x).ld, rt->data_bf16(y), rt->t(y).ld, rt->stream));
  else
    ROC_CHECK(roc_activation_fwd(model.local_rows(), (int)inputs[0].dims[0], (int)actiMode, rt->data(x), rt->t(x).ld,
                                 rt->data(y), rt->t(y).ld, rt->stream));
}
void Activation::backward(const Model& model) {
  if (fusedInto >= 0) return;   // mask applied by the fused indegree_norm backward
  RuntimeImpl* rt = model.ctx;
  if (!rt->t(inputs[0].region).requiresGrad) return;
  const int x = inputs[0].region, y = outputs[0].region;
  const int rows = model.local_rows(), H = (int)inputs[0].dims[0], acc = resetInputGrads[0] ? 0 : 1;
  if (rt->t(y).isBf16)   // the mask of the stored bf16 y
    ROC_CHECK(roc_activation_bwd_y_bf16(rows, H, (int)actiMode, rt->data_bf16(y), rt->t(y).ld, rt->grad(y), rt->t(y).ld,
                                        rt->grad(x), rt->t(x).ld, acc, rt->stream));
  else
    ROC_CHECK(roc_activation_bwd(rows, H, (int)actiMode, rt->data(y), rt->t(y).ld, rt->grad(y), rt->t(y).ld,
                                 rt->grad(x), rt->t(x).ld, acc, rt->stream));
}

// -------------------------------------------------------------- BatchNorm ---
BatchNorm::BatchNorm(const Model& model, const Tensor& _input, float _momentum, float _eps)
    : GnnOp(_input), momentum(_momentum), eps(_eps), fwdOut(-1), workspace(nullptr), workspaceBytes(0) {
  ROC_ASSERT(_input.type == Tensor::NODE_TENSOR && _input.numDim == 2 && _input.dims[1] == model.myGraph.numNodes);
  if (!(_momentum >= 0.0f && _momentum <= 1.0f)) ROC_FATAL("batch_norm: the momentum must be in [0, 1]");
  if (!(_eps >= 0.0f) || !std::isfinite(_eps)) ROC_FATAL("batch_norm: eps must be finite and >= 0");
  RuntimeImpl* rt = model.ctx;
  const int H = (int)_input.dims[0];
  // constant fills only: the Linears' GlorotUniform draws do not move
  ZerosInitializer zeros;
  gamma = model.create_weight_tensor(H, 1, &zeros);
  beta = model.create_weight_tensor(H, 1, &zeros);
  ROC_CHECK(roc_fill(1, H, 1.0f, rt->data(gamma.region), H, rt->stream));
  float* f = (float*)rt->dmalloc((size_t)4 * H * sizeof(float));
  runMean = f; runVar = f + H; saveA = f + 2 * H; saveB = f + 3 * H;
  ROC_CHECK(roc_fill(1, H, 0.0f, runMean, H, rt->stream));
  ROC_CHECK(roc_fill(1, H, 1.0f, runVar, H, rt->stream));
  saveMean = (double*)rt->dmalloc((size_t)2 * H * sizeof(double));
  saveInvStd = saveMean + H;
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>(H);
}
void BatchNorm::init(const Model& model) {
  const int64_t rows = model.local_rows();
  if (rows < 2) ROC_FATAL("batch_norm: the partition has fewer than 2 rows (no batch variance)");
  workspaceBytes = roc_batchnorm_workspace_bytes(rows, (int)inputs[0].dims[0]);
  workspace = model.ctx->dmalloc(workspaceBytes);
}
void BatchNorm::forward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int x = inputs[0].region, y = fwdOut >= 0 ? fwdOut : outputs[0].region;
  ROC_CHECK(roc_batchnorm_fwd(model.local_rows(), (int)inputs[0].dims[0], rt->data(x), rt->t(x).ld,
                              rt->data(gamma.region), rt->data(beta.region), eps, momentum, runMean, runVar,
                              model.mode == MD_MODE_TRAIN, fwdOut >= 0, rt->data(y), rt->t(y).ld, saveA, saveB, saveMean,
                              saveInvStd, workspace, workspaceBytes, rt->stream));
}
void BatchNorm::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int x = inputs[0].region, y = fwdOut >= 0 ? fwdOut : outputs[0].region;
  float* dX = rt->t(x).requiresGrad ? rt->grad(x) : nullptr;
  ROC_CHECK(roc_batchnorm_bwd(model.local_rows(), (int)inputs[0].dims[0], rt->data(x), rt->t(x).ld, rt->grad(y),
                              rt->t(y).ld, fwdOut >= 0, rt->data(gamma.region), saveA, saveB, saveMean, saveInvStd,
                              rt->grad(gamma.region), rt->grad(beta.region), dX, rt->t(x).ld, resetInputGrads[0] ? 0 : 1,
                              workspace, workspaceBytes, rt->stream));
}

// -------------------------------------------------------------- LayerNorm ---
LayerNorm::LayerNorm(const Model& model, const Tensor& _input, float _eps)
    : GnnOp(_input), eps(_eps), fwdOut(-1), workspace(nullptr), workspaceBytes(0) {
  ROC_ASSERT(_input.type == Tensor::NODE_TENSOR && _input.numDim == 2 && _input.dims[1] == model.myGraph.numNodes);
  if (!(_eps >= 0.0f) || !std::isfinite(_eps)) ROC_FATAL("layer_norm: eps must be finite and >= 0");
  RuntimeImpl* rt = model.ctx;
  const int H = (int)_input.dims[0];
  // constant fills only: the Linears' GlorotUniform draws do not move
  ZerosInitializer zeros;
  gamma = model.create_weight_tensor(H, 1, &zeros);
  beta = model.create_weight_tensor(H, 1, &zeros);
  ROC_CHECK(roc_fill(1, H, 1.0f, rt->data(gamma.region), H, rt->stream));
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>(H);
}
void LayerNorm::init(const Model& model) {
  workspaceBytes = roc_layernorm_workspace_bytes(model.local_rows(), (int)inputs[0].dims[0]);
  workspace = model.ctx->dmalloc(workspaceBytes);
}
void LayerNorm::forward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int x = inputs[0].region, y = fwdOut >= 0 ? fwdOut : outputs[0].region;
  ROC_CHECK(roc_layernorm_fwd(model.local_rows(), (int)inputs[0].dims[0], rt->data(x), rt->t(x).ld,
                              rt->data(gamma.region), rt->data(beta.region), eps, fwdOut >= 0, rt->data(y),
                              rt->t(y).ld, rt->stream));
}
void LayerNorm::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int x = inputs[0].region, y = fwdOut >= 0 ? fwdOut : outputs[0].region;
  float* dX = rt->t(x).requiresGrad ? rt->grad(x) : nullptr;
  ROC_CHECK(roc_layernorm_bwd(model.local_rows(), (int)inputs[0].dims[0], rt->data(x), rt->t(x).ld, rt->grad(y),
                              rt->t(y).ld, fwdOut >= 0, rt->data(gamma.region), rt->data(beta.region), eps,
                              rt->grad(gamma.region), rt->grad(beta.region), dX, rt->t(x).ld,
                              resetInputGrads[0] ? 0 : 1, workspace, workspaceBytes, rt->stream));
}

// ---------------------------------------------------------------- Element ---
Element::Element(const Model& model, const Tensor& input0, const Tensor& input1, ElementType _elementType)
    : GnnOp(input0, input1), elementType(_elementType) {
  ROC_ASSERT(input0.numDim == input1.numDim);   // element.cc:33-36
  for (int i = 0; i < input0.numDim; i++) ROC_ASSERT(input0.dims[i] == input1.dims[i]);
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)input0.dims[0]);
}
void Element::init(const Model&) {}
void Element::forward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  ROC_ASSERT(elementType == EW_TYPE_ADD);
  ROC_CHECK(roc_add_fwd(model.local_rows(), (int)inputs[0].dims[0], rt->data(inputs[0].region),
                        rt->t(inputs[0].region).ld, rt->data(inputs[1].region), rt->t(inputs[1].region).ld,
                        rt->data(outputs[0].region), rt->t(outputs[0].region).ld, rt->stream));
}
void Element::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  ROC_ASSERT(elementType == EW_TYPE_ADD);   // element_kernel.cu:102-104
  float* dA = rt->t(inputs[0].region).requiresGrad ? rt->grad(inputs[0].region) : NULL;
  float* dB = rt->t(inputs[1].region).requiresGrad ? rt->grad(inputs[1].region) : NULL;
  ROC_CHECK(roc_add_bwd(model.local_rows(), (int)inputs[0].dims[0], rt->grad(outputs[0].region),
                        rt->t(outputs[0].region).ld, dA, rt->t(inputs[0].region).ld, resetInputGrads[0] ? 0 : 1, dB,
                        rt->t(inputs[1].region).ld, resetInputGrads[1] ? 0 : 1, rt->stream));
}

// -------------------------------------------------------------- ScaledAdd ---
ScaledAdd::ScaledAdd(const Model& model, const Tensor& a, const Tensor& b, float _alpha, float _beta)
    : GnnOp(a, b), alpha(_alpha), beta(_beta) {
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)a.dims[0]);
}
void ScaledAdd::init(const Model&) {}
void ScaledAdd::forward(const Model& model) {
  if (fusedInto >= 0) return;   // applied by the scatter_gather's store
  RuntimeImpl* rt = model.ctx;
  const int a = inputs[0].region, b = inputs[1].region, y = outputs[0].region;
  ROC_CHECK(roc_scaled_add_fwd(model.local_rows(), (int)inputs[0].dims[0], alpha, rt->data(a), rt->t(a).ld, beta,
                               rt->data(b), rt->t(b).ld, rt->data(y), rt->t(y).ld, rt->stream));
}
void ScaledAdd::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  const int a = inputs[0].region, b = inputs[1].region, y = outputs[0].region;
  float* dA = rt->t(a).requiresGrad ? rt->grad(a) : NULL;
  float* dB = rt->t(b).requiresGrad ? rt->grad(b) : NULL;
  ROC_CHECK(roc_scaled_add_bwd(model.local_rows(), (int)inputs[0].dims[0], rt->grad(y), rt->t(y).ld, alpha, dA,
                               rt->t(a).ld, resetInputGrads[0] ? 0 : 1, beta, dB, rt->t(b).ld,
                               resetInputGrads[1] ? 0 : 1, rt->stream));
}

// ---------------------------------------------------------------- Dropout ---
Dropout::Dropout(const Model& model, const Tensor& _input, float _rate, int _seed)
    : GnnOp(_input), rate(_rate), seed(_seed), opIndex(0), sharesWithScaledAdd(false), scratch(nullptr) {
  ROC_ASSERT(_input.numDim == 2);
  ROC_ASSERT(_input.type == Tensor::NODE_TENSOR);
  numOutputs = 1;
  outputs[0] = model.create_node_tensor<DATATYPE>((int)_input.dims[0]);
}
void Dropout::init(const Model&) {}
void Dropout::forward(const Model& model) {
  if (fusedInto >= 0) return;   // applied by the consuming Linear while it loads X
  RuntimeImpl* rt = model.ctx;
  // train: masked scale (dropout_kernel.cu:98-99); infer: plain copy (:159-180)
  const DropDraw d = drop_draw(model, *this);
  if (rt->t(inputs[0].region).isBf16) {   // bf16 in, fp32 out; rate 0 is the widening copy
    ROC_CHECK(roc_dropout_fwd_bf16(model.local_rows(), (int)inputs[0].dims[0], model.myGraph.rowLeft, d.rate, d.key,
                                   rt->trainStep, rt->data_bf16(inputs[0].region), rt->t(inputs[0].region).ld,
                                   rt->data(outputs[0].region), rt->t(outputs[0].region).ld, rt->stream));
    return;
  }
  ROC_CHECK(roc_dropout_fwd(model.local_rows(), (int)inputs[0].dims[0], model.myGraph.rowLeft, d.rate, d.key,
                            rt->trainStep, rt->data(inputs[0].region), rt->t(inputs[0].region).ld,
                            rt->data(outputs[0].region), rt->t(outputs[0].region).ld, rt->stream));
}
void Dropout::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  if (!rt->t(inputs[0].region).requiresGrad) return;   // leaf input (Q8)
  ROC_ASSERT(resetInputGrads[0] || (sharesWithScaledAdd && fusedInto < 0));   // dropout_kernel.cu:119
  if (fusedInto >= 0) return;       // the consuming Linear's dX epilogue already wrote this gradient
  // the kernel overwrites the input gradient; one another op already wrote (only where a scaled_add also reads the
  // input: GCNII's x0) gets its part in scratch, added afterwards
  const int in = inputs[0].region;
  float* dst = grad_or_scratch(model, in, resetInputGrads[0], scratch);
  const DropDraw d = drop_draw(model, *this);
  ROC_CHECK(roc_dropout_bwd(model.local_rows(), (int)inputs[0].dims[0], model.myGraph.rowLeft, d.rate, d.key,
                            rt->trainStep, rt->grad(outputs[0].region), rt->t(outputs[0].region).ld, dst,
                            rt->t(in).ld, rt->stream));
  if (!resetInputGrads[0]) add_scratch(model, in, scratch);
}

// The [INFER] line of softmax_kernel.cu:141-152 (printed once per partition, quirk Q20), to stderr AND stdout, as the
// reference does (scripts scrape either).  With the multi-label metrics a second line gives each split's micro-F1.
static void print_infer(int epoch, const roc_perf_metrics& p, const roc_multilabel_metrics* ml) {
  FILE* sinks[2] = {stderr, stdout};
  for (FILE* f : sinks) {
    fprintf(f,
            "\t[INFER][%d] train_loss: %.4lf  train_accuracy: %.2lf%%(%d/%d)  val_accuracy: %.2lf%%(%d/%d)  "
            "test_accuracy: %.2lf%%(%d/%d)\n",
            epoch, p.trainLoss, p.trainCorrect * 100.0f / p.trainAll, p.trainCorrect, p.trainAll,
            p.valCorrect * 100.0f / p.valAll, p.valCorrect, p.valAll, p.testCorrect * 100.0f / p.testAll,
            p.testCorrect, p.testAll);
    if (ml) {
      double f1[3];
      for (int s = 0; s < 3; s++) {
        const double d = 2.0 * (double)ml->tp[s] + (double)ml->fp[s] + (double)ml->fn[s];
        f1[s] = d > 0 ? 2.0 * (double)ml->tp[s] / d : NAN;
      }
      fprintf(f, "\t[INFER][%d] train_micro_f1: %.4lf  val_micro_f1: %.4lf  test_micro_f1: %.4lf\n", epoch, f1[0],
              f1[1], f1[2]);
    }
  }
  fflush(stdout);
}

// ---------------------------------------------------- SoftmaxCrossEntropy ---
SoftmaxCrossEntropy::SoftmaxCrossEntropy(const Model&, const Tensor& _logit, const Tensor& _label, const Tensor& _mask)
    : GnnOp(_logit, _label, _mask), epoch_num(0), gradOut(-1) {
  ROC_ASSERT(_logit.numDim == 2);   // softmax.cc:36-39
  ROC_ASSERT(_label.numDim == 2);
  ROC_ASSERT(_label.dims[0] == _logit.dims[0]);
  ROC_ASSERT(_label.dims[1] == _logit.dims[1]);
  numOutputs = 0;
}
void SoftmaxCrossEntropy::init(const Model&) {}
void SoftmaxCrossEntropy::forward(const Model& model) {
  mode = model.mode;
  if (model.mode == MD_MODE_TRAIN) {
    // Do nothing in training forward (softmax.cc:48-49)
  } else {
    backward(model);   // softmax.cc:50-54: inference reuses the backward task for metrics
  }
}
void SoftmaxCrossEntropy::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  mode = model.mode;
  if (mode == MD_MODE_TRAIN) epoch_num++;
  ROC_ASSERT(inputs[2].region >= 0);   // softmax_kernel.cu:157-160: masks are required
  const int C = (int)inputs[0].dims[0];
  TensorImpl& lab = rt->t(inputs[1].region);
  if (lab.labelBits)
    ROC_FATAL("softmax_cross_entropy: the label tensor holds multi-labels (set_multilabels); the softmax takes one "
              "class per row (set_labels / set_tensor)");
  rt->lossKind = ROC_HOST_OP_SOFTMAX_CROSS_ENTROPY;
  ROC_CHECK(cudaMemsetAsync(rt->d_perf, 0, sizeof(roc_perf_metrics), rt->stream));
  const int32_t* mask = reinterpret_cast<const int32_t*>(rt->data(inputs[2].region));
  if (gradOut >= 0) {
    // the logits come from an InDegreeNorm: its backward (grad / sqrt(deg)) is applied here and the
    // result goes straight into the gradient the ScatterGather backward reads
    const Graph& g = model.myGraph;
    PushPipe pipe(model, mode == MD_MODE_TRAIN ? gradOut : -1, /*grad=*/true);
    const float* Z = rt->data(inputs[0].region);
    const int64_t ldZ = rt->t(inputs[0].region).ld;
    const float* L = lab.labelIdx ? NULL : rt->data(inputs[1].region);
    const int64_t ldL = lab.labelIdx ? 0 : lab.ld;
    float* G = rt->grad(gradOut);
    const int64_t ldG = rt->t(gradOut).ld;
    for (size_t k = 0; k < pipe.blocks(); k++) {
      const int64_t r0 = pipe.row0(k), nr = pipe.rows(k, model.local_rows());
      ROC_CHECK(roc_softmax_xent_bwd_norm(nr, C, Z + r0 * ldZ, ldZ, L ? L + r0 * ldL : NULL, ldL,
                                          lab.labelIdx ? lab.labelIdx + r0 : NULL, mask + r0, G + r0 * ldG, ldG,
                                          g.d_rowEnd + r0, pipe.colLeft(k), rt->d_perf, rt->stream));
      pipe.pushed(k, G, ldG, C);
    }
  } else if (lab.labelIdx) {
    ROC_CHECK(roc_softmax_xent_bwd_idx(model.local_rows(), C, rt->data(inputs[0].region), rt->t(inputs[0].region).ld,
                                       lab.labelIdx, mask, rt->grad(inputs[0].region), rt->t(inputs[0].region).ld,
                                       rt->d_perf, rt->stream));
  } else {
    ROC_CHECK(roc_softmax_xent_bwd(model.local_rows(), C, rt->data(inputs[0].region), rt->t(inputs[0].region).ld,
                                   rt->data(inputs[1].region), lab.ld, mask, rt->grad(inputs[0].region),
                                   rt->t(inputs[0].region).ld, rt->d_perf, rt->stream));
  }
  if (mode == MD_MODE_INFER && model.printMetrics) print_infer(epoch_num, model.last_metrics(), nullptr);
}

// ---------------------------------------------------- SigmoidCrossEntropy ---
SigmoidCrossEntropy::SigmoidCrossEntropy(const Model&, const Tensor& _logit, const Tensor& _label, const Tensor& _mask)
    : GnnOp(_logit, _label, _mask), epoch_num(0), gradOut(-1) {
  ROC_ASSERT(_logit.numDim == 2);
  ROC_ASSERT(_label.numDim == 2);
  if (_label.dims[0] != _logit.dims[0])
    ROC_FATAL("sigmoid_cross_entropy: the label tensor's width (classes) differs from the logits'");
  ROC_ASSERT(_label.dims[1] == _logit.dims[1]);
  numOutputs = 0;
}
void SigmoidCrossEntropy::init(const Model&) {}
void SigmoidCrossEntropy::forward(const Model& model) {
  mode = model.mode;
  if (model.mode == MD_MODE_INFER) backward(model);   // as the softmax: nothing in training, metrics in inference
}
void SigmoidCrossEntropy::backward(const Model& model) {
  RuntimeImpl* rt = model.ctx;
  mode = model.mode;
  if (mode == MD_MODE_TRAIN) epoch_num++;
  ROC_ASSERT(inputs[2].region >= 0);   // masks are required
  const int C = (int)inputs[0].dims[0];
  const TensorImpl& lab = rt->t(inputs[1].region);
  if (!lab.labelBits)
    ROC_FATAL("sigmoid_cross_entropy: the label tensor has no multi-labels (set them with set_multilabels)");
  rt->lossKind = ROC_HOST_OP_SIGMOID_CROSS_ENTROPY;
  ROC_CHECK(cudaMemsetAsync(rt->d_multilabel, 0, sizeof(roc_multilabel_metrics), rt->stream));
  // one partition: the fused norm backward divides by the in-degree of the whole CSR (rowEnd from colLeft)
  const int rg = gradOut >= 0 ? gradOut : inputs[0].region;
  ROC_CHECK(roc_sigmoid_xent_bwd(model.local_rows(), C, rt->data(inputs[0].region), rt->t(inputs[0].region).ld,
                                 lab.labelBits, (C + 31) / 32, reinterpret_cast<const int32_t*>(rt->data(inputs[2].region)),
                                 rt->grad(rg), rt->t(rg).ld, gradOut >= 0 ? model.myGraph.d_rowEnd : NULL,
                                 model.myGraph.colLeft, rt->d_multilabel, rt->stream));
  rt->multilabelRan = true;
  if (mode == MD_MODE_INFER && model.printMetrics) {
    roc_multilabel_metrics ml;
    model.last_multilabel_metrics(&ml);
    print_infer(epoch_num, model.last_metrics(), &ml);
  }
}

// ----------------------------------------------------------- initializers ---
// initializer.cc:31-46 + initializer_kernel.cu:22-51: cuRAND's default XORWOW
// generator seeded with the next std::rand(), uniform (0,1] over the weight's
// linear memory order, then W = 2*s*u - s.  cuRAND is called at init only, so
// the weights match the reference bit for bit for a given -seed.
void GlorotUniform::init(const Model* model, const Tensor* p) {
  RuntimeImpl* rt = model->ctx;
  ROC_ASSERT(p->numDim == 2);
  int num = std::rand();
  const int inputDim = (int)p->dims[0], outputDim = (int)p->dims[1];
  const size_t vol = (size_t)inputDim * outputDim;
  float scale = sqrt(6.0 / (inputDim + outputDim));
  curandGenerator_t gen;
  ROC_CHECK(curandCreateGenerator(&gen, CURAND_RNG_PSEUDO_DEFAULT));
  ROC_CHECK(curandSetStream(gen, rt->stream));
  ROC_CHECK(curandSetPseudoRandomGeneratorSeed(gen, (unsigned long long)num));
  float* w = rt->data(p->region);
  ROC_CHECK(curandGenerateUniform(gen, w, vol));
  ROC_CHECK(roc_scale((int64_t)vol, -scale, scale, w, rt->stream));
  ROC_CHECK(cudaStreamSynchronize(rt->stream));
  curandDestroyGenerator(gen);
}

void ZerosInitializer::init(const Model* model, const Tensor* p) {
  RuntimeImpl* rt = model->ctx;
  ROC_ASSERT(p->numDim == 2);
  TensorImpl& x = rt->t(p->region);
  ROC_CHECK(roc_fill(x.rows, x.H, 0.0f, rt->data(p->region), x.ld, rt->stream));
}

// -------------------------------------------------------------- optimizer ---
// optimizer.cc:22-70: m and v per parameter, zero-initialised; must be built
// after every linear() call (it walks model->parameters).
AdamOptimizer::AdamOptimizer(const Model* _model, double _alpha, double _beta1, double _beta2, double _weight_decay,
                             double _epsilon)
    : Optimizer(_model), alpha(_alpha), beta1(_beta1), beta2(_beta2), weight_decay(_weight_decay),
      epsilon(_epsilon), alpha_t(_alpha), beta1_t(1.0f), beta2_t(1.0f) {
  RuntimeImpl* rt = _model->ctx;
  ZerosInitializer zeros;
  for (size_t i = 0; i < model->parameters.size(); i++) {
    const Tensor& p = model->parameters[i];
    Tensor t = p;
    t.region = rt->new_tensor((int64_t)p.dims[1], (int)p.dims[0], (int64_t)p.dims[0], false, true);
    v_regions[p.region] = t.region;
    zeros.init(_model, &t);
    t.region = rt->new_tensor((int64_t)p.dims[1], (int)p.dims[0], (int64_t)p.dims[0], false, true);
    m_regions[p.region] = t.region;
    zeros.init(_model, &t);
  }
}

void AdamOptimizer::set_weight_decay(double _weight_decay) { weight_decay = _weight_decay; }

// optimizer.cc:79-85
void AdamOptimizer::next(void) {
  beta1_t *= beta1;
  beta2_t *= beta2;
  alpha_t = alpha * sqrt(1 - beta2_t) / (1 - beta1_t);
}

// optimizer.cc:87-119 + optimizer_kernel.cu:66-103 (the gradient was already summed
// over partitions by Model::update's all-reduce)
void AdamOptimizer::update(const Tensor* p) {
  RuntimeImpl* rt = model->ctx;
  ROC_ASSERT(v_regions.find(p->region) != v_regions.end());
  ROC_ASSERT(m_regions.find(p->region) != m_regions.end());
  const int64_t count = (int64_t)p->dims[0] * (int64_t)p->dims[1];
  ROC_CHECK(roc_adam_update(count, (float)alpha_t, (float)beta1, (float)beta2, (float)weight_decay, (float)epsilon,
                            rt->grad(p->region), rt->data(m_regions[p->region]), rt->data(v_regions[p->region]),
                            rt->data(p->region), rt->stream));
}

// ------------------------------------------------------------------- CLI ----
// Same flags as gnn.cc:114-179, including "-dr" being taken by dropout before
// decay-rate can see it (quirk Q19).
void parse_input_args(char** argv, int argc, Config& config) {
  for (int i = 1; i < argc; i++) {
    const std::string a(argv[i]);
    const bool more = i + 1 < argc;
    if (a == "-seed" && more) config.seed = atoi(argv[++i]);
    else if ((a == "-ng" || a == "-ll:gpu") && more) config.numGPUs = atoi(argv[++i]);
    else if ((a == "-e" || a == "-epoch") && more) config.numEpochs = atoi(argv[++i]);
    else if (a == "-lr" && more) config.learning_rate = atof(argv[++i]);
    else if ((a == "-dropout" || a == "-dr") && more) config.dropout_rate = atof(argv[++i]);
    else if ((a == "-decay" || a == "-wd") && more) config.weight_decay = atof(argv[++i]);
    else if (a == "-decay-rate" && more) config.decay_rate = atof(argv[++i]);
    else if ((a == "-decay-step" || a == "-ds") && more) config.decay_steps = atoi(argv[++i]);
    else if (a == "-file" && more) config.filename = std::string(argv[++i]);
    else if (a == "-verbose" || a == "-v") config.verbose = true;
    else if (a == "-layers" && more) {
      std::stringstream ss((std::string(argv[++i])));
      std::string word;
      config.layers.clear();
      while (std::getline(ss, word, '-')) config.layers.push_back(std::stoi(word));
    }
  }
}
