/*
 * roc_gnn.h — the Model / op-builder surface of ROC's gnn.h (gnn.h:105-222,
 * optimizer.h:25-50, initializer.h) over a thin C++ host: one process per GPU,
 * CUDA streams, HBM-resident tensors, NCCL for the two exchange steps.  The
 * Legion runtime, GnnMapper, TensorAccessor staging and ResourceManager are
 * gone; `Context` / `Runtime` remain as plain handles so the reference's model
 * script (gnn.cc:65-111) compiles against this header unchanged:
 *
 *     Graph graph(ctx, runtime, config);
 *     Model model(graph, ctx, runtime);
 *     Tensor input = model.create_node_tensor<DATATYPE>(config.layers[0]);
 *     ... model.dropout / linear / indegree_norm / scatter_gather / relu / add ...
 *     model.softmax_cross_entropy(t, label, mask);
 *     AdamOptimizer* optimizer = new AdamOptimizer(&model, config.learning_rate);
 *     optimizer->set_weight_decay(config.weight_decay);
 *     model.optimizer = optimizer;  model.init(config);
 *     loop: optimizer->alpha *= decay;  train_mode; zero_gradients; forward; backward; update
 *
 * Names, argument meaning, enum values and error behaviour (assert / exit(1))
 * follow the reference; every class cites the reference definition it mirrors.
 * The device work is done by the C-ABI kernel layer in roc_b200.h.
 */
#ifndef ROC_GNN_H_
#define ROC_GNN_H_

#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "roc_b200.h"

typedef uint32_t V_ID;   /* types.h:5 */
typedef uint64_t E_ID;   /* types.h:6 */
typedef float DATATYPE;  /* types.h:7 */

#define MAX_FILE_LEN 64        /* gnn.h:27 (kept for parity; paths are not truncated here) */
#define MAX_NUM_PARTS 64       /* gnn.h:28 */
#define MAX_NUM_INPUTS 8       /* gnn.h:30 */
#define MAX_NUM_OUTPUTS 8      /* gnn.h:31 */
#define MAX_NUM_DIM 4          /* gnn.h:32 */
#define FILE_HEADER_SIZE (sizeof(E_ID) + sizeof(V_ID)) /* gnn.h:33 */

enum AggrType { AGGR_AVG, AGGR_MAX, AGGR_MIN, AGGR_SUM };            /* gnn.h:75-80 */
enum ActiMode { AC_MODE_NONE, AC_MODE_RELU, AC_MODE_SIGMOID, AC_MODE_ELU };   /* gnn.h:82-86, + ELU */
enum ElementType { EW_TYPE_ADD, EW_TYPE_MUL };                         /* gnn.h:88-91 */
enum ModelMode { MD_MODE_TRAIN, MD_MODE_INFER };                       /* gnn.h:93-96 */
enum MaskType { MASK_TRAIN, MASK_VAL, MASK_TEST, MASK_NONE };          /* gnn.h:98-103 */

namespace roc { namespace host { struct RuntimeImpl; struct TensorImpl; struct Comm; } }

/* Stand-ins for Legion's handles.  A Runtime owns the process's GPU, stream,
 * device allocations and (for numParts > 1) the NCCL communicator. */
typedef roc::host::RuntimeImpl* Context;

class Runtime {
public:
  /* device: CUDA ordinal for this process; myPart / numParts: which vertex-range
   * partition this process owns (one process per GPU). */
  explicit Runtime(int device = 0, int myPart = 0, int numParts = 1);
  ~Runtime();
  Context context() const { return impl; }
  /* NCCL bootstrap (only place NCCL appears): rank 0 creates the id, the
   * launcher broadcasts the 128 bytes, every rank calls init_nccl. */
  static bool nccl_unique_id(unsigned char id[128]);
  bool init_nccl(const unsigned char id[128]);
  void synchronize();
  roc::host::RuntimeImpl* impl;
private:
  Runtime(const Runtime&);
  Runtime& operator=(const Runtime&);
};

struct Config {  /* gnn.h:105-113 */
  int numGPUs, numMachines, totalGPUs, numEpochs, decay_steps, seed;
  bool verbose;
  float learning_rate, weight_decay, dropout_rate;
  float decay_rate;
  std::string filename;
  std::vector<int> layers;
  Config();
};

struct Graph {  /* gnn.h:120-130; ctor = gnn.cc:751-872 (reads <file>.add_self_edge.lux) */
  Graph(Context _ctx, Runtime* _runtime, const Config& config);
  /* Same partitioning / device CSR from arrays already in host memory
   * (host_rowEnd: N global END offsets; host_colSrc: all E sources). */
  Graph(Context _ctx, Runtime* _runtime, V_ID numNodes, E_ID numEdges,
        const E_ID* host_rowEnd, const V_ID* host_colSrc);
  V_ID numNodes;
  E_ID numEdges;
  int numParts, numMachines;
  int maxHidden;
  /* this process's partition (the rects of rowPtrLP / colIdxLP for its colour) */
  int myPart;
  V_ID rowLeft, rowRight;
  E_ID colLeft, colRight;
  std::vector<V_ID> vbounds;   /* [numParts][2] */
  std::vector<E_ID> ebounds;   /* [numParts][2] */
  /* device CSR (replaces rowPtrLR / colIdxLR): END offsets + lean sources */
  E_ID* d_rowEnd;
  V_ID* d_colSrc;
  roc_sg_plan* plan;
  /* numParts > 1: halo exchange structures (derived and private; see roc_halo_* in roc_b200.h).
   * The plan is then built on the remapped col ([own rows | halo rows]); d_colSrc stays canonical. */
  roc_halo* halo;
  V_ID numHalo;
  std::vector<size_t> recvCounts, recvOffs, sendCounts, sendOffs;   /* rows, per peer partition */
  V_ID* d_sendRows;      /* local rows other partitions read, grouped by requester */
  size_t numSendRows;
  /* Peer-write exchange (roc_push_rows): the same send list sorted by source row, each entry with the partition
   * that reads it and its row in that partition's [own | halo] slab; cut into row blocks so that a producer
   * (Linear, softmax) can push block k while it computes block k + 1. */
  V_ID* d_pushRows;
  unsigned char* d_pushPeer;
  V_ID* d_pushDst;
  std::vector<V_ID> pushBlockRow;       /* [blocks + 1] first local row of each block */
  std::vector<size_t> pushBlockOff;     /* [blocks + 1] offsets into the sorted send list */
  std::vector<E_ID> pushBlockColLeft;   /* [blocks] global END offset of the row before the block */
  /* Copy-engine exchange: block k's entries of the requester-grouped send list (d_packSel[packBlockOff[k] ..]),
   * and, per requester q, where block k starts inside q's contiguous run (packPeerOff[q * (blocks + 1) + k]). */
  V_ID* d_packSel;
  std::vector<size_t> packBlockOff;
  std::vector<size_t> packPeerOff;
  std::vector<V_ID> peerSlab0;          /* [parts] first row of this partition's rows in partition q's [own | halo] slab */
private:
  void build(Context ctx, const E_ID* host_rowEnd, const V_ID* slice_colSrc);
};

struct Tensor {  /* gnn.h:132-158 */
  enum Type { NODE_TENSOR = 1, EDGE_TENSOR = 2, GRAPH_TENSOR = 3, WEIGHT_TENSOR = 4, INVALID_TENSOR = 9 };
  Tensor(void) : type(INVALID_TENSOR), numDim(0), region(-1) { dims[0] = dims[1] = dims[2] = dims[3] = 0; }
  Tensor(Type _type) : type(_type), numDim(0), region(-1) { dims[0] = dims[1] = dims[2] = dims[3] = 0; }
  Type type;
  int numDim;
  E_ID dims[MAX_NUM_DIM];   /* dims[0] = hidden width, dims[1] = numNodes (node tensors); [in][out] (weights) */
  int region;               /* handle into the Runtime's tensor table (replaces LogicalRegion) */
};

class Model;
class GnnOp;

class Initializer {  /* initializer.h */
public:
  Initializer(void) {}
  virtual ~Initializer(void) {}
  virtual void init(const Model* model, const Tensor* tensor) = 0;
};
class GlorotUniform : public Initializer {  /* initializer.cc:31-46, initializer_kernel.cu:22-51 */
public:
  void init(const Model* model, const Tensor* tensor);
};
class ZerosInitializer : public Initializer {  /* initializer.cc:54-70 */
public:
  void init(const Model* model, const Tensor* tensor);
};

class Optimizer {  /* optimizer.h:25-32 */
public:
  Optimizer(const Model* _model) : model(_model) {}
  virtual ~Optimizer() {}
  virtual void next(void) = 0;
  virtual void update(const Tensor* p) = 0;
  const Model* model;
};

class AdamOptimizer : public Optimizer {  /* optimizer.h:34-50, optimizer.cc:22-119 */
public:
  AdamOptimizer(const Model* _model, double _alpha = 0.001f, double _beta1 = 0.9f,
                double _beta2 = 0.999f, double _weight_decay = 0.0f, double _epsilon = 1e-8);
  void next(void);
  void update(const Tensor* p);
  void set_weight_decay(double _weight_decay);
  double alpha, beta1, beta2, weight_decay, epsilon;
  double alpha_t, beta1_t, beta2_t;
  std::map<int, int> v_regions, m_regions;   /* weight region -> moment buffers */
};

class Model {  /* gnn.h:162-203 */
public:
  Model(const Graph& _graph, Context _ctx, Runtime* _runtime);
  Tensor add(const Tensor& _input1, const Tensor& _input2);
  Tensor dropout(const Tensor& _input, float rate, int seed = 0);
  Tensor scatter_gather(const Tensor& _input);
  /* With an aggregator (not in gnn.h, which declares AggrType but only sums).  AGGR_SUM is the one-argument form.
   * AGGR_AVG appends scatter_gather -> indegree_norm -> indegree_norm (x / sqrt(deg) / sqrt(deg): the mean to within
   * one fp32 rounding, the wiring of GraphSAGE-mean).  AGGR_MAX / AGGR_MIN: per feature, the max / min over the
   * in-neighbours (roc_sg_minmax_forward_planned); the backward sends each output gradient to the first source that
   * held the extreme.  That is the true gradient only on a symmetric graph without duplicate edges: init() refuses
   * a graph whose rows do not have strictly increasing sources.  Single partition only (exit(1) otherwise). */
  Tensor scatter_gather(const Tensor& _input, AggrType aggr);
  /* Edge dropout (not in gnn.h): the sum aggregation with each in-edge dropped at rate `dropout` in train mode and a
   * kept one scaled by 1 / (1 - dropout) (roc_sg_forward_dropout_planned), the APPNP paper's dropout of the propagation
   * matrix and PyG APPNP(dropout=).  keep(i<-j) is drawn per step from Philox keyed by the pair (i <- j) with key
   * (seed << 32) | the op's position and the model's train step, as Model::dropout draws its own, so every such op
   * draws its own mask each step.  Degrees stay the full graph's (the epilogue fusions with indegree_norm and the
   * teleport fusion apply as to the plain sum): dropout on the normalised adjacency entries, not DropEdge's
   * renormalisation on the sampled graph.  The backward is the dropped sum over the output gradient with the reverse
   * pairs' decisions (quirk Q1: exact on a symmetric graph), or with set_exact_backward the dropped transposed sum
   * (roc_sg_transpose_sum_backward_dropout).  Infer mode and dropout = 0 run the plain sum.  The input stays fp32 under
   * set_bf16_aggregation.  Exits for an aggregator other than AGGR_SUM with dropout > 0, a rate outside [0, 1), or more
   * than one partition. */
  Tensor scatter_gather(const Tensor& _input, AggrType aggr, float dropout, int seed = 0);
  /* Attention aggregation (GAT; roc_sg_attn_forward_planned): `scores` has 2 * heads columns, [s_dst | s_src] per
   * head; the output has the input's width, each head's block of H / heads columns weighted by that head's
   * softmax over the row's in-edges.  Its backward is a gather over the same CSR (quirk Q1): exact for the
   * destination scores, the true gradient of the rest on a symmetric graph.  Never fused with neighbouring ops.
   * Single partition only (exit(1) otherwise).  dropout > 0: attention dropout at that rate in train mode
   * (roc_sg_attn_forward_dropout_planned), each step's keep mask drawn from Philox with key (seed << 32) | the op's
   * position and the model's train step, as Model::dropout draws its own; infer mode and dropout = 0 run the plain
   * calls.  A rate outside [0, 1) exits. */
  Tensor attention_gather(const Tensor& input, const Tensor& scores, int heads, float negativeSlope = 0.2f,
                          float dropout = 0.0f, int seed = 0);
  /* GATv2's dynamic attention (roc_sg_attn_v2_forward_planned): per destination v and head k over v's in-edges u,
   *   e[v,u,k] = sum_f a[k][f] * LeakyReLU(xl[u][kF+f] + xr[v][kF+f]),  p = softmax_u(e),
   *   out[v][kF:(k+1)F] = sum_u p[v,u,k] * xl[u][kF:(k+1)F]
   * xl (the values) and xr (the targets) have H = heads * F columns, H <= 256, heads <= 8; they may be one tensor
   * (PyG's share_weights), whose gradient then takes both parts.  Appends one parameter `a` of parameter_shape
   * (heads, F), drawn by GlorotUniform (uniform in +-sqrt(6 / (heads + F)), PyG's glorot of GATv2Conv.att).  A mode of
   * attention_gather: op_info reports it as one.  Its backward runs over the same CSR (exact on a symmetric graph), or
   * over the transpose with set_exact_backward.  Never fused; set_bf16_aggregation leaves both inputs fp32.  Exits on
   * different widths, H % heads != 0, H > 256, heads > 8, bf16 inputs, a bad slope, or more than one partition. */
  Tensor dynamic_attention_gather(const Tensor& xl, const Tensor& xr, int heads, float negativeSlope = 0.2f);
  /* Softmax aggregation with one temperature t (roc_sg_softmax_forward_planned; PyG SoftmaxAggregation, GENConv's
   * default aggregator): per destination v and column f over v's in-edges u, p = softmax_u(t * x[u][f]) and
   * out[v][f] = sum_u p * x[u][f] (0 for a row with no in-edge).  t = 0 is the mean, a large t approaches the max.
   * learnTemperature: t is a parameter of parameter_shape (1, 1), appended here and filled with `temperature` (no
   * random draw, so the Linears' GlorotUniform draws do not move), trained by Adam with the model's weight decay;
   * otherwise t is a constant and the backward skips dt.  A mode of attention_gather: op_info reports it as one.  Its
   * backward runs over the same CSR (exact on a symmetric graph), or over the transpose with set_exact_backward; it adds
   * into its input's gradient when another op wrote it first.  Never fused; set_bf16_aggregation leaves its input fp32.
   * Exits on a temperature that is not finite, a bf16 input (at init()), or more than one partition. */
  Tensor softmax_gather(const Tensor& x, float temperature = 1.0f, bool learnTemperature = false);
  /* Dot-product attention (roc_sg_attn_dot_forward_planned; the graph transformer layer, PyG TransformerConv's
   * attention): per destination v and head k over v's in-edges u, s = scale * q[v]_k . k[u]_k, p = softmax_u(s) and
   * out[v]_k = sum_u p * v[u]_k (0 for a row with no in-edge).  q, k and v have H = heads * F columns, H <= 256,
   * heads <= 8, and any of them may be the same tensor (its gradient then takes every part).  scale is neither 0 nor
   * non-finite (PyG's 1 / sqrt(F) is the caller's: Model.dot_attention_gather computes it).  No parameter.  A mode of
   * attention_gather: op_info reports it as one.  Training forwards keep m | 1/Z per head; inference forwards write
   * none.  Its backward runs over the same CSR (exact on a symmetric graph), or over the transpose with
   * set_exact_backward; it adds into an input's gradient when another op wrote it first.  Never fused;
   * set_bf16_aggregation leaves q, k and v fp32.  Exits on unequal widths, H % heads != 0, H > 256, heads > 8, a bad
   * scale, bf16 inputs, or more than one partition. */
  Tensor dot_attention_gather(const Tensor& q, const Tensor& k, const Tensor& v, int heads, float scale);
  /* The per-head GAT scores of `input` (H = heads * F columns; roc_attn_scores_fwd / _bwd): a [rows][2 * heads] output
   * [s_dst | s_src], head k's scores the dot products of its own F columns with its a_dst and a_src.  Appends one
   * parameter A, a weight tensor of dims {F, 2 * heads} (row k: a_dst of head k, row heads + k: its a_src), drawn by the
   * GlorotUniform of a Linear F -> 2 * heads.  Reads a bf16 input only when set_bf16_aggregation made it so.  Exits
   * when H % heads != 0 or H > 1024.  Single partition only (exit(1) otherwise). */
  Tensor attention_scores(const Tensor& input, int heads);
  /* Edge-weighted aggregation (roc_sg_weighted_forward_planned): out[v] = sum over v's in-edges e of
   * edgeWeights[e] * input[src(e)].  edgeWeights is an edge tensor (create_edge_tensor).  Its backward is exact on any
   * graph: init() builds the graph's transpose once (roc_sg_transpose) the first time a model has such an op, and the
   * input gradient runs over it.  The edge tensor's gradient is computed only after set_edge_grad(edges, true).
   * Never fused with neighbouring ops.  Single partition only (exit(1) otherwise). */
  Tensor scatter_gather(const Tensor& input, const Tensor& edgeWeights);
  /* Opt-in gradient of an edge tensor (off by default, like the raw features').  When on, backward() leaves in its
   * gradient twin the sum, over every weighted scatter_gather that reads it, of sum_h outGrad[v][h] * input[src][h]
   * per edge (roc_sg_edge_dot_planned): the first op to run backward overwrites it and the others add, so the
   * previous step's value is never kept.  Call it before init() when the op's input needs no gradient of its own. */
  void set_edge_grad(const Tensor& edges, bool on);
  void softmax_cross_entropy(const Tensor& logits, const Tensor& labels, const Tensor& mask);
  /* Multi-label sigmoid cross-entropy (roc_sigmoid_xent_bwd): labels set by set_multilabels, one 0/1 label per class.
   * Like the softmax it does nothing in the training forward, and in infer mode its forward runs the kernel for the
   * metrics only.  Single partition only (exit(1) otherwise). */
  void sigmoid_cross_entropy(const Tensor& logits, const Tensor& labels, const Tensor& mask);
  Tensor indegree_norm(const Tensor& _input);
  Tensor linear(const Tensor& _input, int outDim, ActiMode activation, Initializer* initializer = NULL);
  Tensor relu(const Tensor& _input);
  Tensor sigmoid(const Tensor& _input);
  /* ELU with alpha = 1 (roc_activation_fwd with ROC_AC_MODE_ELU); never fused with another op.  A Linear cannot apply
   * it (linear() exits on AC_MODE_ELU).  Row-local like relu, so not refused on more than one partition, but untested
   * there. */
  Tensor elu(const Tensor& _input);
  /* Scaled add (roc_scaled_add_fwd / _bwd): fmaf(alpha, a, beta * b), the initial residual of APPNP and GCNII.  Exits
   * on unequal shapes, a non-finite alpha or beta, or a == b.  With fusion on and one partition, init() fuses it into
   * the store of a sum scatter_gather whose indegree_norm feeds only it, as its first input (fuse_teleport in model.cc).
   * Row-local like elu, so not refused on more than one partition, but untested there. */
  Tensor scaled_add(const Tensor& a, const Tensor& b, float alpha, float beta);
  /* Batch normalisation over every local row (torch.nn.BatchNorm1d; roc_batchnorm_fwd / roc_batchnorm_bwd).  Appends
   * two parameters, gamma (filled with 1) then beta (0), each a weight tensor of dims {H, 1}; creating them draws no
   * random numbers.  A training forward normalises by the batch statistics and updates the running mean (start 0) and
   * variance (start 1); an infer-mode forward uses the running statistics and updates nothing.  init() refuses a
   * partition of fewer than 2 rows.  Single partition only (exit(1) otherwise). */
  Tensor batch_norm(const Tensor& input, float momentum = 0.1f, float eps = 1e-5f);
  /* Layer normalisation over the columns of each local row (torch.nn.LayerNorm(H, eps); roc_layernorm_fwd /
   * roc_layernorm_bwd).  Appends two parameters, gamma (filled with 1) then beta (0), each a weight tensor of dims
   * {H, 1}, trained by the optimizer as batch_norm's are; creating them draws no random numbers.  The same forward runs
   * in train and infer mode (no running statistics), and any row count is accepted.  op_info reports it as a
   * batch_norm, the normalisation kind, and a relu that alone reads its output is fused into it as into a batch_norm.
   * Exits on a negative or non-finite eps.  Single partition only (exit(1) otherwise). */
  Tensor layer_norm(const Tensor& input, float eps = 1e-5f);
  /* DT = DATATYPE (fp32), int (masks), or __nv_bfloat16 (<cuda_bf16.h>): a leaf feature matrix stored in bf16, rounded
   * to nearest even, rows of round_up(H, 8) elements.  It never has a gradient and is never an op's output; linear and
   * dropout read it (bit-identical to the same model on an fp32 input holding the widened values), and init() refuses
   * any other op that reads it.  Untested at more than one partition. */
  template <typename DT> Tensor create_node_tensor(int _numHidden) const;
  /* gnn.h:178, gnn.cc:534-560: one value per edge of this partition, dims = {numHidden, numEdges}, stored as a dense
   * fp32 array in the CSR's edge order, with a gradient twin allocated on first use.  Only DT = float and
   * numHidden == 1 (exit(1) otherwise).  set_tensor / get_tensor move its local edge count of values. */
  template <typename DT> Tensor create_edge_tensor(int numHidden) const;
  Tensor create_weight_tensor(int _inDim, int _outDim, Initializer* initializer) const;
  void load_features(const Tensor& input, const std::string& filename);
  void load_labels(const Tensor& label, const std::string& filename);
  void load_train_mask(const Tensor& mask, const std::string& filename);
  bool init(const Config& config);
  void train_mode(void);
  void infer_mode(void);
  void forward(void);
  void backward(void);
  void update(void);
  void zero_gradients(void);

  /* ---- additions (not in gnn.h): host<->device access to this partition's rows ---- */
  /* Copy `rows_local x H` values between a dense host buffer and the tensor.  A bf16 tensor takes and returns fp32
   * rows (set: rounded to nearest even on the device; get: widened exactly); grad = true is an error on a bf16 leaf and
   * reaches the fp32 gradient of a bf16 tensor an op produces (set_bf16_aggregation). */
  void set_tensor(const Tensor& t, const void* host, bool grad = false);
  void get_tensor(const Tensor& t, void* host, bool grad = false) const;
  /* a bf16 tensor's raw bits, `rows_local x H` uint16 values, copied as they are */
  void set_tensor_bf16(const Tensor& t, const uint16_t* host);
  void get_tensor_bf16(const Tensor& t, uint16_t* host) const;
  /* labels as class indices (what load_labels parses, load_task.cu:118-123) */
  void set_labels(const Tensor& label, const int* host_class_idx);
  /* multi-labels for sigmoid_cross_entropy, bit-packed: ceil(H / 32) words per row (bit c % 32 of word c / 32 is
   * label c), rows dense.  Only these words travel; the tensor's fp32 data is not used. */
  void set_multilabels(const Tensor& label, const uint32_t* host_packed_bits);
  /* PerfMetrics of the latest loss pass (after a sigmoid cross-entropy: its loss[0], rows and exact matches) */
  roc_perf_metrics last_metrics(void) const;
  /* the multi-label metrics of the latest sigmoid cross-entropy pass; false before one has run */
  bool last_multilabel_metrics(roc_multilabel_metrics* out) const;
  void set_fusion(bool on) { fuse = on; }
  /* Opt-in exact backward (off by default) for the sum (and so AGGR_AVG), max / min and attention aggregations on
   * directed graphs: their input gradients run over the graph's transpose (roc_sg_transpose_sum_backward,
   * roc_sg_transpose_minmax_backward, roc_sg_attn_backward_exact) instead of the same CSR (quirk Q1, the true gradient
   * only on a symmetric graph).  init() then builds the transpose once, shared with the weighted ops, and max / min
   * accept graphs with duplicate edges.  Call it before init().  Single partition only (exit(1) otherwise). */
  void set_exact_backward(bool on);
  /* Opt-in bf16 aggregation inputs (off by default).  At init(), after fusion, a tensor is stored in bf16 when
   *  - a Linear with AC_MODE_NONE writes it in its forward (its own output, or the output of an indegree_norm fused
   *    into its epilogue) and one sum scatter_gather alone reads it; or
   *  - a Linear with AC_MODE_NONE or an unfused relu writes it, at least one max / min scatter_gather, weighted
   *    scatter_gather or attention_gather reads it as its feature input, and every other reader is one of those or a
   *    Linear reading it as X with no fused dropout (GAT's score Linear) or an attention_scores.
   * Its producer rounds the fp32 result to nearest even as it stores it (a relu's gradient then takes its mask from the
   * stored bf16 value), the aggregations read the rows at half width and compute in fp32, and a Linear reads them as a
   * bf16 X.  The gradient of such a tensor is an ordinary fp32 tensor; every other tensor stays fp32.  Call it before
   * init().  Single partition only (init() exits otherwise). */
  void set_bf16_aggregation(bool on);
  /* the source ids a max / min scatter_gather chose (its `arg`), [rows_local][H] u32; `out` is its output tensor */
  void get_aggr_index(const Tensor& out, uint32_t* host) const;
  /* the running mean and variance (fp32, H values each) of the batch_norm whose output is `out` */
  void get_batch_norm_stats(const Tensor& out, float* mean, float* var) const;
  void set_batch_norm_stats(const Tensor& out, const float* mean, const float* var);
  int64_t local_rows(void) const { return (int64_t)myGraph.rowRight - myGraph.rowLeft + 1; }

public:
  ModelMode mode;
  Graph myGraph;
  Context ctx;
  Runtime* runtime;
  Optimizer* optimizer;
  std::vector<Tensor> parameters;
  std::vector<GnnOp*> layers;
  int epoch_num;
  bool fuse;          /* fuse linear->norm and SG->norm->relu into kernel epilogues (default on) */
  bool printMetrics;  /* print the [INFER] accuracy line like softmax_kernel.cu:141-152 (default on) */
  bool exactBackward; /* set_exact_backward (default off) */
  bool bf16Aggregation; /* set_bf16_aggregation (default off) */
};

class GnnOp {  /* gnn.h:205-222 */
public:
  GnnOp(const Tensor& input);
  GnnOp(const Tensor& input1, const Tensor& input2);
  GnnOp(const Tensor& input1, const Tensor& input2, const Tensor& input3);
  virtual ~GnnOp() {}
  virtual void init(const Model& model) = 0;
  virtual void forward(const Model& model) = 0;
  virtual void backward(const Model& model) = 0;
public:
  int numInputs, numOutputs;
  ModelMode mode;
  Tensor inputs[MAX_NUM_INPUTS], outputs[MAX_NUM_OUTPUTS];
  bool trainableInputs[MAX_NUM_INPUTS];
  bool resetInputGrads[MAX_NUM_INPUTS];
  /* host-side scheduling state (not in gnn.h) */
  int fusedInto;    /* >= 0: this op's work is done by layers[fusedInto] */
};

class ScatterGather : public GnnOp {  /* gnn.h:225-242, scattergather.cc */
public:
  ScatterGather(const Model& model, const Tensor& input, AggrType aggr = AGGR_SUM);
  virtual void init(const Model& model);
  virtual void forward(const Model& model);
  virtual void backward(const Model& model);
  AggrType aggr;     /* AGGR_SUM, or AGGR_MAX / AGGR_MIN (never fused with neighbouring ops) */
  uint32_t* arg;     /* max / min: [Nloc][argLd] source id behind each output value (first forward; Runtime arena) */
  int64_t argLd;
  int epilogue;      /* ROC_SG_EPI_* the forward store applies (set by Model::init fusion) */
  int bwdEpilogue;   /* same for the backward launch */
  int fwdOut, bwdOut;/* region the fused forward / backward writes (-1: own output / input grad) */
  int teleT;         /* >= 0: a scaled_add fused into the store (roc_sg_forward_teleport_planned) reads this region as t */
  float teleAlpha, teleBeta;   /*   ... with these coefficients */
  float dropRate;    /* edge dropout of the sum in train mode (0: none; Model::scatter_gather(input, aggr, dropout, seed)) */
  int seed;
  int opIndex;       /* position in the model: the Philox key is (seed << 32) | opIndex, as a Dropout's */
private:
  float drop_rate(const Model& model) const;
  const uint8_t* keep_mask(const Model& model, const roc_sg_plan* plan, roc_vid_t selfBase, int rowIsSource) const;
};

class AttentionGather : public GnnOp {  /* not in the reference: Model::attention_gather */
public:
  AttentionGather(const Model& model, const Tensor& input, const Tensor& scores, int heads, float slope, float dropRate,
                  int seed);
  /* the dynamic (GATv2) mode: inputs xl, xr (Model::dynamic_attention_gather) */
  AttentionGather(const Model& model, const Tensor& xl, const Tensor& xr, int heads, float slope);
  /* the softmax aggregation mode: input x (Model::softmax_gather) */
  AttentionGather(const Model& model, const Tensor& x, float temperature, bool learnTemperature);
  /* the dot-product mode: inputs q, k, v (Model::dot_attention_gather) */
  AttentionGather(const Model& model, const Tensor& q, const Tensor& k, const Tensor& v, int heads, float scale);
  virtual void init(const Model& model);
  virtual void forward(const Model& model);
  virtual void backward(const Model& model);
  int heads;
  float slope;
  float dropRate;    /* attention dropout in train mode (0: none) */
  int seed;
  int opIndex;       /* position in the model: the Philox key is (seed << 32) | opIndex, as a Dropout's */
  uint8_t* keep;     /* [E] keep bytes of the last training forward, in the plan's edge order (Runtime arena) */
  uint8_t* keep2;    /* [E] the backward's input-gradient pass's: reverse pairs, or the transposed plan's order */
  float* stats;      /* [Nloc][statsLd] m | 1/Z per head of the last forward (Runtime arena) */
  int64_t statsLd;
  float* scratch[3]; /* gradients of an input that accumulates (or needs none), written here first (Runtime arena) */
  bool dynamic;      /* GATv2's dynamic attention: inputs[0] = xl, inputs[1] = xr, parameter a */
  Tensor a;          /* dynamic: parameter, dims {heads, F} (memory a[k][f] at f * heads + k) */
  bool softmax;      /* the softmax aggregation: inputs[0] = x, stats [Nloc][statsLd] m | 1/Z per column */
  bool learnTemperature;   /* softmax: t is the parameter `temperature` */
  Tensor temperature;      /* softmax with learnTemperature: parameter, dims {1, 1} */
  float* tConst;     /* softmax without it: t in one device float (Runtime arena) */
  bool dot;          /* dot-product attention: inputs[0] = q, inputs[1] = k, inputs[2] = v */
  float scale;       /* dot: the logits' scale */
private:
  float drop_rate(const Model& model) const;
  uint64_t drop_key() const;
  void keep_mask(const Model& model, const roc_sg_plan* plan, roc_vid_t selfBase, int rowIsSource, uint8_t*& buf);
  void dynamic_backward(const Model& model);
  void softmax_backward(const Model& model);
  void dot_backward(const Model& model);
};

class AttentionScores : public GnnOp {  /* not in the reference: Model::attention_scores */
public:
  AttentionScores(const Model& model, const Tensor& input, int heads);
  virtual void init(const Model& model);
  virtual void forward(const Model& model);
  virtual void backward(const Model& model);
  int heads;
  Tensor a;          /* parameter, dims {F, 2 * heads} */
  void* workspace;   /* roc_attn_scores_workspace_bytes (Runtime arena) */
  size_t workspaceBytes;
};

class WeightedScatterGather : public GnnOp {  /* not in the reference: Model::scatter_gather(input, edgeWeights) */
public:
  WeightedScatterGather(const Model& model, const Tensor& input, const Tensor& edgeWeights);
  virtual void init(const Model& model);
  virtual void forward(const Model& model);
  virtual void backward(const Model& model);
  float* scratch;    /* the input gradient when another op already wrote it (added afterwards; Runtime arena) */
};

class InDegreeNorm : public GnnOp {  /* gnn.h:244-261, graphnorm.cc */
public:
  InDegreeNorm(const Model& model, const Tensor& input);
  virtual void init(const Model& model);
  virtual void forward(const Model& model);
  virtual void backward(const Model& model);
  int reluOut;      /* a relu fused into the forward: its output region, whose grad the backward reads and whose
                       values' mask it applies (-1: none; the backward reads its own output's grad) */
  bool bwdFused;    /* backward done in another op's epilogue (a Linear's dX or the loss) */
  bool sharesWithScaledAdd;   /* a scaled_add also reads the input: the backward may add to its gradient (init) */
  float* scratch;   /* the input gradient when another op already wrote it (added afterwards; Runtime arena) */
};

class Linear : public GnnOp {  /* gnn.h:263-285, linear.cc */
public:
  Linear(const Model& model, const Tensor& input, int outDim, ActiMode _activaiton, Initializer* initializer);
  void init(const Model& model);
  void forward(const Model& model);
  void backward(const Model& model);
public:
  ActiMode activation;
  Tensor weight;
  int flags;        /* ROC_LINEAR_* (norm epilogue fused) */
  int fwdOut;       /* region the forward writes (-1: own output) */
  int dropOp;       /* >= 0: layers[dropOp] is the Dropout feeding this op, applied while X is loaded */
  uint32_t* dropMask;      /* packed keep-mask of that dropout, [rows][dropLd] (roc_dropout_mask) */
  int64_t dropLd;
  /* dX epilogue fusions: relu mask of region dxReluOf's values, then / sqrt(deg); dX goes to dxOut's grad */
  int dxReluOf;     /* -1: none */
  bool dxNorm;
  int dxOut;        /* -1: the input's own grad */
};

class Activation : public GnnOp {  /* gnn.h:287-302, activation.cc */
public:
  Activation(const Model& model, const Tensor& input, ActiMode _actiMode);
  void init(const Model& model);
  void forward(const Model& model);
  void backward(const Model& model);
public:
  ActiMode actiMode;
};

class Element : public GnnOp {  /* gnn.h:304-319, element.cc */
public:
  Element(const Model& model, const Tensor& input0, const Tensor& input1, ElementType _elementType);
  void init(const Model& model);
  void forward(const Model& model);
  void backward(const Model& model);
public:
  ElementType elementType;
};

class ScaledAdd : public GnnOp {  /* not in the reference: Model::scaled_add */
public:
  ScaledAdd(const Model& model, const Tensor& a, const Tensor& b, float alpha, float beta);
  void init(const Model& model);
  void forward(const Model& model);
  void backward(const Model& model);
public:
  float alpha, beta;
};

class Dropout : public GnnOp {  /* gnn.h:321-344, dropout.cc */
public:
  Dropout(const Model& model, const Tensor& input, float rate, int seed);
  virtual void init(const Model& model);
  virtual void forward(const Model& model);
  virtual void backward(const Model& model);
public:
  float rate;
  int seed;
  int opIndex;      /* position in the model: distinguishes the Philox streams of the layers */
  bool sharesWithScaledAdd;   /* a scaled_add also reads the input: the backward may add to its gradient (init) */
  float* scratch;   /* the input gradient when another op already wrote it (added afterwards; Runtime arena) */
};

class BatchNorm : public GnnOp {  /* not in the reference: Model::batch_norm */
public:
  BatchNorm(const Model& model, const Tensor& input, float momentum, float eps);
  virtual void init(const Model& model);
  virtual void forward(const Model& model);
  virtual void backward(const Model& model);
public:
  float momentum, eps;
  Tensor gamma, beta;   /* parameters, dims {H, 1} */
  int fwdOut;           /* a relu fused into the forward (Model::init): its output region, which the forward writes and
                           whose gradient the backward reads (-1: none) */
  /* Runtime arena, H values each: running statistics; a, b of the last training forward; its mean and invstd */
  float *runMean, *runVar, *saveA, *saveB;
  double *saveMean, *saveInvStd;
  void* workspace;      /* roc_batchnorm_workspace_bytes */
  size_t workspaceBytes;
};

class LayerNorm : public GnnOp {  /* not in the reference: Model::layer_norm */
public:
  LayerNorm(const Model& model, const Tensor& input, float eps);
  virtual void init(const Model& model);
  virtual void forward(const Model& model);
  virtual void backward(const Model& model);
public:
  float eps;
  Tensor gamma, beta;   /* parameters, dims {H, 1} */
  int fwdOut;           /* a relu fused into the forward, as BatchNorm::fwdOut (-1: none) */
  void* workspace;      /* roc_layernorm_workspace_bytes */
  size_t workspaceBytes;
};

class SoftmaxCrossEntropy : public GnnOp {  /* gnn.h:346-363, softmax.cc */
public:
  SoftmaxCrossEntropy(const Model& model, const Tensor& logits, const Tensor& labels, const Tensor& mask);
  virtual void init(const Model& model);
  virtual void forward(const Model& model);
  virtual void backward(const Model& model);
public:
  int epoch_num;
  int gradOut;      /* >= 0: write the logits' grad / sqrt(deg) into this region's grad (fused norm backward) */
};

class SigmoidCrossEntropy : public GnnOp {  /* not in the reference: Model::sigmoid_cross_entropy */
public:
  SigmoidCrossEntropy(const Model& model, const Tensor& logits, const Tensor& labels, const Tensor& mask);
  virtual void init(const Model& model);
  virtual void forward(const Model& model);
  virtual void backward(const Model& model);
public:
  int epoch_num;
  int gradOut;      /* >= 0: write the logits' grad / sqrt(deg) into this region's grad (fused norm backward) */
};

/* CLI of the reference driver, gnn.cc:114-179 (same flags, same `-dr` quirk). */
void parse_input_args(char** argv, int argc, Config& config);

#endif /* ROC_GNN_H_ */
