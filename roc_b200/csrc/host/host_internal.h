// host_internal.h — internals of the thin C++ host (not part of the public API).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "roc_gnn.h"
#include "roc_host.h"

namespace roc {
namespace host {

// FatalError / checkCUDA of the reference (cuda_helper.h:6-29): print and exit(1).
[[noreturn]] void fatal(const char* what, const char* file, int line);
#define ROC_FATAL(msg) ::roc::host::fatal((msg), __FILE__, __LINE__)
#define ROC_CHECK(call)                                                            \
  do {                                                                             \
    int rc_ = (int)(call);                                                         \
    if (rc_ != 0) {                                                                \
      char b_[640];                                                                \
      snprintf(b_, sizeof(b_), "%s failed with code %d", #call, rc_);              \
      ROC_FATAL(b_);                                                               \
    }                                                                              \
  } while (0)
#define ROC_ASSERT(cond)                                                           \
  do { if (!(cond)) ROC_FATAL("assertion failed: " #cond); } while (0)

struct TensorImpl {
  int64_t rows = 0;       // local rows (node tensors) or outDim (weights)
  int H = 0;              // logical width (node: hidden; weight: inDim, stored [out][in])
  int64_t ld = 0;         // floats between rows (H rounded up to 4 for node tensors)
  bool isInt = false;     // create_node_tensor<int> (mask)
  bool isBf16 = false;    // create_node_tensor<__nv_bfloat16>: a leaf feature matrix held as bf16 bits, ld elements
                          // per row (H rounded up to 8); or, with Model::set_bf16_aggregation, a Linear output that
                          // only a sum ScatterGather reads (its gradient stays fp32, with the same ld).  The bits are
                          // reached only through RuntimeImpl::data_bf16, never as float*
  bool isWeight = false;
  bool requiresGrad = false;
  bool produced = false;  // output of some op
  int64_t haloData = 0;   // extra rows after the local ones: halo slab of a ScatterGather input
  int64_t haloGrad = 0;   // same for the gradient twin (backward ScatterGather reads it)
  float* data = nullptr;  // lazily allocated (node tensors)
  float* grad = nullptr;
  int32_t* labelIdx = nullptr;   // compact labels when loaded through load_labels / set_labels
  uint32_t* labelBits = nullptr; // bit-packed multi-labels (set_multilabels): ceil(H / 32) words per row
  // peer-write halo exchange: this tensor's buffers on the other partitions' GPUs (CUDA IPC mappings, index = part)
  std::vector<float*> peerData, peerGrad;
  bool freshData = false, freshGrad = false;   // the producer already pushed this step's boundary rows
};

// NCCL through dlopen so the library has no link-time NCCL dependency and, inside
// a torch process, binds to the libnccl.so.2 torch already loaded.
struct Comm {
  void* lib = nullptr;
  void* comm = nullptr;
  int rank = 0, world = 1;
  bool load();
  static bool unique_id(unsigned char id[128]);
  bool init(int rank, int world, const unsigned char id[128]);
  // recvbuf[offsets[r] .. +counts[r]) <- rank r's sendbuf (counts in floats)
  int allgatherv(const float* sendbuf, float* recvbuf, const std::vector<size_t>& counts,
                 const std::vector<size_t>& offsets, cudaStream_t st);
  int allreduce_sum(float* buf, size_t count, cudaStream_t st);
  int allreduce_sum_i32(int* buf, size_t count, cudaStream_t st);
  int allgather_i32(const int* sendbuf, int* recvbuf, size_t countPerRank, cudaStream_t st);
  int barrier(int* scratch, cudaStream_t st);   // one-int all-reduce: completes once every rank's stream got here
  // all-to-all-v by grouped ncclSend / ncclRecv (counts and offsets in elements; no self transfer)
  int alltoallv(const void* sendbuf, const std::vector<size_t>& sendCounts, const std::vector<size_t>& sendOffs,
                void* recvbuf, const std::vector<size_t>& recvCounts, const std::vector<size_t>& recvOffs,
                bool isFloat, cudaStream_t st);
  void destroy();
};

struct RuntimeImpl {
  int device = 0, myPart = 0, numParts = 1;
  cudaStream_t stream = nullptr;       // the compute stream: every op enqueues here
  cudaStream_t commStream = nullptr;   // peer-write pushes of the halo exchange run here, beside the producer
  cudaEvent_t evProduced = nullptr, evPushed = nullptr;
  bool p2p = false;                    // halo exchange into peer-mapped slabs (else staged rows + NCCL all-to-all-v)
  bool p2pCopyEngines = true;          // ... by pack + cudaMemcpyAsync per peer (DMA engines, no SMs); false: roc_push_rows
  std::vector<cudaStream_t> peerStreams;   // one per partition: the copies to different peers run on different engines
  std::vector<cudaEvent_t> peerDone;       // last copy of the current exchange on that stream
  cudaEvent_t evPacked = nullptr;
  bool exchInFlight = false;           // copies of the previous exchange may still read the send buffer
  int pushSMs = 0;                     // SMs a pipelined producer leaves free for the push kernel (0: none)
  int pushGridSMs = 0;                 // SMs the pipelined push kernel's grid is sized for (-1: pushSMs, 0: whole chip)
  int* d_barrier = nullptr;
  std::vector<TensorImpl> tensors;
  std::vector<void*> allocs;
  Comm comm;
  bool commReady = false;
  // shared scratch
  float* gatherBuf = nullptr; size_t gatherFloats = 0;   // [numNodes][maxLd]: all-gather fallback (ROC_B200_HALO=0)
  float* sendBuf = nullptr; size_t sendFloats = 0;       // packed rows other partitions asked for
  void ensure_sendbuf(size_t floats);
  void* linWs = nullptr; size_t linWsBytes = 0;           // split-K workspace of Linear backward
  void* staging = nullptr; size_t stagingBytes = 0;       // H2D staging for dense host rows -> padded rows
  float* flatGrad = nullptr; size_t flatGradCount = 0;    // all dW, one all-reduce
  roc_sg_transpose* sgTranspose = nullptr;                // the graph's transpose: exact backward, weighted ops
  uint8_t* sgKeep = nullptr;                              // [E] edge dropout's keep bytes, refilled by each dropped sum
  roc_perf_metrics* d_perf = nullptr;
  roc_perf_metrics h_perf{};
  roc_multilabel_metrics* d_multilabel = nullptr;   // what the sigmoid cross-entropy accumulates
  bool multilabelRan = false;   // d_multilabel holds a sigmoid cross-entropy's metrics
  int lossKind = -1;   // ROC_HOST_OP_* of the loss that ran last (-1: none yet); last_metrics reads its metrics
  uint32_t trainStep = 0;
  // optional per-launch timing of the ScatterGather kernels (bench.py's roofline leg)
  struct SgTiming { int H; cudaEvent_t a, b; };
  bool profileSg = false;
  std::vector<SgTiming> sgTimings;
  void sg_begin(int H);
  void sg_end();
  // ROC_B200_OPPROF=1: device time of every op's forward / backward on the compute stream, averaged over the
  // steps and printed by rank 0 when the Runtime goes away (where does a step's time go at N GPUs?)
  struct OpTiming { int layer; int dir; cudaEvent_t a, b; };
  bool opProf = false;
  bool opTrace = false;
  std::vector<OpTiming> opTimings;
  std::vector<std::string> opNames;
  void op_begin(int layer, int dir);
  void op_end();
  void op_report();

  void* dmalloc(size_t bytes);
  void dfree_all();
  int new_tensor(int64_t rows, int H, int64_t ld, bool isInt, bool isWeight);
  float* data(int region);   // allocates on first use, zero-filled; a bf16 tensor is an error
  float* grad(int region);   // a bf16 leaf has no gradient: an error
  uint16_t* data_bf16(int region);   // the bf16 tensor's bits, allocated on first use, zero-filled
  // append `halo` rows to the data / grad buffer of x (re-allocating and copying if it already exists)
  void grow_halo(TensorImpl& x, bool grad, int64_t halo);
  // map the other partitions' copies of x's data / grad buffer (collective: every rank calls it for the same tensor)
  bool open_peers(TensorImpl& x, bool grad);
  TensorImpl& t(int region) { return tensors[(size_t)region]; }
  void ensure_gather(size_t floats);
  void ensure_lin_ws(size_t bytes);
  void ensure_staging(size_t bytes);
};

inline int64_t round_up4(int64_t x) { return (x + 3) / 4 * 4; }
inline int64_t round_up8(int64_t x) { return (x + 7) / 8 * 8; }

// an op's ROC_HOST_OP_* kind (roc_host_op_info), and each kind's name in refusals and the per-op trace / profile
int op_kind(const GnnOp* op);
extern const char* const opKindNames[ROC_HOST_OP_SCALED_ADD + 1];

}  // namespace host
}  // namespace roc
