// runtime.cc — Runtime: the process's GPU, stream, device memory and NCCL communicator.
// Replaces what Legion/Realm + GnnMapper + ResourceManager provided to the reference
// (gnn_mapper.cc, resourcemanager.cc, load_task.cu:296-376): here it is one
// cudaSetDevice, one stream and plain device allocations that live as long as the Runtime.
#include <dlfcn.h>
#include <nccl.h>
#include <algorithm>
#include <cstring>
#include <map>

#include "host_internal.h"

namespace roc {
namespace host {

void fatal(const char* what, const char* file, int line) {
  fprintf(stderr, "%s\n%s:%d\nAborting...\n", what, file, line);
  fflush(stderr);
  exit(1);
}

void* RuntimeImpl::dmalloc(size_t bytes) {
  void* p = nullptr;
  if (bytes == 0) bytes = 16;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    char b[160];
    snprintf(b, sizeof(b), "cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
    ROC_FATAL(b);
  }
  allocs.push_back(p);
  return p;
}

void RuntimeImpl::dfree_all() {
  for (void* p : allocs) cudaFree(p);
  allocs.clear();
}

int RuntimeImpl::new_tensor(int64_t rows, int H, int64_t ld, bool isInt, bool isWeight) {
  TensorImpl ti;
  ti.rows = rows; ti.H = H; ti.ld = ld; ti.isInt = isInt; ti.isWeight = isWeight;
  tensors.push_back(ti);
  return (int)tensors.size() - 1;
}

float* RuntimeImpl::data(int region) {
  TensorImpl& x = t(region);
  if (x.isBf16) ROC_FATAL("a bf16 node tensor was read as fp32: only linear and dropout take bf16 input");
  if (!x.data) {
    size_t bytes = (size_t)(x.rows + x.haloData) * (size_t)x.ld * sizeof(float);
    x.data = (float*)dmalloc(bytes);
    ROC_CHECK(cudaMemsetAsync(x.data, 0, bytes ? bytes : 16, stream));
  }
  return x.data;
}

uint16_t* RuntimeImpl::data_bf16(int region) {
  TensorImpl& x = t(region);
  ROC_ASSERT(x.isBf16);
  if (!x.data) {
    size_t bytes = (size_t)x.rows * (size_t)x.ld * sizeof(uint16_t);
    x.data = (float*)dmalloc(bytes);   // the untyped buffer; every access goes through this accessor
    ROC_CHECK(cudaMemsetAsync(x.data, 0, bytes ? bytes : 16, stream));
  }
  return reinterpret_cast<uint16_t*>(x.data);
}

float* RuntimeImpl::grad(int region) {
  TensorImpl& x = t(region);
  if (x.isBf16 && !x.produced) ROC_FATAL("a bf16 leaf tensor has no gradient");   // a produced one has an fp32 twin
  if (!x.grad) {
    size_t bytes = (size_t)(x.rows + x.haloGrad) * (size_t)x.ld * sizeof(float);
    x.grad = (float*)dmalloc(bytes);
    ROC_CHECK(cudaMemsetAsync(x.grad, 0, bytes ? bytes : 16, stream));
  }
  return x.grad;
}

void RuntimeImpl::grow_halo(TensorImpl& x, bool isGrad, int64_t halo) {
  int64_t& have = isGrad ? x.haloGrad : x.haloData;
  float*& buf = isGrad ? x.grad : x.data;
  if (halo <= have) return;
  if (buf) {
    const size_t oldBytes = (size_t)(x.rows + have) * (size_t)x.ld * sizeof(float);
    const size_t newBytes = (size_t)(x.rows + halo) * (size_t)x.ld * sizeof(float);
    float* nb = (float*)dmalloc(newBytes);
    ROC_CHECK(cudaMemsetAsync(nb, 0, newBytes, stream));
    ROC_CHECK(cudaMemcpyAsync(nb, buf, oldBytes, cudaMemcpyDeviceToDevice, stream));
    buf = nb;   // the old buffer stays in the arena until the Runtime goes away
  }
  have = halo;
}

// Collective.  Every rank exports the buffer's CUDA IPC handle, the handles are all-gathered over NCCL and each
// rank maps the other ranks' buffers; returns false (the caller falls back to the NCCL exchange) if a mapping fails.
bool RuntimeImpl::open_peers(TensorImpl& x, bool isGrad) {
  std::vector<float*>& peers = isGrad ? x.peerGrad : x.peerData;
  if (!peers.empty()) return true;
  float* mine = isGrad ? x.grad : x.data;
  ROC_ASSERT(mine != nullptr);
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
  cudaIpcMemHandle_t h;
  int ok = cudaIpcGetMemHandle(&h, mine) == cudaSuccess ? 1 : 0;
  if (!ok) { cudaGetLastError(); memset(&h, 0, sizeof(h)); }
  const int P = numParts;
  int* d_h = (int*)dmalloc(sizeof(int) * 17 * (size_t)(P + 1));
  int hostMine[17];
  memcpy(hostMine, &h, 64); hostMine[16] = ok;
  std::vector<int> all((size_t)17 * P);
  ROC_CHECK(cudaMemcpyAsync(d_h, hostMine, sizeof(hostMine), cudaMemcpyHostToDevice, stream));
  ROC_CHECK(comm.allgather_i32(d_h, d_h + 17, 17, stream));
  ROC_CHECK(cudaMemcpyAsync(all.data(), d_h + 17, sizeof(int) * 17 * (size_t)P, cudaMemcpyDeviceToHost, stream));
  ROC_CHECK(cudaStreamSynchronize(stream));
  bool good = true;
  for (int q = 0; q < P; q++) good = good && all[(size_t)17 * q + 16] == 1;
  std::vector<float*> mapped((size_t)P, nullptr);
  if (good) {
    for (int q = 0; q < P && good; q++) {
      if (q == myPart) { mapped[(size_t)q] = mine; continue; }
      cudaIpcMemHandle_t hq;
      memcpy(&hq, &all[(size_t)17 * q], 64);
      void* p = nullptr;
      if (cudaIpcOpenMemHandle(&p, hq, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); good = false; }
      mapped[(size_t)q] = (float*)p;
    }
  }
  // every rank must take the same path: agree on the outcome
  int flag = good ? 0 : 1;
  ROC_CHECK(cudaMemcpyAsync(d_h, &flag, sizeof(int), cudaMemcpyHostToDevice, stream));
  ROC_CHECK(comm.allreduce_sum_i32(d_h, 1, stream));
  ROC_CHECK(cudaMemcpyAsync(&flag, d_h, sizeof(int), cudaMemcpyDeviceToHost, stream));
  ROC_CHECK(cudaStreamSynchronize(stream));
  if (flag != 0) {
    for (int q = 0; q < P; q++) if (q != myPart && mapped[(size_t)q]) cudaIpcCloseMemHandle(mapped[(size_t)q]);
    return false;
  }
  peers = mapped;
  return true;
}

void RuntimeImpl::ensure_gather(size_t floats) {
  if (floats <= gatherFloats) return;
  gatherBuf = (float*)dmalloc(floats * sizeof(float));   // old one stays in the arena (freed at exit)
  gatherFloats = floats;
}

void RuntimeImpl::sg_begin(int H) {
  if (!profileSg) return;
  SgTiming t; t.H = H;
  ROC_CHECK(cudaEventCreate(&t.a)); ROC_CHECK(cudaEventCreate(&t.b));
  ROC_CHECK(cudaEventRecord(t.a, stream));
  sgTimings.push_back(t);
}
void RuntimeImpl::sg_end() {
  if (!profileSg || sgTimings.empty()) return;
  ROC_CHECK(cudaEventRecord(sgTimings.back().b, stream));
}

void RuntimeImpl::op_begin(int layer, int dir) {
  if (opTrace) {   // ROC_B200_TRACE=1: name every op before it runs and synchronise after it (which op hangs / faults?)
    fprintf(stderr, "[roc_b200 trace] part %d %s layer %d %s ...\n", myPart, dir == 0 ? "fwd" : (dir == 1 ? "bwd" : "upd"), layer,
            (layer >= 0 && (size_t)layer < opNames.size()) ? opNames[(size_t)layer].c_str() : "-");
    fflush(stderr);
  }
  if (!opProf) return;
  OpTiming t; t.layer = layer; t.dir = dir;
  ROC_CHECK(cudaEventCreate(&t.a)); ROC_CHECK(cudaEventCreate(&t.b));
  ROC_CHECK(cudaEventRecord(t.a, stream));
  opTimings.push_back(t);
}
void RuntimeImpl::op_end() {
  if (opTrace) {
    cudaError_t e = cudaStreamSynchronize(stream);
    fprintf(stderr, "[roc_b200 trace] part %d    done (%s)\n", myPart, cudaGetErrorString(e));
    fflush(stderr);
  }
  if (!opProf || opTimings.empty()) return;
  ROC_CHECK(cudaEventRecord(opTimings.back().b, stream));
}
void RuntimeImpl::op_report() {
  if (!opProf || opTimings.empty()) return;
  cudaDeviceSynchronize();
  std::map<std::pair<int, int>, std::pair<double, int>> acc;
  for (OpTiming& t : opTimings) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) { auto& e = acc[{t.layer, t.dir}]; e.first += ms; e.second += 1; }
    cudaEventDestroy(t.a); cudaEventDestroy(t.b);
  }
  opTimings.clear();
  if (myPart != 0) return;
  double tot = 0;
  fprintf(stderr, "[roc_b200] op profile (ms per call on the compute stream, part 0 of %d):\n", numParts);
  for (auto& kv : acc) {
    const double ms = kv.second.first / kv.second.second;
    tot += ms;
    const int l = kv.first.first;
    fprintf(stderr, "  %-3s layer %2d %-22s %8.3f  (%d calls)\n", kv.first.second == 0 ? "fwd" : (kv.first.second == 1 ? "bwd" : "upd"), l,
            (l >= 0 && (size_t)l < opNames.size()) ? opNames[(size_t)l].c_str() : "-", ms, kv.second.second);
  }
  fprintf(stderr, "  sum %8.3f ms\n", tot);
}

void RuntimeImpl::ensure_sendbuf(size_t floats) {
  if (floats <= sendFloats) return;
  sendBuf = (float*)dmalloc(floats * sizeof(float));
  sendFloats = floats;
}

void RuntimeImpl::ensure_staging(size_t bytes) {
  if (bytes <= stagingBytes) return;
  staging = dmalloc(bytes);
  stagingBytes = bytes;
}

void RuntimeImpl::ensure_lin_ws(size_t bytes) {
  if (bytes <= linWsBytes) return;
  linWs = dmalloc(bytes);
  linWsBytes = bytes;
}

// ------------------------------------------------------------------- NCCL ---
namespace {
struct NcclFns {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*);
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
  ncclResult_t (*CommDestroy)(ncclComm_t);
  ncclResult_t (*GroupStart)();
  ncclResult_t (*GroupEnd)();
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
  const char* (*GetErrorString)(ncclResult_t);
};
NcclFns g_nccl;
void* g_ncclLib = nullptr;

bool load_nccl() {
  if (g_ncclLib) return true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (const char* n : names) {
    h = dlopen(n, RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);   // prefer one already in the process (torch's)
    if (h) break;
  }
  if (!h)
    for (const char* n : names) { h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (h) break; }
  if (!h) { fprintf(stderr, "roc_b200: cannot load libnccl: %s\n", dlerror()); return false; }
#define SYM(field, name) \
  *(void**)(&g_nccl.field) = dlsym(h, name); \
  if (!g_nccl.field) { fprintf(stderr, "roc_b200: libnccl lacks %s\n", name); return false; }
  SYM(GetUniqueId, "ncclGetUniqueId");
  SYM(CommInitRank, "ncclCommInitRank");
  SYM(CommDestroy, "ncclCommDestroy");
  SYM(GroupStart, "ncclGroupStart");
  SYM(GroupEnd, "ncclGroupEnd");
  SYM(Broadcast, "ncclBroadcast");
  SYM(AllReduce, "ncclAllReduce");
  SYM(AllGather, "ncclAllGather");
  SYM(Send, "ncclSend");
  SYM(Recv, "ncclRecv");
  SYM(GetErrorString, "ncclGetErrorString");
#undef SYM
  g_ncclLib = h;
  return true;
}
}  // namespace

bool Comm::load() { return load_nccl(); }

bool Comm::unique_id(unsigned char id[128]) {
  if (!load_nccl()) return false;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId u;
  if (g_nccl.GetUniqueId(&u) != ncclSuccess) return false;
  memcpy(id, &u, 128);
  return true;
}

bool Comm::init(int r, int w, const unsigned char id[128]) {
  if (!load_nccl()) return false;
  ncclUniqueId u;
  memcpy(&u, id, 128);
  ncclComm_t c;
  ncclResult_t rc = g_nccl.CommInitRank(&c, w, u, r);
  if (rc != ncclSuccess) {
    fprintf(stderr, "roc_b200: ncclCommInitRank: %s\n", g_nccl.GetErrorString(rc));
    return false;
  }
  comm = c; rank = r; world = w;
  return true;
}

int Comm::allgatherv(const float* sendbuf, float* recvbuf, const std::vector<size_t>& counts,
                     const std::vector<size_t>& offsets, cudaStream_t st) {
  // NCCL has no all-gather-v: one grouped broadcast per owner, landing each slab at
  // its row offset of the gathered matrix.
  ncclComm_t c = (ncclComm_t)comm;
  if (g_nccl.GroupStart() != ncclSuccess) return -1;
  for (int r = 0; r < world; r++) {
    if (counts[r] == 0) continue;
    ncclResult_t rc = g_nccl.Broadcast(r == rank ? (const void*)sendbuf : (const void*)(recvbuf + offsets[r]),
                                       recvbuf + offsets[r], counts[r], ncclFloat, r, c, st);
    if (rc != ncclSuccess) { g_nccl.GroupEnd(); return -2; }
  }
  return g_nccl.GroupEnd() == ncclSuccess ? 0 : -3;
}

int Comm::allreduce_sum(float* buf, size_t count, cudaStream_t st) {
  return g_nccl.AllReduce(buf, buf, count, ncclFloat, ncclSum, (ncclComm_t)comm, st) == ncclSuccess ? 0 : -1;
}

int Comm::allreduce_sum_i32(int* buf, size_t count, cudaStream_t st) {
  return g_nccl.AllReduce(buf, buf, count, ncclInt32, ncclSum, (ncclComm_t)comm, st) == ncclSuccess ? 0 : -1;
}

int Comm::allgather_i32(const int* sendbuf, int* recvbuf, size_t countPerRank, cudaStream_t st) {
  return g_nccl.AllGather(sendbuf, recvbuf, countPerRank, ncclInt32, (ncclComm_t)comm, st) == ncclSuccess ? 0 : -1;
}

int Comm::barrier(int* scratch, cudaStream_t st) {
  return g_nccl.AllReduce(scratch, scratch, 1, ncclInt32, ncclSum, (ncclComm_t)comm, st) == ncclSuccess ? 0 : -1;
}

int Comm::alltoallv(const void* sendbuf, const std::vector<size_t>& sendCounts, const std::vector<size_t>& sendOffs,
                    void* recvbuf, const std::vector<size_t>& recvCounts, const std::vector<size_t>& recvOffs,
                    bool isFloat, cudaStream_t st) {
  // one grouped ncclSend + ncclRecv per peer: NVSwitch gives every pair full bandwidth, so the
  // group is a single fused transfer; 4-byte elements either way
  ncclComm_t c = (ncclComm_t)comm;
  const ncclDataType_t dt = isFloat ? ncclFloat : ncclUint32;
  const char* sb = static_cast<const char*>(sendbuf);
  char* rb = static_cast<char*>(recvbuf);
  if (g_nccl.GroupStart() != ncclSuccess) return -1;
  for (int q = 0; q < world; q++) {
    if (q == rank) continue;
    if (sendCounts[q] && g_nccl.Send(sb + sendOffs[q] * 4, sendCounts[q], dt, q, c, st) != ncclSuccess) { g_nccl.GroupEnd(); return -2; }
    if (recvCounts[q] && g_nccl.Recv(rb + recvOffs[q] * 4, recvCounts[q], dt, q, c, st) != ncclSuccess) { g_nccl.GroupEnd(); return -3; }
  }
  return g_nccl.GroupEnd() == ncclSuccess ? 0 : -4;
}

void Comm::destroy() {
  if (comm && g_ncclLib) g_nccl.CommDestroy((ncclComm_t)comm);
  comm = nullptr;
}

}  // namespace host
}  // namespace roc

using namespace roc::host;

Runtime::Runtime(int device, int myPart, int numParts) {
  impl = new RuntimeImpl();
  impl->device = device; impl->myPart = myPart; impl->numParts = numParts;
  if (numParts < 1 || myPart < 0 || myPart >= numParts || numParts > MAX_NUM_PARTS)
    ROC_FATAL("Runtime: bad partition index / count");
  if (roc_device_count() <= 0)
    ROC_FATAL("roc_b200: no CUDA device visible - this engine has no CPU fallback");
  ROC_CHECK(cudaSetDevice(device));
  {
    // The compute stream outranks the exchange stream: when a producer block and the push of the previous block
    // become runnable together, the producer's CTAs (a whole SM each) are placed first and the push kernel takes
    // the SMs the producer left free — the other way round its small CTAs would sit on every SM and keep the
    // producer out.
    int lo = 0, hi = 0;   // numerically lower = higher priority
    ROC_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    const char* pe = getenv("ROC_B200_PUSH_PRIO");          // experiments: 0 = equal priorities
    const bool prio = !(pe && pe[0] == '0');
    ROC_CHECK(cudaStreamCreateWithPriority(&impl->stream, cudaStreamNonBlocking, prio ? hi : lo));
    ROC_CHECK(cudaStreamCreateWithPriority(&impl->commStream, cudaStreamNonBlocking, lo));
  }
  ROC_CHECK(cudaEventCreateWithFlags(&impl->evProduced, cudaEventDisableTiming));
  ROC_CHECK(cudaEventCreateWithFlags(&impl->evPushed, cudaEventDisableTiming));
  ROC_CHECK(cudaEventCreateWithFlags(&impl->evPacked, cudaEventDisableTiming));
  for (int q = 0; q < numParts && numParts > 1; q++) {
    cudaStream_t ps = nullptr; cudaEvent_t pe = nullptr;
    ROC_CHECK(cudaStreamCreateWithFlags(&ps, cudaStreamNonBlocking));
    ROC_CHECK(cudaEventCreateWithFlags(&pe, cudaEventDisableTiming));
    impl->peerStreams.push_back(ps); impl->peerDone.push_back(pe);
  }
  impl->d_barrier = (int*)impl->dmalloc(sizeof(int));
  ROC_CHECK(cudaMemsetAsync(impl->d_barrier, 0, sizeof(int), impl->stream));
  if (const char* e = getenv("ROC_B200_PUSH_SMS")) impl->pushSMs = std::max(0, atoi(e));
  if (const char* e = getenv("ROC_B200_OPPROF")) impl->opProf = e[0] == '1';
  if (const char* e = getenv("ROC_B200_TRACE")) impl->opTrace = e[0] == '1';
  if (const char* e = getenv("ROC_B200_PUSH_GRID")) impl->pushGridSMs = atoi(e);   // experiments: SMs the pipelined push grid is sized for (0 = chip)
  {
    // The stream-ordered allocations of the kernel layer (the GEMMs' split-weight scratch) come from the device's
    // default pool; by default it hands unused memory back at every synchronisation and the next step pays the
    // driver allocation again (one slow step in every few).  Keep it.
    cudaMemPool_t pool = nullptr;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess && pool) {
      uint64_t keep = UINT64_MAX;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    cudaGetLastError();
  }
  impl->d_perf = (roc_perf_metrics*)impl->dmalloc(sizeof(roc_perf_metrics));
  ROC_CHECK(cudaMemsetAsync(impl->d_perf, 0, sizeof(roc_perf_metrics), impl->stream));
}

Runtime::~Runtime() {
  if (!impl) return;
  cudaSetDevice(impl->device);
  cudaDeviceSynchronize();
  impl->op_report();
  for (TensorImpl& x : impl->tensors) {
    for (size_t q = 0; q < x.peerData.size(); q++) if ((int)q != impl->myPart && x.peerData[q]) cudaIpcCloseMemHandle(x.peerData[q]);
    for (size_t q = 0; q < x.peerGrad.size(); q++) if ((int)q != impl->myPart && x.peerGrad[q]) cudaIpcCloseMemHandle(x.peerGrad[q]);
  }
  impl->comm.destroy();
  roc_sg_transpose_destroy(impl->sgTranspose);
  impl->dfree_all();
  for (cudaStream_t ps : impl->peerStreams) cudaStreamDestroy(ps);
  for (cudaEvent_t pe : impl->peerDone) cudaEventDestroy(pe);
  if (impl->evPacked) cudaEventDestroy(impl->evPacked);
  if (impl->evProduced) cudaEventDestroy(impl->evProduced);
  if (impl->evPushed) cudaEventDestroy(impl->evPushed);
  if (impl->commStream) cudaStreamDestroy(impl->commStream);
  if (impl->stream) cudaStreamDestroy(impl->stream);
  delete impl;
}

bool Runtime::nccl_unique_id(unsigned char id[128]) { return Comm::unique_id(id); }

bool Runtime::init_nccl(const unsigned char id[128]) {
  ROC_CHECK(cudaSetDevice(impl->device));
  if (impl->numParts == 1) return true;
  impl->commReady = impl->comm.init(impl->myPart, impl->numParts, id);
  return impl->commReady;
}

void Runtime::synchronize() { ROC_CHECK(cudaStreamSynchronize(impl->stream)); }
