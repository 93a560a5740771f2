/*
 * ref_harness.cu — launch harness for the REFERENCE's own CUDA kernels.
 *
 * TEST INFRASTRUCTURE (second parity witness + "reference kernel on the same
 * H100" timing column).  Nothing under roc_b200/ uses it.
 *
 * The reference cannot be built whole (every TU includes legion.h; the Legion
 * submodule is absent), but its __global__ kernel bodies have no Legion
 * dependence.  oracle/Makefile cuts those line ranges out of the sources where
 * they lie under /root/reference into oracle/_ref/gen/ *.inc (git-ignored build
 * output, never committed) and this file #includes them behind a typedef shim
 * that restates the handful of definitions they need:
 *   types.h:5-15 (V_ID/E_ID/DATATYPE/NodeStruct/EdgeStruct),
 *   cuda_helper.h:31-45 (CUDA_KERNEL_LOOP/CUDA_NUM_THREADS/BLOCK_SIZE_LIMIT/GET_BLOCKS),
 *   gnn.h:88-103 (ElementType, MaskType), legion's coord_t (long long).
 * Each launcher uses the reference's own grid shape and argument order, citing
 * the launch site.  All pointers are DEVICE pointers.
 */
#include <cuda_runtime.h>
#include <cublas_v2.h>
#include <cudnn.h>
#include <curand.h>
#include <assert.h>
#include <stdint.h>
#include <stdio.h>
#include <cub/cub.cuh>

typedef uint32_t V_ID;
typedef uint64_t E_ID;
typedef float DATATYPE;
typedef long long coord_t;
struct NodeStruct { E_ID index; };
struct EdgeStruct { V_ID src, dst; };
enum ElementType { EW_TYPE_ADD, EW_TYPE_MUL };
enum MaskType { MASK_TRAIN, MASK_VAL, MASK_TEST, MASK_NONE };
#define CUDA_KERNEL_LOOP(i, n) \
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += blockDim.x * gridDim.x)
const int CUDA_NUM_THREADS = 512;
const int BLOCK_SIZE_LIMIT = 32768;
inline int GET_BLOCKS(const int N) {
  int ret = (N + CUDA_NUM_THREADS - 1) / CUDA_NUM_THREADS;
  return (ret > BLOCK_SIZE_LIMIT) ? BLOCK_SIZE_LIMIT : ret;
}

#include "_ref/gen/cuda_helper_kernels.inc"   /* cuda_helper.cu:2-36 */
#include "_ref/gen/aggre_coop_kernel.inc"     /* scattergather_kernel.cu:20-76 */
#include "_ref/gen/norm_coop_kernel.inc"      /* graphnorm_kernel.cu:19-57 */
#include "_ref/gen/softmax_kernels.inc"       /* softmax_kernel.cu:19-79 */
#include "_ref/gen/optimizer_kernels.inc"     /* optimizer_kernel.cu:22-63 */
#include "_ref/gen/op_kernel.inc"             /* element_kernel.cu:19-39 */
#include "_ref/gen/relu_backward.inc"         /* linear_kernel.cu:120-127 */
#include "_ref/gen/init_graph_kernel.inc"     /* load_task.cu:271-294 */

#define RC(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

static cublasHandle_t g_blas = nullptr;
static cudnnHandle_t g_dnn = nullptr;
static int ensure_handles() {
  if (!g_blas && cublasCreate(&g_blas) != CUBLAS_STATUS_SUCCESS) return -1;
  if (!g_dnn && cudnnCreate(&g_dnn) != CUDNN_STATUS_SUCCESS) return -2;
  return 0;
}

extern "C" {

/* scattergather_kernel.cu:141-143 */
int roc_ref_scatter_gather(V_ID rowLeft, V_ID rowRight, E_ID colLeft, int hiddenDim,
                           const void* row_ptrs, const void* col_idxs,
                           const float* input, float* output) {
  long long vol = (long long)(rowRight - rowLeft + 1) * hiddenDim;
  aggre_coop_kernel<<<GET_BLOCKS((int)vol), CUDA_NUM_THREADS>>>(
      rowLeft, rowRight, colLeft, hiddenDim, (const NodeStruct*)row_ptrs,
      (const EdgeStruct*)col_idxs, input, output);
  RC(cudaGetLastError());
  return 0;
}

/* graphnorm_kernel.cu:111-113 */
int roc_ref_indegree_norm(V_ID rowLeft, V_ID rowRight, E_ID colLeft, int hiddenDim,
                          const void* row_ptrs, const float* input, float* output) {
  norm_coop_kernel<<<GET_BLOCKS(rowRight - rowLeft + 1), CUDA_NUM_THREADS>>>(
      rowLeft, rowRight, colLeft, hiddenDim, (const NodeStruct*)row_ptrs, input, output);
  RC(cudaGetLastError());
  return 0;
}

/* load_task.cu:329-330 */
int roc_ref_init_graph(V_ID rowLeft, V_ID rowRight, E_ID colLeft, void* rowPtrs,
                       void* colIdxs, const E_ID* rawRows, const V_ID* rawCols) {
  init_graph_kernel<<<GET_BLOCKS(rowRight - rowLeft + 1), CUDA_NUM_THREADS>>>(
      rowLeft, rowRight, colLeft, (NodeStruct*)rowPtrs, (EdgeStruct*)colIdxs, rawRows, rawCols);
  RC(cudaGetLastError());
  return 0;
}

/* linear_kernel.cu:76-80 (+ in-place cuDNN ReLU :98-100) */
int roc_ref_linear_fwd(int nloc, int inDim, int outDim, const float* W,
                       const float* X, float* Y, int relu) {
  if (ensure_handles()) return -1;
  float alpha = 1.0f, beta = 0.0f;
  if (cublasSgemm(g_blas, CUBLAS_OP_T, CUBLAS_OP_N, outDim, nloc, inDim, &alpha, W,
                  inDim, X, inDim, &beta, Y, outDim) != CUBLAS_STATUS_SUCCESS)
    return -3;
  if (relu) {
    cudnnTensorDescriptor_t t; cudnnActivationDescriptor_t a;
    cudnnCreateActivationDescriptor(&a); cudnnCreateTensorDescriptor(&t);
    int dims[] = {nloc, outDim, 1}; int strides[] = {outDim, 1, 1};
    cudnnSetTensorNdDescriptor(t, CUDNN_DATA_FLOAT, 3, dims, strides);
    cudnnSetActivationDescriptor(a, CUDNN_ACTIVATION_RELU, CUDNN_PROPAGATE_NAN, 0.0);
    cudnnStatus_t s = cudnnActivationForward(g_dnn, a, &alpha, t, Y, &beta, t, Y);
    cudnnDestroyTensorDescriptor(t); cudnnDestroyActivationDescriptor(a);
    if (s != CUDNN_STATUS_SUCCESS) return -4;
  }
  return 0;
}

/* linear_kernel.cu:206-207 (reluBackward), :220-224 (dW), :227-231 (dX) */
int roc_ref_linear_bwd(int nloc, int inDim, int outDim, const float* W, const float* X,
                       const float* Y, float* dY, float* dW, float* dX, int relu) {
  if (ensure_handles()) return -1;
  float alpha = 1.0f;
  if (relu) {
    int vol = nloc * outDim;
    reluBackward<<<GET_BLOCKS(vol), CUDA_NUM_THREADS>>>(dY, Y, vol);
  }
  if (cublasSgemm(g_blas, CUBLAS_OP_N, CUBLAS_OP_T, inDim, outDim, nloc, &alpha, X, inDim,
                  dY, outDim, &alpha, dW, inDim) != CUBLAS_STATUS_SUCCESS) return -3;
  if (dX && cublasSgemm(g_blas, CUBLAS_OP_N, CUBLAS_OP_N, inDim, nloc, outDim, &alpha, W,
                        inDim, dY, outDim, &alpha, dX, inDim) != CUBLAS_STATUS_SUCCESS) return -4;
  RC(cudaGetLastError());
  return 0;
}

/* activation_kernel.cu:50-66 (fwd) / :114-132 (bwd, beta = alpha = 1) ; mode 1 relu 2 sigmoid */
int roc_ref_activation(int nloc, int H, int mode, int backward, const float* x_or_y,
                       const float* dy, const float* x, float* out) {
  if (ensure_handles()) return -1;
  cudnnTensorDescriptor_t t; cudnnActivationDescriptor_t a;
  cudnnCreateActivationDescriptor(&a); cudnnCreateTensorDescriptor(&t);
  int dims[] = {nloc, H, 1}; int strides[] = {H, 1, 1};
  cudnnSetTensorNdDescriptor(t, CUDNN_DATA_FLOAT, 3, dims, strides);
  cudnnSetActivationDescriptor(a, mode == 1 ? CUDNN_ACTIVATION_RELU : CUDNN_ACTIVATION_SIGMOID,
                               CUDNN_PROPAGATE_NAN, 0.0);
  float alpha = 1.0f, beta = 0.0f;
  cudnnStatus_t s;
  if (!backward)
    s = cudnnActivationForward(g_dnn, a, &alpha, t, x_or_y, &beta, t, out);
  else
    s = cudnnActivationBackward(g_dnn, a, &alpha, t, x_or_y, t, dy, t, x, &alpha, t, out);
  cudnnDestroyTensorDescriptor(t); cudnnDestroyActivationDescriptor(a);
  return s == CUDNN_STATUS_SUCCESS ? 0 : -4;
}

/* softmax_kernel.cu:124-156: cudnnSoftmaxForward -> calc_loss -> softmax_backward.
 * perf: device PerfMetrics, zeroed here like :128-134. */
int roc_ref_softmax_xent_bwd(int nloc, int C, const float* logits, const float* labels,
                             const int* mask, float* logitsGrad, void* perf_host) {
  if (ensure_handles()) return -1;
  cudnnTensorDescriptor_t d; cudnnCreateTensorDescriptor(&d);
  int dims[] = {nloc, C, 1, 1}; int strides[] = {C, 1, 1, 1};
  cudnnSetTensorNdDescriptor(d, CUDNN_DATA_FLOAT, 4, dims, strides);
  float alpha = 1.0f, beta = 0.0f;
  cudnnStatus_t s = cudnnSoftmaxForward(g_dnn, CUDNN_SOFTMAX_ACCURATE, CUDNN_SOFTMAX_MODE_INSTANCE,
                                        &alpha, d, logits, &beta, d, logitsGrad);
  cudnnDestroyTensorDescriptor(d);
  if (s != CUDNN_STATUS_SUCCESS) return -4;
  PerfMetrics* perf; PerfMetrics z; memset(&z, 0, sizeof(z));
  RC(cudaMalloc(&perf, sizeof(PerfMetrics)));
  RC(cudaMemcpy(perf, &z, sizeof(PerfMetrics), cudaMemcpyHostToDevice));
  calc_loss<<<GET_BLOCKS(nloc), CUDA_NUM_THREADS>>>(logitsGrad, labels, mask, perf, C, nloc);
  RC(cudaMemcpy(perf_host, perf, sizeof(PerfMetrics), cudaMemcpyDeviceToHost));
  softmax_backward<<<GET_BLOCKS(nloc * C), CUDA_NUM_THREADS>>>(logitsGrad, labels, mask, C, nloc);
  RC(cudaGetLastError());
  cudaFree(perf);
  return 0;
}

/* optimizer_kernel.cu:88-101: replica sum then adam_update */
int roc_ref_adam_update(int count, int numReplicas, float alpha_t, float beta1, float beta2,
                        float weight_decay, float epsilon, float* WGrad, float* M, float* V, float* W) {
  for (int i = 1; i < numReplicas; i++)
    add_kernel<<<GET_BLOCKS(count), CUDA_NUM_THREADS>>>(count, 1.0f, WGrad + (size_t)i * count, WGrad);
  adam_update<<<GET_BLOCKS(count), CUDA_NUM_THREADS>>>(count, alpha_t, beta1, beta2, weight_decay,
                                                      epsilon, WGrad, M, V, W);
  RC(cudaGetLastError());
  return 0;
}

/* element_kernel.cu:62-64 (fwd add), :96-99 (bwd: dst += src) */
int roc_ref_add_fwd(long long n, const float* a, const float* b, float* y) {
  op_kernel<<<GET_BLOCKS((int)n), CUDA_NUM_THREADS>>>(a, b, y, n, EW_TYPE_ADD);
  RC(cudaGetLastError());
  return 0;
}
int roc_ref_add_inplace(long long n, float* dst, const float* src) {
  add_kernel<<<GET_BLOCKS((int)n), CUDA_NUM_THREADS>>>(dst, src, (coord_t)n);
  RC(cudaGetLastError());
  return 0;
}

/* initializer_kernel.cu:38-48: cuRAND XORWOW uniform, then scale_kernel(-s, s) */
int roc_ref_glorot(int inDim, int outDim, int seed, float* W) {
  long long vol = (long long)inDim * outDim;
  float scale = sqrt(6.0 / (inDim + outDim));
  curandGenerator_t gen;
  if (curandCreateGenerator(&gen, CURAND_RNG_PSEUDO_DEFAULT) != CURAND_STATUS_SUCCESS) return -5;
  curandSetPseudoRandomGeneratorSeed(gen, seed);
  if (curandGenerateUniform(gen, W, vol) != CURAND_STATUS_SUCCESS) return -6;
  scale_kernel<<<GET_BLOCKS((int)vol), CUDA_NUM_THREADS>>>(W, (coord_t)vol, -scale, scale);
  curandDestroyGenerator(gen);
  RC(cudaDeviceSynchronize());
  return 0;
}

int roc_ref_sync(void) { RC(cudaDeviceSynchronize()); return 0; }

} /* extern "C" */
