// linear.cu — C-ABI entry points of the Linear op and the kernel dispatcher.
// Replaces Linear::forward_task / backward_task (linear_kernel.cu:19-118, 129-245).
#include <cstdlib>
#include <cstring>
#include "common.cuh"

namespace roc {
int simt_dw_splits(int64_t rows, int inDim, int outDim);
// X / ldX of the forward and dW: fp32, or bf16 (raw bits) when xBf16
int simt_linear_fwd(int64_t rows, int inDim, int outDim, const void* X, bool xBf16, int64_t ldX, const float* W,
                    void* Y, bool yBf16, int64_t ldY, int relu, const uint64_t* rowEnd, uint64_t colLeft,
                    const DropMask* dm, cudaStream_t st);
int simt_linear_dx(int64_t rows, int inDim, int outDim, const float* dY, int64_t ldDY, const float* W, float* dX,
                   int64_t ldDX, int accumulate, const DropMask* dm, const float* reluOf, int64_t ldR,
                   const uint64_t* rowEnd, uint64_t colLeft, cudaStream_t st);
int simt_linear_dw(int64_t rows, int inDim, int outDim, const void* X, bool xBf16, int64_t ldX, const float* dY,
                   int64_t ldDY, float* dW, float* workspace, size_t wsBytes, const DropMask* dm, cudaStream_t st,
                   roc_gemm_info* info);
int relu_bwd_inplace(int64_t rows, int H, const float* Y, int64_t ldY, float* dY, int64_t ldDY, cudaStream_t st);

// tensor-core path (linear_tc.cu, linear_tc_dw.cu); each returns ROC_ERR_UNSUPPORTED when the
// shape / alignment is outside what the wgmma kernels take.
// They describe the launch they made in *info (roc_last_gemm_info).
// Y is fp32, or bf16 (raw bits) when yBf16
int tc_linear_fwd(int64_t rows, int inDim, int outDim, const void* X, bool xBf16, int64_t ldX, const float* W,
                  void* Y, bool yBf16, int64_t ldY, int relu, const uint64_t* rowEnd, uint64_t colLeft,
                  const DropMask* dm, cudaStream_t st, roc_gemm_info* info);
int tc_linear_dx(int64_t rows, int inDim, int outDim, const float* dY, int64_t ldDY, const float* W, float* dX,
                 int64_t ldDX, int accumulate, const DropMask* dm, const float* reluOf, int64_t ldR,
                 const uint64_t* rowEnd, uint64_t colLeft, cudaStream_t st, roc_gemm_info* info);
size_t tc_dw_workspace_bytes(int64_t rows, int inDim, int outDim);
int tc_linear_dw(int64_t rows, int inDim, int outDim, const void* X, bool xBf16, int64_t ldX, const float* dY,
                 int64_t ldDY, float* dW, float* workspace, size_t wsBytes, const DropMask* dm, cudaStream_t st,
                 roc_gemm_info* info);

// which kernel served the calling thread's last Linear GEMM of each kind, and how it was launched (test hook: the
// tensor-core path returns ROC_ERR_UNSUPPORTED for shapes it does not take and the dispatcher then uses SIMT — a test
// that means to check the tensor cores, or one instantiation / pipeline regime of them, must be able to see that it did)
static thread_local roc_gemm_info t_last[3] = {};   // fwd, dW, dX; path 0 none, 1 tensor cores (wgmma), 2 SIMT

// GEMM `which` on the tensor cores, or on the exact-fp32 SIMT kernels when they do not take it (ROC_ERR_UNSUPPORTED)
// or ROC_B200_GEMM=simt is set ("notc" is the same switch under its older name, still set by existing scripts and
// tests).  The switch is read on every call, so a test can cross-check the two paths call by call.  Each path fills in
// what it knows of its launch.
template <class Tc, class Simt>
static int run_gemm(int which, Tc&& tc, Simt&& simt) {
  const char* e = getenv("ROC_B200_GEMM");
  const bool forced = e && (strcmp(e, "simt") == 0 || strcmp(e, "notc") == 0);
  roc_gemm_info info{};
  int rc = forced ? ROC_ERR_UNSUPPORTED : tc(&info);
  if (rc == ROC_ERR_UNSUPPORTED) {
    info = roc_gemm_info{};
    info.path = 2;
    rc = simt(&info);
  } else {
    info.path = 1;
  }
  t_last[which] = info;
  return rc;
}
}  // namespace roc

using namespace roc;

// A dropout mask is usable when rate in (0, 1); rate == 0 is the identity (infer mode).
static int mask_args(const uint32_t* mask, int64_t ldMask, float rate, int inDim, DropMask* dm, const DropMask** out) {
  *out = nullptr;
  if (rate < 0.f || rate >= 1.f) return ROC_ERR_INVALID;
  if (rate == 0.f) return ROC_OK;
  if (!mask || ldMask < (inDim + 31) / 32 || (ldMask % 4)) return ROC_ERR_INVALID;
  dm->bits = mask; dm->ld = ldMask; dm->scale = 1.0f / (1.0f - rate);   // the scale of roc_dropout_fwd
  *out = dm;
  return ROC_OK;
}

static int linear_fwd_impl(int64_t rows, int inDim, int outDim, const void* X, bool xBf16, int64_t ldX,
                           const float* W, float* Y, int64_t ldY, int activation, int flags, const roc_eid_t* rowEnd,
                           roc_eid_t colLeft, const DropMask* dm, roc_stream_t stream) {
  if (!X || !W || !Y || rows < 0 || inDim <= 0 || outDim <= 0 || ldX < inDim || ldY < outDim) return ROC_ERR_INVALID;
  if (activation != ROC_AC_MODE_NONE && activation != ROC_AC_MODE_RELU) return ROC_ERR_UNSUPPORTED;  // linear_kernel.cu:96
  if ((flags & ROC_LINEAR_NORM_EPILOGUE) && !rowEnd) return ROC_ERR_INVALID;
  const bool yBf16 = (flags & ROC_LINEAR_Y_BF16) != 0;
  if (yBf16 && (ldY % 8)) return ROC_ERR_INVALID;
  if (rows == 0) return ROC_OK;
  const uint64_t* re = (flags & ROC_LINEAR_NORM_EPILOGUE) ? rowEnd : nullptr;
  const int relu = activation == ROC_AC_MODE_RELU;
  cudaStream_t st = as_stream(stream);
  return run_gemm(
      0,
      [&](roc_gemm_info* i) {
        return tc_linear_fwd(rows, inDim, outDim, X, xBf16, ldX, W, Y, yBf16, ldY, relu, re, colLeft, dm, st, i);
      },
      [&](roc_gemm_info*) {
        return simt_linear_fwd(rows, inDim, outDim, X, xBf16, ldX, W, Y, yBf16, ldY, relu, re, colLeft, dm, st);
      });
}

extern "C" int roc_linear_fwd(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX, const float* W,
                              float* Y, int64_t ldY, int activation, int flags, const roc_eid_t* rowEnd,
                              roc_eid_t colLeft, roc_stream_t stream) {
  return linear_fwd_impl(rows, inDim, outDim, X, false, ldX, W, Y, ldY, activation, flags, rowEnd, colLeft, nullptr,
                         stream);
}

extern "C" int roc_linear_fwd_dropout(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX,
                                      const float* W, float* Y, int64_t ldY, int activation, int flags,
                                      const roc_eid_t* rowEnd, roc_eid_t colLeft, const uint32_t* mask,
                                      int64_t ldMask, float rate, roc_stream_t stream) {
  DropMask dm; const DropMask* use;
  int rc = mask_args(mask, ldMask, rate, inDim, &dm, &use);
  if (rc != ROC_OK) return rc;
  return linear_fwd_impl(rows, inDim, outDim, X, false, ldX, W, Y, ldY, activation, flags, rowEnd, colLeft, use,
                         stream);
}

extern "C" int roc_linear_fwd_bf16(int64_t rows, int inDim, int outDim, const uint16_t* X, int64_t ldX,
                                   const float* W, float* Y, int64_t ldY, int activation, int flags,
                                   const roc_eid_t* rowEnd, roc_eid_t colLeft, const uint32_t* mask, int64_t ldMask,
                                   float rate, roc_stream_t stream) {
  DropMask dm; const DropMask* use = nullptr;
  if (mask || rate != 0.f) {
    int rc = mask_args(mask, ldMask, rate, inDim, &dm, &use);
    if (rc != ROC_OK) return rc;
  }
  return linear_fwd_impl(rows, inDim, outDim, X, true, ldX, W, Y, ldY, activation, flags, rowEnd, colLeft, use,
                         stream);
}

extern "C" size_t roc_linear_bwd_workspace_bytes(int64_t rows, int inDim, int outDim) {
  if (rows <= 0 || inDim <= 0 || outDim <= 0) return 0;
  size_t a = (size_t)simt_dw_splits(rows, inDim, outDim) * (size_t)inDim * (size_t)outDim * sizeof(float);
  size_t b = tc_dw_workspace_bytes(rows, inDim, outDim);
  return a > b ? a : b;
}

static int linear_bwd_impl(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX, const float* W,
                           const float* Y, int64_t ldY, float* dY, int64_t ldDY, float* dW, float* dX,
                           int64_t ldDX, int activation, int accumulate_dX, void* workspace,
                           size_t workspaceBytes, const DropMask* dm, const float* dxReluOf, int64_t ldReluOf,
                           const roc_eid_t* dxRowEnd, roc_eid_t colLeft, roc_stream_t stream, int parts = 0) {
  if (parts != 0 && (activation != ROC_AC_MODE_NONE || (parts != ROC_LINEAR_BWD_ONLY_DX && parts != ROC_LINEAR_BWD_ONLY_DW)))
    return ROC_ERR_INVALID;
  if (parts == ROC_LINEAR_BWD_ONLY_DX && !dX) return ROC_ERR_INVALID;
  if (parts == ROC_LINEAR_BWD_ONLY_DW) { dX = nullptr; dxReluOf = nullptr; dxRowEnd = nullptr; }
  if ((dxReluOf || dxRowEnd) && !dX) return ROC_ERR_INVALID;
  if (dxReluOf && ldReluOf < inDim) return ROC_ERR_INVALID;
  if (!X || !W || !dY || !dW || rows < 0 || inDim <= 0 || outDim <= 0 || ldX < inDim || ldDY < outDim)
    return ROC_ERR_INVALID;
  if (dX && ldDX < inDim) return ROC_ERR_INVALID;
  if (activation != ROC_AC_MODE_NONE && activation != ROC_AC_MODE_RELU) return ROC_ERR_UNSUPPORTED;
  if (rows == 0) return ROC_OK;
  cudaStream_t st = as_stream(stream);
  if (activation == ROC_AC_MODE_RELU) {
    if (!Y || ldY < outDim) return ROC_ERR_INVALID;
    int rc = relu_bwd_inplace(rows, outDim, Y, ldY, dY, ldDY, st);
    if (rc != ROC_OK) return rc;
  }
  if (!workspace) return ROC_ERR_INVALID;
  float* ws = (float*)workspace;
  if (parts != ROC_LINEAR_BWD_ONLY_DX) {
    int rc = run_gemm(
        1,
        [&](roc_gemm_info* i) {
          return tc_linear_dw(rows, inDim, outDim, X, false, ldX, dY, ldDY, dW, ws, workspaceBytes, dm, st, i);
        },
        [&](roc_gemm_info* i) {
          return simt_linear_dw(rows, inDim, outDim, X, false, ldX, dY, ldDY, dW, ws, workspaceBytes, dm, st, i);
        });
    if (rc != ROC_OK) return rc;
  }
  if (dX)
    return run_gemm(
        2,
        [&](roc_gemm_info* i) {
          return tc_linear_dx(rows, inDim, outDim, dY, ldDY, W, dX, ldDX, accumulate_dX, dm, dxReluOf, ldReluOf,
                              dxRowEnd, colLeft, st, i);
        },
        [&](roc_gemm_info*) {
          return simt_linear_dx(rows, inDim, outDim, dY, ldDY, W, dX, ldDX, accumulate_dX, dm, dxReluOf, ldReluOf,
                                dxRowEnd, colLeft, st);
        });
  return ROC_OK;
}

extern "C" int roc_linear_bwd(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX, const float* W,
                              const float* Y, int64_t ldY, float* dY, int64_t ldDY, float* dW, float* dX,
                              int64_t ldDX, int activation, int accumulate_dX, void* workspace,
                              size_t workspaceBytes, roc_stream_t stream) {
  return linear_bwd_impl(rows, inDim, outDim, X, ldX, W, Y, ldY, dY, ldDY, dW, dX, ldDX, activation, accumulate_dX,
                         workspace, workspaceBytes, nullptr, nullptr, 0, nullptr, 0, stream);
}

extern "C" int roc_linear_bwd_dropout(int64_t rows, int inDim, int outDim, const float* X, int64_t ldX,
                                      const float* W, const float* Y, int64_t ldY, float* dY, int64_t ldDY,
                                      float* dW, float* dX, int64_t ldDX, int activation, int accumulate_dX,
                                      void* workspace, size_t workspaceBytes, const uint32_t* mask,
                                      int64_t ldMask, float rate, roc_stream_t stream) {
  DropMask dm; const DropMask* use;
  int rc = mask_args(mask, ldMask, rate, inDim, &dm, &use);
  if (rc != ROC_OK) return rc;
  return linear_bwd_impl(rows, inDim, outDim, X, ldX, W, Y, ldY, dY, ldDY, dW, dX, ldDX, activation, accumulate_dX,
                         workspace, workspaceBytes, use, nullptr, 0, nullptr, 0, stream);
}

// Everything roc_linear_bwd / roc_linear_bwd_dropout do, plus the backward of the ops that sit
// between X's producer and this Linear folded into the dX epilogue (see roc_linear_bwd_args).
extern "C" int roc_linear_bwd_fused(const roc_linear_bwd_args* a, roc_stream_t stream) {
  if (!a) return ROC_ERR_INVALID;
  DropMask dm; const DropMask* use = nullptr;
  if (a->dropMask || a->dropRate != 0.f) {
    int rc = mask_args(a->dropMask, a->ldMask, a->dropRate, a->inDim, &dm, &use);
    if (rc != ROC_OK) return rc;
  }
  return linear_bwd_impl(a->rows, a->inDim, a->outDim, a->X, a->ldX, a->W, a->Y, a->ldY, a->dY, a->ldDY, a->dW,
                         a->dX, a->ldDX, a->activation, a->accumulate_dX, a->workspace, a->workspaceBytes, use,
                         a->dxReluOf, a->ldReluOf, a->dxNormRowEnd, a->colLeft, stream, a->parts);
}

extern "C" int roc_linear_dw_bf16(int64_t rows, int inDim, int outDim, const uint16_t* X, int64_t ldX,
                                  const float* Y, int64_t ldY, float* dY, int64_t ldDY, float* dW, int activation,
                                  void* workspace, size_t workspaceBytes, const uint32_t* mask, int64_t ldMask,
                                  float rate, roc_stream_t stream) {
  DropMask dm; const DropMask* use = nullptr;
  if (mask || rate != 0.f) {
    int rc = mask_args(mask, ldMask, rate, inDim, &dm, &use);
    if (rc != ROC_OK) return rc;
  }
  if (!X || !dY || !dW || !workspace || rows < 0 || inDim <= 0 || outDim <= 0 || ldX < inDim || ldDY < outDim)
    return ROC_ERR_INVALID;
  if (activation != ROC_AC_MODE_NONE && activation != ROC_AC_MODE_RELU) return ROC_ERR_UNSUPPORTED;
  if (rows == 0) return ROC_OK;
  cudaStream_t st = as_stream(stream);
  if (activation == ROC_AC_MODE_RELU) {   // as roc_linear_bwd: dY = (Y > 0) ? dY : 0 in place
    if (!Y || ldY < outDim) return ROC_ERR_INVALID;
    int rc = relu_bwd_inplace(rows, outDim, Y, ldY, dY, ldDY, st);
    if (rc != ROC_OK) return rc;
  }
  float* ws = (float*)workspace;
  return run_gemm(
      1,
      [&](roc_gemm_info* i) {
        return tc_linear_dw(rows, inDim, outDim, X, true, ldX, dY, ldDY, dW, ws, workspaceBytes, use, st, i);
      },
      [&](roc_gemm_info* i) {
        return simt_linear_dw(rows, inDim, outDim, X, true, ldX, dY, ldDY, dW, ws, workspaceBytes, use, st, i);
      });
}

extern "C" int roc_last_gemm_path(int which) { return (which >= 0 && which < 3) ? t_last[which].path : 0; }

extern "C" int roc_last_gemm_info(int which, roc_gemm_info* info) {
  if (which < 0 || which >= 3 || !info) return ROC_ERR_INVALID;
  *info = t_last[which];
  return ROC_OK;
}
