// tc_common.cuh — sm_90a building blocks written as inline PTX: mbarrier, TMA
// (cp.async.bulk.tensor), warpgroup MMA (wgmma) and its shared-memory descriptor.
// Formats follow the PTX ISA (wgmma matrix descriptor, register fragment layouts).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace roc {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// One lane of a converged warp (elect.sync).  The TMA issuing loops run warp-converged and branch on
// this only around the issue itself, so ptxas knows the operands are warp-uniform.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, px;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
// warp index as a value ptxas knows to be warp-uniform
__device__ __forceinline__ int uniform_warp_idx() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0); }

// ---------------------------------------------------------------- mbarrier ---
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!ok);
}
// make generic-proxy smem writes visible to the async proxy (TMA / wgmma reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// --------------------------------------------------------------------- TMA ---
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load: coordinates {c0 = innermost (elements), c1 = row}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}

// -------------------------------------------------------------------- wgmma ---
// Warpgroup MMA (sm_90a): the 128 threads of a warpgroup issue together; the accumulator lives in
// their registers (m64nNk8 f32: warp w of the group holds rows 16w..16w+15, thread lane l holds rows
// 16w + l/4 and 16w + l/4 + 8, columns 8j + 2(l%4) and +1 for each n8 block j).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// An MMA reads its register A fragment asynchronously, after the instruction has issued.  A fake use of the
// fragments placed after the wgmma_wait_all that retires their MMAs keeps the compiler from handing those
// registers to other values (the next k-step's fragments, say) while the MMAs may still read them.
template <int A, int B, int C>
__device__ __forceinline__ void keep_live(const uint32_t (&r)[A][B][C]) {
#pragma unroll
  for (int i = 0; i < A; i++)
#pragma unroll
    for (int j = 0; j < B; j++)
#pragma unroll
      for (int k = 0; k < C; k++) asm volatile("" ::"r"(r[i][j][k]) : "memory");
}
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[16]) {
#pragma unroll
  for (int i = 0; i < 16; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 32] += A[64 x 8] * B[32 x 8]^T, kind tf32 with fp32 accumulate.  A comes from registers
// (thread lane l of warp w: a0 = (16w + l/4, l%4), a1 = row + 8, a2 = col + 4, a3 = both), B from
// shared memory through a descriptor (K-major, 128-byte swizzle).
__device__ __forceinline__ void wgmma_m64n32k8_tf32(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
      : "memory");
}
// The same at N = 64 and N = 128: B is 2 or 4 of the n32 B tiles stacked along N (rows 32c.. of the K-major tile),
// and the accumulator is the n32 accumulators of those tiles concatenated (n8 block j in d[4j..4j+3]).
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
      ",%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "{%32,%33,%34,%35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
      : "memory");
}
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
      ",%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
      ",%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
      ",%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
      "{%64,%65,%66,%67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
      : "memory");
}
// D[64 x 32 NC] += A * B^T on the NC n32 accumulators d[c] (NC = 1, 2, 4) as one MMA
template <int NC>
__device__ __forceinline__ void wgmma_m64nNk8_tf32(float (&d)[NC][16], const uint32_t (&a)[4], uint64_t bdesc) {
  if constexpr (NC == 1) wgmma_m64n32k8_tf32(d[0], a, bdesc);
  else if constexpr (NC == 2) wgmma_m64n64k8_tf32(reinterpret_cast<float (&)[32]>(d), a, bdesc);
  else wgmma_m64n128k8_tf32(reinterpret_cast<float (&)[64]>(d), a, bdesc);
}

// -------------------------------------------------------------- descriptors ---
// wgmma shared-memory matrix descriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46),
// base offset [49,52) (0: every tile here starts 1024-byte aligned), layout [62,64) (1 = SWIZZLE_128B).
// A K-major tf32 operand written by TMA with CU_TENSOR_MAP_SWIZZLE_128B: rows of 32 floats (128 bytes),
// 8-row atoms of 1024 bytes (SBO); LBO is unused for swizzled K-major layouts.  The k8 step inside the
// 128-byte row advances the start address by 32 bytes (the hardware applies the swizzle to the
// absolute address).
__device__ __forceinline__ uint64_t make_sdesc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1u << 16;
  d |= (uint64_t)(1024u >> 4) << 32;
  d |= 1ull << 62;
  return d;
}

// split of an fp32 value into a TF32 head (10-bit mantissa, truncated) and the exact remainder
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xFFFFE000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}

// ------------------------------------------------------ host: tensor maps -----
// cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// fp32 row-major [rows][cols] with `ld` floats between rows; box = [boxRows][boxCols],
// 128-byte swizzle (boxCols * 4 must be 128), out-of-bounds elements read as zero.
inline bool make_tmap_32b_2d(CUtensorMap* m, CUtensorMapDataType dt, const void* base, uint64_t rows, uint64_t cols,
                             uint64_t ld, uint32_t boxRows, uint32_t boxCols, CUtensorMapSwizzle swizzle,
                             CUtensorMapL2promotion promo = CU_TENSOR_MAP_L2_PROMOTION_L2_256B) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 4};
  cuuint32_t box[2] = {boxCols, boxRows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                  promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}
inline bool make_tmap_f32_2d(CUtensorMap* m, const float* base, uint64_t rows, uint64_t cols, uint64_t ld,
                             uint32_t boxRows, uint32_t boxCols,
                             CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  return make_tmap_32b_2d(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, rows, cols, ld, boxRows, boxCols, swizzle);
}
// uint32 row-major [rows][cols] (the packed dropout mask), no swizzle
inline bool make_tmap_u32_2d(CUtensorMap* m, const uint32_t* base, uint64_t rows, uint64_t cols, uint64_t ld,
                             uint32_t boxRows, uint32_t boxCols) {
  return make_tmap_32b_2d(m, CU_TENSOR_MAP_DATA_TYPE_UINT32, base, rows, cols, ld, boxRows, boxCols,
                          CU_TENSOR_MAP_SWIZZLE_NONE);
}

}  // namespace tc
}  // namespace roc
