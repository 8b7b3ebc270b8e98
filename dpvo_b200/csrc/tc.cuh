// The one home of the inline-PTX wrappers of the kernels: shared-memory addresses, mbarriers, TMA and 1-D bulk copies,
// cp.async, named barriers, mma.sync and wgmma, used by chain.cu, gemm.cu, softagg.cu, corr.cu, corr_bin.cu,
// corr_tc.cu, encoder.cu and update_ops.cu.  Also declares the host-side tensor-map encoder (common.cu).
#pragma once
#include "common.cuh"
#include <cuda.h>          // CUtensorMap types only; the encoder is fetched from the driver at run time

namespace dpvo {

// ---- PTX wrappers ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
// makes the initialised mbarriers visible to the async proxy (TMA, bulk copies) and to the other CTAs of the cluster
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.shared::cta.b64 st, [%0];\n}\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n}\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// also takes the barrier's shared-memory address (smem_u32), for callers that keep it in a register
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { mbar_wait(smem_u32(bar), parity); }
// bounded wait: a broken hand-shake traps (launch failure) instead of hanging the device.  try_wait suspends the
// thread for a hardware-defined interval per attempt, so the bound is tens of milliseconds at the very least.  No
// printf here: a function call between wgmma instructions would serialise the MMA pipeline of the caller.
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  for (uint32_t it = 0; it < (1u << 26); ++it) {
    uint32_t ok;
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
    if (ok) return;
  }
  __trap();
}
// register budget per thread of a warpgroup (all four warps execute it): producers give registers back to consumers
template <int N> __device__ __forceinline__ void warpgroup_reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N)); }
template <int N> __device__ __forceinline__ void warpgroup_reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N)); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
// 2-D TMA tile load, completion signalled on an mbarrier (SASS: UTMALDG)
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n" ::"r"(dst),
               "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* tmap, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];\n" ::"r"(dst),
               "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
               : "memory");
}
// 1-D bulk copy of `bytes` (a multiple of 16) global -> shared, completion signalled on the mbarrier at shared-memory
// address bar: a caller that issues several copies per barrier, from several lanes, then keeps one 32-bit register
// live rather than a 64-bit generic pointer
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
// 2-D TMA tile load multicast to the CTAs of the cluster in cta_mask: the tile lands at the same shared-memory offset in
// each of them and completes its bytes on the mbarrier at the same offset in each
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t dst, const void* tmap, int c0, int c1, uint64_t* bar, uint16_t cta_mask) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%2, %3}], [%4], %5;\n"
               ::"r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "h"(cta_mask)
               : "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster (the own rank included).  Used to
// hand back a stage that was read by wgmma (retired by wgmma.wait_group) and is overwritten by TMA: no generic-proxy
// accesses to order, so the default .release.cta semantics suffice; .release.cluster would add a MEMBAR.GPU per arrive
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile("{\n.reg .b32 ra;\nmapa.shared::cluster.u32 ra, %0, %1;\nmbarrier.arrive.shared::cluster.b64 _, [ra];\n}\n"
               ::"r"(smem_u32(bar)), "r"(cta)
               : "memory");
}
// L2 prefetch of a 2-D tile (no shared-memory destination, no completion to wait for)
__device__ __forceinline__ void tma_prefetch_l2_2d(const void* tmap, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];\n" ::"l"(tmap), "r"(c0), "r"(c1) : "memory");
}
// 2-D TMA tile store smem -> global (SASS: UTMASTG), tracked by the issuing thread's bulk async-group
__device__ __forceinline__ void tma_store_2d(const void* tmap, int c0, int c1, uint32_t src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];\n" ::"l"(tmap), "r"(c0), "r"(c1), "r"(src)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;\n" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;\n" ::"n"(N) : "memory"); }
// ---- warp MMA (mma.sync): D[16x8] += A[16x16] B[16x8], fp16 operands, fp32 accumulate -----------------------
__device__ __forceinline__ void mma_m16n8k16(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// ---- warpgroup MMA (wgmma, sm_90a) ------------------------------------------------------------
// A warpgroup (four consecutive warps, the first a multiple of four) issues the MMA collectively; the fp32
// accumulator of an m64nN tile lives in its registers: thread (warp w of the group, lane l) holds rows
// 16 w + l / 4 and 16 w + l / 4 + 8, columns 8 j + 2 (l % 4) + {0, 1}, as d[4 j + {0, 1}] and d[4 j + {2, 3}].
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// the accumulator registers are outputs of the asynchronous MMAs until wgmma_wait retires them: keep the compiler from
// moving their uses across the wait
template <int R> __device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void wgmma_m64n192k16(float (&d)[96], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %98, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95}, %96, %97, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor (wgmma): start address >> 4 | LBO (unused for swizzled
// K-major, canonical value 1) | SBO = 8 rows * 128 B | layout type 1 (SWIZZLE_128B) in bits 62-63.  The tile base must be
// 1024-byte aligned; the K offset of a 16-element step inside the 128-byte atom is added to the start address (+2 = 32 B).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(nthreads) : "memory"); }

// ---- host: tensor maps ---------------------------------------------------------------------------------------
// Encodes a TMA descriptor of an fp16 tensor of `rank` dimensions, innermost first (byte strides of dimensions 1 ..
// rank - 1), loaded in boxes of box[] elements with the 128-byte swizzle; unit element strides, 256-byte L2
// promotion, out-of-bounds elements read as zero.  Returns DPVO_OK, or DPVO_ERR_CUDA with the error text prefixed by op.
int encode_tmap(CUtensorMap* m, const char* op, int rank, const void* ptr, const cuuint64_t* dims, const cuuint64_t* strides,
                const cuuint32_t* box);
// row-major fp16 [rows, cols] with a row stride of ld elements, in boxes of box_rows rows x 64 columns (128 bytes)
inline int encode_tmap_2d(CUtensorMap* m, const char* op, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  return encode_tmap(m, op, 2, ptr, dims, strides, box);
}

}  // namespace dpvo
