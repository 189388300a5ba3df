// Hopper (sm_90a) PTX wrappers shared by the fast3r_b200 kernels: mbarrier, TMA (cp.async.bulk.tensor),
// warpgroup MMA (wgmma.mma_async) and its shared-memory matrix descriptors.  Hand-written inline PTX; the descriptor
// bit layout follows the PTX ISA "matrix descriptor format" table for wgmma.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace f3r {

#define F3R_DEVICE __device__ __forceinline__

F3R_DEVICE uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

F3R_DEVICE uint32_t lane_id() { return threadIdx.x & 31; }

F3R_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------ mbarrier
F3R_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
F3R_DEVICE void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
F3R_DEVICE void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

F3R_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
F3R_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
F3R_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Blocks until the phase with the given parity has completed.
F3R_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// Same, for waits that are not latency critical (TMA producers several stages ahead): sleeps between polls so that the
// spinning warp does not take issue slots from the math warps that share its scheduler.
F3R_DEVICE void mbar_wait_relaxed(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) asm volatile("nanosleep.u32 64;");
}

// ------------------------------------------------------------------ TMA loads (tile mode)
F3R_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
F3R_DEVICE void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
F3R_DEVICE void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
F3R_DEVICE void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}

// ------------------------------------------------------------------ TMA stores (smem -> global, bulk_group completion)
F3R_DEVICE void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// global[tile] += smem[tile]  (element-wise add performed by the memory system; fp32 tensor map)
F3R_DEVICE void tma_reduce_add_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
F3R_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
F3R_DEVICE void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
F3R_DEVICE void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ------------------------------------------------------------------ programmatic dependent launch
// Kernels of the hot chain are launched with cudaLaunchAttributeProgrammaticStreamSerialization (f3r::pdl_enabled()): the
// next kernel's CTAs may become resident, run their prologue (barrier init, descriptor prefetch) and park
// at pdl_wait() while the previous kernel drains its last wave.  pdl_wait() returns when ALL memory operations of the
// preceding grid are complete and visible, so every access to global memory must come after it; pdl_launch_dependents()
// only allows the successor to be scheduled early.  Without the launch attribute both are no-ops.
F3R_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
F3R_DEVICE void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ------------------------------------------------------------------ thread-block clusters
F3R_DEVICE uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
F3R_DEVICE uint32_t cluster_id_x() { uint32_t r; asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r)); return r; }
F3R_DEVICE uint32_t num_clusters_x() { uint32_t r; asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r)); return r; }
F3R_DEVICE void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ------------------------------------------------------------------ wgmma
// Shared-memory matrix descriptor, 128-byte swizzle, rows of 128 bytes (64 bf16), 8-row groups 1024 B apart
// (tiles 1024-byte aligned, so the base-offset field stays 0).
//  K-major  (operand rows = M/N index, 64 contiguous K elements per row): LBO unused (1), SBO = 1024 B;
//           a 16-element K step inside the swizzle row is +32 B, i.e. +2 in the (addr >> 4) field.
//  MN-major (smem rows = K index, 64 contiguous M/N elements per row):    LBO unused (1), SBO = 1024 B;
//           a 16-element K step is 16 rows = +2048 B, i.e. +128 in the (addr >> 4) field.
F3R_DEVICE uint64_t make_smem_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);   // start address, bits [0,14)
  d |= static_cast<uint64_t>(1) << 16;                      // leading byte offset >> 4 (unused with 128B swizzle)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;              // stride byte offset >> 4
  d |= static_cast<uint64_t>(1) << 62;                      // SWIZZLE_128B
  return d;
}
F3R_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
F3R_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
F3R_DEVICE void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory"); }
// Keeps the compiler from moving accesses of accumulator registers across wgmma issue / wait points.
template <int kN>
F3R_DEVICE void fence_regs(float (&d)[kN]) {
#pragma unroll
  for (int i = 0; i < kN; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Accumulator fragment of an m64nN wgmma (per warpgroup): warp w of the warpgroup holds rows 16w + lane/4 (+8);
// d[4j + 2h + e] is row 16w + lane/4 + 8h, column 8j + 2 (lane % 4) + e.

// The 16-bit operand type of the tensor-core kernels: T = __nv_bfloat16 (the default) or __half, with the same
// fragment layouts and the same fp32 accumulation; only the instruction's .bf16 / .f16 type differs.
template <typename T>
constexpr bool is_f16 = std::is_same<T, __half>::value;

// D[64 x 128] (+)= A[smem] * B[smem]^T (both K-major unless trans_b: B MN-major)
#define F3R_WGMMA_SS_N128(TY) \
  asm volatile( \
      "{\n\t.reg .pred p;\n\t" \
      "setp.ne.b32 p, %66, 0;\n\t" \
      "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, %67;\n\t}\n" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
      : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(kTransB))
template <int kTransB, typename T = __nv_bfloat16>
F3R_DEVICE void wgmma_ss_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  if constexpr (is_f16<T>) F3R_WGMMA_SS_N128("f16");
  else F3R_WGMMA_SS_N128("bf16");
}

// D[64 x 256] (+)= A[smem] * B[smem]^T (both K-major unless trans_b: B MN-major)
#define F3R_WGMMA_SS_N256(TY) \
  asm volatile( \
      "{\n\t.reg .pred p;\n\t" \
      "setp.ne.b32 p, %130, 0;\n\t" \
      "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, %131;\n\t}\n" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127]) \
      : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(kTransB))
template <int kTransB, typename T = __nv_bfloat16>
F3R_DEVICE void wgmma_ss_n256(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  if constexpr (is_f16<T>) F3R_WGMMA_SS_N256("f16");
  else F3R_WGMMA_SS_N256("bf16");
}

// D[64 x 64] (+)= A[registers: 4 x packed bf16x2 per thread] * B[smem] (B MN-major if kTransB)
#define F3R_WGMMA_RS_N64(TY) \
  asm volatile( \
      "{\n\t.reg .pred p;\n\t" \
      "setp.ne.b32 p, %37, 0;\n\t" \
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}\n" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate), "n"(kTransB))
template <int kTransB, typename T = __nv_bfloat16>
F3R_DEVICE void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  if constexpr (is_f16<T>) F3R_WGMMA_RS_N64("f16");
  else F3R_WGMMA_RS_N64("bf16");
}

// ------------------------------------------------------------------ misc math
F3R_DEVICE uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);  // .x = lo (low 16 bits), .y = hi
  return *reinterpret_cast<uint32_t*>(&v);
}
F3R_DEVICE float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
F3R_DEVICE float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }
F3R_DEVICE uint32_t pack_f16(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);  // cvt.rn.f16x2.f32; .x = lo (low 16 bits), .y = hi
  return *reinterpret_cast<uint32_t*>(&v);
}
F3R_DEVICE float f16_lo(uint32_t v) { return __half2float(__ushort_as_half(static_cast<unsigned short>(v & 0xFFFFu))); }
F3R_DEVICE float f16_hi(uint32_t v) { return __half2float(__ushort_as_half(static_cast<unsigned short>(v >> 16))); }

// Conversions of one 16-bit element type: pack two fp32 values (round to nearest even) into a 32-bit pair, and unpack
// its low / high element.
template <typename T>
struct Half16 {
  static F3R_DEVICE uint32_t pack(float lo, float hi) { return pack_bf16(lo, hi); }
  static F3R_DEVICE float lo(uint32_t v) { return bf16_lo(v); }
  static F3R_DEVICE float hi(uint32_t v) { return bf16_hi(v); }
};
template <>
struct Half16<__half> {
  static F3R_DEVICE uint32_t pack(float lo, float hi) { return pack_f16(lo, hi); }
  static F3R_DEVICE float lo(uint32_t v) { return f16_lo(v); }
  static F3R_DEVICE float hi(uint32_t v) { return f16_hi(v); }
};
F3R_DEVICE float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

}  // namespace f3r
