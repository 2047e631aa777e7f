// Shared helpers for the sm_90a kernels: error plumbing, PTX wrappers (mbarrier, TMA, wgmma),
// exact-rounding fp32 intrinsics.  No torch types anywhere below the C-ABI (include/frcnn_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>

namespace frcnn {

// ---- error plumbing: every C-ABI entry returns an int status; message kept per thread -------
enum Status : int {
  OK = 0, ERR_CUDA = -1, ERR_ARG = -2, ERR_NO_DEVICE = -3, ERR_DRIVER_ENTRY = -4, ERR_CAPACITY = -5
};
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define FRCNN_CUDA(expr)                                                        \
  do {                                                                          \
    cudaError_t _e = (expr);                                                    \
    if (_e != cudaSuccess) return ::frcnn::cuda_fail(_e, #expr, __FILE__, __LINE__); \
  } while (0)

#define FRCNN_LAUNCH_CHECK() FRCNN_CUDA(cudaGetLastError())

#define FRCNN_REQUIRE(cond, ...)                    \
  do {                                              \
    if (!(cond)) {                                  \
      ::frcnn::set_error(__VA_ARGS__);              \
      return ::frcnn::ERR_ARG;                      \
    }                                               \
  } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// ---- device-side PTX wrappers -------------------------------------------------------------
#if defined(__CUDACC__)

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// mbarrier ------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive that the compiler must order after the computation of `dep` (an otherwise unused register operand)
__device__ __forceinline__ void mbar_arrive_after(uint64_t* bar, uint32_t dep) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0]; // after %1" ::"r"(smem_u32(bar)), "r"(dep) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%0], %1;\n\t"
      "@P bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}\n" ::"r"(addr), "r"(parity) : "memory");
}

// ---- development watchdog (builds with -DFRCNN_WATCHDOG only: libfrcnn_b200_wd.so) -------------------------------------
// A barrier-protocol bug in a warp-specialised kernel shows up as a hang, which on a leased GPU box is a lost call with no
// information.  In watchdog builds every tagged wait gives up after ~0.2 s, records who waited on what, and raises a
// device-wide abort flag that makes every other tagged wait fall through, so the kernel terminates (with garbage) and the
// host can read the record through frcnn_debug_watchdog().  Normal builds compile MBAR_WAIT to the plain wait.
#ifdef FRCNN_WATCHDOG
static __device__ unsigned int g_watchdog[16];   // per translation unit (only conv_gemm.cu uses it)
//   // [0] abort flag, [1] count, [2..7] first record: block, thread, tag, parity, kbt, spare
__device__ __forceinline__ void mbar_wait_wd(uint64_t* bar, uint32_t parity, uint32_t tag, uint32_t aux) {
  const uint32_t addr = smem_u32(bar);
  long long t0 = 0;
  for (uint32_t it = 0;; ++it) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
                 : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
    if (ok) return;
    if ((it & 63u) == 63u) {
      if (*(volatile unsigned int*)&g_watchdog[0]) return;
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 400000000LL) {
        if (atomicAdd(&g_watchdog[1], 1u) == 0u) {
          g_watchdog[2] = blockIdx.x; g_watchdog[3] = threadIdx.x; g_watchdog[4] = tag; g_watchdog[5] = parity; g_watchdog[6] = aux;
        }
        __threadfence();
        atomicExch(&g_watchdog[0], 1u);
        return;
      }
    }
  }
}
#define MBAR_WAIT(bar, parity, tag, aux) mbar_wait_wd(bar, parity, tag, (uint32_t)(aux))
#else
#define MBAR_WAIT(bar, parity, tag, aux) mbar_wait(bar, parity)
#endif

// TMA ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// wgmma (sm_90a warpgroup MMA) ------------------------------------------------------------------
// K-major, SWIZZLE_128B shared-memory matrix descriptor (8-row x 128 B atoms, 1024 B apart; the tile is 1024-B aligned).
// Stepping K inside the 128-byte swizzle row is a plain advance of the start-address field.
__device__ __forceinline__ uint64_t wgmma_sw128_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;                  // LBO: unused for swizzled K-major
  d |= (uint64_t)(1024u >> 4) << 32;       // SBO: 8 rows x 128 B
  d |= (uint64_t)1 << 62;                  // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of an accumulator register across an asynchronous wgmma and its wait
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// D[64 x N] (+)= A[64 x K] * B[N x K]^T, fp32 accumulate in registers; A from registers (the m64k16 / m64k8 fragment of this
// thread), B from shared memory (descriptor).  scale_d = 0 starts a fresh sum.
template <int N> __device__ __forceinline__ void wgmma_f16_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d);
template <int N> __device__ __forceinline__ void wgmma_tf32_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_f16_rs<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_f16_rs<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32_rs<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32_rs<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d));
}
// register re-allocation between warp roles: every warp of a warpgroup (4 consecutive warps) executes the same one
template <int R> __device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// two fp32 -> packed fp16x2 (lo half = a, hi half = b), round to nearest even, IEEE overflow: |x| >= 65520 becomes +-Inf
// and NaN stays NaN, so an activation outside the fp16 range poisons the output instead of being clamped to a finite value
__device__ __forceinline__ uint32_t pack_f16x2_rn(float a, float b) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}

// read-only global loads the compiler may neither duplicate nor sink (asm volatile): used where the loads must be
// issued early, all together, to hide their latency (conv epilogue)
__device__ __forceinline__ float4 ld_nc_f4_pinned(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float2 ld_nc_f2_pinned(const float* p) {
  float2 v;
  asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
  return v;
}
// the same, predicated: no memory access (and zeros) when `pred` is false
__device__ __forceinline__ float2 ld_nc_f2_pinned_if(const float* p, bool pred) {
  float2 v = make_float2(0.f, 0.f);
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %3, 0;\n\t@q ld.global.nc.v2.f32 {%0, %1}, [%2];\n\t}\n"
               : "+f"(v.x), "+f"(v.y) : "l"(p), "r"((int)pred));
  return v;
}
__device__ __forceinline__ float ld_nc_f32_pinned(const float* p) {
  float v;
  asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}

// 128-bit load from a 32-bit shared-space address
__device__ __forceinline__ float4 lds_f4(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr));
  return v;
}

// programmatic dependent launch: let the next kernel in the stream start its prologue early / wait for the previous one's data
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// same rounding (nearest, ties away from zero) for finite inputs in two integer ops: add half a tf32 ulp to the magnitude
// bits, clear the low 13 bits.  cvt.rna.tf32 additionally special-cases Inf/NaN (an extra compare + select per element),
// which the operand splitter -- it shares its scheduler with the MMA-issuing warp -- does not need.
__device__ __forceinline__ float to_tf32_fast(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}

// round-to-nearest fp32 -> tf32 (result is an fp32 bit pattern with the low 13 mantissa bits clear)
__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

#endif  // __CUDACC__
}  // namespace frcnn
