// Hopper warpgroup MMA (wgmma.mma_async) wrappers, one per tile width N (the PTX instruction names every
// accumulator register).  m64nNk16 bf16 and m64nNk32 e4m3, fp32 accumulators in registers: the fragment d[N/2] of
// thread t holds rows (t/32)*16 + (t%32)/4 (+8) and columns 8j + 2*(t%4) (+1).
#pragma once
#include <stdint.h>

namespace b2b {

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// accumulator operand lists: "+f"(d[i]) ... and the matching "%i, ..." register names
#define B2B_WD4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define B2B_WD8(i) B2B_WD4(i), B2B_WD4(i + 4)
#define B2B_WD16(i) B2B_WD8(i), B2B_WD8(i + 8)
#define B2B_WD32(i) B2B_WD16(i), B2B_WD16(i + 16)
#define B2B_WD64(i) B2B_WD32(i), B2B_WD32(i + 32)
#define B2B_WD128(i) B2B_WD64(i), B2B_WD64(i + 64)
#define B2B_WS8 "%0, %1, %2, %3, %4, %5, %6, %7"
#define B2B_WS16 B2B_WS8 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define B2B_WS32 B2B_WS16 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define B2B_WS64 B2B_WS32 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define B2B_WS128 B2B_WS64 ", %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"

#define B2B_WGMMA(N, R, IA, IB, IC, IA1, IA2, IA3, IB4, IC5)                                                     \
  template <>                                                                                                    \
  struct Wgmma<N> {                                                                                              \
    static __device__ __forceinline__ void bf16_ss(float (&d)[R], uint64_t a, uint64_t b, uint32_t acc) {        \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #IC ", 0;\nwgmma.mma_async.sync.aligned.m64n" #N          \
                   "k16.f32.bf16.bf16 {" B2B_WS##R "}, %" #IA ", %" #IB ", p, 1, 1, 0, 0;\n}\n"                   \
                   : B2B_WD##R(0) : "l"(a), "l"(b), "r"(acc));                                                    \
    }                                                                                                            \
    static __device__ __forceinline__ void e4m3_ss(float (&d)[R], uint64_t a, uint64_t b, uint32_t acc) {        \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #IC ", 0;\nwgmma.mma_async.sync.aligned.m64n" #N          \
                   "k32.f32.e4m3.e4m3 {" B2B_WS##R "}, %" #IA ", %" #IB ", p, 1, 1;\n}\n"                         \
                   : B2B_WD##R(0) : "l"(a), "l"(b), "r"(acc));                                                    \
    }                                                                                                            \
    /* A from registers (bf16 pairs in the accumulator-fragment order), B MN-major */                            \
    static __device__ __forceinline__ void bf16_rs_tb(float (&d)[R], const uint32_t (&a)[4], uint64_t b,         \
                                                      uint32_t acc) {                                            \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #IC5 ", 0;\nwgmma.mma_async.sync.aligned.m64n" #N         \
                   "k16.f32.bf16.bf16 {" B2B_WS##R "}, {%" #IA ", %" #IA1 ", %" #IA2 ", %" #IA3 "}, %" #IB4           \
                   ", p, 1, 1, 1;\n}\n"                                                                            \
                   : B2B_WD##R(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));               \
    }                                                                                                            \
  };

template <int N> struct Wgmma;
B2B_WGMMA(16, 8, 8, 9, 10, 9, 10, 11, 12, 13)
B2B_WGMMA(32, 16, 16, 17, 18, 17, 18, 19, 20, 21)
B2B_WGMMA(64, 32, 32, 33, 34, 33, 34, 35, 36, 37)
B2B_WGMMA(128, 64, 64, 65, 66, 65, 66, 67, 68, 69)
B2B_WGMMA(256, 128, 128, 129, 130, 129, 130, 131, 132, 133)
#undef B2B_WGMMA

}  // namespace b2b
