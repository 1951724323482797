// fpmath.cuh — floating-point primitives with pinned rounding/flush behaviour.
//
// The reference kernels are NVRTC-compiled with --use_fast_math and then LTO-linked by
// nvJitLink WITHOUT -ftz (include/CudaModularProgram.h:84-98,225). The SASS that results on
// sm_90 (inspected with cuobjdump on oracle/_ref/*.cubin) therefore mixes
//   * plain mul/add/fma  -> FMUL / FADD / FFMA     (round-to-nearest, denormals kept)
//   * a / b              -> MUFU.RCP + FMUL.FTZ    (div.approx.ftz, front-end lowered)
//   * pow(2, l)          -> MUFU.EX2               (ex2.approx.ftz)
//   * float -> uint      -> F2I.FTZ.U32.TRUNC      (cvt.rzi.ftz.u32.f32, saturating)
// Results that are compared bit-for-bit with the reference (octree quantisation, voxel
// centres, projected depth and pixel coordinates) are computed with these wrappers, which
// emit exactly those instructions and cannot be re-contracted by ptxas (.rn is explicit).
#pragma once
#include <stdint.h>

namespace fpx {

__device__ __forceinline__ float add(float a, float b) {
    float r; asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
__device__ __forceinline__ float sub(float a, float b) {
    float r; asm("sub.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
__device__ __forceinline__ float mul(float a, float b) {
    float r; asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
__device__ __forceinline__ float mul_ftz(float a, float b) {
    float r; asm("mul.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
__device__ __forceinline__ float fma(float a, float b, float c) {
    float r; asm("fma.rn.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c)); return r;
}
__device__ __forceinline__ float rcp(float a) {          // MUFU.RCP
    float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r;
}
__device__ __forceinline__ float ex2(float a) {          // MUFU.EX2
    float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r;
}
__device__ __forceinline__ float lg2(float a) {          // MUFU.LG2
    float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r;
}
__device__ __forceinline__ float sqrt_approx(float a) {  // MUFU.SQRT
    float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r;
}
// a / b as the reference computes it: a * MUFU.RCP(b), product flushed
__device__ __forceinline__ float div_fast(float a, float b) { return mul_ftz(a, rcp(b)); }

__device__ __forceinline__ uint32_t f2u(float a) {       // F2I.FTZ.U32.TRUNC (saturating, NaN -> 0)
    uint32_t r; asm("cvt.rzi.ftz.u32.f32 %0, %1;" : "=r"(r) : "f"(a)); return r;
}
__device__ __forceinline__ int32_t f2i(float a) {        // F2I.FTZ.TRUNC
    int32_t r; asm("cvt.rzi.ftz.s32.f32 %0, %1;" : "=r"(r) : "f"(a)); return r;
}
__device__ __forceinline__ float u2f(uint32_t a) {       // I2FP.F32.U32
    float r; asm("cvt.rn.f32.u32 %0, %1;" : "=f"(r) : "r"(a)); return r;
}
__device__ __forceinline__ double dfma(double a, double b, double c) {
    double r; asm("fma.rn.f64 %0, %1, %2, %3;" : "=d"(r) : "d"(a), "d"(b), "d"(c)); return r;
}
__device__ __forceinline__ double dmul(double a, double b) {
    double r; asm("mul.rn.f64 %0, %1, %2;" : "=d"(r) : "d"(a), "d"(b)); return r;
}
__device__ __forceinline__ double dadd(double a, double b) {
    double r; asm("add.rn.f64 %0, %1, %2;" : "=d"(r) : "d"(a), "d"(b)); return r;
}
__device__ __forceinline__ int32_t d2i(double a) {       // F2I.F64.TRUNC
    int32_t r; asm("cvt.rzi.s32.f64 %0, %1;" : "=r"(r) : "d"(a)); return r;
}

}  // namespace fpx
