// hadamard.cuh -- element loads / stores of ct_hadamard_transform, shared by the kernel (hadamard.cu) and its CPU twin (cpu_twin.cu)
// so that both convert the same way: 16-bit inputs widen exactly, fp64 results reach 16-bit outputs through fp32 (two roundings, as
// torch's CPU conversion does).
#pragma once

#include "common.cuh"

namespace ctb {

// element dtype <-> C
template <int DT> struct Elem;
template <> struct Elem<CT_F32> {
    using T = float;
    template <class C> __host__ __device__ static C load(T v) { return (C)v; }
    __host__ __device__ static T store(float v) { return v; }
    __host__ __device__ static T store(double v) { return (float)v; }
};
template <> struct Elem<CT_BF16> {
    using T = __nv_bfloat16;
    template <class C> __host__ __device__ static C load(T v) { return (C)__bfloat162float(v); }
    __host__ __device__ static T store(float v) { return __float2bfloat16_rn(v); }
    __host__ __device__ static T store(double v) { return __float2bfloat16_rn((float)v); }
};
template <> struct Elem<CT_F16> {
    using T = __half;
    template <class C> __host__ __device__ static C load(T v) { return (C)__half2float(v); }
    __host__ __device__ static T store(float v) { return __float2half_rn(v); }
    __host__ __device__ static T store(double v) { return __float2half_rn((float)v); }
};

}  // namespace ctb
