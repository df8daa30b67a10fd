// The two activation-operand formats of the GEMM and attention kernels (csrc/ops.h), as the elementwise and attention kernels write
// them.  `plane` is the number of elements per plane and `o` the element offset of the first value; N consecutive values go out as one
// vector store per plane (N = 8: 16 bytes of fp16, N = 4: 8 bytes, N = 2: 4 bytes).
//   fmt 0, fp16 planes:  hi = rn(v) and, with nplanes == 2, lo = rn(v - hi) one plane further.  The GEMM epilogue (gemm_tc.cu) writes
//                        the same hi / lo planes with its own stores.
//   fmt 1, f8 image:     fp16 plane of v * 2^A16 (saturating), then the two e4m3 byte planes (v - hi) * 2^LO8 and hi * 2^HI8, where hi
//                        is the value the fp16 plane represents (ds_gemm_desc.f8).  Powers of two: the roundings are those of v.
#pragma once
#include "ops.h"
#include <cuda_fp16.h>
#include <cuda_fp8.h>

namespace dsb {

__device__ __forceinline__ void split_h16(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}

// fp16 hi / lo planes of two values: one packed convert each way (hi = rn(v), lo = rn(v - hi), as split_h16)
__device__ __forceinline__ void split_h16_pair(float v0, float v1, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(v0, v1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

// f8 image of two values.  Packed arithmetic (two values per instruction wherever the ISA has it): v * 2^A16 -> f16x2 convert -> clamp
// as half2 (a value beyond the fp16 range converts to inf and is clamped back: the same result as clamping first) -> hi byte plane
// straight from the half2 (cvt.e4m3x2.f16x2 of hi * 2^(HI8 - A16), exact: a power of two) -> lo = fma(hi, -2^(LO8 - A16), v * 2^LO8)
// = (v - hi / 2^A16) * 2^LO8 with one rounding.  7 instructions per value instead of 11 (gn_apply with this store is otherwise bound by
// instruction issue).
__device__ __forceinline__ void f8_image_pair(float v0, float v1, uint32_t& hi16, unsigned short& lo8, unsigned short& hi8) {
    constexpr float kA16 = (float)(1 << DS_F8_SH_A16), kLo8 = (float)(1 << DS_F8_SH_LO8);
    constexpr float kLoA = (float)(1 << (DS_F8_SH_LO8 - DS_F8_SH_A16));
    static_assert(DS_F8_SH_A16 >= DS_F8_SH_HI8 && DS_F8_SH_LO8 >= DS_F8_SH_A16, "operand scales");
    const __half2 lim = __float2half2_rn(65504.f);
    __half2 h = __floats2half2_rn(v0 * kA16, v1 * kA16);
    h = __hmin2(__hmax2(h, __hneg2(lim)), lim);
    hi16 = *reinterpret_cast<const uint32_t*>(&h);
    const float2 hf = __half22float2(h);
    lo8 = __nv_cvt_float2_to_fp8x2(make_float2(fmaf(hf.x, -kLoA, v0 * kLo8), fmaf(hf.y, -kLoA, v1 * kLo8)), __NV_SATFINITE, __NV_E4M3);
    const __half2 h8 = __hmul2(h, __float2half2_rn(1.0f / (float)(1 << (DS_F8_SH_A16 - DS_F8_SH_HI8))));
    hi8 = __nv_cvt_halfraw2_to_fp8x2(*reinterpret_cast<const __half2_raw*>(&h8), __NV_SATFINITE, __NV_E4M3);
}

// one vector store of BYTES bytes
template <int BYTES> struct StoreVec;
template <> struct StoreVec<4> { using T = uint32_t; };
template <> struct StoreVec<8> { using T = uint2; };
template <> struct StoreVec<16> { using T = uint4; };

template <int N>
__device__ __forceinline__ void store_planes(__half* base, long long plane, long long o, const float* v, int nplanes) {
    using V = typename StoreVec<2 * N>::T;
    __align__(2 * N) uint32_t hi[N / 2];
    __align__(2 * N) uint32_t lo[N / 2];
#pragma unroll
    for (int j = 0; j < N / 2; ++j) split_h16_pair(v[2 * j], v[2 * j + 1], hi[j], lo[j]);
    *reinterpret_cast<V*>(base + o) = *reinterpret_cast<const V*>(hi);
    if (nplanes > 1) *reinterpret_cast<V*>(base + plane + o) = *reinterpret_cast<const V*>(lo);
}

template <int N>
__device__ __forceinline__ void store_f8(__half* base, long long plane, long long o, const float* v) {
    using V16 = typename StoreVec<2 * N>::T;
    using V8 = typename StoreVec<N>::T;
    __align__(2 * N) uint32_t hi[N / 2];
    __align__(N) unsigned short lo8[N / 2];
    __align__(N) unsigned short hi8[N / 2];
#pragma unroll
    for (int j = 0; j < N / 2; ++j) f8_image_pair(v[2 * j], v[2 * j + 1], hi[j], lo8[j], hi8[j]);
    *reinterpret_cast<V16*>(base + o) = *reinterpret_cast<const V16*>(hi);
    unsigned char* b8 = reinterpret_cast<unsigned char*>(base + plane);
    *reinterpret_cast<V8*>(b8 + o) = *reinterpret_cast<const V8*>(lo8);
    *reinterpret_cast<V8*>(b8 + plane + o) = *reinterpret_cast<const V8*>(hi8);
}

// N = 4 or 8 values in format fmt (0 or 1; nplanes is 2 for the f8 image, which reuses the two-plane footprint)
template <int N>
__device__ __forceinline__ void store_operand(__half* base, long long plane, long long o, const float* v, int nplanes, int fmt) {
    if (fmt == 1) store_f8<N>(base, plane, o, v);
    else store_planes<N>(base, plane, o, v, nplanes);
}

}  // namespace dsb
