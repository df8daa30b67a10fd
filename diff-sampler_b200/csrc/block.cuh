// Block-wide primitives of the one-CTA-per-row kernels (optimal.cu, prdc.cu).  Each combines values in an order fixed by thread and
// warp index alone, which is what makes those kernels' outputs bit-identical from call to call.
#pragma once
#include <cuda_runtime.h>

namespace dsb {

struct SumOp {
    template <class T> __device__ T operator()(T a, T b) const { return a + b; }
};
struct MaxOp {
    template <class T> __device__ T operator()(T a, T b) const { return a > b ? a : b; }
};

// Block-wide reduction over NW warps: butterfly within each warp, then every thread folds the warp totals 0, 1, ... itself.
template <int NW, class T, class Op>
__device__ __forceinline__ T block_reduce(T v, Op op, T* sh) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();                                   // `sh` may still be read by the previous reduction
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    T r = sh[0];
#pragma unroll
    for (int i = 1; i < NW; ++i) r = op(r, sh[i]);
    return r;
}

// Block argmax (kMax) or argmin over NW warps; equal values go to the lower index.  The winner is returned to every thread.
template <int NW, bool kMax>
__device__ __forceinline__ void block_argbest(float& v, int& idx, float* shf, int* shi) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, idx, o);
        if ((kMax ? v2 > v : v2 < v) || (v2 == v && i2 < idx)) { v = v2; idx = i2; }
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { shf[threadIdx.x >> 5] = v; shi[threadIdx.x >> 5] = idx; }
    __syncthreads();
    v = shf[0]; idx = shi[0];
    for (int i = 1; i < NW; ++i)
        if ((kMax ? shf[i] > v : shf[i] < v) || (shf[i] == v && shi[i] < idx)) { v = shf[i]; idx = shi[i]; }
}

// Appends index i of every flagged thread of one NW x 32-wide tile to list[n ..] in index order (warp ballots) and returns the new
// length, the same in every thread.  With kCap > 0 only positions below kCap are written, while the length keeps counting, so the
// caller can tell that the list overflowed.  The caller synchronises before reading the list.
template <int NW, int kCap = 0>
__device__ __forceinline__ int block_compact(bool f, int i, int* list, int n, int* shi) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    __syncthreads();
    if (lane == 0) shi[w] = __popc(bal);
    __syncthreads();
    int before = n, tile = 0;
    for (int ww = 0; ww < NW; ++ww) {
        if (ww < w) before += shi[ww];
        tile += shi[ww];
    }
    before += __popc(bal & ((1u << lane) - 1u));
    if (f && (kCap == 0 || before < kCap)) list[before] = i;
    return n + tile;
}

}  // namespace dsb
