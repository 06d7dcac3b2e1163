// Layout / precision preparation kernels: fp32 master copies -> padded 16-bit tensor-core operands.
//
// Restates on the device the per-call host work of the reference prologue: fp32 casts (rank_implicit.py:70-71),
// subject gather (:236), COSINE object norms with the zero guard (:98-105, :238-240), whitelist row gather (:220).
#pragma once
#include "common.cuh"

namespace b200 {

// One warp per row: fp32 L2 norm accumulated in fp64 (zero -> 1e-10, rank_implicit.py:103-104), plus the global maxima
// needed for the fp16 scale and for the certificate bound (non-negative floats order like their bit patterns).
// TX: the stored object type (float, __half, __nv_bfloat16), widened on load.
template <typename TX>
__global__ void row_stats_kernel(const TX* __restrict__ x, int64_t n, int d, int normalise, float* __restrict__ norms,
                                 unsigned* __restrict__ g_absmax_bits, unsigned* __restrict__ g_maxnorm_bits) {
    const int lane = threadIdx.x & 31;
    const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row >= n) return;
    double ss = 0.0;
    float amax = 0.f;
    for (int j = lane; j < d; j += 32) {
        const float v = to_f32(x[row * d + j]);
        ss = fma((double)v, (double)v, ss);
        amax = fmaxf(amax, fabsf(v));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ss += __shfl_xor_sync(B200_FULL_MASK, ss, o);
        amax = fmaxf(amax, __shfl_xor_sync(B200_FULL_MASK, amax, o));
    }
    float nrm = (float)sqrt(ss);
    const float raw_norm = nrm;
    if (nrm == 0.f) nrm = 1e-10f;
    if (lane == 0) {
        if (norms) norms[row] = nrm;
        // COSINE objects are stored pre-divided by their norm: |x/norm| <= 1 and |row|_2 ~ 1
        const float am = normalise ? amax / nrm : amax;
        const float mn = normalise ? (raw_norm == 0.f ? 0.f : 1.0000005f) : raw_norm;
        if (isfinite(am)) atomicMax(g_absmax_bits, __float_as_uint(am));
        if (isfinite(mn)) atomicMax(g_maxnorm_bits, __float_as_uint(mn));
    }
}

template <typename T>
__device__ __forceinline__ T to_tc(float v);
template <>
__device__ __forceinline__ __half to_tc<__half>(float v) {
    return __float2half_rn(v);
}
template <>
__device__ __forceinline__ __nv_bfloat16 to_tc<__nv_bfloat16>(float v) {
    return __float2bfloat16_rn(v);
}

// Power-of-two exponent e such that amax * 2^e lies in [2^13, 2^14); 0 when amax is 0 or not finite.  Both operand types
// are scaled: fp16 for its narrow range, bf16 because the tensor cores do not keep fp32-subnormal (bf16-subnormal)
// operands, so a tiny unscaled row would lose its scores entirely while eps, relative to the row's norm, stays tight.
__host__ __device__ __forceinline__ int fp16_scale_exp(float amax) {
    if (!(amax > 0.f) || !isfinite(amax)) return 0;
    int ex;
    frexpf(amax, &ex);  // amax = m * 2^ex, m in [0.5, 1)  ->  amax in [2^(ex-1), 2^ex)
    return 14 - ex;
}

// One warp per output row: out[row, 0:d_pad] = T( x[src_row, :] (/ norm) * 2^e ), zero padded in rows and columns.
// PER_ROW_EXP: e is chosen per row (subjects) and written to row_exp; otherwise `fixed_exp` (objects) is used.
// TX: the type of x (fp32 subjects; objects in their stored type), widened on load.
template <typename TX, typename T, bool PER_ROW_EXP>
__global__ void convert_rows_kernel(const TX* __restrict__ x, const int64_t* __restrict__ row_map,
                                    const int32_t* __restrict__ sel_rows, int64_t n, int64_t n_pad, int d, int d_pad,
                                    const float* __restrict__ norms, int fixed_exp, T* __restrict__ out,
                                    int32_t* __restrict__ row_exp) {
    const int lane = threadIdx.x & 31;
    const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row >= n_pad) return;
    T* o = out + row * d_pad;
    if (row >= n) {
        for (int j = lane; j < d_pad; j += 32) o[j] = to_tc<T>(0.f);
        return;
    }
    const int64_t lrow = sel_rows ? (int64_t)sel_rows[row] : row;  // compact batch row -> logical row -> physical row
    const int64_t src = row_map ? row_map[lrow] : lrow;
    const TX* xr = x + src * d;
    const float inv = norms ? norms[src] : 1.f;
    int e = fixed_exp;
    if (PER_ROW_EXP) {
        float amax = 0.f;
        for (int j = lane; j < d; j += 32) amax = fmaxf(amax, fabsf(to_f32(xr[j])));
#pragma unroll
        for (int o2 = 16; o2 > 0; o2 >>= 1) amax = fmaxf(amax, __shfl_xor_sync(B200_FULL_MASK, amax, o2));
        e = fp16_scale_exp(amax);
        if (lane == 0) row_exp[row] = e;
    }
    for (int j = lane; j < d_pad; j += 32) {
        float v = 0.f;
        if (j < d) {
            v = to_f32(xr[j]);
            if (norms) v = v / inv;
            v = ldexpf(v, e);
        }
        o[j] = to_tc<T>(v);
    }
}

// Whitelist gather of 16-bit operand rows: out[p, :] = in[pos2obj[p], :] (16-byte chunks), zero rows beyond n_pos.
__global__ void gather_rows16_kernel(const uint4* __restrict__ in, const int32_t* __restrict__ pos2obj, int64_t n_pos,
                                     int64_t n_pad, int chunks_per_row, uint4* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pad * chunks_per_row) return;
    const int64_t p = i / chunks_per_row;
    const int c = (int)(i - p * chunks_per_row);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (p < n_pos) v = in[(int64_t)pos2obj[p] * chunks_per_row + c];
    out[i] = v;
}

// fp16 / bf16 factors handed over as device tensors -> fp32 (exact widening).
__global__ void widen16_kernel(const void* __restrict__ in, int is_bf16, int64_t n, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = is_bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(in)[i]) : __half2float(reinterpret_cast<const __half*>(in)[i]);
}

__global__ void fill_f32_kernel(float* __restrict__ out, int64_t n, float v) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = v;
}

__global__ void iota_kernel(int32_t* __restrict__ out, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (int32_t)i;
}

// [n, d] row-major -> [d, n] row-major fp32 (32 x 32 tiles through shared memory); TX: the stored type, widened on load.
template <typename TX>
__global__ void transpose_kernel(const TX* __restrict__ in, int64_t n, int d, float* __restrict__ out) {
    __shared__ float tile[32][33];
    const int64_t r0 = (int64_t)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int64_t r = r0 + i;
        const int c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < n && c < d) ? to_f32(in[r * d + c]) : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i;
        const int64_t r = r0 + threadIdx.x;
        if (c < d && r < n) out[(int64_t)c * n + r] = tile[threadIdx.x][i];
    }
}

}  // namespace b200
