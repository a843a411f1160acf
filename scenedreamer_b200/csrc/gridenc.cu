// a6/a7: stand-alone multi-resolution hash / tiled grid encoder, float32 and (autocast) float16 tables, sm_90a.
//
// Behavioural contract = _gridencoder.grid_encode_forward / grid_encode_backward of the reference
// (gridencoder/src/gridencoder.cu:423-478 wrappers; :75-224 kernel_grid, :227-314
// kernel_grid_backward, :317-343 kernel_input_backward; index math :35-72).  This is the drop-in
// boundary op; the render hot path itself uses the fused kernel in render_fused.cu.
//
// GPU mapping (HBM/L2-gather bound, no tensor cores): one thread per (sample, level); the C
// features of a corner are fetched with ONE vector load (2x LDG.128 for C=8) instead of C scalar
// loads; the backward scatters with vector reductions (red.global.add.v4.f32, sm_90+) -- 2 per
// corner for C=8 instead of 8 scalar atomics; blocks are level-major (blockIdx.y = level) so a
// wave of CTAs keeps one level's table slice hot in the 126 MB L2.
//
// T = __half is the reference's autocast path (grid.py:38-39 converts the table to half when C is even; the binding
// dispatches on the table's dtype, gridencoder.cu:442-444): table, outputs, dy_dx, grad and grad_inputs are half, the
// coordinates stay float32.  The reference computes it with c10::Half, whose every operator returns through a float
// and rounds back (Half += float rounds the addend FIRST, then the sum; Half - Half and Half * Half round their result) --
// `hr()` below marks each of those roundings, so forward and dy_dx are bit-identical; the table gradient accumulates with
// half2 atomics (:299-305) and is order-dependent in both implementations.
#include <cuda_fp16.h>

#include <cstdlib>

#include "common.cuh"

namespace {

__device__ __constant__ uint32_t kPrimes[7] = {1u, 2654435761u, 805459861u, 3674653429u,
                                               2097192037u, 1434869437u, 2165219737u};

template <uint32_t D>
__device__ __forceinline__ uint32_t grid_index(uint32_t gridtype, bool align_corners, uint32_t hashmap_size,
                                               uint32_t resolution, const uint32_t (&pg)[D]) {
    uint32_t stride = 1, index = 0;
#pragma unroll
    for (uint32_t d = 0; d < D; d++) {
        if (stride <= hashmap_size) {
            index += pg[d] * stride;
            stride *= align_corners ? resolution : (resolution + 1);
        }
    }
    if (gridtype == 0 && stride > hashmap_size) {
        uint32_t h = 0;
#pragma unroll
        for (uint32_t d = 0; d < D; d++) h ^= pg[d] * kPrimes[d];
        index = h;
    }
    return index % hashmap_size;
}

template <uint32_t C>
__device__ __forceinline__ void load_feat(const float *__restrict__ g, float (&v)[C]) {
    if constexpr (C == 8) {
        const float4 a = __ldg(reinterpret_cast<const float4 *>(g));
        const float4 b = __ldg(reinterpret_cast<const float4 *>(g) + 1);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else if constexpr (C == 4) {
        const float4 a = __ldg(reinterpret_cast<const float4 *>(g));
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    } else if constexpr (C == 2) {
        const float2 a = __ldg(reinterpret_cast<const float2 *>(g));
        v[0] = a.x; v[1] = a.y;
    } else {
        v[0] = __ldg(g);
    }
}
// half features: one vector load of C halves (16 B for C = 8), widened to float registers
template <uint32_t C>
__device__ __forceinline__ void load_feat(const __half *__restrict__ g, float (&v)[C]) {
    static_assert(C % 2 == 0, "half tables: even C only (grid.py:38)");
    uint32_t w[C / 2];
    if constexpr (C == 8) {
        const uint4 a = __ldg(reinterpret_cast<const uint4 *>(g));
        w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
    } else if constexpr (C == 4) {
        const uint2 a = __ldg(reinterpret_cast<const uint2 *>(g));
        w[0] = a.x; w[1] = a.y;
    } else {
        w[0] = __ldg(reinterpret_cast<const uint32_t *>(g));
    }
#pragma unroll
    for (uint32_t k = 0; k < C / 2; k++) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&w[k]));
        v[2 * k] = f.x;
        v[2 * k + 1] = f.y;
    }
}
template <uint32_t C>
__device__ __forceinline__ void store_feat(float *__restrict__ o, const float (&v)[C]) {
#pragma unroll
    for (uint32_t c = 0; c < C; c++) o[c] = v[c];
}
template <uint32_t C>
__device__ __forceinline__ void store_feat(__half *__restrict__ o, const float (&v)[C]) {   // v already holds half values
    uint32_t w[C / 2];
#pragma unroll
    for (uint32_t k = 0; k < C / 2; k++) {
        const __half2 h = __floats2half2_rn(v[2 * k], v[2 * k + 1]);
        w[k] = *reinterpret_cast<const uint32_t *>(&h);
    }
    if constexpr (C == 8) *reinterpret_cast<uint4 *>(o) = make_uint4(w[0], w[1], w[2], w[3]);
    else if constexpr (C == 4) *reinterpret_cast<uint2 *>(o) = make_uint2(w[0], w[1]);
    else *reinterpret_cast<uint32_t *>(o) = w[0];
}
// one c10::Half rounding (float -> half -> float); identity for float tables
template <typename T>
__device__ __forceinline__ float hr(float x) {
    if constexpr (sizeof(T) == 2) return __half2float(__float2half_rn(x));
    else return x;
}

template <uint32_t D>
__device__ __forceinline__ bool locate(const float *__restrict__ x, float scale, bool align_corners,
                                       float (&pos)[D], uint32_t (&pg)[D]) {
    bool oob = false;
#pragma unroll
    for (uint32_t d = 0; d < D; d++) {
        const float v = x[d];
        if (v < 0 || v > 1) oob = true;
        pos[d] = v * scale + (align_corners ? 0.0f : 0.5f);
        const float fl = floorf(pos[d]);
        pg[d] = (uint32_t)fl;
        pos[d] -= (float)pg[d];
    }
    return oob;
}

template <typename T, uint32_t D, uint32_t C, int MINB>
__global__ void __launch_bounds__(256, MINB)
grid_forward_kernel(const float *__restrict__ inputs, const T *__restrict__ grid,
                    const int *__restrict__ offsets, T *__restrict__ outputs, uint32_t B, uint32_t L,
                    float S, uint32_t H, bool calc_grad_inputs, T *__restrict__ dy_dx, uint32_t gridtype,
                    bool align_corners)
{
    constexpr bool kHalf = sizeof(T) == 2;
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint32_t level = blockIdx.y;
    grid += (size_t)(uint32_t)offsets[level] * C;
    T *out = outputs + ((size_t)level * B + b) * C;
    const uint32_t hashmap_size = offsets[level + 1] - offsets[level];
    const float scale = exp2f(level * S) * H - 1.0f;
    const uint32_t resolution = (uint32_t)ceilf(scale) + 1;

    float pos[D];
    uint32_t pg[D];
    const bool oob = locate<D>(inputs + (size_t)b * D, scale, align_corners, pos, pg);
    if (oob) {
        float zero[C];
#pragma unroll
        for (uint32_t c = 0; c < C; c++) zero[c] = 0;
        store_feat<C>(out, zero);
        if (calc_grad_inputs) {
            T *dd = dy_dx + ((size_t)b * L + level) * D * C;
#pragma unroll
            for (uint32_t k = 0; k < D; k++) store_feat<C>(dd + k * C, zero);
        }
        return;
    }
    float res[C];
#pragma unroll
    for (uint32_t c = 0; c < C; c++) res[c] = 0;

    if constexpr (!kHalf) {
        // float32: ONE pass over the 2^D corners feeds the interpolation and all D derivative rows.  d out / d x_gd is
        // scale * sum over corners of (+-1 by the corner's side along gd) * (product of the OTHER axes' weights) * feature;
        // the reference walks the corners once more per axis (160 more gathers per (sample, level) at D = 5,
        // gridencoder.cu:180-222) -- same sum, different association (parity 1e-6 relative, tests/test_gpu_ops.py).
        // The interpolation itself keeps the reference's order of operations exactly.
        float rg[D][C];
#pragma unroll
        for (uint32_t gd = 0; gd < D; gd++)
#pragma unroll
            for (uint32_t c = 0; c < C; c++) rg[gd][c] = 0;
#pragma unroll
        for (uint32_t idx = 0; idx < (1u << D); idx++) {
            float wd[D], pre[D + 1];
            uint32_t pl[D];
            pre[0] = 1;
#pragma unroll
            for (uint32_t d = 0; d < D; d++) {
                if ((idx & (1u << d)) == 0) { wd[d] = 1 - pos[d]; pl[d] = pg[d]; }
                else { wd[d] = pos[d]; pl[d] = pg[d] + 1; }
                pre[d + 1] = pre[d] * wd[d];
            }
            const uint32_t index = grid_index<D>(gridtype, align_corners, hashmap_size, resolution, pl);
            float v[C];
            load_feat<C>(grid + (size_t)index * C, v);
#pragma unroll
            for (uint32_t c = 0; c < C; c++) res[c] += pre[D] * v[c];
            if (calc_grad_inputs) {
                float suf = 1;
#pragma unroll
                for (int gd = (int)D - 1; gd >= 0; gd--) {
                    const float e = pre[gd] * suf;
                    const float coef = (idx & (1u << gd)) ? e : -e;
#pragma unroll
                    for (uint32_t c = 0; c < C; c++) rg[gd][c] += coef * v[c];
                    suf *= wd[gd];
                }
            }
        }
        store_feat<C>(out, res);
        if (calc_grad_inputs) {
            T *dd = dy_dx + ((size_t)b * L + level) * D * C;
#pragma unroll
            for (uint32_t gd = 0; gd < D; gd++) {
#pragma unroll
                for (uint32_t c = 0; c < C; c++) rg[gd][c] *= scale;
                store_feat<C>(dd + gd * C, rg[gd]);
            }
        }
        return;
    }

    // float16 tables: the reference's loop structure, every c10::Half rounding in place (bit-identical results)
#pragma unroll
    for (uint32_t idx = 0; idx < (1u << D); idx++) {
        float w = 1;
        uint32_t pl[D];
#pragma unroll
        for (uint32_t d = 0; d < D; d++) {
            if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
            else { w *= pos[d]; pl[d] = pg[d] + 1; }
        }
        const uint32_t index = grid_index<D>(gridtype, align_corners, hashmap_size, resolution, pl);
        float v[C];
        load_feat<C>(grid + (size_t)index * C, v);
#pragma unroll
        for (uint32_t c = 0; c < C; c++) res[c] = hr<T>(res[c] + hr<T>(w * v[c]));      // Half += float (:166)
    }
    store_feat<C>(out, res);

    if (calc_grad_inputs) {
        T *dd = dy_dx + ((size_t)b * L + level) * D * C;
#pragma unroll
        for (uint32_t gd = 0; gd < D; gd++) {
            float rg[C];
#pragma unroll
            for (uint32_t c = 0; c < C; c++) rg[c] = 0;
#pragma unroll
            for (uint32_t idx = 0; idx < (1u << (D - 1)); idx++) {
                float w = scale;
                uint32_t pl[D];
#pragma unroll
                for (uint32_t nd = 0; nd < D - 1; nd++) {
                    const uint32_t d = (nd >= gd) ? (nd + 1) : nd;
                    if ((idx & (1u << nd)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                pl[gd] = pg[gd];
                const uint32_t il = grid_index<D>(gridtype, align_corners, hashmap_size, resolution, pl);
                pl[gd] = pg[gd] + 1;
                const uint32_t ir = grid_index<D>(gridtype, align_corners, hashmap_size, resolution, pl);
                float vl[C], vr[C];
                load_feat<C>(grid + (size_t)il * C, vl);
                load_feat<C>(grid + (size_t)ir * C, vr);
#pragma unroll
                for (uint32_t c = 0; c < C; c++) rg[c] = hr<T>(rg[c] + hr<T>(w * hr<T>(vr[c] - vl[c])));   // (:213)
            }
            store_feat<C>(dd + gd * C, rg);
        }
    }
}

template <uint32_t C>
__device__ __forceinline__ void red_add(float *__restrict__ g, const float (&v)[C]) {
    if constexpr (C == 8) {
        atomicAdd(reinterpret_cast<float4 *>(g), make_float4(v[0], v[1], v[2], v[3]));
        atomicAdd(reinterpret_cast<float4 *>(g) + 1, make_float4(v[4], v[5], v[6], v[7]));
    } else if constexpr (C == 4) {
        atomicAdd(reinterpret_cast<float4 *>(g), make_float4(v[0], v[1], v[2], v[3]));
    } else if constexpr (C == 2) {
        atomicAdd(reinterpret_cast<float2 *>(g), make_float2(v[0], v[1]));
    } else {
        atomicAdd(g, v[0]);
    }
}

// half table gradient: (__half)(w * g) pairs added with half2 atomics, as the reference does (:299-305)
template <uint32_t C>
__device__ __forceinline__ void red_add(__half *__restrict__ g, const float (&v)[C]) {
#pragma unroll
    for (uint32_t c = 0; c < C; c += 2) atomicAdd(reinterpret_cast<__half2 *>(g + c), __floats2half2_rn(v[c], v[c + 1]));
}

template <typename T, uint32_t D, uint32_t C>
__global__ void __launch_bounds__(256)
grid_backward_kernel(const T *__restrict__ grad, const float *__restrict__ inputs,
                     const int *__restrict__ offsets, T *__restrict__ grad_grid, uint32_t B, uint32_t L,
                     float S, uint32_t H, uint32_t gridtype, bool align_corners)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint32_t level = blockIdx.y;
    grad_grid += (size_t)(uint32_t)offsets[level] * C;
    const uint32_t hashmap_size = offsets[level + 1] - offsets[level];
    const float scale = exp2f(level * S) * H - 1.0f;
    const uint32_t resolution = (uint32_t)ceilf(scale) + 1;
    float pos[D];
    uint32_t pg[D];
    if (locate<D>(inputs + (size_t)b * D, scale, align_corners, pos, pg)) return;  // grad pre-zeroed
    float g[C];
    load_feat<C>(grad + ((size_t)level * B + b) * C, g);
#pragma unroll
    for (uint32_t idx = 0; idx < (1u << D); idx++) {
        float w = 1;
        uint32_t pl[D];
#pragma unroll
        for (uint32_t d = 0; d < D; d++) {
            if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
            else { w *= pos[d]; pl[d] = pg[d] + 1; }
        }
        const uint32_t index = grid_index<D>(gridtype, align_corners, hashmap_size, resolution, pl);
        float v[C];
#pragma unroll
        for (uint32_t c = 0; c < C; c++) v[c] = w * g[c];
        red_add<C>(grad_grid + (size_t)index * C, v);
    }
}

template <typename T, uint32_t D, uint32_t C>
__global__ void __launch_bounds__(256)
input_backward_kernel(const T *__restrict__ grad, const T *__restrict__ dy_dx,
                      T *__restrict__ grad_inputs, uint32_t B, uint32_t L)
{
    const uint32_t t = threadIdx.x + blockIdx.x * blockDim.x;
    if (t >= B * D) return;
    const uint32_t b = t / D, d = t - b * D;
    const T *dd = dy_dx + (size_t)b * L * D * C;
    float r = 0;
    for (uint32_t l = 0; l < L; l++) {
        float g[C], y[C];
        load_feat<C>(grad + ((size_t)l * B + b) * C, g);
        load_feat<C>(dd + (l * D + d) * C, y);
#pragma unroll
        for (uint32_t c = 0; c < C; c++) {
            if constexpr (sizeof(T) == 2) r = hr<T>(r + hr<T>(g[c] * y[c]));      // Half += Half * Half (:338)
            else r += g[c] * y[c];
        }
    }
    if constexpr (sizeof(T) == 2) grad_inputs[t] = __float2half_rn(r);
    else grad_inputs[t] = r;
}

template <uint32_t D, uint32_t C, typename T>
int launch_fwd(const float *in, const T *emb, const int *off, T *out, uint32_t B, uint32_t L, float S,
               uint32_t H, bool calc, T *dy_dx, uint32_t gt, bool ac, cudaStream_t st) {
    dim3 grid(sdb_div_up(B, 256u), L);
    // the float32 kernel with dy_dx holds D*C + C accumulators and 2^D gathers in flight: two CTAs per SM cap it at 128
    // registers (a few spills).  Two was the faster choice at D=5, C=8 on the previous GPU generation; carried over, not
    // re-measured on H100.  SDB_GRIDENC_MINB=1 selects the other build.
    static const int minb = [] { const char *e = getenv("SDB_GRIDENC_MINB"); return e ? atoi(e) : 2; }();
    if (minb == 2 && D * C >= 32)
        grid_forward_kernel<T, D, C, 2><<<grid, 256, 0, st>>>(in, emb, off, out, B, L, S, H, calc, dy_dx, gt, ac);
    else
        grid_forward_kernel<T, D, C, 1><<<grid, 256, 0, st>>>(in, emb, off, out, B, L, S, H, calc, dy_dx, gt, ac);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}
template <uint32_t D, uint32_t C, typename T>
int launch_bwd(const T *grad, const float *in, const int *off, T *gg, uint32_t B, uint32_t L, float S,
               uint32_t H, bool calc, const T *dy_dx, T *gi, uint32_t gt, bool ac, cudaStream_t st) {
    dim3 grid(sdb_div_up(B, 256u), L);
    grid_backward_kernel<T, D, C><<<grid, 256, 0, st>>>(grad, in, off, gg, B, L, S, H, gt, ac);
    SDB_CHECK_LAUNCH();
    if (calc) {
        input_backward_kernel<T, D, C><<<sdb_div_up(B * D, 256u), 256, 0, st>>>(grad, dy_dx, gi, B, L);
        SDB_CHECK_LAUNCH();
    }
    return SDB_OK;
}

}  // namespace

#define SDB_DISPATCH_DC(FN, ...)                                          \
    switch (D * 16 + C) {                                                 \
        case 2 * 16 + 1: return FN<2, 1>(__VA_ARGS__);                    \
        case 2 * 16 + 2: return FN<2, 2>(__VA_ARGS__);                    \
        case 2 * 16 + 4: return FN<2, 4>(__VA_ARGS__);                    \
        case 2 * 16 + 8: return FN<2, 8>(__VA_ARGS__);                    \
        case 3 * 16 + 1: return FN<3, 1>(__VA_ARGS__);                    \
        case 3 * 16 + 2: return FN<3, 2>(__VA_ARGS__);                    \
        case 3 * 16 + 4: return FN<3, 4>(__VA_ARGS__);                    \
        case 3 * 16 + 8: return FN<3, 8>(__VA_ARGS__);                    \
        case 4 * 16 + 1: return FN<4, 1>(__VA_ARGS__);                    \
        case 4 * 16 + 2: return FN<4, 2>(__VA_ARGS__);                    \
        case 4 * 16 + 4: return FN<4, 4>(__VA_ARGS__);                    \
        case 4 * 16 + 8: return FN<4, 8>(__VA_ARGS__);                    \
        case 5 * 16 + 1: return FN<5, 1>(__VA_ARGS__);                    \
        case 5 * 16 + 2: return FN<5, 2>(__VA_ARGS__);                    \
        case 5 * 16 + 4: return FN<5, 4>(__VA_ARGS__);                    \
        case 5 * 16 + 8: return FN<5, 8>(__VA_ARGS__);                    \
        default: return SDB_EUNSUPPORTED;                                 \
    }

extern "C" int sdb_grid_encode_forward(
    const float *d_inputs, const float *d_embeddings, const int32_t *d_offsets, float *d_outputs,
    uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
    int calc_grad_inputs, float *d_dy_dx, uint32_t gridtype, int align_corners, void *stream)
{
    if (!d_inputs || !d_embeddings || !d_offsets || !d_outputs) return SDB_EINVAL;
    if (calc_grad_inputs && !d_dy_dx) return SDB_EINVAL;
    if (B == 0 || L == 0) return SDB_OK;
    SDB_DISPATCH_DC(launch_fwd, d_inputs, d_embeddings, d_offsets, d_outputs, B, L, S, H, calc_grad_inputs != 0,
                    d_dy_dx, gridtype, align_corners != 0, (cudaStream_t)stream)
}

extern "C" int sdb_grid_encode_backward(
    const float *d_grad, const float *d_inputs, const float *d_embeddings, const int32_t *d_offsets,
    float *d_grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
    int calc_grad_inputs, const float *d_dy_dx, float *d_grad_inputs, uint32_t gridtype,
    int align_corners, void *stream)
{
    (void)d_embeddings;
    if (!d_grad || !d_inputs || !d_offsets || !d_grad_embeddings) return SDB_EINVAL;
    if (calc_grad_inputs && (!d_dy_dx || !d_grad_inputs)) return SDB_EINVAL;
    if (B == 0 || L == 0) return SDB_OK;
    SDB_DISPATCH_DC(launch_bwd, d_grad, d_inputs, d_offsets, d_grad_embeddings, B, L, S, H, calc_grad_inputs != 0,
                    d_dy_dx, d_grad_inputs, gridtype, align_corners != 0, (cudaStream_t)stream)
}

#define SDB_DISPATCH_DC_EVEN(FN, ...)                                     \
    switch (D * 16 + C) {                                                 \
        case 2 * 16 + 2: return FN<2, 2>(__VA_ARGS__);                    \
        case 2 * 16 + 4: return FN<2, 4>(__VA_ARGS__);                    \
        case 2 * 16 + 8: return FN<2, 8>(__VA_ARGS__);                    \
        case 3 * 16 + 2: return FN<3, 2>(__VA_ARGS__);                    \
        case 3 * 16 + 4: return FN<3, 4>(__VA_ARGS__);                    \
        case 3 * 16 + 8: return FN<3, 8>(__VA_ARGS__);                    \
        case 4 * 16 + 2: return FN<4, 2>(__VA_ARGS__);                    \
        case 4 * 16 + 4: return FN<4, 4>(__VA_ARGS__);                    \
        case 4 * 16 + 8: return FN<4, 8>(__VA_ARGS__);                    \
        case 5 * 16 + 2: return FN<5, 2>(__VA_ARGS__);                    \
        case 5 * 16 + 4: return FN<5, 4>(__VA_ARGS__);                    \
        case 5 * 16 + 8: return FN<5, 8>(__VA_ARGS__);                    \
        default: return SDB_EUNSUPPORTED;                                 \
    }

// float16 tables (the reference under autocast; even C only -- grid.py:38 keeps odd C in float32)
extern "C" int sdb_grid_encode_forward_f16(
    const float *d_inputs, const void *d_embeddings, const int32_t *d_offsets, void *d_outputs,
    uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
    int calc_grad_inputs, void *d_dy_dx, uint32_t gridtype, int align_corners, void *stream)
{
    if (!d_inputs || !d_embeddings || !d_offsets || !d_outputs) return SDB_EINVAL;
    if (calc_grad_inputs && !d_dy_dx) return SDB_EINVAL;
    if (B == 0 || L == 0) return SDB_OK;
    SDB_DISPATCH_DC_EVEN(launch_fwd, d_inputs, (const __half *)d_embeddings, d_offsets, (__half *)d_outputs, B, L, S, H,
                         calc_grad_inputs != 0, (__half *)d_dy_dx, gridtype, align_corners != 0, (cudaStream_t)stream)
}

extern "C" int sdb_grid_encode_backward_f16(
    const void *d_grad, const float *d_inputs, const void *d_embeddings, const int32_t *d_offsets,
    void *d_grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
    int calc_grad_inputs, const void *d_dy_dx, void *d_grad_inputs, uint32_t gridtype,
    int align_corners, void *stream)
{
    (void)d_embeddings;
    if (!d_grad || !d_inputs || !d_offsets || !d_grad_embeddings) return SDB_EINVAL;
    if (calc_grad_inputs && (!d_dy_dx || !d_grad_inputs)) return SDB_EINVAL;
    if (B == 0 || L == 0) return SDB_OK;
    SDB_DISPATCH_DC_EVEN(launch_bwd, (const __half *)d_grad, d_inputs, d_offsets, (__half *)d_grad_embeddings, B, L, S, H,
                         calc_grad_inputs != 0, (const __half *)d_dy_dx, (__half *)d_grad_inputs, gridtype, align_corners != 0,
                         (cudaStream_t)stream)
}
