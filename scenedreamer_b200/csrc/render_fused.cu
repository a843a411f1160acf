// Fused per-pixel render for sm_90a: depth sampling -> label lookup -> hash-grid features ->
// style-modulated sigma/colour MLP on wgmma tensor cores -> front-to-back compositing + sky blend,
// plus the per-ray sky MLP on the same tensor-core engine.
//
// Behavioural contract = Generator._forward_perpix of the reference and the tile loop around it
// (imaginaire/generators/scenedreamer.py:285-428, :600-628) with its callees
//   mc_utils.sample_depth_batched        mc_utils.py:82-151     (a2)
//   NaN guard / world coords / labels    scenedreamer.py:350-363 (a3, a4)
//   normalise + scene code + GridEncoder scenedreamer.py:298-303, gridencoder.cu:75-170 (a5, a6)
//   LightningMLP / ModLinear             model_utils/layers.py:92-126, :241-271 (a8)
//   PE + SKYMLP                          voxlib/positional_encoding_kernel.cu:40-75, gancraft_base.py:150-169 (a9)
//   volum_rendering_relu + blending      mc_utils.py:154-161, scenedreamer.py:373-413 (a10, a11)
//
// Design (DESIGN.md has the long version)
//   * persistent CTAs (one per SM); a work item is a 16x8-pixel ray tile = 128 rays = the M of every
//     GEMM; row r of every GEMM is ray r, the tile is walked sample by sample (s = 0..S-1),
//     so compositing is a per-thread running sum (no cross-thread reduction, any S);
//   * warp roles: 8 epilogue warps (accumulator row -> LeakyReLU -> 16-bit operand in smem; sigma tap;
//     compositing; warps 0-3 own columns 0..127, warps 4-7 columns 128..255 of the same 128 rows),
//     one MMA warpgroup (wgmma in 64x64 blocks), 8 gather warps (hash-grid fetch for the NEXT sample step
//     while the MLP of the current one runs; results wait in registers until the operand buffer is free),
//     one producer warpgroup (one thread streams the weights into a 4-slot ring with 1-D bulk TMA copies);
//   * accumulators: a layer's fp32 [128 x 256] result (128 KB) fits neither next to the operand buffers in
//     shared memory nor in the registers the three roles share.  The column blocks that finish after the
//     layer's MMAs have read their operand columns are staged there in fp32 (half of a hidden layer, all of
//     the last; hand_plan), the others go to a per-CTA buffer pair in global memory (L2-resident, ping-pong
//     by layer parity), and the epilogue reads its rows from either; MMA and epilogue hand a layer over per
//     64-row block, so the epilogue of one row block runs while the MMAs of the other do;
//   * fc_1's bias and the label embedding ride in layer 0's GEMM: its operand has 16 extra K columns
//     (one-hot label + constant 1), the weight image carries bias / embedding rows there -- exactly
//     the reference's fc_m_a(onehot) product; the biases of the later layers (style beta included) are
//     fp32 adds where the MMA warpgroup writes a block out, so the epilogue is LeakyReLU + 16-bit split only;
//   * the 16-bit activations stay on chip: ONE in-place 128x256 operand buffer in shared memory; the
//     per-sample L2 traffic is the table gather plus the accumulator round trip above;
//   * precision: 0 = one fp16 pass; 1 / 2 = bf16 / fp16 "x3" split (x_hi*W_hi + x_lo*W_hi + x_hi*W_lo:
//     ~2^-16 resp. ~2^-21 relative, i.e. fp32-grade for the 1e-3 parity bar); accumulation is fp32;
//   * sky-only tiles never reach the render kernel: a pre-pass writes their outputs and compacts the
//     list of live tiles (their compositing weights are exactly zero, scenedreamer.py:376).
//   * early termination + dynamic tile scheduling (inference): a tile stops marching once every live ray is opaque
//     (one-step-delayed decision, see ESTOP below); further tiles are drawn from a global counter;
//   * training: the TRAIN variants additionally leave a per-sample record in HBM, and the same engine runs the
//     data-gradient chains (MODE kBwd / kSkyBwd: transposed weights, LeakyReLU' from recorded sign words);
//     render_train.cu holds the rest of the backward (compositing, table scatter, weight-gradient GEMMs).
#include <stdlib.h>

#include <map>
#include <mutex>
#include <utility>

#include "rf_common.cuh"

namespace rf {

int32_t *g_debug_buffer = nullptr;

// ---- sampling (a2/a3) ------------------------------------------------------------------------------
struct Sample { float depth, nd; int idx; };

__device__ __forceinline__ Sample sample_at(const Params &p, const float *st, int row, int k, const float *frac,
                                            long long ray) {
    const float total = st[kStTotal * kRows + row];
    float r0, r1;
    if (p.uniforms == nullptr) {          // deterministic: linspace fractions * total (mc_utils.py:118-126)
        r0 = __fmul_rn(frac[k], total);
        r1 = __fmul_rn(frac[k + 1], total);
    } else {                              // stratified: (u / nsamples + k / nsamples) * total (:122-126)
        // a ray without intervals samples at 0 whatever u is; rows of a tile outside the image are such rays, and their `ray`
        // lies past the image (past the end of the uniforms for the last one), so their u is not read
        const float ns = (float)(p.S + 1);
        const bool any = total > 0.0f;
        const float u0 = any ? __ldg(p.uniforms + ray * (p.S + 1) + k) : 0.0f;
        const float u1 = any ? __ldg(p.uniforms + ray * (p.S + 1) + k + 1) : 0.0f;
        r0 = __fmul_rn(__fadd_rn(__fdiv_rn(u0, ns), frac[k]), total);
        r1 = __fmul_rn(__fadd_rn(__fdiv_rn(u1, ns), frac[k + 1]), total);
    }
    Sample s;
    const float mid = __fmul_rn(__fadd_rn(r1, r0), 0.5f);     // (a + b) / 2 (:134)
    s.nd = __fsub_rn(r1, r0);                                   // :135
    int idx = 0;
#pragma unroll
    for (int j = 0; j < kMaxM; j++)
        if (j < p.M && mid > st[(kStAccu + j) * kRows + row]) idx++;   // :139 (strict >)
    if (idx > p.M - 1) idx = p.M - 1;
    s.idx = idx;
    float d = __fadd_rn(st[(kStHeads + idx) * kRows + row], mid);      // :145-149
    if (!(fabsf(d) <= 3.402823466e38f)) d = 0.0f;                      // NaN / inf -> 0 (scenedreamer.py:350-352)
    s.depth = d;
    return s;
}

// per-ray sampling state (mc_utils.py:102-107, :141-143) of pixel `pix` of image `img` into row `row` of state buffer st: the
// accumulated interval lengths, the interval heads, the total length, the labels (4 bits per interval) and the ray direction.
// A pixel outside the image (!valid) gets the state of a ray without intervals.  Returns the first and the last voxel id.
struct RayVoxels { int32_t first, last; };
__device__ __forceinline__ RayVoxels ray_state(const Params &p, float *st, int row, int img, long long pix, bool valid) {
    const long long hw = (long long)p.H * p.W, ray = img * hw + pix;
    float accu = 0.0f, cum = 0.0f, entry0 = 0.0f, prev_exit = 0.0f;
    uint32_t labs = 0;
    RayVoxels v{0, 0};
#pragma unroll
    for (int j = 0; j < kMaxM; j++) {
        if (j < p.M) {
            float en = 0.0f, ex = 0.0f;
            int32_t id = 0;
            if (valid) {
                id = __ldg(p.voxel_id + ray * p.M + j);
                en = __ldg(p.depth2 + ((long long)img * 2 + 0) * hw * p.M + pix * p.M + j);
                ex = __ldg(p.depth2 + ((long long)img * 2 + 1) * hw * p.M + pix * p.M + j);
            }
            float d = __fsub_rn(ex, en);                       // mc_utils.py:102-104
            if (d != d) d = 0.0f;
            accu = (j == 0) ? d : __fadd_rn(accu, d);
            st[(kStAccu + j) * kRows + row] = accu;
            if (j == 0) {
                entry0 = en;
                st[(kStHeads + 0) * kRows + row] = en;
            } else {                                           // :141-143
                const float dd = __fsub_rn(en, prev_exit);
                cum = (j == 1) ? dd : __fadd_rn(cum, dd);
                st[(kStHeads + j) * kRows + row] = __fadd_rn(cum, entry0);
            }
            prev_exit = ex;
            const int lid = (id >= 0 && id < p.n_lut) ? __ldg(p.lut + id) : 0;
            labs |= ((uint32_t)lid & 15u) << (4 * j);
            if (j == 0) v.first = id;
            v.last = id;
        }
    }
    st[kStTotal * kRows + row] = fminf(accu, p.sample_depth);   // :107
    st[kStLab * kRows + row] = __uint_as_float(labs);
#pragma unroll
    for (int k = 0; k < 3; k++) st[(kStDir + k) * kRows + row] = valid ? __ldg(p.raydirs + ray * 3 + k) : 0.0f;
    return v;
}

// world position of the sample at depth t on the ray (dir, ori) -> grid coordinate x[0..2] in [0,1] inside the volume, with
// the reference's operation order (scenedreamer.py:354, :299; grid.py:144): p = dir*t + ori; p / dim * 2 - 1; (x + 1) / 2.
// Returns whether the sample lies outside the volume (gridencoder.cu:98-104).
__device__ __forceinline__ bool grid_coord(const Params &p, const float (&dir)[3], const float (&ori)[3], float t, float (&x)[5]) {
    bool out = false;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float pw = __fadd_rn(__fmul_rn(dir[k], t), ori[k]);
        const float nrm = __fsub_rn(__fmul_rn(__fdiv_rn(pw, p.vdim[k]), 2.0f), 1.0f);
        x[k] = __fmul_rn(__fadd_rn(nrm, 1.0f), 0.5f);
        if (x[k] < 0.0f || x[k] > 1.0f) out = true;
    }
    return out;
}

// compositing weight of one sample (mc_utils.py:155): w = (1 - exp(-e)) * exp(-E) with e = relu(sigma) * interval and E the
// sum of e over the samples in front of it (Eexcl, advanced by e)
__device__ __forceinline__ float sample_weight(float sigma, float nd, float dists_scale, float &Eexcl) {
    const float e = __fmul_rn(fmaxf(sigma, 0.0f), __fmul_rn(nd, dists_scale));
    const float a = 1.0f - expf(-e);
    const float b = expf(-Eexcl);
    Eexcl = __fadd_rn(Eexcl, e);
    return a * b;
}

// the sample's weight w into the ray's opacity and depth sums.  depth = sum w*t with t of several hundred voxels: 1e-3
// absolute is ~16 ulp of the running sum, so the 24..64-term sum is carried compensated (exact product error + two-sum);
// costs 8 flops per sample
__device__ __forceinline__ void composite_add(float w, float depth, float &Wsum, float &Dsum, float &Dcomp) {
    Wsum += w;
    const float pr = __fmul_rn(w, depth);
    const float pe = __fmaf_rn(w, depth, -pr);
    const float sn = __fadd_rn(Dsum, pr);
    const float bv = __fsub_rn(sn, Dsum);
    Dcomp = __fadd_rn(Dcomp, __fadd_rn(__fadd_rn(__fsub_rn(Dsum, __fsub_rn(sn, bv)), __fsub_rn(pr, bv)), pe));
    Dsum = sn;
}

// the sample's colour c into the ray's running sum (scenedreamer.py:407-408)
template <int NC>
__device__ __forceinline__ void colour_add(float w, const float (&c)[NC], float (&outc)[NC]) {
#pragma unroll
    for (int j = 0; j < NC; j++) {
        const float rgb = fminf(fmaxf(c[j], -1.0f), 1.0f) + 1.0f;
        outc[j] = fmaf(w, rgb, outc[j]);
    }
}

// output of a finished ray (scenedreamer.py:380-413): channels c0 .. c0 + NC - 1 of its composited colour outc blended with the
// sky -- the image's mean sky where the ray reaches the ground or its last voxel is not air (nosky), else its own -- and, with
// `head`, its depth and opacity
template <int NC>
__device__ __forceinline__ void finish_ray(const Params &p, int img, long long ray, bool nosky, int c0, const float (&outc)[NC],
                                           float Wsum, float depth, bool head) {
    const float sky_w = 1.0f - Wsum;
    const float4 *skp = reinterpret_cast<const float4 *>((nosky ? p.sky_avg + (long long)img * kOutC : p.sky + ray * kOutC) + c0);
    float4 *dst = reinterpret_cast<float4 *>(p.net_out + ray * kOutC + c0);
#pragma unroll
    for (int q = 0; q < NC / 4; q++) {
        const float4 sk = __ldg(skp + q);
        float4 o;
        o.x = (outc[4 * q + 0] + sky_w * (fminf(fmaxf(sk.x, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        o.y = (outc[4 * q + 1] + sky_w * (fminf(fmaxf(sk.y, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        o.z = (outc[4 * q + 2] + sky_w * (fminf(fmaxf(sk.z, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        o.w = (outc[4 * q + 3] + sky_w * (fminf(fmaxf(sk.w, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        dst[q] = o;
    }
    if (head) {
        if (p.depth_out) p.depth_out[ray] = depth;
        if (p.total_weight) p.total_weight[ray] = Wsum;
    }
}

// ---- gather (a5/a6) ----------------------------------------------------------------------------------
// One level of the hash-grid encoder at x (gridencoder.cu:133-170): the 5-D raw table (32 corners) or the pre-blended 3-D
// table (8 corners).  GU < 8 (3-D only) unrolls the corner loop GU times, so that at most 2 * GU gathers of a lane are in
// flight: the ray-slot kernel's gather shares the LSU with the epilogue's operand stores, and a fully unrolled level queues 16
// scattered LDG.128 per lane -- up to 4,096 L1 wavefronts ahead of every epilogue store.  Same arithmetic per feature.
template <bool RAW5D, int GU = 8>
__device__ __forceinline__ void encode_level(const float *__restrict__ tbl, uint32_t mask, float scale, const float (&x)[5],
                                             float (&res)[8]) {
    static_assert(GU == 8 || !RAW5D, "the 5-D corner loop is always fully unrolled");
    constexpr int D = RAW5D ? 5 : 3;
    float f[D];
    uint32_t g[D];
#pragma unroll
    for (int d = 0; d < D; d++) grid_cell(x[d], scale, g[d], f[d]);
#pragma unroll
    for (int c = 0; c < 8; c++) res[c] = 0.0f;
    if constexpr (RAW5D) {
        const uint32_t h0[2] = {g[0], g[0] + 1u};
        const uint32_t h1[2] = {g[1] * kPrime1, (g[1] + 1u) * kPrime1};
        const uint32_t h2[2] = {g[2] * kPrime2, (g[2] + 1u) * kPrime2};
        const uint32_t h3[2] = {g[3] * kPrime3, (g[3] + 1u) * kPrime3};
        const uint32_t h4[2] = {g[4] * kPrime4, (g[4] + 1u) * kPrime4};
#pragma unroll
        for (int idx = 0; idx < 32; idx++) {
            const int b0 = idx & 1, b1 = (idx >> 1) & 1, b2 = (idx >> 2) & 1, b3 = (idx >> 3) & 1, b4 = (idx >> 4) & 1;
            float w = b0 ? f[0] : 1.0f - f[0];
            w *= b1 ? f[1] : 1.0f - f[1];
            w *= b2 ? f[2] : 1.0f - f[2];
            w *= b3 ? f[3] : 1.0f - f[3];
            w *= b4 ? f[4] : 1.0f - f[4];
            const uint32_t index = (h0[b0] ^ h1[b1] ^ h2[b2] ^ h3[b3] ^ h4[b4]) & mask;
            float v[8];
            ld8(tbl + (size_t)index * 8, v);
#pragma unroll
            for (int c = 0; c < 8; c++) res[c] = fmaf(w, v[c], res[c]);
        }
    } else {
#pragma unroll(GU)
        for (int idx = 0; idx < 8; idx++) {
            float w;
            const uint32_t index = corner3(mask, g, f, idx, w);
            float v[8];
            ld8(tbl + (size_t)index * 8, v);
#pragma unroll
            for (int c = 0; c < 8; c++) res[c] = fmaf(w, v[c], res[c]);
        }
    }
}

// 8 fp32 values -> one 16-byte chunk of 16-bit operand (hi) and, for the x3 split, the residual (lo)
// PREC: 0 = fp16 single pass, 1 = bf16 hi/lo split, 2 = fp16 hi/lo split
template <int PREC>
__device__ __forceinline__ void split8(const float (&v)[8], uint4 &hi, uint4 &lo) {
    uint32_t h[4], l[4];
    if constexpr (PREC == 2) {
        // hi = fp16(v) (RN), lo = fp16(v - hi): 22 significant bits (|err| ~ 2^-22 |v|); needs |v| < 65504
#pragma unroll
        for (int q = 0; q < 4; q++) {
            h[q] = tc05::pack2<false>(v[2 * q], v[2 * q + 1]);
            const float2 hf = tc05::unpack2<false>(h[q]);
            l[q] = tc05::pack2<false>(v[2 * q] - hf.x, v[2 * q + 1] - hf.y);
        }
    } else if constexpr (PREC == 1) {
        // hi = v truncated to bf16 (exactly representable), lo = bf16(v - hi): |err| <= 2^-16 |v|
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint32_t a = __float_as_uint(v[2 * q]), b = __float_as_uint(v[2 * q + 1]);
            h[q] = __byte_perm(a, b, 0x7632);
            const float la = v[2 * q] - __uint_as_float(a & 0xFFFF0000u);
            const float lb = v[2 * q + 1] - __uint_as_float(b & 0xFFFF0000u);
            l[q] = tc05::pack2<true>(la, lb);
        }
    } else {
#pragma unroll
        for (int q = 0; q < 4; q++) { h[q] = tc05::pack2<false>(v[2 * q], v[2 * q + 1]); l[q] = 0; }
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

template <int PREC> __device__ __forceinline__ uint32_t one16() { return PREC == 1 ? 0x3F80u : 0x3C00u; }   // 1.0

// layer-0 operand chunks of the hash-grid features at x: the 8 levels of this thread's column half (level half + 2 i), zero
// outside the volume.  rec(level, res) is handed the fp32 features of every level.
template <bool RAW5D, int GU, int PREC, class Rec>
__device__ __forceinline__ void encode_features(const Params &p, uint32_t mask, const float *sScale, int half, const float (&x)[5],
                                                bool oob, uint4 (&fh)[8], uint4 (&fl)[8], Rec &&rec) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int level = half + 2 * i;
        float res[8];
        if (oob) {
#pragma unroll
            for (int c = 0; c < 8; c++) res[c] = 0.0f;
        } else {
            encode_level<RAW5D, GU>(p.table + ((size_t)level << p.log2_T) * 8, mask, sScale[level], x, res);
        }
        split8<PREC>(res, fh[i], fl[i]);
        rec(level, res);
    }
}

// K-extension of layer 0, the 8 columns 128 + 8 half ..: one-hot label (columns 128..142) and the constant-1 bias column 143
// == the reference's fc_m_a(onehot) product and fc_1's bias (layers.py:102-105)
__device__ __forceinline__ uint4 label_chunk(uint32_t label, int half, uint32_t one) {
    const int k = (int)label - 8 * half;                     // position inside this thread's 8-wide chunk
    const uint32_t v = (k >= 0 && k < 8) ? one << (16 * (k & 1)) : 0u, q = k >> 1;
    return make_uint4(q == 0 ? v : 0u, q == 1 ? v : 0u, q == 2 ? v : 0u, (q == 3 ? v : 0u) | (half == 1 ? one << 16 : 0u));   // | column 143
}

// this thread's part of row `row` of the layer-0 operand: the feature chunks of its 8 levels and its K-extension chunk
template <bool X3>
__device__ __forceinline__ void store_layer0(uint8_t *sHhi, uint8_t *sHlo, int row, int half, const uint4 (&fh)[8],
                                             const uint4 (&fl)[8], uint4 ext) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const uint32_t off = tc05::chunk_off(kRows, row, half + 2 * i);
        *reinterpret_cast<uint4 *>(sHhi + off) = fh[i];
        if constexpr (X3) *reinterpret_cast<uint4 *>(sHlo + off) = fl[i];
    }
    const uint32_t off = tc05::chunk_off(kRows, row, kFeat / 8 + half);
    *reinterpret_cast<uint4 *>(sHhi + off) = ext;
    if constexpr (X3) *reinterpret_cast<uint4 *>(sHlo + off) = make_uint4(0, 0, 0, 0);
}

// ---- the kernel ------------------------------------------------------------------------------------
// RAYQ (inference render only): the 128 MMA rows of the CTA are independent RAY SLOTS instead of the pixels of one 16x8 tile.
// Every slot has its own (ray, sample step) cursor; when its ray is finished -- all S samples marched or, with early termination,
// transmittance below the threshold -- the slot takes the next ray of a frame-wide queue of live rays (compacted by
// prepass_rays_kernel, in tile order so that neighbouring slots stay spatially coherent).  Dead rays never occupy a row and a
// tile no longer marches until its slowest ray is opaque: per C2 frame 4.4-4.7 M + ~0.5 M (one wasted step per terminated ray)
// instead of 6.5-6.8 M samples are shaded (tools/ray_stats.py).  The CTA runs ONE open-ended "tile": the loop control of all four
// roles is the early-termination mechanism below (stop_step decided by the epilogue two steps ahead).
template <int PREC, bool RAW5D, int MODE, bool TRAIN, bool RAYQ = false, int GU = 8>
__global__ void __launch_bounds__(kThreads, 1)
mlp_kernel(const Params p)
{
    static_assert(!RAYQ || (MODE == kRender && !TRAIN && !RAW5D), "ray slots: inference render over the pre-blended table");
    constexpr bool SKY = MODE == kSky, BWD = MODE == kBwd || MODE == kSkyBwd, SKYBWD = MODE == kSkyBwd;
    constexpr bool ONE_STEP = SKY || SKYBWD;     // per-RAY networks: every tile of the frame, one step per tile
    constexpr int NACT = Net<MODE>::NACT;
    static_assert(!TRAIN || ((MODE == kRender || MODE == kSky) && !RAW5D), "the training record is written by the forward networks");
    static_assert(!BWD || PREC == 1, "the gradient chains run in the range-safe bf16x3 mode");
    constexpr bool X3 = PREC != 0;
    constexpr bool BF16 = PREC == 1;
    constexpr Smem SM = smem_map();
    constexpr int PARTS = X3 ? 2 : 1;
    constexpr int NH = Net<MODE>::NH, NL = Net<MODE>::NL;
    static_assert(SM.total <= 232448, "shared memory map exceeds the 227 KB a CTA can have");
    static_assert(Net<MODE>::NBIAS <= Net<kRender>::NBIAS, "bias table slot");
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *sHhi = smem + SM.h_hi;
    uint8_t *sHlo = smem + SM.h_lo;
    uint8_t *sRing = smem + SM.ring;
    float *sF = reinterpret_cast<float *>(smem + SM.fsec);
    float *sBias = reinterpret_cast<float *>(smem + SM.bias);
    float *sScale = reinterpret_cast<float *>(smem + SM.scales);
    float *sFrac = reinterpret_cast<float *>(smem + SM.frac);
    float *sSig = reinterpret_cast<float *>(smem + SM.sig);
    float *sState = reinterpret_cast<float *>(smem + SM.state);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + SM.bars);
    uint32_t *sWalk = reinterpret_cast<uint32_t *>(smem + SM.walk);
    // the weight ring: 16 KB slots, each holding one stage (k16 slabs of one 64-column block, block_stages / stage_slabs)
    constexpr uint32_t kSlot = 16384, kSlabB = 2048 * PARTS;       // ring slot; one k16 slab of a 64-column block
    constexpr int kSps = kSlot / kSlabB;                           // slabs per ring slot
    constexpr int kStepStages = step_stages<MODE>(kSps);
    // the column-block walk of layer 0, of a hidden layer and of the last layer, and where the epilogue finds each block
    // (hand_plan)
    constexpr uint32_t kWalk0 = hand_plan<MODE>(0).walk, kWalkH = hand_plan<MODE>(1).walk, kWalkL = hand_plan<MODE>(NL - 1).walk;
    constexpr uint32_t kSrc0 = hand_plan<MODE>(0).src, kSrcH = hand_plan<MODE>(1).src, kSrcL = hand_plan<MODE>(NL - 1).src;
    static_assert(SKYBWD || hand_all_staged<MODE>(NL - 1), "the epilogue reads the last layer from the operand buffer only");
    // Early termination (north star: "early termination"; inference render only).  stop_step[buf] = number of sample
    // steps the tile in state buffer `buf` executes (S until decided).  The epilogue decides during the compositing of
    // step s ("every live ray has transmittance < early_T") and sets s + 2: by the time ANY role starts step s + 2 it
    // has synchronised (through the barriers it already waits on) with an epilogue that is past that compositing, so
    // all roles read the same value and execute the same number of steps -- the barrier phase arithmetic, which only
    // depends on the global executed-step counter n, stays consistent.
    constexpr bool ESTOP = MODE == kRender && !TRAIN;
    volatile int *sStop = reinterpret_cast<volatile int *>(smem + SM.stop);
    volatile int *sVote = sStop + 2;
    int *sVoted = const_cast<int *>(sStop) + 4;  // row blocks that have voted on step s (index s & 1)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // the render gradient chain has no dependency between the sample steps of a tile: there every (tile, step) is its own
    // work item (work_mult = S, one step each), which balances a few hundred tiles over 148 CTAs far better than whole tiles
    const int wmult = (MODE == kBwd && p.work_mult > 1) ? p.work_mult : 1;
    const int n_work = RAYQ ? (int)gridDim.x : (ONE_STEP ? p.n_tiles : *p.n_live * wmult);
    // the render chain over one image of a multi-view record: its work items start at record item view[0] * wmult (the record
    // lists live tiles grouped by image); read per work item rather than kept in a register across the roles' loops
    auto rec_work = [&](int work) {
        if constexpr (MODE != kBwd) return work;
        int first;
        asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(first) : "l"(p.view));      // volatile: re-read where used, not held
        return work + first * wmult;
    };
    constexpr bool STATE = MODE == kRender;      // per-ray sampling state (gather -> epilogue hand-off) exists
    const int S = ONE_STEP ? 1 : p.S;
    const int SL = RAYQ ? 0x3fffffff : S;        // steps of one work item: open-ended for ray slots (ended through sStop)
    // ray-slot bookkeeping lives in the second state buffer (unused in this mode): per-step row info ring, done flags, cursors
    uint4 *sInfo = reinterpret_cast<uint4 *>(sState + kStFloats * kRows);          // [4][128]: depth, interval, ray, code
    int *sDone = reinterpret_cast<int *>(sInfo + 4 * kRows);                        // [2][128]: ray + 1 finished early at step (s & 1)
    int2 *sCur = reinterpret_cast<int2 *>(sDone + 2 * kRows);                       // [128]: (ray, sample step) of every slot
    volatile int *sExh = reinterpret_cast<volatile int *>(sCur + kRows);            // [4]: queue exhausted as of step (s & 3); [4] = seen
    static_assert(4 * kRows * 16 + 2 * kRows * 4 + kRows * 8 + 32 <= kStFloats * kRows * 4, "ray-slot bookkeeping fits the second state buffer");

    // ---- one-time setup ----
    if (tid == 0) {
        for (int i = 0; i < 4; i++) tc05::mbar_init(&bars[B_WFULL + i], 1);
        tc05::mbar_init(&bars[B_FEAT], kGatherThreads);
        tc05::mbar_init(&bars[B_HFREE], 1);
        for (int rb = 0; rb < 2; rb++) {
            tc05::mbar_init(&bars[B_OPND + rb], kEpiThreads / 2);
            tc05::mbar_init(&bars[B_ACC + rb], 1);
            tc05::mbar_init(&bars[B_OUTRDY + rb], 1);
            tc05::mbar_init(&bars[B_EPIDONE + rb], kEpiThreads / 2);
            tc05::mbar_init(&bars[B_EPIDONE + 2 + rb], kEpiThreads / 2);
        }
        for (int i = 0; i < 2; i++) { tc05::mbar_init(&bars[B_STRDY + i], kRows); tc05::mbar_init(&bars[B_STFREE + i], kEpiThreads); }
        tc05::mbar_init(&bars[B_COMP], kEpiThreads);
        for (int i = 0; i < 4; i++) tc05::mbar_init(&bars[B_WEMPTY + i], 4);
        tc05::fence_mbar_init();
        // the ring stages of one sample step, the same for every step and image: per layer and row block, the layer's column
        // blocks in the order the MMA warpgroup walks them (hand_plan), each block's bytes (contiguous in the pack, wpack_off)
        // cut at stage boundaries.  Entry = pack offset / 2 KB | bytes / 2 KB << 16, so that a refill is one shared load
        // (walking the layers per refill took most of its time).
        int k = 0;
        for (int l = 0; l < NL; l++) {
            const int nK = layerK<MODE>(l) / 16, ncb = layerN<MODE>(l) / 64, nsb = block_stages(nK, kSps);
            const uint32_t walk = l == 0 ? kWalk0 : (l == NL - 1 ? kWalkL : kWalkH);
            for (int rb = 0; rb < 2; rb++)
                for (int pos = 0; pos < ncb; pos++) {
                    const int c = (walk >> (8 * pos)) & 3u;
                    uint32_t po = (uint32_t)(layerOff<MODE>(l, PARTS) + (int64_t)c * nK * kSlabB);
                    for (int js = 0; js < nsb; js++) {
                        const uint32_t bytes = (uint32_t)stage_slabs(nK, kSps, js) * kSlabB;
                        sWalk[k++] = (po >> 11) | ((bytes >> 11) << 16);
                        po += bytes;
                    }
                }
        }
    }
    if (tid < 2) { sStop[tid] = RAYQ ? 0x7fffffff : kMaxS + 1; sVote[tid] = 0; sVoted[tid] = 0; }
    if constexpr (RAYQ) {
        for (int i = tid; i < kRows; i += kThreads) { sCur[i] = make_int2(-1, 0); sDone[i] = 0; sDone[kRows + i] = 0; }
        if (tid < 5) sExh[tid] = 0;
    }
    // Work distribution over the persistent CTAs.  Static (work = blockIdx + it * grid) unless the launcher hands in a
    // counter: then the first tile is static and every further one is drawn from the counter by ONE thread of the
    // most-ahead role (gather thread 0) and published through a 4-deep shared ring; the other roles pick the it-th
    // entry up when they get there (spin on the published count).  Tiles differ in cost once early termination is on,
    // and 2,800 tiles over 148 CTAs leave a 19-vs-18 tail even when they do not.
    volatile int *sWork = reinterpret_cast<volatile int *>(smem + SM.sched);
    volatile int *sPub = sWork + 4;
    if (tid == 0) *sPub = 0;
    const bool dyn = STATE && !RAYQ && p.work_counter != nullptr;
    auto fetch_work = [&](int it) -> int {
        if (!dyn) {
            const int w = (int)blockIdx.x + it * (int)gridDim.x;
            return w < n_work ? w : -1;
        }
        while (*sPub <= it) {
        }
        return sWork[it & 3];
    };
    if (STATE) {
        for (int i = tid; i < kLevels; i += kThreads) sScale[i] = exp2f(i * p.level_S) * p.base_res - 1.0f;   // gridencoder.cu:126
        for (int i = tid; i <= p.S; i += kThreads) sFrac[i] = p.fractions[i];
    }
    __syncthreads();
    const uint32_t mask = SKY ? 0u : ((1u << p.log2_T) - 1u);

    if (warp < 8) {
        set_maxnreg<kRegsEpi>();
        // =========================== EPILOGUE / COMPOSITING WARPS ===========================
        const int row = tid & (kRows - 1), half = tid >> 7;          // column half: 128*half .. +127
        // 64-row block of this thread (warps 0,1,4,5 / 2,3,6,7): its hand-offs with the MMA warpgroup and its compositing
        // barrier (named barrier 4 + rb) are per row block, so the two blocks can run up to half a layer apart
        const int rb = row >> 6;
        const bool rb_lead = (tid & 191) == 0;                       // thread 0 / 64: one per row block
        // early-termination vote of step s: a row-block leader calls this once its block's votes are in; the second of the two
        // blocks gets true and decides for the CTA from the votes of both
        auto last_vote = [&](int s) {
            __threadfence_block();
            const bool last = atomicAdd(&sVoted[s & 1], 1) == 1;
            if (last) {
                sVoted[s & 1] = 0;
                __threadfence_block();
            }
            return last;
        };
        const float *acc_cta = p.acc + (size_t)blockIdx.x * 2 * kRows * kAccCols;  // this CTA's two accumulator buffers (acc_off)
        uint32_t n = 0;                 // global step counter
        int loaded_img = -1;
        for (int it = 0;; it++) {
            const int work = fetch_work(it);
            if (work < 0) break;
            const int tile = RAYQ ? 0 : (ONE_STEP ? work : p.tile_list[rec_work(work) / wmult]);
            const TileCoord tc = tile_coord(p, tile);
            const int buf = it & 1;
            const float *st = sState + buf * kStFloats * kRows;
            if (Net<MODE>::TAIL && loaded_img != tc.img) {
                // sigma head of this image's pack -> shared memory (epilogue threads are the only readers)
                const float *packF = reinterpret_cast<const float *>(p.pack + (long long)tc.img * p.pack_stride +
                                                                     layerOff<MODE>(NL, PARTS));
                asm volatile("bar.sync 1, 256;" ::: "memory");
                for (int i = tid; i < kFTotal; i += kEpiThreads) sF[i] = __ldg(packF + i);
                asm volatile("bar.sync 1, 256;" ::: "memory");
                loaded_img = tc.img;
            }
            const int y = tc.y0 + (row >> 4), x = tc.x0 + (row & 15);
            const bool in_img = (y < p.H) && (x < p.W);
            const long long ray = ((long long)tc.img * p.H + y) * p.W + x;
            uint32_t flags = in_img ? 4u : 0u, labs = 0;
            float dir0 = 0.0f, ori0 = 0.0f;
            if (STATE && !RAYQ) {
                tc05::mbar_wait(&bars[B_STRDY + buf], (it >> 1) & 1);
                flags = __float_as_uint(st[kStFlags * kRows + row]);
                labs = __float_as_uint(st[kStLab * kRows + row]);
                dir0 = st[(kStDir + 0) * kRows + row];
                ori0 = __ldg(p.cam_ori + tc.img * 3);
            }
            (void)labs;
            const bool live = flags & 1u, valid = flags & 4u;
            float outc[32];
#pragma unroll
            for (int c = 0; c < 32; c++) outc[c] = 0.0f;
            float Wsum = 0.0f, Dsum = 0.0f, Dcomp = 0.0f, Eexcl = 0.0f;
            bool is_gnd = false;

            int s_done = S;           // steps actually executed for this tile
            int skip_ray = -1;        // RAYQ: the ray this slot finished early at the previous step (its next sample is already in flight)
            (void)skip_ray;
            for (int s = 0; s < SL; s++, n++) {
                if (ESTOP && s >= 2 && s >= sStop[buf]) { s_done = s; break; }
                Sample sm{0.0f, 0.0f, 0};
                if (STATE && !RAYQ) {
                    sm = sample_at(p, st, row, s, sFrac, ray);
                    is_gnd = is_gnd || (__fadd_rn(__fmul_rn(dir0, sm.depth), ori0) <= 1.0f);   // scenedreamer.py:354,380
                }
                float sig_part = 0.0f;
                // training record addressing: step = (work item, sample), slot = (step, tile row)
                const long long step_id = (long long)work * S + s;
                const long long slot = step_id * kRows + row;
                float dsig = 0.0f;
                if constexpr (MODE == kBwd) dsig = __ldg(p.tr.dsig + slot);
                (void)slot; (void)dsig;
#pragma unroll 1
                for (int l = 0; l < NH; l++) {
                    const uint32_t g = n * NL + l;                   // global layer counter -> accumulator buffer
                    const float *acc = acc_cta + (g & 1u) * kRows * kAccCols;
                    // the column blocks of this layer that the MMA warpgroup staged in the operand buffer, in place (hand_plan)
                    const uint32_t hsrc = l == 0 ? kSrc0 : kSrcH;
                    // kBwd: LeakyReLU sign words of the forward activation A_{6-l} this layer's data gradient passes
                    // through (prefetched before the accumulator wait)
                    uint4 mw = make_uint4(0u, 0u, 0u, 0u);
                    if constexpr (BWD)
                        mw = __ldg(reinterpret_cast<const uint4 *>(p.tr.mask + (((long long)rec_work(work) * S + s) * kNumAct + (NACT - 1 - l)) * kRows * 8 + row * 8 + half * 4));
                    if ((tid & 127) == 0) SDB_MARK(half, 1, n, l);
                    tc05::mbar_wait(&bars[B_ACC + rb], (n * NH + l) & 1);
                    if ((tid & 127) == 0) SDB_MARK(half, 2, n, l);
                    if (rb_lead) SDB_STAMP(n, l, 4 + 2 * rb);
#pragma unroll 1
                    for (int c0 = 0; c0 < 128; c0 += 32) {
                        // a 32-column chunk in two 16-column halves (16 live accumulator registers instead of 32: the
                        // compositing state of the tile stays in registers next to them)
                        uint32_t rec[16];            // TRAIN / chain: bf16 (round-to-nearest) copy of the chunk for the record
                        uint32_t mword = 0;          // TRAIN: LeakyReLU sign bits of the chunk
                        (void)rec; (void)mword;
                        const uint32_t word = c0 == 0 ? mw.x : (c0 == 32 ? mw.y : (c0 == 64 ? mw.z : mw.w));
                        (void)word;
                        // one source per 64-column block: the thread's own slots of the operand buffer (read here, then
                        // overwritten below with the 16-bit operand), or the L2 buffer
                        const bool staged = (hsrc >> (4 * ((half * 128 + c0) >> 6))) & 15u;
#pragma unroll
                        for (int hh = 0; hh < 2; hh++) {
                            float v[16];
                            if (staged) stg_ld<16>(sHhi, sHlo, row, half * 128 + c0 + 16 * hh, v);
                            else acc_ld<16>(acc, row, half * 128 + c0 + 16 * hh, v);
                            if constexpr (BWD) {
                                if (MODE == kBwd && l == 2) {   // dA4 += dsigma * fc_sigma.weight (sigma taps A4, layers.py:115)
                                    const float *ws = sF + kFWsig + half * 128 + c0 + 16 * hh;
#pragma unroll
                                    for (int j = 0; j < 16; j++) v[j] = fmaf(dsig, ws[j], v[j]);
                                }
                                // dZ = dA * LeakyReLU'(z): slope 1 where the forward activation was > 0, else 0.2
#pragma unroll
                                for (int j = 0; j < 16; j++) v[j] = ((word >> (16 * hh + j)) & 1u) ? v[j] : 0.2f * v[j];
                            } else {
#pragma unroll
                                for (int j = 0; j < 16; j++) v[j] = fmaxf(v[j], 0.2f * v[j]);          // LeakyReLU(0.2)
                                if (MODE == kRender && l == 3) {   // sigma = fc_sigma(f) after fc_4's activation (layers.py:115)
                                    const float *ws = sF + kFWsig + half * 128 + c0 + 16 * hh;
#pragma unroll
                                    for (int j = 0; j < 16; j++) sig_part = fmaf(v[j], ws[j], sig_part);
                                }
                            }
                            if constexpr (TRAIN || BWD) {
#pragma unroll
                                for (int q = 0; q < 8; q++) rec[8 * hh + q] = tc05::pack2<true>(v[2 * q], v[2 * q + 1]);
                            }
                            if constexpr (TRAIN) {
#pragma unroll
                                for (int j = 0; j < 16; j++) mword |= (v[j] > 0.0f ? 1u : 0u) << (16 * hh + j);
                            }
#pragma unroll
                            for (int q = 0; q < 2; q++) {
                                uint4 hi, lo;
                                const float(&v8)[8] = *reinterpret_cast<const float(*)[8]>(&v[8 * q]);
                                split8<PREC>(v8, hi, lo);
                                const uint32_t off = tc05::chunk_off(kRows, row, half * 16 + (c0 >> 3) + 2 * hh + q);
                                *reinterpret_cast<uint4 *>(sHhi + off) = hi;
                                if constexpr (X3) *reinterpret_cast<uint4 *>(sHlo + off) = lo;
                            }
                        }
                        if constexpr (TRAIN || BWD) {
                            // forward: A_{l+1}[slot][128*half + c0 ..], backward: dZ_{6-l}[slot][...]
                            // (tiled record: a warp's 32 rows of one 8-column chunk are 512 contiguous bytes)
                            uint16_t *arr = TRAIN ? p.tr.act + (long long)l * p.tr.slot_cap * kActCols
                                                  : p.tr.dz + (long long)(NACT - 1 - l) * p.tr.slot_cap * kHidden;
                            constexpr int nch = (TRAIN ? kActCols : kHidden) / 8;
                            const int ch0 = (half * 128 + c0) >> 3;
#pragma unroll
                            for (int q = 0; q < 4; q++)
                                *reinterpret_cast<uint4 *>(rec_chunk(arr, slot, nch, ch0 + q)) =
                                    make_uint4(rec[4 * q], rec[4 * q + 1], rec[4 * q + 2], rec[4 * q + 3]);
                        }
                        if constexpr (TRAIN) p.tr.mask[((step_id * kNumAct + l) * kRows + row) * 8 + half * 4 + (c0 >> 5)] = mword;
                    }
                    // the next layer's operand rows of this row block are written (the MMA warpgroup may start on them), and
                    // these rows of accumulator buffer (g & 1) are free again
                    tc05::fence_proxy_async_smem();
                    tc05::mbar_arrive(&bars[B_OPND + rb]);
                    tc05::mbar_arrive(&bars[B_EPIDONE + (g & 1u) * 2 + rb]);
                    if (rb_lead) SDB_STAMP(n, l, 5 + 2 * rb);
                    if (MODE == kRender && l == 3) sSig[half * kRows + row] = sig_part;
                    if constexpr (TRAIN) {   // the constant-1 column that turns the weight-gradient GEMM's column 256 into the bias gradient
                        if (half == 0) {
                            uint16_t *arr = p.tr.act + (long long)l * p.tr.slot_cap * kActCols;
                            *reinterpret_cast<uint4 *>(rec_chunk(arr, slot, kActCols / 8, kHidden / 8)) = make_uint4(0x3F80u, 0u, 0u, 0u);
                            *reinterpret_cast<uint4 *>(rec_chunk(arr, slot, kActCols / 8, kHidden / 8 + 1)) = make_uint4(0u, 0u, 0u, 0u);
                        }
                    }
                }
                // ---- colour layer ----
                const uint32_t go = n * NL + NH;
                if ((tid & 127) == 0) SDB_MARK(half, 3, n, NH);
                tc05::mbar_wait(&bars[B_OUTRDY + rb], n & 1);
                if ((tid & 127) == 0) SDB_MARK(half, 4, n, NH);
                if (rb_lead) SDB_STAMP(n, NH, 4 + 2 * rb);
                if constexpr (SKYBWD) {
                    // last layer of the sky chain: dA1 [128 x 256] -> dZ1 = dA1 * LeakyReLU'(z1) -> bf16 record only
                    const uint4 mw = __ldg(reinterpret_cast<const uint4 *>(p.tr.mask + ((step_id * kNumAct + 0) * kRows + row) * 8 + half * 4));
#pragma unroll 1
                    for (int c0 = 0; c0 < 128; c0 += 32) {
                        float v[32];
                        const int col = half * 128 + c0;
                        const uint32_t src = (kSrcL >> (4 * (col >> 6))) & 15u;
                        if (src) stg_ld<32>(sHhi, sHlo, row, 64 * (int)(src - 1) + (col & 63), v);
                        else acc_ld<32>(acc_cta + (go & 1u) * kRows * kAccCols, row, col, v);
                        const uint32_t word = c0 == 0 ? mw.x : (c0 == 32 ? mw.y : (c0 == 64 ? mw.z : mw.w));
#pragma unroll
                        for (int j = 0; j < 32; j++) v[j] = ((word >> j) & 1u) ? v[j] : 0.2f * v[j];
                        const int ch0 = (half * 128 + c0) >> 3;
#pragma unroll
                        for (int q = 0; q < 4; q++)
                            *reinterpret_cast<uint4 *>(rec_chunk(p.tr.dz, slot, kHidden / 8, ch0 + q)) =
                                make_uint4(tc05::pack2<true>(v[8 * q], v[8 * q + 1]), tc05::pack2<true>(v[8 * q + 2], v[8 * q + 3]),
                                           tc05::pack2<true>(v[8 * q + 4], v[8 * q + 5]), tc05::pack2<true>(v[8 * q + 6], v[8 * q + 7]));
                    }
                    tc05::mbar_arrive(&bars[B_EPIDONE + (go & 1u) * 2 + rb]);
                    if (rb_lead) SDB_STAMP(n, NH, 5 + 2 * rb);
                    continue;
                }
                // the last layer is staged whole, clear of the gather's columns (hand_plan): colour block 0 at region 3 (this half's
                // 32 columns), kBwd block `half` (this half's 64 columns) at its region
                float c[32];
                const int ccol = BWD ? 64 * (int)(((kSrcL >> (4 * half)) & 15u) - 1) : 64 * (int)((kSrcL & 15u) - 1) + half * 32;
                stg_ld<32>(sHhi, sHlo, row, ccol, c);
                if constexpr (BWD) {
                    // d(hash-grid features) [128 rays x 128]: this half owns 64 columns -> fp32 record for the table backward
                    float c2[32];
                    stg_ld<32>(sHhi, sHlo, row, ccol + 32, c2);
                    tc05::mbar_arrive(&bars[B_EPIDONE + (go & 1u) * 2 + rb]);
                    if (rb_lead) SDB_STAMP(n, NH, 5 + 2 * rb);
                    float *dst = p.tr.dx0 + slot * kFeat + half * 64;
#pragma unroll
                    for (int q = 0; q < 4; q++) st_global_v8f(dst + 8 * q, &c[8 * q]);
#pragma unroll
                    for (int q = 0; q < 4; q++) st_global_v8f(dst + 32 + 8 * q, &c2[8 * q]);
                    continue;
                }
                tc05::mbar_arrive(&bars[B_EPIDONE + (go & 1u) * 2 + rb]);
                if (rb_lead) SDB_STAMP(n, NH, 5 + 2 * rb);
                if constexpr (SKY) {
#pragma unroll
                    for (int j = 0; j < 32; j++) outc[j] = c[j];
                } else if constexpr (RAYQ) {
                    // ---- compositing of ray slots (a10/a11): every row is its own ray at its own sample step ----
                    tc05::named_sync(4 + rb, 128);                          // sSig of both column halves of these rows
                    const float sigma = (sSig[row] + sSig[kRows + row]) + sF[kFBsig];
                    const uint4 info = sInfo[(s & 3) * kRows + row];            // published by the gather role for this step
                    const int rq = (int)info.z;
                    const uint32_t code = info.w;                                // bits 0-7 sample step, 8 first, 9 last, 11 sky_mask, 12 is_gnd (any sample)
                    const int s_ray = (int)(code & 0xffu);
                    const bool act = rq >= 0 && rq != skip_ray;
                    if (act && (code & 0x100u)) {
#pragma unroll
                        for (int j = 0; j < 32; j++) outc[j] = 0.0f;
                        Wsum = 0.0f; Dsum = 0.0f; Dcomp = 0.0f; Eexcl = 0.0f;
                    }
                    float w = 0.0f;
                    bool fin = false;
                    if (act) {
                        const float depth = __uint_as_float(info.x), nd = __uint_as_float(info.y);
                        w = sample_weight(sigma, nd, p.dists_scale, Eexcl);
                        composite_add(w, depth, Wsum, Dsum, Dcomp);
                        if (half == 0 && p.weights_out) p.weights_out[(long long)rq * S + s_ray] = w;
                        fin = (code & 0x200u) || (p.early_T > 0.0f && expf(-Eexcl) < p.early_T);
                    }
                    colour_add(w, c, outc);
                    if (act && fin) {
                        // this slot's ray is finished
                        const bool nosky = !(code & 0x800u) || (code & 0x1000u);
                        finish_ray(p, 0, rq, nosky, half * 32, outc, Wsum, __fadd_rn(Dsum, Dcomp), half == 0);
                        skip_ray = (code & 0x200u) ? -1 : rq;
                    }
                    // early finishes are reported to the gather role (it replaces the ray two steps on); natural ends it sees itself
                    if (half == 0) sDone[(s & 1) * kRows + row] = (act && fin && !(code & 0x200u)) ? rq + 1 : 0;
                    // is the CTA done?  every slot idle or finished AND the queue was already empty when this step was built
                    {
                        const bool idle = !act || fin;
                        const bool wall = __all_sync(0xffffffffu, idle);
                        if (lane == 0 && !wall) sVote[s & 1] = 1;
                        tc05::named_sync(4 + rb, 128);
                        if (rb_lead && last_vote(s)) {
                            if (sVote[s & 1] == 0 && sExh[s & 3] != 0 && sStop[0] > s + 2) sStop[0] = s + 2;
                            sVote[s & 1] = 0;
                        }
                    }
                    tc05::mbar_arrive(&bars[B_COMP]);                      // compositing of step s is complete (done flags visible)
                } else {
                    // ---- compositing (a10/a11) ----
                    tc05::named_sync(4 + rb, 128);                          // sSig of both column halves of these rows
                    const float sigma = (sSig[row] + sSig[kRows + row]) + sF[kFBsig];
                    float w = sample_weight(sigma, sm.nd, p.dists_scale, Eexcl);
                    w = live ? w : 0.0f;                                                              // scenedreamer.py:376
                    composite_add(w, sm.depth, Wsum, Dsum, Dcomp);
                    if constexpr (TRAIN) {   // what the compositing backward needs: sigma, scaled interval, colour head output
                        if (half == 0) { p.tr.sig[slot] = sigma; p.tr.nds[slot] = __fmul_rn(sm.nd, p.dists_scale); }
                        float *cd = p.tr.c + slot * kOutC + half * 32;
#pragma unroll
                        for (int q = 0; q < 4; q++) st_global_v8f(cd + 8 * q, &c[8 * q]);
                    }
                    if (half == 0 && valid) {
                        if (p.weights_out) p.weights_out[ray * S + s] = w;
                        if (p.rdepth_out) p.rdepth_out[ray * S + s] = sm.depth;
                    }
                    if (ESTOP && p.early_T > 0.0f) {
                        // vote: is every ray of the tile finished (sky-only / outside the image, or opaque)?
                        const bool done = !live || expf(-Eexcl) < p.early_T;
                        const bool wall = __all_sync(0xffffffffu, done);
                        if (lane == 0 && !wall) sVote[s & 1] = 1;
                        tc05::named_sync(4 + rb, 128);
                        if (rb_lead && last_vote(s)) {
                            if (sVote[s & 1] == 0 && sStop[buf] > S) sStop[buf] = s + 2;
                            sVote[s & 1] = 0;
                        }
                    }
                    colour_add(w, c, outc);
                }
            }
            if constexpr (SKY) {
                // ---- sky features out + per-tile column sums for the frame-global mean (scenedreamer.py:597) ----
                if (valid) {
                    float4 *dst = reinterpret_cast<float4 *>(p.sky_out + ray * kOutC + half * 32);
#pragma unroll
                    for (int q = 0; q < 8; q++) dst[q] = make_float4(outc[4 * q], outc[4 * q + 1], outc[4 * q + 2], outc[4 * q + 3]);
                }
                float *red = sSig;      // [4 quadrant warps][64] partial sums, then 64 threads finish
                asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
                for (int j = 0; j < 32; j++) {
                    float v = valid ? outc[j] : 0.0f;
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                    if (lane == 0) red[(warp & 3) * kOutC + half * 32 + j] = v;
                }
                asm volatile("bar.sync 1, 256;" ::: "memory");
                if (tid < kOutC)
                    p.sky_partial[(long long)tile * kOutC + tid] =
                        (red[tid] + red[kOutC + tid]) + (red[2 * kOutC + tid] + red[3 * kOutC + tid]);
            } else if constexpr (RAYQ) {
                if (tid == 0 && p.steps_done != nullptr) atomicAdd(p.steps_done, s_done);      // CTA steps of 128 slots each
            } else if constexpr (!BWD) {
                if constexpr (ESTOP) {
                    // samples the tile did not shade: their weights are below early_T (reported as 0); the ground test of
                    // the sky-leak logic (scenedreamer.py:380) still looks at every sample position
                    for (int s = s_done; s < S; s++) {
                        const Sample sm = sample_at(p, st, row, s, sFrac, ray);
                        is_gnd = is_gnd || (__fadd_rn(__fmul_rn(dir0, sm.depth), ori0) <= 1.0f);
                        if (half == 0 && valid) {
                            if (p.weights_out) p.weights_out[ray * S + s] = 0.0f;
                            if (p.rdepth_out) p.rdepth_out[ray * S + s] = sm.depth;
                        }
                    }
                }
                if (tid == 0 && p.steps_done != nullptr) atomicAdd(p.steps_done, s_done);
                // ---- finalize the tile ----
                const bool sky_mask = flags & 2u;
                const bool nosky = (!sky_mask) || is_gnd;
                if constexpr (TRAIN) {
                    if (half == 0) p.tr.rayflags[(long long)work * kRows + row] = (live ? 1u : 0u) | (nosky ? 2u : 0u) | (valid ? 4u : 0u);
                }
                if (valid) finish_ray(p, tc.img, ray, nosky, half * 32, outc, Wsum, __fadd_rn(Dsum, Dcomp), half == 0);
                tc05::mbar_arrive(&bars[B_STFREE + buf]);
            }
        }
    } else if (warp < kGatherWarp0) {
      set_maxnreg<kRegsCtl>();
      // =========================== MMA WARPGROUP ===========================
      // Layer l of a sample step: D[128 x N] = H[128 x K] * W_l^T, one 64-row block rb after the other, each in 64-column
      // blocks (the sum over K in registers) written once -- staged in operand columns no MMA of the layer reads any more, or
      // else to this CTA's fp32 accumulator buffer (g & 1) in global memory (hand_plan) -- where the epilogue reads its rows.
      // A row block is handed over as soon as it is written, so the epilogue of one row block runs
      // while the MMAs of the other do.  Weights go through a 4-slot ring of 16 KB stages (4 k16 slabs of one 64-column block
      // at x3, 8 at x1; a hidden-layer block at x3 fills the whole ring), one bulk copy each (wpack_off); the producer
      // warpgroup keeps the ring full, the weights are streamed once per row block.  Named barrier 3 is this warpgroup's
      // (1, 4, 5: epilogue, 2: gather).
      //
      // Numerics: slabs 0..7 of a block and slabs 8..nK-1 are two fresh tensor-core sums d0, d1 (numerics groups), and the
      // block is RN(d0 + d1), or d0 when nK <= 8: the tensor core's own accumulation does not round to nearest, and over a
      // whole x3 layer that moved the full-frame depth outside its parity bound.  Layers 1 .. NL-1 of the forward networks
      // then add their fp32 bias (the pack's table: hi + lo of the 16-bit parts, what a bias K slab would have summed on the
      // tensor core, exactly) with one more round-to-nearest add.  Two 32-register sets X, Y alternate: block c's group 0 is
      // in X, its group 1 goes to Y; once both are done X = RN(RN(X + Y) + b), the next block's group 0 is issued into Y and X is
      // stored while it runs, then the next block's group 1 goes to X, and so on.  A block staged late (kHDelayed) waits for
      // the next block's group 0 to retire before its store, and that block's group 1 is issued after it.  The blocks are
      // walked in hand_plan order (a hidden layer: 2, 3, 0, 1); each is the same sum whatever the order.  Every stage is its own
      // commit group, so its ring slot is released (each warp arrives on the slot's empty barrier once its wait_group says the
      // stage's MMAs are done) and refilled with a stage of the next block by the producer.
      const int t = tid - kMmaWarp0 * 32;
      static_assert(block_stages(kHidden / 16, kSps) <= 4 && block_stages(kRenderK0 / 16, kSps) <= 4,
                    "the stages of one column block fit the 4-slot ring");
      constexpr bool BIAS = Net<MODE>::NBIAS > 0;
      uint32_t n = 0, q = 0, qr = 0;                                 // ring stages issued to the tensor cores / retired
      int loaded_img = -1;
      for (int it = 0;; it++) {
          const int work = fetch_work(it);
          if (work < 0) break;
          const int tile = RAYQ ? 0 : (ONE_STEP ? work : p.tile_list[rec_work(work) / wmult]);
          const int img = tile_coord(p, tile).img;
          if (BIAS && loaded_img != img) {
              // bias table of this image's pack -> shared memory (this warpgroup is its only reader)
              const float *packB = reinterpret_cast<const float *>(p.pack + (long long)img * p.pack_stride + biasOff<MODE>(PARTS));
              tc05::named_sync(3, 128);
              for (int i = t; i < Net<MODE>::NBIAS; i += 128) sBias[i] = __ldg(packB + i);
              tc05::named_sync(3, 128);
              loaded_img = img;
          }
          for (int s = 0; s < SL; s++, n++) {
              if (ESTOP && s >= 2 && s >= sStop[it & 1]) break;
#pragma unroll 1
              for (int l = 0; l < NL; l++) {
                  const uint32_t g = n * NL + l, buf = g & 1u;
                  const int N = layerN<MODE>(l), nK = layerK<MODE>(l) / 16;
                  const int ncb = N / 64, nsb = block_stages(nK, kSps), ns0 = group0_stages(nK, kSps);
#pragma unroll 1
                  for (int rb = 0; rb < 2; rb++) {
                      if (t == 0) SDB_MARK(2, 1, n, l);
                      // these rows of accumulator buffer `buf` were last read by the epilogue of global layer g - 2
                      if (g >= 2) tc05::mbar_wait(&bars[B_EPIDONE + buf * 2 + rb], ((g >> 1) - 1) & 1);
                      if (l == 0) {
                          if (rb == 0) tc05::mbar_wait(&bars[B_FEAT], n & 1);
                      } else {
                          tc05::mbar_wait(&bars[B_OPND + rb], (n * NH + l - 1) & 1);   // operand rows from the previous epilogue
                      }
                      if (t == 0) SDB_MARK(2, 2, n, l);
                      if (t == 0) SDB_STAMP(n, l, 2 * rb);
                      TSplit ts;
                      ts.start();
                      // element offset of this row block in the accumulator buffers (p.acc is re-read at the store: a 64-bit
                      // pointer held across the block loop would not fit the registers next to the two accumulator sets)
                      const uint32_t dst = (blockIdx.x * 2 + buf) * kRows * kAccCols + acc_off(rb * 64, 0);
                      const uint32_t walk = l == 0 ? kWalk0 : (l == NL - 1 ? kWalkL : kWalkH);
                      float x[32], y[32];
                      // issue the MMAs of stages [js0, js1) of the current block into d, one commit group per stage; the first
                      // slab of stage js0 starts a fresh sum (js0 = the first stage of a numerics group)
                      auto issue = [&](float (&d)[32], int js0, int js1) {
                          for (int js = js0; js < js1; js++) {
                              const uint32_t slot = q & 3u;
                              tc05::mbar_wait(&bars[B_WFULL + slot], (q >> 2) & 1u);
                              ts.lap(kSplitFull);
                              const uint32_t sb = tc05::smem_u32(sRing + slot * kSlot);
                              const int kk0 = stage_slab0(nK, kSps, js), ns = stage_slabs(nK, kSps, js);
                              tc05::wgmma_fence();
#pragma unroll
                              for (int i = 0; i < kSps; i++) {
                                  if (i >= ns) break;
                                  const uint32_t aoff = (uint32_t)(kk0 + i) * 2 * kLboA + rb * 1024;
                                  const uint64_t ah = tc05::make_smem_desc(tc05::smem_u32(sHhi) + aoff, kLboA, kSbo);
                                  const uint64_t bh = tc05::make_smem_desc(sb + i * kSlabB, 1024, kSbo);
                                  tc05::wgmma_m64n64k16<BF16, 0, 0>(d, ah, bh, (js > js0 || i > 0) ? 1u : 0u);
                                  if constexpr (X3) {
                                      const uint64_t al = tc05::make_smem_desc(tc05::smem_u32(sHlo) + aoff, kLboA, kSbo);
                                      tc05::wgmma_m64n64k16<BF16, 0, 0>(d, al, bh, 1u);
                                      tc05::wgmma_m64n64k16<BF16, 0, 0>(d, ah, bh + (2048 >> 4), 1u);
                                  }
                              }
                              tc05::wgmma_commit();
                              q++;
                              ts.lap(kSplitIssue);
                          }
                      };
                      // wait for the `pending` stages in flight, oldest first; this warp is done with a stage's ring slot as
                      // soon as its MMAs are
                      auto retire = [&](int pending) {
                          auto release = [&]() {
                              ts.lap(kSplitWait);
                              if (lane == 0) tc05::mbar_arrive(&bars[B_WEMPTY + (qr & 3u)]);
                              qr++;
                              ts.lap(kSplitRelease);
                          };
#pragma unroll 1
                          for (int k = pending - 1; k > 0; k--) {
                              tc05::wgmma_wait_n(k);
                              release();
                          }
                          // always: ptxas serialises every wgmma of the kernel if one path may read an accumulator set in flight
                          tc05::wgmma_wait<0>();
                          if (pending > 0) release();
                      };
                      bool g0_done = false;          // the current block's group 0 has retired (the block before it was staged late)
                      // the pos-th block of the walk: its group 0 is in flight in a.  Issue group 1 into b, retire the block's
                      // stages, reduce into a, start the next block's group 0 in b and store a.
                      auto block = [&](float (&a)[32], float (&b)[32], int pos) {
                          const uint32_t w = walk >> (8 * pos);
                          const int c = (int)(w & 3u);
                          issue(b, ns0, nsb);
                          retire(g0_done ? nsb - ns0 : nsb);
                          g0_done = false;
                          tc05::wgmma_fence_acc(a);
                          tc05::wgmma_fence_acc(b);
                          if (nsb > ns0) {
#pragma unroll
                              for (int i = 0; i < 32; i++) a[i] = __fadd_rn(a[i], b[i]);
                          }
                          // the thread's fragment position, re-read here: held across the block loop it was spilled
                          uint32_t ft;
                          asm volatile("mov.u32 %0, %%tid.x;" : "=r"(ft));
                          ft -= kMmaWarp0 * 32;
                          if (BIAS && l > 0) {
                              const float *bias = sBias + (l - 1) * kHidden + c * 64;
#pragma unroll
                              for (int i = 0; i < 32; i += 2) {
                                  const float2 bb = *reinterpret_cast<const float2 *>(bias + tc05::frag_col(ft, i));
                                  a[i] = __fadd_rn(a[i], bb.x);
                                  a[i + 1] = __fadd_rn(a[i + 1], bb.y);
                              }
                          }
                          ts.lap(kSplitReduce);
                          if (pos + 1 < ncb) issue(b, 0, ns0);
                          if (!(w & kHStaged)) {
#ifndef SDB_AB_NO_ACC
                              // in the buffer's layout (acc_off) a warp's 8-byte stores of one (j, h) fragment pair are two whole
                              // 128-byte lines: 8 rows of two 4-column chunks, where the row-major buffer took 8 partial lines.
                              // Pair (j, h) of the thread sits 8 j columns (two chunks: 128 floats) and 8 h rows (32 floats) past
                              // its pair (0, 0), so the 16 stores share one address
                              float *out = p.acc + (dst + (uint32_t)(c & 1) * 4096u + acc_off(tc05::frag_row(ft, 0), tc05::frag_col(ft, 0)));
#pragma unroll
                              for (int i = 0; i < 32; i += 2)
                                  *reinterpret_cast<float2 *>(out + (i >> 2) * 128 + ((i >> 1) & 1) * 32) = make_float2(a[i], a[i + 1]);
#endif
                          } else {
                              // Staged in operand region r of this row block's rows.  The stores overwrite operand rows this
                              // warpgroup's wgmma read: every MMA that reads the region has retired in this warp (wait_group), and
                              // with kHBarrier the four warps meet first, so no warp's MMAs still read it -- no warp relies on
                              // another reading only its own 16 A rows.
                              if (w & kHDelayed) {
                                  retire(ns0);        // the next block's group 0, the region's last reader
                                  g0_done = true;
                              }
                              // layer 0 may stage in the region where the last layer of step n - 1 left its output (and its
                              // epilogue overwrites those rows): the epilogue of that layer has read both halves first
                              if (l == 0 && (w & kHFirst) && g >= 1)
                                  tc05::mbar_wait(&bars[B_EPIDONE + ((g - 1) & 1u) * 2 + rb], ((g - 1) >> 1) & 1u);
                              if (w & kHBarrier) tc05::named_sync(3, 128);
                              // pair (j, h) of chunk 8 r + j, row 16 warp + lane / 4 + 8 h: lanes 0-1 of a quad hold its floats
                              // 0-3 (hi slot), lanes 2-3 its floats 4-7 (lo slot), so 8 rows of a quad column are 128
                              // contiguous bytes of either part: conflict-free 8-byte stores
                              const uint32_t sa = tc05::smem_u32(smem) + ((ft & 2u) ? SM.h_lo : SM.h_hi) + (ft & 1u) * 8u +
                                                  tc05::chunk_off(kRows, rb * 64 + tc05::frag_row(ft, 0), 8u * ((w >> 4) & 3u));
#pragma unroll
                              for (int i = 0; i < 32; i += 2)
                                  tc05::st_shared_v2f(sa + (i >> 2) * kRows * 16 + ((i >> 1) & 1) * 128, a[i], a[i + 1]);
                          }
                          ts.lap(kSplitStore);
                      };
                      issue(x, 0, ns0);
#pragma unroll 1
                      for (int pos = 0; pos < ncb; pos += 2) {
                          block(x, y, pos);
                          if (pos + 1 < ncb) block(y, x, pos + 1);
                      }
                      __threadfence_block();
                      tc05::named_sync(3, 128);
                      ts.lap(kSplitBarrier);
                      if (t == 0) SDB_STAMP(n, l, 2 * rb + 1);
                      if (t == 0) SDB_STAMP_SPLIT(n, l, rb, ts);
                      if (t == 0) {
                          if (l == NL - 1) {
                              tc05::mbar_arrive(&bars[B_OUTRDY + rb]);
                              if (rb == 1) tc05::mbar_arrive(&bars[B_HFREE]);
                          } else {
                              tc05::mbar_arrive(&bars[B_ACC + rb]);
                          }
                      }
                  }
              }
          }
      }
    } else if (warp < kProducerWarp0) {
        // =========================== GATHER WARPS (layer-0 operand producers) ===========================
        set_maxnreg<kRegsGather>();
        const int gt = tid - kGatherWarp0 * 32;
        const int row = gt & (kRows - 1), half = gt >> 7;
        uint32_t n = 0;
        for (int it = 0;; it++) {
            if (dyn && gt == 0) {
                // publish the it-th work item of this CTA (slot it & 3 was last used by tile it - 4, which every role has
                // left: this thread is past the STFREE wait of tile it - 2)
                int w = (int)blockIdx.x;
                if (it > 0) w = atomicAdd(p.work_counter, 1) + (int)gridDim.x;
                sWork[it & 3] = w < n_work ? w : -1;
                __threadfence_block();
                *sPub = it + 1;
            }
            const int work = fetch_work(it);
            if (work < 0) break;
            const int tile = RAYQ ? 0 : (ONE_STEP ? work : p.tile_list[rec_work(work) / wmult]);
            const TileCoord tc = tile_coord(p, tile);
            const int y = tc.y0 + (row >> 4), x = tc.x0 + (row & 15);
            const bool valid = (y < p.H) && (x < p.W);
            const long long pix = (long long)y * p.W + x, hw = (long long)p.H * p.W;
            const long long ray = (long long)tc.img * hw + pix;
            if constexpr (SKY) {
                // ---- positional encoding of the ray direction (positional_encoding_kernel.cu:58-72): 5 degrees + orig ----
                uint4 ch[6], cl[6];
                if (half == 0) {
                    float pe[kSkyK0];
#pragma unroll
                    for (int k = 0; k < kSkyK0; k++) pe[k] = 0.0f;
                    if (valid) {
#pragma unroll
                        for (int d = 0; d < 3; d++) {
                            const float v = __ldg(p.raydirs + ray * 3 + d);
#pragma unroll
                            for (int i = 0; i < 5; i++) {
                                const float rad = v * 3.14159265358979323846f * exp2f((float)i);
                                float sn, cs;
                                sincosf(rad, &sn, &cs);
                                pe[(2 * i) * 3 + d] = sn;
                                pe[(2 * i + 1) * 3 + d] = cs;
                            }
                            pe[30 + d] = v;
                        }
                    }
                    pe[kSkyK0 - 1] = 1.0f;      // bias column
#pragma unroll
                    for (int c = 0; c < 6; c++) {
                        const float(&v8)[8] = *reinterpret_cast<const float(*)[8]>(&pe[8 * c]);
                        split8<PREC>(v8, ch[c], cl[c]);
                    }
                    if constexpr (TRAIN) {   // bf16 copy of the layer-0 operand: X0[slot][48] (fc1 weight / bias gradient)
                        const long long slot0 = (long long)work * kRows + row;
#pragma unroll
                        for (int q = 0; q < kSkyK0 / 8; q++)
                            *reinterpret_cast<uint4 *>(rec_chunk(p.tr.x0, slot0, kSkyK0 / 8, q)) =
                                make_uint4(tc05::pack2<true>(pe[8 * q], pe[8 * q + 1]), tc05::pack2<true>(pe[8 * q + 2], pe[8 * q + 3]),
                                           tc05::pack2<true>(pe[8 * q + 4], pe[8 * q + 5]), tc05::pack2<true>(pe[8 * q + 6], pe[8 * q + 7]));
                    }
                }
                if (gt == 0) SDB_MARK(4, 3, n, it);
                if (n > 0) tc05::mbar_wait_backoff(&bars[B_HFREE], (n - 1) & 1);
                if (half == 0) {
#pragma unroll
                    for (int c = 0; c < 6; c++) {
                        const uint32_t off = tc05::chunk_off(kRows, row, c);
                        *reinterpret_cast<uint4 *>(sHhi + off) = ch[c];
                        if constexpr (X3) *reinterpret_cast<uint4 *>(sHlo + off) = cl[c];
                    }
                }
                tc05::fence_proxy_async_smem();
                tc05::mbar_arrive(&bars[B_FEAT]);
                n++;
            } else if constexpr (BWD) {
                // ---- layer-0 operand of the gradient chain: dL/dc [128 rays x 64] fp32 from the compositing backward ----
                for (int s = 0; s < S; s++, n++) {
                    const long long slot = ((long long)work * S + s) * kRows + row;
                    // render chain: dL/dc in slot order; sky chain: dL/dsky in RAY order (zero outside the image)
                    const float4 *src = reinterpret_cast<const float4 *>(p.tr.dc + (SKYBWD ? ray : slot) * kOutC + half * 32);
                    const bool have = SKYBWD ? valid : true;
                    uint4 gh[4], gl[4];
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        float4 a = make_float4(0.0f, 0.0f, 0.0f, 0.0f), b = a;
                        if (have) { a = __ldg(src + 2 * q); b = __ldg(src + 2 * q + 1); }
                        const float v8[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                        split8<PREC>(v8, gh[q], gl[q]);
                        if constexpr (SKYBWD)     // bf16 copy in slot order: operand of the fc_out_c weight-gradient GEMM
                            *reinterpret_cast<uint4 *>(rec_chunk(p.tr.dc16, slot, kOutC / 8, half * 4 + q)) =
                                make_uint4(tc05::pack2<true>(a.x, a.y), tc05::pack2<true>(a.z, a.w), tc05::pack2<true>(b.x, b.y),
                                           tc05::pack2<true>(b.z, b.w));
                    }
                    if (gt == 0) SDB_MARK(4, 3, n, it);
                    if (n > 0) tc05::mbar_wait_backoff(&bars[B_HFREE], (n - 1) & 1);
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const uint32_t off = tc05::chunk_off(kRows, row, half * 4 + q);
                        *reinterpret_cast<uint4 *>(sHhi + off) = gh[q];
                        if constexpr (X3) *reinterpret_cast<uint4 *>(sHlo + off) = gl[q];
                    }
                    tc05::fence_proxy_async_smem();
                    tc05::mbar_arrive(&bars[B_FEAT]);
                }
            } else if constexpr (RAYQ) {
                // ---- ray slots: this role owns the cursors; it refills a slot whose ray has marched all S samples, or was
                //      reported finished by the compositing of two steps ago, from the frame-wide queue of live rays ----
                float *st = sState;                                   // state buffer 0, private to this role in this mode
                const int n_rays = __ldg(p.n_live);                   // live rays listed by prepass_rays_kernel
                const int32_t *rlist = p.tile_list;                   // ... in tile order (ray index inside the image)
                const float ori[3] = {__ldg(p.cam_ori + 0), __ldg(p.cam_ori + 1), __ldg(p.cam_ori + 2)};
                float x5[5];
                x5[3] = __fmul_rn(__fadd_rn(__ldg(p.genc + 0), 1.0f), 0.5f);   // grid.py:144 on dims 3,4
                x5[4] = __fmul_rn(__fadd_rn(__ldg(p.genc + 1), 1.0f), 0.5f);
                for (int s = 0;; s++, n++) {
                    if (s >= 2) {
                        tc05::mbar_wait_backoff(&bars[B_COMP], (uint32_t)(s - 2) & 1u, 32);    // done flags (and stop decision) of step s - 2
                        if (s >= sStop[0]) break;
                    }
                    if (gt == 0) SDB_STAMP(n, 7, 0);                   // (timeline row 7 = this role, preparing step n)
                    if (half == 0) {
                        const int2 cur = sCur[row];
                        int rq = cur.x, sr = cur.y + 1;
                        const bool need = rq < 0 || sr >= S || (s >= 2 && sDone[(s & 1) * kRows + row] == rq + 1);
                        if (need) {
                            rq = -1;
                            sr = 0;
                            if (sExh[4] == 0) {
                                const int idx = atomicAdd(p.work_counter, 1);
                                if (idx < n_rays) rq = __ldg(rlist + idx);
                                else sExh[4] = 1;
                            }
                            uint32_t code0 = 0;
                            if (rq >= 0) {
                                const RayVoxels vox = ray_state(p, st, row, 0, rq, true);      // one image: ray = pixel
                                const float dx = st[(kStDir + 0) * kRows + row];
                                // the ground test of the sky-leak logic looks at EVERY sample position (scenedreamer.py:380), also at
                                // those an early finish will skip; per-sample outputs of skipped samples: weight 0, depth as sampled
                                bool gnd = false;
                                for (int k = 0; k < S; k++) {
                                    const Sample sk = sample_at(p, st, row, k, sFrac, rq);
                                    gnd = gnd || (__fadd_rn(__fmul_rn(dx, sk.depth), ori[0]) <= 1.0f);
                                    if (p.rdepth_out) p.rdepth_out[(long long)rq * S + k] = sk.depth;
                                    if (p.weights_out) p.weights_out[(long long)rq * S + k] = 0.0f;
                                }
                                code0 = (vox.last == 0 ? 0x800u : 0u) | (gnd ? 0x1000u : 0u);
                            }
                            st[kStFlags * kRows + row] = __uint_as_float(code0);
                        }
                        sCur[row] = make_int2(rq, sr);
                    }
                    asm volatile("bar.sync 2, 256;" ::: "memory");
                    if (gt == 0) SDB_STAMP(n, 7, 1);
                    const int2 cur = sCur[row];
                    const bool act = cur.x >= 0;
                    const uint32_t labs = __float_as_uint(st[kStLab * kRows + row]);
                    Sample sm{0.0f, 0.0f, 0};
                    bool oob = true;
                    uint4 fh[8], fl[8];
                    if (act) {
                        sm = sample_at(p, st, row, cur.y, sFrac, cur.x);
                        const float dir[3] = {st[(kStDir + 0) * kRows + row], st[(kStDir + 1) * kRows + row], st[(kStDir + 2) * kRows + row]};
                        oob = grid_coord(p, dir, ori, sm.depth, x5);
                    }
                    encode_features<RAW5D, GU, PREC>(p, mask, sScale, half, x5, oob, fh, fl, [](int, const float (&)[8]) {});
                    const uint4 ext = label_chunk((labs >> (4 * sm.idx)) & 15u, half, one16<PREC>());
                    if (half == 0) {
                        const uint32_t code = __float_as_uint(st[kStFlags * kRows + row]) | (uint32_t)cur.y | (cur.y == 0 ? 0x100u : 0u) |
                                              (cur.y == S - 1 ? 0x200u : 0u);
                        sInfo[(s & 3) * kRows + row] = make_uint4(__float_as_uint(sm.depth), __float_as_uint(sm.nd), (uint32_t)cur.x, code);
                    }
                    if (gt == 0) sExh[s & 3] = sExh[4];               // after the bar.sync: every fetch of this step has been made
                    if (gt == 0) SDB_STAMP(n, 7, 2);
                    if (n > 0) tc05::mbar_wait_backoff(&bars[B_HFREE], (n - 1) & 1);
                    if (gt == 0) SDB_STAMP(n, 7, 3);
                    if (s >= 2 && s >= sStop[0]) break;                // the CTA ended before this step: drop the features
                    store_layer0<X3>(sHhi, sHlo, row, half, fh, fl, ext);
                    tc05::fence_proxy_async_smem();
                    tc05::mbar_arrive(&bars[B_FEAT]);
                }
            } else {
                const int buf = it & 1;
                float *st = sState + buf * kStFloats * kRows;
                // ---- per-ray sampling state (first 128 gather threads) ----
                if (gt == 0) SDB_MARK(4, 1, n, it);
                if (it >= 2) tc05::mbar_wait_backoff(&bars[B_STFREE + buf], ((it >> 1) - 1) & 1);
                if (gt == 0) sStop[buf] = kMaxS + 1;           // undecided (published with the state: bar.sync 2 + STRDY below)
                if (half == 0) {
                    const RayVoxels vox = ray_state(p, st, row, tc.img, pix, valid);
                    const uint32_t flags = (valid && vox.first != 0 ? 1u : 0u) | (vox.last == 0 ? 2u : 0u) | (valid ? 4u : 0u);
                    st[kStFlags * kRows + row] = __uint_as_float(flags);
                }
                asm volatile("bar.sync 2, 256;" ::: "memory");
                if (half == 0) tc05::mbar_arrive(&bars[B_STRDY + buf]);
                const bool live = __float_as_uint(st[kStFlags * kRows + row]) & 1u;
                const uint32_t labs = __float_as_uint(st[kStLab * kRows + row]);
                const float dir[3] = {st[(kStDir + 0) * kRows + row], st[(kStDir + 1) * kRows + row], st[(kStDir + 2) * kRows + row]};
                const float ori[3] = {__ldg(p.cam_ori + tc.img * 3 + 0), __ldg(p.cam_ori + tc.img * 3 + 1), __ldg(p.cam_ori + tc.img * 3 + 2)};
                float x5[5];
                x5[3] = __fmul_rn(__fadd_rn(__ldg(p.genc + tc.img * 2 + 0), 1.0f), 0.5f);   // grid.py:144 on dims 3,4
                x5[4] = __fmul_rn(__fadd_rn(__ldg(p.genc + tc.img * 2 + 1), 1.0f), 0.5f);

                for (int s = 0; s < S; s++, n++) {
                    uint4 fh[8], fl[8];
                    const Sample sm = sample_at(p, st, row, s, sFrac, ray);
                    const bool outside = grid_coord(p, dir, ori, sm.depth, x5);
                    const bool oob = !live || outside;
                    const uint32_t label = (labs >> (4 * sm.idx)) & 15u;
                    if constexpr (TRAIN) {
                        // the sample's record entries that need no features, written before the gather so that the grid
                        // position and the label are not held across it: the position (x3) and X0 columns 128..143 (the
                        // one-hot label and the constant 1, bf16)
                        const long long slot = ((long long)work * S + s) * kRows + row;
                        if (half == 0) p.tr.x3[slot] = make_float4(x5[0], x5[1], x5[2], oob ? -1.0f : 1.0f);
                        *reinterpret_cast<uint4 *>(rec_chunk(p.tr.x0, slot, kX0Cols / 8, kFeat / 8 + half)) = label_chunk(label, half, one16<1>());
                    }
                    encode_features<RAW5D, 8, PREC>(p, mask, sScale, half, x5, oob, fh, fl, [&](int level, const float (&res)[8]) {
                        if constexpr (TRAIN) {   // bf16 copy of the features: X0[slot][8*level ..] (operand of the fc_1 weight gradient)
                            const long long slot = ((long long)work * S + s) * kRows + row;
                            *reinterpret_cast<uint4 *>(rec_chunk(p.tr.x0, slot, kX0Cols / 8, level)) =
                                make_uint4(tc05::pack2<true>(res[0], res[1]), tc05::pack2<true>(res[2], res[3]),
                                           tc05::pack2<true>(res[4], res[5]), tc05::pack2<true>(res[6], res[7]));
                        }
                    });
                    const uint4 ext = label_chunk(label, half, one16<PREC>());
                    if (gt == 0) SDB_MARK(4, 3, n, it);
                    if (n > 0) tc05::mbar_wait_backoff(&bars[B_HFREE], (n - 1) & 1);
                    if (gt == 0) SDB_MARK(4, 4, n, it);
                    if (ESTOP && s >= 2 && s >= sStop[buf]) break;           // the tile ended before this step: drop the features
                    store_layer0<X3>(sHhi, sHlo, row, half, fh, fl, ext);
                    tc05::fence_proxy_async_smem();
                    tc05::mbar_arrive(&bars[B_FEAT]);
                }
            }
        }
    } else {
        // =========================== WEIGHT PRODUCER ===========================
        // One thread keeps the weight ring full, so that no MMA warp waits for a refill: every stage of a step's table (sWalk),
        // in order, goes to ring slot q & 3 once the four MMA warps have released the slot's previous stage (B_WEMPTY), with
        // expect_tx and one bulk copy onto B_WFULL.  It walks the MMA warpgroup's work and step loops and issues exactly the
        // stages that warpgroup consumes, so no copy is in flight when the CTA exits.
        set_maxnreg<kRegsProd>();
        if (warp == kProducerWarp0 && elect_one()) {
            uint32_t n = 0, q = 0;                                    // global step counter, ring stages issued
            uint32_t waited = 0;                                      // (timeline build) cycles in empty-barrier waits of step n
            auto wait_empty = [&]() {
                if (q < 4) return;                                    // the ring starts empty
                const uint32_t c = SDB_CLOCK();
                tc05::mbar_wait(&bars[B_WEMPTY + (q & 3u)], ((q >> 2) - 1) & 1u);
                waited += SDB_CLOCK() - c;
            };
            for (int it = 0;; it++) {
                const int work = fetch_work(it);
                if (work < 0) break;
                const int tile = RAYQ ? 0 : (ONE_STEP ? work : p.tile_list[rec_work(work) / wmult]);
                const uint8_t *pack = p.pack + (long long)tile_coord(p, tile).img * p.pack_stride;
                for (int s = 0; s < SL; s++, n++) {
                    SDB_MARK(3, 1, n, it);
                    waited = 0;
                    // The stop test of step s reads what the compositing of step s - 2 decided, so it follows the wait for
                    // the slot of the step's first stage.  That slot's previous stage is one of the last four of step s - 1,
                    // all in its colour layer (4 stages or more), and each MMA warp released it after its B_OPND waits of
                    // step s - 1 (both row blocks, from layer 1 on).  A row block's operand rows of step s - 1 are handed over
                    // after its compositing of step s - 2.  A later compositing sets sStop to s + 1 or more, which does not
                    // change the test; the reset for the tile two ahead (gather, after STFREE of this one) comes after the
                    // MMA warpgroup has run a step of the next tile, whose stages this thread issues after this test.
                    wait_empty();
                    if (ESTOP && s >= 2 && s >= sStop[it & 1]) break;
                    for (int k = 0; k < kStepStages; k++, q++) {
                        if (k > 0) wait_empty();
                        const uint32_t e = sWalk[k], bytes = (e >> 16) << 11, slot = q & 3u;
                        tc05::mbar_arrive_expect_tx(&bars[B_WFULL + slot], bytes);
                        tc05::bulk_g2s(sRing + slot * kSlot, pack + ((e & 0xffffu) << 11), bytes, &bars[B_WFULL + slot]);
                    }
                    SDB_STAMP_PROD(n, waited);
                }
            }
        }
    }
}

// ---- pre-pass: live-tile list + outputs of sky-only tiles -----------------------------------------
// outputs of a sky-only ray: its weights are zero, all its samples sit at the camera origin (scenedreamer.py:350-354,376)
__device__ __forceinline__ void sky_only_ray(const Params &p, int img, long long ray) {
    const bool is_gnd = __ldg(p.cam_ori + img * 3) <= 1.0f;
    const float none[kOutC] = {};
    finish_ray(p, img, ray, is_gnd, 0, none, 0.0f, 0.0f, true);
    for (int s = 0; s < p.S; s++) {
        if (p.weights_out) p.weights_out[ray * p.S + s] = 0.0f;
        if (p.rdepth_out) p.rdepth_out[ray * p.S + s] = 0.0f;
    }
}

__global__ void __launch_bounds__(kRows)
prepass_kernel(const Params p, int32_t *tile_list, int32_t *n_live)
{
    const int tile = blockIdx.x, row = threadIdx.x;
    const TileCoord tc = tile_coord(p, tile);
    const int y = tc.y0 + (row >> 4), x = tc.x0 + (row & 15);
    const bool valid = (y < p.H) && (x < p.W);
    const long long ray = ((long long)tc.img * p.H + y) * p.W + x;
    const bool live = valid && (__ldg(p.voxel_id + ray * p.M) != 0);
    const int any = __syncthreads_or(live ? 1 : 0);
    if (any) {
        if (row == 0) {
            const int w = atomicAdd(n_live, 1);
            tile_list[w] = tile;
            if (p.tr.tile_work) p.tr.tile_work[tile] = w;
        }
        return;
    }
    if (row == 0 && p.tr.tile_work) p.tr.tile_work[tile] = -1;
    if (valid) sky_only_ray(p, tc.img, ray);
}

// ---- training pre-pass: the live-tile list grouped by image, so that the backward can take the record one image at a time.
// Record header (int32): [0] live tiles of all images, [1 + 2i] first live-list position of image i, [2 + 2i] its live tiles.
// train_prepass_kernel counts per image and leaves each live tile's rank inside its image in tile_work; train_list_kernel
// turns the counts into offsets and the ranks into list positions.
__global__ void __launch_bounds__(kRows)
train_prepass_kernel(const Params p, int32_t *hdr)
{
    const int tile = blockIdx.x, row = threadIdx.x;
    const TileCoord tc = tile_coord(p, tile);
    const int y = tc.y0 + (row >> 4), x = tc.x0 + (row & 15);
    const bool valid = (y < p.H) && (x < p.W);
    const long long ray = ((long long)tc.img * p.H + y) * p.W + x;
    const bool live = valid && (__ldg(p.voxel_id + ray * p.M) != 0);
    if (__syncthreads_or(live ? 1 : 0)) {
        if (row == 0) p.tr.tile_work[tile] = atomicAdd(hdr + 2 + 2 * tc.img, 1);
        return;
    }
    if (row == 0) p.tr.tile_work[tile] = -1;
    if (valid) sky_only_ray(p, tc.img, ray);
}

__global__ void __launch_bounds__(256)
train_list_kernel(const Params p, int32_t *hdr, int32_t *tile_list)
{
    const int tile = blockIdx.x * 256 + threadIdx.x;
    if (tile == 0) {
        int first = 0;
        for (int i = 0; i < p.n_img; i++) { hdr[1 + 2 * i] = first; first += hdr[2 + 2 * i]; }
        hdr[0] = first;
    }
    if (tile >= p.n_tiles) return;
    const int rank = p.tr.tile_work[tile];
    if (rank < 0) return;
    const int img = tile / (p.tiles_x * p.tiles_y);
    int w = rank;
    for (int i = 0; i < img; i++) w += hdr[2 + 2 * i];
    p.tr.tile_work[tile] = w;
    tile_list[w] = tile;
}

// ---- pre-pass of the ray-slot kernel: queue of live rays (tile order) + outputs of every ray that hits nothing ----
__global__ void __launch_bounds__(kRows)
prepass_rays_kernel(const Params p, int32_t *ray_list, int32_t *n_rays)
{
    __shared__ int s_cnt[4], s_base;
    const int tile = blockIdx.x, row = threadIdx.x, warp = row >> 5, lane = row & 31;
    const TileCoord tc = tile_coord(p, tile);
    const int y = tc.y0 + (row >> 4), x = tc.x0 + (row & 15);
    const bool valid = (y < p.H) && (x < p.W);
    const long long ray = ((long long)tc.img * p.H + y) * p.W + x;
    const bool live = valid && (__ldg(p.voxel_id + ray * p.M) != 0);
    const unsigned bal = __ballot_sync(0xffffffffu, live);
    if (lane == 0) s_cnt[warp] = __popc(bal);
    __syncthreads();
    if (row == 0) {
        const int tot = s_cnt[0] + s_cnt[1] + s_cnt[2] + s_cnt[3];
        s_base = tot ? atomicAdd(n_rays, tot) : 0;
    }
    __syncthreads();
    if (live) {
        int pre = __popc(bal & ((1u << lane) - 1u));
        for (int w = 0; w < warp; w++) pre += s_cnt[w];
        ray_list[s_base + pre] = (int32_t)ray;
        return;
    }
    if (valid) sky_only_ray(p, tc.img, ray);
}

// frame-global sky mean from the per-tile partial sums, fixed summation order (deterministic): 16 groups of 64
// threads each add every 16th tile in order, then the 16 partial sums are added in order
constexpr int kMeanGroups = 16;
__global__ void __launch_bounds__(kOutC * kMeanGroups)
sky_mean_kernel(const float *__restrict__ partial, float *__restrict__ sky_avg, int tiles_per_img, float inv_count)
{
    __shared__ float red[kMeanGroups][kOutC];
    const int img = blockIdx.x, c = threadIdx.x & (kOutC - 1), grp = threadIdx.x / kOutC;
    const float *pp = partial + (long long)img * tiles_per_img * kOutC + c;
    float acc = 0.0f;
    for (int t = grp; t < tiles_per_img; t += kMeanGroups) acc += pp[(long long)t * kOutC];
    red[grp][c] = acc;
    __syncthreads();
    if (grp == 0) {
        float a = 0.0f;
#pragma unroll
        for (int k = 0; k < kMeanGroups; k++) a += red[k][c];
        sky_avg[img * kOutC + c] = a * inv_count;
    }
}

// ---- per-scene pre-blend of the two constant encoder dims -------------------------------------------
__global__ void __launch_bounds__(256)
preblend_kernel(const float *__restrict__ table, float *__restrict__ table3, int L, int log2_T, float level_S, int base_res,
                const float *__restrict__ genc)
{
    const uint32_t T = 1u << log2_T, mask = T - 1u;
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= (size_t)L * T) return;
    const uint32_t level = (uint32_t)(i >> log2_T), e = (uint32_t)i & mask;
    const float scale = exp2f(level * level_S) * base_res - 1.0f;
    float f[2];
    uint32_t g[2];
#pragma unroll
    for (int d = 0; d < 2; d++) grid_cell(__fmul_rn(__fadd_rn(genc[d], 1.0f), 0.5f), scale, g[d], f[d]);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const float *tl = table + ((size_t)level << log2_T) * 8;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const GencCorner k = genc_corner(g, f, j);
        const float w = k.w3 * k.w4;
        float v[8];
        ld8(tl + (size_t)((e ^ k.key) & mask) * 8, v);
#pragma unroll
        for (int c = 0; c < 8; c++) acc[c] = fmaf(w, v[c], acc[c]);
    }
    float4 *o = reinterpret_cast<float4 *>(table3 + i * 8);
    o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// ---- weight packer ---------------------------------------------------------------------------------
// fp32 value of the 16-bit part(s) the pack stores for v: hi (+ lo = v - hi at precision 1 / 2).  hi + lo is exact in fp32
// (lo holds the bits below hi's), so it is what the tensor core sums for 1 * hi + 0 * hi + 1 * lo.
template <int PREC>
__device__ __forceinline__ float packed_value(float v) {
    if constexpr (PREC == 1) {
        const float hi = __bfloat162float(__float2bfloat16_rn(v));
        return __fadd_rn(hi, __bfloat162float(__float2bfloat16_rn(v - hi)));
    } else if constexpr (PREC == 2) {
        const float hi = __half2float(__float2half_rn(v));
        return __fadd_rn(hi, __half2float(__float2half_rn(v - hi)));
    } else {
        return __half2float(__float2half_rn(v));
    }
}

// One thread per (layer, n, k) element of the weight matrices, then one per fp32 entry (sigma head, bias table).
//   render: layer 0 [256 x 144]: cols 0..127 fc_1.weight, 128+lab emb[lab][n], 143 fc_1.bias;
//           layers 1..5 [256 x 256]: W*alpha; colour [64 x 256]: W; bias table: beta of fc_2..fc_6, fc_out_c.bias
//   sky:    layer 0 [256 x 48]: cols 0..32 fc1.weight, 47 bias (fc1.bias + fc_z_a(z)); layers 1..4, colour, bias table as above
template <int PREC, bool SKY>
__global__ void __launch_bounds__(256)
pack_kernel(const float *w0, const float *b0, const float *emb, int n_labels, const float *wh, const float *bh,
            const float *wsig, const float *bsig, const float *wout, const float *bout, uint8_t *pack)
{
    constexpr int MODE = SKY ? kSky : kRender;
    constexpr bool X3 = PREC != 0;
    constexpr int PARTS = X3 ? 2 : 1;
    constexpr int NL = Net<MODE>::NL;
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    long long nW = 0;
    for (int l = 0; l < NL; l++) nW += (long long)layerK<MODE>(l) * layerN<MODE>(l);
    if (t < nW) {
        long long r = t;
        int l = 0;
        while (r >= (long long)layerK<MODE>(l) * layerN<MODE>(l)) { r -= (long long)layerK<MODE>(l) * layerN<MODE>(l); l++; }
        const int K = layerK<MODE>(l);
        const int nn = (int)(r / K), k = (int)(r % K);
        float v = 0.0f;
        if (l == 0) {
            if (SKY) {
                if (k < 33) v = w0[(long long)nn * 33 + k];
                else if (k == kSkyK0 - 1) v = b0[nn];
            } else {
                if (k < kFeat) v = w0[(long long)nn * kFeat + k];
                else if (k == kRenderK0 - 1) v = b0[nn];
                else if (k - kFeat < n_labels) v = emb[(long long)(k - kFeat) * kHidden + nn];
            }
        } else if (l == NL - 1) {
            v = wout[(long long)nn * kHidden + k];
        } else {
            v = wh[((long long)(l - 1) * kHidden + nn) * kHidden + k];
        }
        uint8_t *base = pack + layerOff<MODE>(l, PARTS);
        const int nK = K / 16;
        if constexpr (PREC == 1) {
            const __nv_bfloat16 hi = __float2bfloat16_rn(v);
            const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
            *reinterpret_cast<__nv_bfloat16 *>(base + wpack_off(nK, PARTS, nn, k, 0)) = hi;
            *reinterpret_cast<__nv_bfloat16 *>(base + wpack_off(nK, PARTS, nn, k, 1)) = lo;
        } else if constexpr (PREC == 2) {
            const __half hi = __float2half_rn(v);
            const __half lo = __float2half_rn(v - __half2float(hi));
            *reinterpret_cast<__half *>(base + wpack_off(nK, PARTS, nn, k, 0)) = hi;
            *reinterpret_cast<__half *>(base + wpack_off(nK, PARTS, nn, k, 1)) = lo;
        } else {
            *reinterpret_cast<__half *>(base + wpack_off(nK, PARTS, nn, k, 0)) = __float2half_rn(v);
        }
        return;
    }
    long long u = t - nW;
    if (!SKY) {
        if (u < kFTotal) {
            float *F = reinterpret_cast<float *>(pack + layerOff<MODE>(NL, PARTS));
            float v = 0.0f;
            if (u < kHidden) v = wsig[u];
            else if (u == kFBsig) v = bsig[0];
            F[u] = v;
            return;
        }
        u -= kFTotal;
    }
    if (u >= Net<MODE>::NBIAS) return;
    const int l = 1 + (int)(u / kHidden), nn = (int)(u % kHidden);
    const float v = l == NL - 1 ? bout[nn] : bh[(long long)(l - 1) * kHidden + nn];
    reinterpret_cast<float *>(pack + biasOff<MODE>(PARTS))[u] = packed_value<PREC>(v);
}

template <bool SKY>
int launch_pack(const float *w0, const float *b0, const float *emb, int n_labels, const float *wh, const float *bh,
                const float *wsig, const float *bsig, const float *wout, const float *bout, int precision, void *pack,
                cudaStream_t st) {
    constexpr int MODE = SKY ? kSky : kRender;
    long long n = (SKY ? 0 : kFTotal) + Net<MODE>::NBIAS;
    for (int l = 0; l < Net<MODE>::NL; l++) n += (long long)layerK<MODE>(l) * layerN<MODE>(l);
    const int blocks = (int)((n + 255) / 256);
    if (precision == 1)
        pack_kernel<1, SKY><<<blocks, 256, 0, st>>>(w0, b0, emb, n_labels, wh, bh, wsig, bsig, wout, bout, (uint8_t *)pack);
    else if (precision == 2)
        pack_kernel<2, SKY><<<blocks, 256, 0, st>>>(w0, b0, emb, n_labels, wh, bh, wsig, bsig, wout, bout, (uint8_t *)pack);
    else
        pack_kernel<0, SKY><<<blocks, 256, 0, st>>>(w0, b0, emb, n_labels, wh, bh, wsig, bsig, wout, bout, (uint8_t *)pack);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

// Per-CTA fp32 accumulator buffers of the fused kernels ([grid][2][128][128], L2-resident), one per (device, stream): launches
// on one stream are ordered, so they can share it; launches on different streams get different buffers.  A buffer is
// allocated (or grown) on the first launch that needs it and kept for the life of the process.  Allocation is refused while
// the stream is being captured into a CUDA graph: run one launch of the same size outside the capture first.
static int acc_buffers(int grid, cudaStream_t st, float **out) {
    static std::mutex mu;
    static std::map<std::pair<int, cudaStream_t>, std::pair<float *, int>> bufs;
    int dev = 0;
    SDB_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(mu);
    std::pair<float *, int> &b = bufs[std::make_pair(dev, st)];
    if (b.second < grid) {
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        SDB_CUDA(cudaStreamIsCapturing(st, &cs));
        if (cs != cudaStreamCaptureStatusNone) return SDB_EUNSUPPORTED;
        if (b.first) SDB_CUDA(cudaFree(b.first));
        b = std::make_pair((float *)nullptr, 0);
        SDB_CUDA(cudaMalloc(&b.first, (size_t)grid * 2 * kRows * kAccCols * sizeof(float)));
        b.second = grid;
    }
    *out = b.first;
    return SDB_OK;
}

template <int PREC, bool RAW5D, int MODE, bool TRAIN = false, bool RAYQ = false, int GU = 8>
int launch_mlp(const Params &p_in, int grid, cudaStream_t st) {
    Params p = p_in;
    const int e = acc_buffers(grid, st, &p.acc);
    if (e != SDB_OK) return e;
    const size_t smem = smem_map().total;
    cudaFuncAttributes fa;
    SDB_CUDA(cudaFuncGetAttributes(&fa, mlp_kernel<PREC, RAW5D, MODE, TRAIN, RAYQ, GU>));
    if (fa.numRegs < kRegsLaunch) return SDB_EUNSUPPORTED;   // setmaxnreg pool would be too small: refuse rather than hang
    SDB_CUDA(cudaFuncSetAttribute(mlp_kernel<PREC, RAW5D, MODE, TRAIN, RAYQ, GU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mlp_kernel<PREC, RAW5D, MODE, TRAIN, RAYQ, GU><<<grid, kThreads, smem, st>>>(p);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

int launch_train_forward(const Params &p, int precision, int grid, cudaStream_t st) {
    return precision == 0 ? launch_mlp<0, false, kRender, true>(p, grid, st) : launch_mlp<2, false, kRender, true>(p, grid, st);
}
int launch_bwd_chain(const Params &p, int grid, cudaStream_t st) { return launch_mlp<1, false, kBwd>(p, grid, st); }
int launch_sky_train_forward(const Params &p, int grid, cudaStream_t st) { return launch_mlp<2, false, kSky, true>(p, grid, st); }
int launch_sky_bwd_chain(const Params &p, int grid, cudaStream_t st) { return launch_mlp<1, false, kSkyBwd>(p, grid, st); }
int launch_train_prepass(const Params &p, int32_t *hdr, int32_t *tile_list, cudaStream_t st) {
    SDB_CUDA(cudaMemsetAsync(hdr, 0, (size_t)(1 + 2 * p.n_img) * 4, st));
    train_prepass_kernel<<<p.n_tiles, kRows, 0, st>>>(p, hdr);
    SDB_CHECK_LAUNCH();
    train_list_kernel<<<(p.n_tiles + 255) / 256, 256, 0, st>>>(p, hdr, tile_list);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}
int launch_prepass(const Params &p, int32_t *ws, cudaStream_t st) {
    SDB_CUDA(cudaMemsetAsync(ws, 0, 16, st));
    prepass_kernel<<<p.n_tiles, kRows, 0, st>>>(p, ws + 4, ws);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

// ---- weight packer of the gradient chain (kBwd): B operands are the transposed forward weights -------
//   layer 0 [256 x 64]: B[n][k] = fc_out_c.weight[k][n];  layers 1..5 [256 x 256]: B[n][k] = W'_{fc_(7-l)}[k][n]
//   (wh[5-l], the style-modulated weight);  layer 6 [128 x 256]: B[n][k] = fc_1.weight[k][n];  fp32 tail: fc_sigma.weight
//   sky chain (kSkyBwd): layer 0 [256 x 64]: fc_out_c^T; layers 1..4 [256 x 256]: fc5^T .. fc2^T (wh[4-l]); no tail
template <int MODE>
__global__ void __launch_bounds__(256)
pack_bwd_kernel(const float *w1, const float *wh, const float *wsig, const float *wout, uint8_t *pack)
{
    constexpr int PARTS = 2, NL = Net<MODE>::NL;
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    long long nW = 0;
    for (int l = 0; l < NL; l++) nW += (long long)layerK<MODE>(l) * layerN<MODE>(l);
    if (t < nW) {
        long long r = t;
        int l = 0;
        while (r >= (long long)layerK<MODE>(l) * layerN<MODE>(l)) { r -= (long long)layerK<MODE>(l) * layerN<MODE>(l); l++; }
        const int K = layerK<MODE>(l);
        const int nn = (int)(r / K), k = (int)(r % K);
        float v;
        if (l == 0) v = wout[(long long)k * kHidden + nn];
        else if (MODE == kBwd && l == NL - 1) v = w1[(long long)k * kFeat + nn];
        else v = wh[((long long)((MODE == kBwd ? 5 : 4) - l) * kHidden + k) * kHidden + nn];
        uint8_t *base = pack + layerOff<MODE>(l, PARTS);
        const __nv_bfloat16 hi = __float2bfloat16_rn(v);
        const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
        *reinterpret_cast<__nv_bfloat16 *>(base + wpack_off(K / 16, PARTS, nn, k, 0)) = hi;
        *reinterpret_cast<__nv_bfloat16 *>(base + wpack_off(K / 16, PARTS, nn, k, 1)) = lo;
        return;
    }
    if (!Net<MODE>::TAIL) return;
    const long long u = t - nW;
    if (u >= kFTotal) return;
    float *F = reinterpret_cast<float *>(pack + layerOff<MODE>(NL, PARTS));
    F[u] = u < kHidden ? wsig[u] : 0.0f;
}

}  // namespace rf

// Diagnostics: a host-mapped (pinned) int32[64] buffer that CTA 0 fills with progress markers.
extern "C" void sdb_debug_set_progress_buffer(void *mapped) { rf::g_debug_buffer = (int32_t *)mapped; }

extern "C" int64_t sdb_mlp_pack_bytes(int32_t precision) { return rf::packBytes<rf::kRender>(precision != 0 ? 2 : 1); }
extern "C" int64_t sdb_sky_pack_bytes(int32_t precision) { return rf::packBytes<rf::kSky>(precision != 0 ? 2 : 1); }

extern "C" int sdb_pack_mlp(const float *d_w1, const float *d_b1, const float *d_emb, int32_t n_labels,
                            const float *d_wh, const float *d_bh, const float *d_wsig, const float *d_bsig,
                            const float *d_wout, const float *d_bout, int32_t precision, void *d_pack, void *stream)
{
    if (!d_w1 || !d_b1 || !d_emb || !d_wh || !d_bh || !d_wsig || !d_bsig || !d_wout || !d_bout || !d_pack) return SDB_EINVAL;
    if (n_labels < 1 || n_labels > rf::kMaxLabels || precision < 0 || precision > 2) return SDB_EINVAL;
    return rf::launch_pack<false>(d_w1, d_b1, d_emb, n_labels, d_wh, d_bh, d_wsig, d_bsig, d_wout, d_bout, precision, d_pack,
                                  (cudaStream_t)stream);
}

extern "C" int64_t sdb_mlp_backward_pack_bytes(void) { return rf::packBytes<rf::kBwd>(2); }

extern "C" int sdb_pack_mlp_backward(const float *d_w1, const float *d_wh, const float *d_wsig, const float *d_wout,
                                     void *d_pack, void *stream)
{
    using namespace rf;
    if (!d_w1 || !d_wh || !d_wsig || !d_wout || !d_pack) return SDB_EINVAL;
    long long n = kFTotal;
    for (int l = 0; l < Net<kBwd>::NL; l++) n += (long long)layerK<kBwd>(l) * layerN<kBwd>(l);
    pack_bwd_kernel<kBwd><<<(int)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_w1, d_wh, d_wsig, d_wout, (uint8_t *)d_pack);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

extern "C" int64_t sdb_sky_backward_pack_bytes(void) { return rf::packBytes<rf::kSkyBwd>(2); }

extern "C" int sdb_pack_sky_mlp_backward(const float *d_wh, const float *d_wout, void *d_pack, void *stream)
{
    using namespace rf;
    if (!d_wh || !d_wout || !d_pack) return SDB_EINVAL;
    long long n = 0;
    for (int l = 0; l < Net<kSkyBwd>::NL; l++) n += (long long)layerK<kSkyBwd>(l) * layerN<kSkyBwd>(l);
    pack_bwd_kernel<kSkyBwd><<<(int)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(nullptr, d_wh, nullptr, d_wout, (uint8_t *)d_pack);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

extern "C" int sdb_pack_sky_mlp(const float *d_w1, const float *d_b1, const float *d_wh, const float *d_bh,
                                const float *d_wout, const float *d_bout, int32_t precision, void *d_pack, void *stream)
{
    if (!d_w1 || !d_b1 || !d_wh || !d_bh || !d_wout || !d_bout || !d_pack) return SDB_EINVAL;
    if (precision < 0 || precision > 2) return SDB_EINVAL;
    return rf::launch_pack<true>(d_w1, d_b1, nullptr, 0, d_wh, d_bh, nullptr, nullptr, d_wout, d_bout, precision, d_pack,
                                 (cudaStream_t)stream);
}

extern "C" int sdb_preblend_table(const float *d_table, float *d_table3, int32_t L, int32_t log2_T, float level_S,
                                  int32_t base_res, const float *d_global_enc, void *stream)
{
    if (!d_table || !d_table3 || !d_global_enc || L < 1 || L > 32 || log2_T < 4 || log2_T > 24) return SDB_EINVAL;
    const size_t n = (size_t)L << log2_T;
    rf::preblend_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_table, d_table3, L, log2_T, level_S,
                                                                                        base_res, d_global_enc);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

static int64_t sdb_num_tiles(int32_t n_img, int32_t H, int32_t W) {
    return (int64_t)n_img * sdb_div_up(H, rf::kTileH) * sdb_div_up(W, rf::kTileW);
}

// workspace (int32 words): [0] live tiles (tile kernel) / live rays (ray-slot kernel), [1] steps executed (x 128 rows), [2] work
// counter / queue head, [3] 1 = the ray-slot kernel ran, [4 .. 4+tiles) live-tile list, then 4 floats: the by-value camera origin
// (when sdb_render_params.d_cam_ori is NULL), then [R] the queue of live rays
extern "C" int64_t sdb_render_workspace_bytes(int32_t n_img, int32_t H, int32_t W) {
    if (n_img <= 0 || H <= 0 || W <= 0) return 0;
    return (sdb_num_tiles(n_img, H, W) + 8 + (int64_t)n_img * H * W) * 4;      // ... + the live-ray queue of the ray-slot kernel
}

namespace rf {
__global__ void set_cam_kernel(float *dst, float a, float b, float c) { dst[0] = a; dst[1] = b; dst[2] = c; }
__global__ void set_flag_kernel(int32_t *dst) { *dst = 1; }
}

extern "C" int64_t sdb_sky_workspace_bytes(int32_t n_img, int32_t H, int32_t W) {
    if (n_img <= 0 || H <= 0 || W <= 0) return 0;
    return sdb_num_tiles(n_img, H, W) * rf::kOutC * 4;
}

// sky forward, optionally (record != nullptr, fp16x3 only) leaving the training record of the pass
static int sky_forward_impl(const float *d_raydirs, int32_t n_img, int32_t H, int32_t W, const void *d_sky_pack,
                            int64_t pack_stride, int32_t precision, float *d_sky, float *d_sky_avg, void *d_workspace,
                            void *d_record, void *stream)
{
    using namespace rf;
    if (!d_raydirs || !d_sky_pack || !d_sky || !d_sky_avg || !d_workspace) return SDB_EINVAL;
    if (n_img <= 0 || H <= 0 || W <= 0) return SDB_EINVAL;
    if (precision < 0 || precision > 2) return SDB_EUNSUPPORTED;
    if (d_record && precision != 2) return SDB_EUNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    Params p{};
    p.n_img = n_img; p.H = H; p.W = W; p.M = 1; p.S = 1;
    p.raydirs = d_raydirs;
    p.pack = (const uint8_t *)d_sky_pack; p.pack_stride = pack_stride;
    p.sky_out = d_sky; p.sky_partial = (float *)d_workspace;
    p.debug = g_debug_buffer;
    p.tiles_x = sdb_div_up(W, kTileW); p.tiles_y = sdb_div_up(H, kTileH);
    p.n_tiles = n_img * p.tiles_x * p.tiles_y;
    const int grid = p.n_tiles < sdb_num_sms() ? p.n_tiles : sdb_num_sms();
    int rc;
    if (d_record) {
        const SkyRecordLayout rl = sky_record_layout(p.n_tiles);
        uint8_t *rec = (uint8_t *)d_record;
        p.tr.slot_cap = (long long)p.n_tiles * kRows;
        p.tr.x0 = reinterpret_cast<uint16_t *>(rec + rl.x0);
        p.tr.act = reinterpret_cast<uint16_t *>(rec + rl.act);
        p.tr.mask = reinterpret_cast<uint32_t *>(rec + rl.mask);
        rc = launch_sky_train_forward(p, grid, st);
    } else if (precision == 1) rc = launch_mlp<1, false, kSky>(p, grid, st);
    else if (precision == 2) rc = launch_mlp<2, false, kSky>(p, grid, st);
    else rc = launch_mlp<0, false, kSky>(p, grid, st);
    if (rc != SDB_OK) return rc;
    sky_mean_kernel<<<n_img, kOutC * kMeanGroups, 0, st>>>(p.sky_partial, d_sky_avg, p.tiles_x * p.tiles_y, 1.0f / ((float)H * (float)W));
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

extern "C" int sdb_sky_forward(const float *d_raydirs, int32_t n_img, int32_t H, int32_t W, const void *d_sky_pack,
                               int64_t pack_stride, int32_t precision, float *d_sky, float *d_sky_avg, void *d_workspace,
                               void *stream)
{
    return sky_forward_impl(d_raydirs, n_img, H, W, d_sky_pack, pack_stride, precision, d_sky, d_sky_avg, d_workspace, nullptr, stream);
}

extern "C" int64_t sdb_sky_train_record_bytes(int32_t n_img, int32_t H, int32_t W) {
    if (n_img <= 0 || H <= 0 || W <= 0) return 0;
    return (int64_t)rf::sky_record_layout(sdb_num_tiles(n_img, H, W)).total;
}

extern "C" int sdb_sky_train_forward(const float *d_raydirs, int32_t n_img, int32_t H, int32_t W, const void *d_sky_pack,
                                     float *d_sky, float *d_sky_avg, void *d_workspace, void *d_record, void *stream)
{
    if (!d_record) return SDB_EINVAL;
    if (n_img != 1) return n_img < 1 ? SDB_EINVAL : SDB_EUNSUPPORTED;
    return sky_forward_impl(d_raydirs, n_img, H, W, d_sky_pack, 0, 2, d_sky, d_sky_avg, d_workspace, d_record, stream);
}

extern "C" int sdb_sky_train_forward_views(const float *d_raydirs, int32_t n_img, int32_t H, int32_t W, const void *d_sky_pack,
                                           int64_t pack_stride, float *d_sky, float *d_sky_avg, void *d_workspace, void *d_record,
                                           void *stream)
{
    if (!d_record || pack_stride < 0 || (n_img > 1 && pack_stride > 0 && pack_stride < rf::packBytes<rf::kSky>(2))) return SDB_EINVAL;
    return sky_forward_impl(d_raydirs, n_img, H, W, d_sky_pack, pack_stride, 2, d_sky, d_sky_avg, d_workspace, d_record, stream);
}

namespace rf {
// validate the ABI struct and translate it into kernel parameters (tile list / outputs still unset)
int params_from_abi(const sdb_render_params *sp, Params &p)
{
    if (!sp) return SDB_EINVAL;
    if (!sp->d_voxel_id || !sp->d_depth2 || !sp->d_raydirs || !sp->d_global_enc || !sp->d_fractions ||
        !sp->d_label_lut || !sp->d_mlp_pack || !sp->d_sky || !sp->d_sky_avg || !sp->d_net_out || !sp->d_workspace)
        return SDB_EINVAL;
    if ((sp->d_table == nullptr) == (sp->d_table3 == nullptr)) return SDB_EINVAL;
    if (sp->n_img <= 0 || sp->H <= 0 || sp->W <= 0) return SDB_EINVAL;
    if (!sp->d_cam_ori && sp->n_img != 1) return SDB_EINVAL;
    if (sp->M < 1 || sp->M > kMaxM || sp->S < 1 || sp->S > kMaxS || sp->L != kLevels || sp->log2_T < 4 || sp->log2_T > 24 ||
        sp->precision < 0 || sp->precision > 2 || sp->n_lut < 1)
        return SDB_EUNSUPPORTED;
    p = Params{};
    p.n_img = sp->n_img; p.H = sp->H; p.W = sp->W; p.M = sp->M; p.S = sp->S;
    p.voxel_id = sp->d_voxel_id; p.depth2 = sp->d_depth2; p.raydirs = sp->d_raydirs; p.cam_ori = sp->d_cam_ori;
    p.genc = sp->d_global_enc;
    for (int k = 0; k < 3; k++) p.vdim[k] = sp->voxel_dims[k];
    p.sample_depth = sp->sample_depth; p.dists_scale = sp->dists_scale;
    p.early_T = sp->early_stop_transmittance > 0.0f ? sp->early_stop_transmittance : 0.0f;
    p.fractions = sp->d_fractions; p.uniforms = sp->d_uniforms;
    p.lut = sp->d_label_lut; p.n_lut = sp->n_lut;
    p.raw5d = sp->d_table != nullptr;
    p.table = p.raw5d ? sp->d_table : sp->d_table3;
    p.log2_T = sp->log2_T; p.level_S = sp->level_S; p.base_res = sp->base_res;
    p.pack = (const uint8_t *)sp->d_mlp_pack; p.pack_stride = sp->mlp_pack_stride;
    p.sky = sp->d_sky; p.sky_avg = sp->d_sky_avg;
    p.net_out = sp->d_net_out; p.depth_out = sp->d_depth_out; p.total_weight = sp->d_total_weight;
    p.weights_out = sp->d_weights_out; p.rdepth_out = sp->d_rand_depth_out;
    p.debug = g_debug_buffer;
    p.tiles_x = sdb_div_up(p.W, kTileW); p.tiles_y = sdb_div_up(p.H, kTileH);
    p.n_tiles = p.n_img * p.tiles_x * p.tiles_y;
    if (!sp->d_cam_ori) p.cam_ori = reinterpret_cast<const float *>((const int32_t *)sp->d_workspace + 4 + p.n_tiles);
    return SDB_OK;
}

// by-value camera origin -> its slot behind the tile list (first thing on the stream of a render call)
int stage_cam_ori(const sdb_render_params *sp, const Params &p, cudaStream_t st)
{
    if (sp->d_cam_ori) return SDB_OK;
    set_cam_kernel<<<1, 1, 0, st>>>(const_cast<float *>(p.cam_ori), sp->cam_ori_value[0], sp->cam_ori_value[1], sp->cam_ori_value[2]);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}
}  // namespace rf

extern "C" int sdb_render_rays_forward(const sdb_render_params *sp, void *stream)
{
    using namespace rf;
    cudaStream_t st = (cudaStream_t)stream;
    Params p;
    {
        const int rc = params_from_abi(sp, p);
        if (rc != SDB_OK) return rc;
    }
    int32_t *ws = (int32_t *)sp->d_workspace;
    p.n_live = ws; p.tile_list = ws + 4; p.steps_done = ws + 1; p.work_counter = ws + 2;
    {
        const int rc = stage_cam_ori(sp, p, st);
        if (rc != SDB_OK) return rc;
    }
    // Ray slots (mlp_kernel<.., RAYQ>): one image over the pre-blended table -- what inference renders.  SDB_RAY_SLOTS=0 keeps the
    // tile kernel (diagnostics / comparison).
    const char *env_rq = getenv("SDB_RAY_SLOTS");
    const bool rayq = !p.raw5d && p.n_img == 1 && !(env_rq && atoi(env_rq) == 0);
    if (rayq) {
        int32_t *ray_list = ws + 8 + p.n_tiles;
        SDB_CUDA(cudaMemsetAsync(ws, 0, 16, st));
        prepass_rays_kernel<<<p.n_tiles, kRows, 0, st>>>(p, ray_list, ws);
        SDB_CHECK_LAUNCH();
        p.tile_list = ray_list;
        // one CTA per SM, but never more CTAs than 128-ray groups the frame could fill (small frames)
        const long long groups = ((long long)p.H * p.W + kRows - 1) / kRows;
        const int grid = groups < sdb_num_sms() ? (int)groups : sdb_num_sms();
        int rc;
        if (sp->precision == 0) rc = launch_mlp<0, false, kRender, false, true>(p, grid, st);
        else if (sp->precision == 1) rc = launch_mlp<1, false, kRender, false, true>(p, grid, st);
        else {
            // gathers in flight per lane: 2 corners (4 LDG.128) by default, a choice measured on the previous GPU generation and not
            // re-measured on H100; SDB_GATHER_UNROLL=8 selects the fully unrolled level
            static const int gu = [] { const char *e = getenv("SDB_GATHER_UNROLL"); return e ? atoi(e) : 2; }();
            if (gu == 8) rc = launch_mlp<2, false, kRender, false, true>(p, grid, st);
            else rc = launch_mlp<2, false, kRender, false, true, 2>(p, grid, st);
        }
        if (rc != SDB_OK) return rc;
        set_flag_kernel<<<1, 1, 0, st>>>(ws + 3);
        SDB_CHECK_LAUNCH();
        return SDB_OK;
    }
    {
        const int rc = launch_prepass(p, ws, st);
        if (rc != SDB_OK) return rc;
    }
    const int grid = p.n_tiles < sdb_num_sms() ? p.n_tiles : sdb_num_sms();
    switch (sp->precision * 2 + (p.raw5d ? 1 : 0)) {
        case 0: return launch_mlp<0, false, kRender>(p, grid, st);
        case 1: return launch_mlp<0, true, kRender>(p, grid, st);
        case 2: return launch_mlp<1, false, kRender>(p, grid, st);
        case 3: return launch_mlp<1, true, kRender>(p, grid, st);
        case 4: return launch_mlp<2, false, kRender>(p, grid, st);
        default: return launch_mlp<2, true, kRender>(p, grid, st);
    }
}
