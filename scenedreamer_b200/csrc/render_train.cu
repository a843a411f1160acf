// Training side of the fused per-pixel path (a7 + the backward of a8/a10/a11), sm_90a.
//
// Behavioural contract = what torch.autograd computes for Generator._forward_perpix in the reference under
// train.py (imaginaire/generators/scenedreamer.py:313-428): gradients of net_out with respect to
//   hash_encoder.embeddings and the scene code     gridencoder.cu:227-343 (kernel_grid_backward, kernel_input_backward)
//   render_net.* (LightningMLP / ModLinear)        model_utils/layers.py:92-126, :241-271
//   the sky features (-> sky_net)                  scenedreamer.py:387-413
// through volum_rendering_relu (mc_utils.py:154-161), clamp and the sky blend (scenedreamer.py:373-413).
//
// GPU mapping ("split-fused", DESIGN.md section 3.6): the forward pass (render_fused.cu, TRAIN variant) leaves a
// per-sample record in HBM (about 3.9 KB per sample -- 6.7 GB for a 256x256x24 training view, a few per cent of the
// 180 GB), then
//   1. composite_backward_kernel  : one warp per ray, lanes over the 64 feature channels / the S samples;
//   2. mlp_kernel<bf16x3, kBwd>   : the data-gradient chain on the same wgmma engine as the forward
//                                   (transposed weights in the ring, LeakyReLU' from recorded sign words);
//   3. table3_backward_kernel     : scatter into the PRE-BLENDED 3-D table (8 corners instead of 32, vector
//                                   red.add), then the transpose of the pre-blend (the same gather kernel:
//                                   XOR-indexing is an involution) and the scene-code gradient;
//   4. weight gradients           : dZ^T * A over all samples on the tensor cores (wgrad.cu): the bf16 records are
//                                   MMA-ready tiles, bulk-copied into shared memory, fp32 accumulators in registers.
#include <stdio.h>
#include <stdlib.h>

#include "rf_common.cuh"
#include "wgrad.cuh"

namespace rf {

// ---- record / workspace layouts --------------------------------------------------------------------
struct RecordLayout { size_t hdr, tile_list, tile_work, rayflags, x3, x0, act, mask, sig, nds, c, total; };
static size_t align_up(size_t v) { return rf_align_up(v); }
static RecordLayout record_layout(long long n_tiles, int S) {
    const size_t cap = (size_t)n_tiles * S * kRows, steps = (size_t)n_tiles * S;
    RecordLayout r{};
    size_t o = 0;
    r.hdr = o; o += 16;
    r.tile_list = o; o = align_up(o + (size_t)n_tiles * 4);      // directly behind the 16-byte header (prepass contract)
    r.tile_work = o; o = align_up(o + (size_t)n_tiles * 4);
    r.rayflags = o; o = align_up(o + (size_t)n_tiles * kRows * 4);
    r.x3 = o; o = align_up(o + cap * 16);
    r.x0 = o; o = align_up(o + cap * kX0Cols * 2);
    r.act = o; o = align_up(o + (size_t)kNumAct * cap * kActCols * 2);
    r.mask = o; o = align_up(o + steps * kNumAct * kRows * 8 * 4);
    r.sig = o; o = align_up(o + cap * 4);
    r.nds = o; o = align_up(o + cap * 4);
    r.c = o; o = align_up(o + cap * kOutC * 4);
    r.total = o;
    return r;
}
static void bind_record(Params &p, uint8_t *rec, const RecordLayout &r) {
    p.n_live = reinterpret_cast<const int32_t *>(rec + r.hdr);
    p.tile_list = reinterpret_cast<const int32_t *>(rec + r.tile_list);
    p.tr.slot_cap = (long long)p.n_tiles * p.S * kRows;
    p.tr.tile_work = reinterpret_cast<int32_t *>(rec + r.tile_work);
    p.tr.rayflags = reinterpret_cast<uint32_t *>(rec + r.rayflags);
    p.tr.x3 = reinterpret_cast<float4 *>(rec + r.x3);
    p.tr.x0 = reinterpret_cast<uint16_t *>(rec + r.x0);
    p.tr.act = reinterpret_cast<uint16_t *>(rec + r.act);
    p.tr.mask = reinterpret_cast<uint32_t *>(rec + r.mask);
    p.tr.sig = reinterpret_cast<float *>(rec + r.sig);
    p.tr.nds = reinterpret_cast<float *>(rec + r.nds);
    p.tr.c = reinterpret_cast<float *>(rec + r.c);
}

struct BwdLayout { size_t dc32, dc16, dsig32, dsig16, dz, dx0, dt3, total; };
static BwdLayout bwd_layout(long long n_tiles, int S, int L, int log2_T) {
    const size_t cap = (size_t)n_tiles * S * kRows;
    BwdLayout b{};
    size_t o = 0;
    b.dc32 = o; o = align_up(o + cap * kOutC * 4);
    b.dc16 = o; o = align_up(o + cap * kOutC * 2);
    b.dsig32 = o; o = align_up(o + cap * 4);
    b.dsig16 = o; o = align_up(o + cap * 8 * 2);
    b.dz = o; o = align_up(o + (size_t)kNumAct * cap * kHidden * 2);
    b.dx0 = o; o = align_up(o + cap * kFeat * 4);
    b.dt3 = o; o = align_up(o + ((size_t)L << log2_T) * 8 * 4);
    b.total = o;
    return b;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ bool in_clamp(float v) { return v >= -1.0f && v <= 1.0f; }   // torch.clamp passes the gradient on [min, max]
__device__ __forceinline__ float clamp1(float v) { return fminf(fmaxf(v, -1.0f), 1.0f) + 1.0f; }

// ---- 1. compositing backward -----------------------------------------------------------------------
// One CTA per ray tile (live or not), one warp per ray at a time; lane = feature channels (2*lane, 2*lane+1) in
// the channel phases and = sample index in the per-sample phases (S <= 64: two samples per lane).
//   forward (scenedreamer.py:373-413):  e_s = relu(sigma_s) * nds_s,  T_s = exp(-sum_{t<s} e_t),
//     w_s = live * (1 - exp(-e_s)) * T_s,  out = sum_s w_s (clamp(c_s)+1) + (1 - sum_s w_s)(clamp(sky)+1) - 1
//   backward:  dL/dw_s = g . (clamp(c_s)+1) - g . (clamp(sky)+1)
//              dL/de_s = dL/dw_s * T_s exp(-e_s) - sum_{t>s} dL/dw_t * w_t
//              dL/dsigma_s = [sigma_s > 0] nds_s dL/de_s,   dL/dc_s = w_s g [c_s in [-1,1]]
//              dL/dsky = (1 - W) g [sky in [-1,1]]  (routed to the ray's sky feature or, where nosky, to sky_avg)
__global__ void __launch_bounds__(256)
composite_backward_kernel(const Params p, const float *__restrict__ g_out, float *__restrict__ dsky,
                          float *__restrict__ dsky_avg, float *__restrict__ dc32, uint16_t *__restrict__ dc16,
                          float *__restrict__ dsig32, uint16_t *__restrict__ dsig16)
{
    __shared__ float s_avg[8][kOutC];
    const int tile = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const TileCoord tc = tile_coord(p, tile);
    const int work = p.tr.tile_work[tile];
    const int S = p.S;
    const unsigned full = 0xffffffffu;
    float avg0 = 0.0f, avg1 = 0.0f;
    const float2 skavg = *reinterpret_cast<const float2 *>(p.sky_avg + (long long)tc.img * kOutC + 2 * lane);

    for (int row = warp; row < kRows; row += 8) {
        const int y = tc.y0 + (row >> 4), x = tc.x0 + (row & 15);
        const bool in_img = (y < p.H) && (x < p.W);
        const long long ray = ((long long)tc.img * p.H + y) * p.W + x;
        float2 g = make_float2(0.0f, 0.0f);
        if (in_img) g = *reinterpret_cast<const float2 *>(g_out + ray * kOutC + 2 * lane);
        if (work < 0) {
            // tile without any voxel hit (prepass_kernel wrote its output): net_out = clamp(sky') , weight 1
            if (!in_img) continue;
            const bool nosky = __ldg(p.cam_ori + tc.img * 3) <= 1.0f;
            const float2 sk = nosky ? skavg : *reinterpret_cast<const float2 *>(p.sky + ray * kOutC + 2 * lane);
            const float d0 = in_clamp(sk.x) ? g.x : 0.0f, d1 = in_clamp(sk.y) ? g.y : 0.0f;
            if (nosky) { avg0 += d0; avg1 += d1; }
            *reinterpret_cast<float2 *>(dsky + ray * kOutC + 2 * lane) = nosky ? make_float2(0.0f, 0.0f) : make_float2(d0, d1);
            continue;
        }
        const uint32_t fl = p.tr.rayflags[(long long)work * kRows + row];
        const bool live = fl & 1u, nosky = fl & 2u, valid = fl & 4u;
        const long long slot0 = (long long)work * S * kRows + row;      // slot of sample s: slot0 + s * 128

        // ---- phase 1: compositing weights, every lane walks the ray; lane s (and s-32) keeps sample s ----
        float w0 = 0, T0 = 0, e0 = 0, sg0 = 0, nd0 = 0, w1 = 0, T1 = 0, e1 = 0, sg1 = 0, nd1 = 0;
        float E = 0.0f, W = 0.0f;
        for (int s = 0; s < S; s++) {
            const float sig = p.tr.sig[slot0 + (long long)s * kRows], nds = p.tr.nds[slot0 + (long long)s * kRows];
            const float e = __fmul_rn(fmaxf(sig, 0.0f), nds);
            const float T = expf(-E);
            const float w = live ? (1.0f - expf(-e)) * T : 0.0f;
            E = __fadd_rn(E, e);
            W += w;
            if (s == lane) { w0 = w; T0 = T; e0 = e; sg0 = sig; nd0 = nds; }
            if (s == lane + 32) { w1 = w; T1 = T; e1 = e; sg1 = sig; nd1 = nds; }
        }
        // ---- sky term ----
        const float2 sk = nosky ? skavg : (valid ? *reinterpret_cast<const float2 *>(p.sky + ray * kOutC + 2 * lane)
                                                 : make_float2(0.0f, 0.0f));
        const float gsky = warp_sum(g.x * clamp1(sk.x) + g.y * clamp1(sk.y));
        // ---- phase 2: dL/dw_s and dL/dc_s ----
        float dw0 = 0.0f, dw1 = 0.0f;
        for (int s = 0; s < S; s++) {
            const long long slot = slot0 + (long long)s * kRows;
            const float2 c = *reinterpret_cast<const float2 *>(p.tr.c + slot * kOutC + 2 * lane);
            const float dot = warp_sum(g.x * clamp1(c.x) + g.y * clamp1(c.y));
            const float dw = live ? dot - gsky : 0.0f;
            const float ws = __shfl_sync(full, s < 32 ? w0 : w1, s & 31);
            const float dcx = in_clamp(c.x) ? ws * g.x : 0.0f, dcy = in_clamp(c.y) ? ws * g.y : 0.0f;
            *reinterpret_cast<float2 *>(dc32 + slot * kOutC + 2 * lane) = make_float2(dcx, dcy);
            *reinterpret_cast<uint32_t *>(rec_chunk(dc16, slot, kOutC / 8, lane >> 2) + 2 * (lane & 3)) = tc05::pack2<true>(dcx, dcy);
            if (s == lane) dw0 = dw;
            if (s == lane + 32) dw1 = dw;
        }
        // ---- phase 3: dL/dsigma_s (lane = sample): suffix sums of dw_t * w_t over t > s ----
        const float P0 = dw0 * w0, P1 = dw1 * w1;          // zero beyond S (never assigned)
        float suf0 = P0, suf1 = P1;                        // inclusive suffix sums inside each group of 32
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float t0 = __shfl_down_sync(full, suf0, o), t1 = __shfl_down_sync(full, suf1, o);
            if (lane + o < 32) { suf0 += t0; suf1 += t1; }
        }
        const float tot1 = __shfl_sync(full, suf1, 0);
        float ex0 = __shfl_down_sync(full, suf0, 1), ex1 = __shfl_down_sync(full, suf1, 1);
        if (lane == 31) { ex0 = 0.0f; ex1 = 0.0f; }
        ex0 += tot1;
        if (lane < S) {
            const float de = dw0 * (T0 * expf(-e0)) - ex0;
            const float ds = sg0 > 0.0f ? de * nd0 : 0.0f;
            const long long slot = slot0 + (long long)lane * kRows;
            dsig32[slot] = ds;
            *reinterpret_cast<uint4 *>(dsig16 + slot * 8) = make_uint4(tc05::pack2<true>(ds, 0.0f), 0u, 0u, 0u);
        }
        if (lane + 32 < S) {
            const float de = dw1 * (T1 * expf(-e1)) - ex1;
            const float ds = sg1 > 0.0f ? de * nd1 : 0.0f;
            const long long slot = slot0 + (long long)(lane + 32) * kRows;
            dsig32[slot] = ds;
            *reinterpret_cast<uint4 *>(dsig16 + slot * 8) = make_uint4(tc05::pack2<true>(ds, 0.0f), 0u, 0u, 0u);
        }
        // ---- sky gradient ----
        if (valid) {
            const float skw = 1.0f - W;
            const float d0 = in_clamp(sk.x) ? skw * g.x : 0.0f, d1 = in_clamp(sk.y) ? skw * g.y : 0.0f;
            if (nosky) { avg0 += d0; avg1 += d1; }
            *reinterpret_cast<float2 *>(dsky + ray * kOutC + 2 * lane) = nosky ? make_float2(0.0f, 0.0f) : make_float2(d0, d1);
        }
    }
    s_avg[warp][2 * lane] = avg0;
    s_avg[warp][2 * lane + 1] = avg1;
    __syncthreads();
    if (threadIdx.x < kOutC) {
        float a = 0.0f;
#pragma unroll
        for (int w = 0; w < 8; w++) a += s_avg[w][threadIdx.x];
        if (a != 0.0f) atomicAdd(dsky_avg + (long long)tc.img * kOutC + threadIdx.x, a);
    }
}

// ---- 3a. scatter d(features) into the pre-blended table gradient --------------------------------------
// thread = (slot, level), level-major grid so that a wave of CTAs works on one 16 MB level slice (L2-resident).
// A warp is 32 neighbouring rays of one tile at one sample step: on the coarse levels they fall into the same cell,
// so their 8 corner rows coincide and a plain scatter serialises on a handful of addresses (the reference's
// kernel_grid_backward has the same hot spot, gridencoder.cu:307-311).  For level < agg_levels the warp therefore
// groups equal row indices with match.any, reduces each group with shuffles and lets the group leader issue the
// two vector reductions; with more than 4 distinct rows in the warp (fine levels) every lane scatters on its own.
__device__ __forceinline__ void red_add8(float *dst, const float (&v)[8]) {
    atomicAdd(reinterpret_cast<float4 *>(dst), make_float4(v[0], v[1], v[2], v[3]));
    atomicAdd(reinterpret_cast<float4 *>(dst) + 1, make_float4(v[4], v[5], v[6], v[7]));
}

__global__ void __launch_bounds__(256)
table3_backward_kernel(const Params p, const float *__restrict__ dx0, float *__restrict__ dt3, int agg_levels)
{
    // the number of live slots is read on the device: the host never waits for the forward pass to size a launch
    const long long n_slots = (long long)__ldg(p.n_live) * p.S * kRows;
    const long long slot = blockIdx.x * 256ll + threadIdx.x;
    const int level = blockIdx.y, lane = threadIdx.x & 31;
    const unsigned full = 0xffffffffu;
    bool active = slot < n_slots;
    float4 x = make_float4(0.0f, 0.0f, 0.0f, -1.0f);
    if (active) x = p.tr.x3[slot];
    active = active && !(x.w < 0.0f);                          // outside the volume / sky-only ray: no table contribution
    float g[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    if (active) {
        ld8(dx0 + slot * kFeat + level * 8, g);
        bool any = false;
#pragma unroll
        for (int c = 0; c < 8; c++) any = any || (g[c] != 0.0f);
        active = any;
    }
    const bool agg = level < agg_levels;                       // block-uniform
    if (!agg && !active) return;
    if (agg && __ballot_sync(full, active) == 0u) return;      // warp-uniform
    const float scale = exp2f(level * p.level_S) * p.base_res - 1.0f;      // gridencoder.cu:126
    const uint32_t mask = (1u << p.log2_T) - 1u;
    const float xs[3] = {x.x, x.y, x.z};
    const Corners3 cn = corners3(mask, scale, xs);
    float *gt = dt3 + ((size_t)level << p.log2_T) * 8;
    if (!agg) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            float v[8];
#pragma unroll
            for (int c = 0; c < 8; c++) v[c] = cn.w[i] * g[c];
            red_add8(gt + (size_t)cn.idx[i] * 8, v);
        }
        return;
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const uint32_t key = active ? cn.idx[i] : 0xffffffffu;      // inactive lanes form their own (ignored) group
        float v[8];
#pragma unroll
        for (int c = 0; c < 8; c++) v[c] = active ? cn.w[i] * g[c] : 0.0f;
        const unsigned grp = __match_any_sync(full, key);
        const int leader = __ffs(grp) - 1;
        unsigned leaders = __ballot_sync(full, lane == leader);
        if (__popc(leaders) > 4) {
            if (active) red_add8(gt + (size_t)key * 8, v);
            continue;
        }
        while (leaders) {
            const int L = __ffs(leaders) - 1;
            leaders &= leaders - 1;
            const unsigned m = __shfl_sync(full, grp, L);
            const bool mine = (m >> lane) & 1u;
            float s[8];
#pragma unroll
            for (int c = 0; c < 8; c++) {
                float t = mine ? v[c] : 0.0f;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(full, t, o);
                s[c] = t;
            }
            if (lane == L && key != 0xffffffffu) red_add8(gt + (size_t)key * 8, s);
        }
    }
}

// ---- 3b. scene-code gradient: dL/dgenc_d = sum_{l,i} dT3[l][i] . sum_j (dw_j/dgenc_d) T[l][i ^ K_j] --------------
// (the chain rule through preblend_kernel of render_fused.cu; the reference obtains the same number from dy_dx of
//  dims 3,4 in kernel_grid / kernel_input_backward, gridencoder.cu:172-224, :317-343)
__global__ void __launch_bounds__(256)
genc_backward_kernel(const float *__restrict__ table, const float *__restrict__ dt3, int L, int log2_T, float level_S,
                     int base_res, const float *__restrict__ genc, float *__restrict__ dgenc)
{
    __shared__ float red[2][8];
    const uint32_t T = 1u << log2_T, mask = T - 1u;
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    float r0 = 0.0f, r1 = 0.0f;
    if (i < (size_t)L * T) {
        float d[8];
        ld8(dt3 + i * 8, d);
        bool any = false;
#pragma unroll
        for (int c = 0; c < 8; c++) any = any || (d[c] != 0.0f);
        if (any) {
            const uint32_t level = (uint32_t)(i >> log2_T), e = (uint32_t)i & mask;
            const float scale = exp2f(level * level_S) * base_res - 1.0f;
            float f[2];
            uint32_t g[2];
#pragma unroll
            for (int k = 0; k < 2; k++) {
                const float x = __fmul_rn(__fadd_rn(genc[k], 1.0f), 0.5f);
                const float pos = fmaf(x, scale, 0.5f);
                g[k] = (uint32_t)floorf(pos);
                f[k] = pos - (float)g[k];
            }
            const float *tl = table + ((size_t)level << log2_T) * 8;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int b3 = j & 1, b4 = j >> 1;
                const uint32_t K = ((g[0] + b3) * kPrime3) ^ ((g[1] + b4) * kPrime4);
                float v[8];
                ld8(tl + (size_t)((e ^ K) & mask) * 8, v);
                float dot = 0.0f;
#pragma unroll
                for (int c = 0; c < 8; c++) dot = fmaf(v[c], d[c], dot);
                r0 += (b3 ? 1.0f : -1.0f) * (b4 ? f[1] : 1.0f - f[1]) * dot;
                r1 += (b3 ? f[0] : 1.0f - f[0]) * (b4 ? 1.0f : -1.0f) * dot;
            }
            r0 *= scale * 0.5f;      // d pos / d genc = scale * d((genc + 1) / 2) / d genc
            r1 *= scale * 0.5f;
        }
    }
    r0 = warp_sum(r0);
    r1 = warp_sum(r1);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[0][warp] = r0; red[1][warp] = r1; }
    __syncthreads();
    if (threadIdx.x < 2) {
        float a = 0.0f;
#pragma unroll
        for (int w = 0; w < 8; w++) a += red[threadIdx.x][w];
        if (a != 0.0f) atomicAdd(dgenc + threadIdx.x, a);
    }
}

// ---- 4. weight gradients: job lists for wgrad.cu ------------------------------------------------------------------
// One job per 128-row M-tile of a layer's output.  A = the layer's input record, Z = the gradient at its pre-activation.
static void add_jobs(WgJob *jobs, int &n, const uint16_t *A, int a_cols, const uint16_t *Z, int z_cols, float *out, int n_out) {
    for (int r0 = 0; r0 < z_cols; r0 += 128) {
        WgJob &j = jobs[n++];
        j = WgJob{};
        j.A = A; j.Z = Z; j.out = out;
        j.a_chunks = a_cols / 8;
        j.z_chunks_total = z_cols / 8; j.z_chunk0 = r0 / 8; j.z_chunks = (z_cols - r0 < 128 ? z_cols - r0 : 128) / 8;
        j.ld_out = a_cols; j.row0 = r0; j.rows = (n_out - r0 < 128 ? n_out - r0 : 128);
    }
}

}  // namespace rf

extern "C" int64_t sdb_render_train_record_bytes(int32_t n_img, int32_t H, int32_t W, int32_t S) {
    using namespace rf;
    if (n_img <= 0 || H <= 0 || W <= 0 || S < 1 || S > kMaxS) return 0;
    const long long n_tiles = (long long)n_img * sdb_div_up(H, kTileH) * sdb_div_up(W, kTileW);
    return (int64_t)record_layout(n_tiles, S).total;
}

extern "C" int64_t sdb_render_backward_workspace_bytes(int32_t n_img, int32_t H, int32_t W, int32_t S, int32_t L, int32_t log2_T) {
    using namespace rf;
    if (n_img <= 0 || H <= 0 || W <= 0 || S < 1 || S > kMaxS || L < 1 || log2_T < 4 || log2_T > 24) return 0;
    const long long n_tiles = (long long)n_img * sdb_div_up(H, kTileH) * sdb_div_up(W, kTileW);
    return (int64_t)bwd_layout(n_tiles, S, L, log2_T).total;
}

// Diagnostics: byte offsets of the record (11 values: hdr, tile_list, tile_work, rayflags, x3, x0, act, mask, sig, nds, c) and of
// the backward workspace (7 values: dc32, dc16, dsig32, dsig16, dz, dx0, dt3), then the two total sizes -- 20 int64 in all.
extern "C" int sdb_debug_train_layout(int32_t n_img, int32_t H, int32_t W, int32_t S, int32_t L, int32_t log2_T, int64_t *out)
{
    using namespace rf;
    if (!out || n_img <= 0 || H <= 0 || W <= 0 || S < 1 || S > kMaxS) return SDB_EINVAL;
    const long long n_tiles = (long long)n_img * sdb_div_up(H, kTileH) * sdb_div_up(W, kTileW);
    const RecordLayout r = record_layout(n_tiles, S);
    const BwdLayout b = bwd_layout(n_tiles, S, L, log2_T);
    const size_t v[20] = {r.hdr, r.tile_list, r.tile_work, r.rayflags, r.x3, r.x0, r.act, r.mask, r.sig, r.nds, r.c,
                          b.dc32, b.dc16, b.dsig32, b.dsig16, b.dz, b.dx0, b.dt3, r.total, b.total};
    for (int i = 0; i < 20; i++) out[i] = (int64_t)v[i];
    return SDB_OK;
}

extern "C" int sdb_render_rays_train_forward(const sdb_render_params *sp, void *d_record, void *stream)
{
    using namespace rf;
    if (!d_record || !sp || !sp->d_cam_ori) return SDB_EINVAL;      // training takes the camera origin from device memory
    cudaStream_t st = (cudaStream_t)stream;
    Params p;
    {
        const int rc = params_from_abi(sp, p);
        if (rc != SDB_OK) return rc;
    }
    if (p.raw5d || sp->precision != 2) return SDB_EUNSUPPORTED;      // record + backward are built on the pre-blended table, fp16x3
    if (p.n_img != 1) return SDB_EUNSUPPORTED;                        // one view (one style code) per record: the weight gradients are per style
    uint8_t *rec = (uint8_t *)d_record;
    const RecordLayout rl = record_layout(p.n_tiles, p.S);
    bind_record(p, rec, rl);
    {
        const int rc = launch_prepass(p, reinterpret_cast<int32_t *>(rec + rl.hdr), st);
        if (rc != SDB_OK) return rc;
    }
    const int grid = p.n_tiles < sdb_num_sms() ? p.n_tiles : sdb_num_sms();
    return launch_train_forward(p, grid, st);
}

extern "C" int sdb_render_rays_backward(const sdb_render_params *sp, const void *d_record, const sdb_render_grads *g, void *stream)
{
    using namespace rf;
    if (!d_record || !g || !sp || !sp->d_cam_ori) return SDB_EINVAL;
    if (!g->d_grad_net_out || !g->d_bwd_pack || !g->d_table || !g->d_grad_table || !g->d_grad_global_enc || !g->d_grad_w1ext ||
        !g->d_grad_wh || !g->d_grad_wsig || !g->d_grad_wout || !g->d_grad_sky || !g->d_grad_sky_avg || !g->d_workspace)
        return SDB_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    Params p;
    {
        const int rc = params_from_abi(sp, p);
        if (rc != SDB_OK) return rc;
    }
    if (p.raw5d || p.n_img != 1) return SDB_EUNSUPPORTED;
    uint8_t *rec = (uint8_t *)const_cast<void *>(d_record);
    const RecordLayout rl = record_layout(p.n_tiles, p.S);
    bind_record(p, rec, rl);
    const BwdLayout bl = bwd_layout(p.n_tiles, p.S, sp->L, p.log2_T);
    uint8_t *ws = (uint8_t *)g->d_workspace;
    float *dc32 = reinterpret_cast<float *>(ws + bl.dc32);
    uint16_t *dc16 = reinterpret_cast<uint16_t *>(ws + bl.dc16);
    float *dsig32 = reinterpret_cast<float *>(ws + bl.dsig32);
    uint16_t *dsig16 = reinterpret_cast<uint16_t *>(ws + bl.dsig16);
    uint16_t *dz = reinterpret_cast<uint16_t *>(ws + bl.dz);
    float *dx0 = reinterpret_cast<float *>(ws + bl.dx0);
    float *dt3 = reinterpret_cast<float *>(ws + bl.dt3);
    p.tr.dc = dc32; p.tr.dsig = dsig32; p.tr.dz = dz; p.tr.dx0 = dx0;
    p.pack = (const uint8_t *)g->d_bwd_pack; p.pack_stride = g->bwd_pack_stride;

    const bool timing0 = getenv("SDB_TIMING") != nullptr;
    cudaEvent_t tev0 = nullptr;
    if (timing0) { cudaEventCreate(&tev0); cudaEventRecord(tev0, st); }
    // The number of live ray tiles of the recorded pass stays ON THE DEVICE (record header): every kernel below is launched over
    // the record's capacity and reads it there, so this call never synchronises -- the host can queue the whole backward (and the
    // torch ops behind it) while the forward kernel is still running, which is what makes the step time independent of host speed.
    const long long cap_items = (long long)p.n_tiles * p.S;
    const size_t table_bytes = ((size_t)sp->L << p.log2_T) * 8 * 4;

    SDB_CUDA(cudaMemsetAsync(g->d_grad_sky_avg, 0, (size_t)p.n_img * kOutC * 4, st));
    SDB_CUDA(cudaMemsetAsync(g->d_grad_global_enc, 0, 8, st));
    SDB_CUDA(cudaMemsetAsync(dt3, 0, table_bytes, st));

    // SDB_TIMING=1: per-stage device times on stderr (diagnostics; synchronises)
    const bool timing = getenv("SDB_TIMING") != nullptr;
    cudaEvent_t tev[8];
    int ntev = 0;
    auto mark = [&]() { if (timing && ntev < 8) { cudaEventCreate(&tev[ntev]); cudaEventRecord(tev[ntev], st); ntev++; } };
    mark();
    // 1. compositing backward (every tile: sky-only tiles still feed dL/dsky)
    composite_backward_kernel<<<p.n_tiles, 256, 0, st>>>(p, g->d_grad_net_out, g->d_grad_sky, g->d_grad_sky_avg, dc32, dc16,
                                                         dsig32, dsig16);
    SDB_CHECK_LAUNCH();
    mark();
    // 2. data-gradient chain on the tensor-core engine: one work item per (live tile, sample step) -- the slot index
    //    (work * 1 + 0) * 128 + row of such an item IS the record's (tile * S + step) * 128 + row
    {
        Params pc = p;
        pc.work_mult = p.S;
        pc.S = 1;
        const int grid = cap_items < sdb_num_sms() ? (int)cap_items : sdb_num_sms();      // work items beyond n_live * S do not exist: CTAs find none
        const int rc = launch_bwd_chain(pc, grid, st);
        if (rc != SDB_OK) return rc;
    }
    mark();
    // 3. table gradient: scatter into the pre-blended table, transpose of the pre-blend, scene code
    {
        dim3 grid((unsigned)((cap_items * kRows + 255) / 256), kLevels);
        // SDB_TABLE_AGG_LEVELS: tuning knob (levels 0..n-1 use the warp-aggregated scatter); the default was chosen on the
        // previous GPU generation and is carried over, not re-measured on H100
        int agg_levels = 12;
        if (const char *e = getenv("SDB_TABLE_AGG_LEVELS")) agg_levels = atoi(e);
        table3_backward_kernel<<<grid, 256, 0, st>>>(p, dx0, dt3, agg_levels);
        SDB_CHECK_LAUNCH();
        int rc = sdb_preblend_table(dt3, g->d_grad_table, sp->L, p.log2_T, p.level_S, p.base_res, p.genc, stream);
        if (rc != SDB_OK) return rc;
        const size_t n = (size_t)sp->L << p.log2_T;
        genc_backward_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g->d_table, dt3, sp->L, p.log2_T, p.level_S, p.base_res,
                                                                          p.genc, g->d_grad_global_enc);
        SDB_CHECK_LAUNCH();
    }
    mark();
    // 4. weight gradients on the tensor cores (every live item, nothing else: no padding rows to zero)
    {
        SDB_CUDA(cudaMemsetAsync(g->d_grad_w1ext, 0, (size_t)kHidden * kX0Cols * 4, st));
        SDB_CUDA(cudaMemsetAsync(g->d_grad_wh, 0, (size_t)5 * kHidden * kActCols * 4, st));
        SDB_CUDA(cudaMemsetAsync(g->d_grad_wsig, 0, (size_t)8 * kActCols * 4, st));
        SDB_CUDA(cudaMemsetAsync(g->d_grad_wout, 0, (size_t)kOutC * kActCols * 4, st));
        const long long cap = p.tr.slot_cap;
        WgJob jobs[kWgMaxJobs];
        int nj = 0;
        add_jobs(jobs, nj, p.tr.x0, kX0Cols, dz, kHidden, g->d_grad_w1ext, kHidden);                                  // fc_1 | fc_m_a | bias
        for (int k = 0; k < 5; k++)                                                                                    // fc_2 .. fc_6
            add_jobs(jobs, nj, p.tr.act + (size_t)k * cap * kActCols, kActCols, dz + (size_t)(k + 1) * cap * kHidden, kHidden,
                     g->d_grad_wh + (size_t)k * kHidden * kActCols, kHidden);
        add_jobs(jobs, nj, p.tr.act + (size_t)5 * cap * kActCols, kActCols, dc16, kOutC, g->d_grad_wout, kOutC);       // fc_out_c
        add_jobs(jobs, nj, p.tr.act + (size_t)3 * cap * kActCols, kActCols, dsig16, 8, g->d_grad_wsig, 8);             // fc_sigma
        const int rc = launch_wgrad(jobs, nj, p.n_live, p.S, cap_items, st);
        if (rc != SDB_OK) return rc;
    }
    mark();
    if (timing) {
        cudaStreamSynchronize(st);
        float ms[8] = {0};
        for (int i = 0; i + 1 < ntev; i++) cudaEventElapsedTime(&ms[i], tev[i], tev[i + 1]);
        float pre = 0.0f;
        if (tev0) { cudaEventElapsedTime(&pre, tev0, tev[0]); cudaEventDestroy(tev0); }
        int32_t n_live = 0;
        cudaMemcpy(&n_live, rec + rl.hdr, 4, cudaMemcpyDeviceToHost);
        fprintf(stderr, "[sdb timing] backward: prologue %.3f ms, compositing %.3f ms, chain %.3f ms, table %.3f ms, weight GEMMs %.3f ms (n_live %d)\n",
                pre, ms[0], ms[1], ms[2], ms[3], n_live);
        for (int i = 0; i < ntev; i++) cudaEventDestroy(tev[i]);
    }
    return SDB_OK;
}

// ---- sky branch (a9) backward: SKYMLP data-gradient chain on the tensor-core engine + weight-gradient GEMMs -------------
// (gancraft_base.py:150-169 under autograd; the positional encoding of the ray direction needs no gradient)
extern "C" int64_t sdb_sky_backward_workspace_bytes(int32_t n_img, int32_t H, int32_t W) {
    using namespace rf;
    if (n_img <= 0 || H <= 0 || W <= 0) return 0;
    return (int64_t)sky_bwd_layout((long long)n_img * sdb_div_up(H, kTileH) * sdb_div_up(W, kTileW)).total;
}

extern "C" int sdb_sky_backward(int32_t n_img, int32_t H, int32_t W, const void *d_record, const float *d_grad_sky,
                                const void *d_bwd_pack, float *d_grad_w1ext, float *d_grad_wh, float *d_grad_wout,
                                void *d_workspace, void *stream)
{
    using namespace rf;
    if (!d_record || !d_grad_sky || !d_bwd_pack || !d_grad_w1ext || !d_grad_wh || !d_grad_wout || !d_workspace) return SDB_EINVAL;
    if (n_img != 1 || H <= 0 || W <= 0) return n_img == 1 ? SDB_EINVAL : SDB_EUNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    Params p{};
    p.n_img = n_img; p.H = H; p.W = W; p.M = 1; p.S = 1;
    p.tiles_x = sdb_div_up(W, kTileW); p.tiles_y = sdb_div_up(H, kTileH);
    p.n_tiles = n_img * p.tiles_x * p.tiles_y;
    p.pack = (const uint8_t *)d_bwd_pack; p.pack_stride = 0;
    p.debug = g_debug_buffer;
    const SkyRecordLayout rl = sky_record_layout(p.n_tiles);
    const SkyBwdLayout bl = sky_bwd_layout(p.n_tiles);
    uint8_t *rec = (uint8_t *)const_cast<void *>(d_record), *ws = (uint8_t *)d_workspace;
    const long long cap = (long long)p.n_tiles * kRows;
    p.tr.slot_cap = cap;
    p.tr.x0 = reinterpret_cast<uint16_t *>(rec + rl.x0);
    p.tr.act = reinterpret_cast<uint16_t *>(rec + rl.act);
    p.tr.mask = reinterpret_cast<uint32_t *>(rec + rl.mask);
    p.tr.dc = d_grad_sky;
    p.tr.dc16 = reinterpret_cast<uint16_t *>(ws + bl.dc16);
    p.tr.dz = reinterpret_cast<uint16_t *>(ws + bl.dz);
    {
        const int grid = p.n_tiles < sdb_num_sms() ? p.n_tiles : sdb_num_sms();
        const int rc = launch_sky_bwd_chain(p, grid, st);
        if (rc != SDB_OK) return rc;
    }
    SDB_CUDA(cudaMemsetAsync(d_grad_w1ext, 0, (size_t)kHidden * kSkyK0 * 4, st));
    SDB_CUDA(cudaMemsetAsync(d_grad_wh, 0, (size_t)4 * kHidden * kActCols * 4, st));
    SDB_CUDA(cudaMemsetAsync(d_grad_wout, 0, (size_t)kOutC * kActCols * 4, st));
    WgJob jobs[kWgMaxJobs];
    int nj = 0;
    add_jobs(jobs, nj, p.tr.x0, kSkyK0, p.tr.dz, kHidden, d_grad_w1ext, kHidden);                                              // fc1 | bias
    for (int k = 0; k < 4; k++)                                                                                               // fc2 .. fc5
        add_jobs(jobs, nj, p.tr.act + (size_t)k * cap * kActCols, kActCols, p.tr.dz + (size_t)(k + 1) * cap * kHidden, kHidden,
                 d_grad_wh + (size_t)k * kHidden * kActCols, kHidden);
    add_jobs(jobs, nj, p.tr.act + (size_t)4 * cap * kActCols, kActCols, p.tr.dc16, kOutC, d_grad_wout, kOutC);                // fc_out_c
    return launch_wgrad(jobs, nj, nullptr, 1, p.n_tiles, st);
}
