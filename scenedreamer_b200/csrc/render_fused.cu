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
//     one MMA warpgroup (wgmma in 64x32 blocks; its thread 0 also streams the weights into a 4-slot ring
//     with 1-D bulk TMA copies), 8 gather warps (hash-grid fetch for the NEXT sample step while the MLP
//     of the current one runs; results wait in registers until the operand buffer is free);
//   * accumulators: a layer's fp32 [128 x 256] result (128 KB) fits neither next to the operand buffers in
//     shared memory nor in the registers the three roles share, so the MMA warpgroup writes it to a
//     per-CTA buffer pair in global memory (L2-resident, ping-pong by layer parity) and the epilogue reads
//     its rows from there; a layer starts when the epilogue has written all of its input;
//   * bias, style beta and the label embedding ride in the GEMM: the operand has 16 extra K columns
//     (one-hot label + constant 1), the weight image carries bias / embedding rows there -- exactly
//     the reference's fc_m_a(onehot) product -- so the epilogue is LeakyReLU + 16-bit split only;
//   * the 16-bit activations stay on chip: ONE in-place 128x272 operand buffer in shared memory; the
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
        const float ns = (float)(p.S + 1);
        const float u0 = __ldg(p.uniforms + ray * (p.S + 1) + k), u1 = __ldg(p.uniforms + ray * (p.S + 1) + k + 1);
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

// ---- gather (a5/a6) ----------------------------------------------------------------------------------
template <bool RAW5D>
__device__ __forceinline__ void encode_level(const float *__restrict__ tbl, uint32_t mask, float scale, const float (&x)[5],
                                             float (&res)[8]) {
    // gridencoder.cu:133-170.  pos = x*scale + 0.5 is one FFMA in the reference's device code.
    constexpr int D = RAW5D ? 5 : 3;
    float f[D];
    uint32_t g[D];
#pragma unroll
    for (int d = 0; d < D; d++) {
        const float pos = fmaf(x[d], scale, 0.5f);
        const float fl = floorf(pos);
        g[d] = (uint32_t)fl;
        f[d] = pos - (float)g[d];
    }
    const uint32_t h0[2] = {g[0], g[0] + 1u};
    const uint32_t h1[2] = {g[1] * kPrime1, (g[1] + 1u) * kPrime1};
    const uint32_t h2[2] = {g[2] * kPrime2, (g[2] + 1u) * kPrime2};
#pragma unroll
    for (int c = 0; c < 8; c++) res[c] = 0.0f;
    if constexpr (RAW5D) {
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
#pragma unroll
        for (int idx = 0; idx < 8; idx++) {
            const int b0 = idx & 1, b1 = (idx >> 1) & 1, b2 = (idx >> 2) & 1;
            float w = b0 ? f[0] : 1.0f - f[0];
            w *= b1 ? f[1] : 1.0f - f[1];
            w *= b2 ? f[2] : 1.0f - f[2];
            const uint32_t index = (h0[b0] ^ h1[b1] ^ h2[b2]) & mask;
            float v[8];
            ld8(tbl + (size_t)index * 8, v);
#pragma unroll
            for (int c = 0; c < 8; c++) res[c] = fmaf(w, v[c], res[c]);
        }
    }
}

// encode_level<false> with at most 2 * GU gathers of a lane in flight (the corner loop is unrolled GU times only): the ray-slot
// kernel's gather shares the LSU with the epilogue's operand stores, and a fully unrolled level queues 16 scattered LDG.128 per
// lane -- up to 4,096 L1 wavefronts ahead of every epilogue store.  Same arithmetic per feature.
template <int GU>
__device__ __forceinline__ void encode_level_thin(const float *__restrict__ tbl, uint32_t mask, float scale, const float (&x)[5],
                                                  float (&res)[8]) {
    float f[3];
    uint32_t g[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        const float pos = fmaf(x[d], scale, 0.5f);
        const float fl = floorf(pos);
        g[d] = (uint32_t)fl;
        f[d] = pos - (float)g[d];
    }
#pragma unroll
    for (int c = 0; c < 8; c++) res[c] = 0.0f;
#pragma unroll(GU)
    for (int idx = 0; idx < 8; idx++) {
        const uint32_t b0 = idx & 1, b1 = (idx >> 1) & 1, b2 = (idx >> 2) & 1;
        float w = b0 ? f[0] : 1.0f - f[0];
        w *= b1 ? f[1] : 1.0f - f[1];
        w *= b2 ? f[2] : 1.0f - f[2];
        const uint32_t index = ((g[0] + b0) ^ ((g[1] + b1) * kPrime1) ^ ((g[2] + b2) * kPrime2)) & mask;
        float v[8];
        ld8(tbl + (size_t)index * 8, v);
#pragma unroll
        for (int c = 0; c < 8; c++) res[c] = fmaf(w, v[c], res[c]);
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
    constexpr Smem SM = smem_map(X3);
    constexpr int PARTS = X3 ? 2 : 1;
    constexpr int NH = Net<MODE>::NH, NL = Net<MODE>::NL;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *sHhi = smem + SM.h_hi;
    uint8_t *sHlo = smem + SM.h_lo;
    uint8_t *sRing = smem + SM.ring;
    float *sF = reinterpret_cast<float *>(smem + SM.fsec);
    float *sScale = reinterpret_cast<float *>(smem + SM.scales);
    float *sFrac = reinterpret_cast<float *>(smem + SM.frac);
    float *sSig = reinterpret_cast<float *>(smem + SM.sig);
    float *sState = reinterpret_cast<float *>(smem + SM.state);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + SM.bars);
    // Early termination (north star: "early termination"; inference render only).  stop_step[buf] = number of sample
    // steps the tile in state buffer `buf` executes (S until decided).  The epilogue decides during the compositing of
    // step s ("every live ray has transmittance < early_T") and sets s + 2: by the time ANY role starts step s + 2 it
    // has synchronised (through the barriers it already waits on) with an epilogue that is past that compositing, so
    // all roles read the same value and execute the same number of steps -- the barrier phase arithmetic, which only
    // depends on the global executed-step counter n, stays consistent.
    constexpr bool ESTOP = MODE == kRender && !TRAIN;
    volatile int *sStop = reinterpret_cast<volatile int *>(smem + SM.stop);
    volatile int *sVote = sStop + 2;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // the render gradient chain has no dependency between the sample steps of a tile: there every (tile, step) is its own
    // work item (work_mult = S, one step each), which balances a few hundred tiles over 148 CTAs far better than whole tiles
    const int wmult = (MODE == kBwd && p.work_mult > 1) ? p.work_mult : 1;
    const int n_work = RAYQ ? (int)gridDim.x : (ONE_STEP ? p.n_tiles : *p.n_live * wmult);
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
        for (int i = 0; i < 16; i++) tc05::mbar_init(&bars[B_CHUNK + i], kEpiThreads / 2);
        tc05::mbar_init(&bars[B_ACC], 1);
        tc05::mbar_init(&bars[B_OUTRDY], 1);
        tc05::mbar_init(&bars[B_EPIDONE], kEpiThreads);
        tc05::mbar_init(&bars[B_EPIDONE + 1], kEpiThreads);
        for (int i = 0; i < 2; i++) { tc05::mbar_init(&bars[B_STRDY + i], kRows); tc05::mbar_init(&bars[B_STFREE + i], kEpiThreads); }
        tc05::mbar_init(&bars[B_COMP], kEpiThreads);
        tc05::fence_mbar_init();
    }
    if (tid < 2) { sStop[tid] = RAYQ ? 0x7fffffff : kMaxS + 1; sVote[tid] = 0; }
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
    // constant K-extension columns of the hidden operand: column 256 = 1.0 (bias), 257..271 = 0
    for (int i = tid; i < 2 * kRows; i += kThreads) {
        const int r = i & (kRows - 1), kc = kHidden / 8 + (i >> 7);
        const uint4 one = make_uint4((i >> 7) == 0 ? one16<PREC>() : 0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4 *>(sHhi + tc05::chunk_off(kRows, r, kc)) = one;
        if constexpr (X3) *reinterpret_cast<uint4 *>(sHlo + tc05::chunk_off(kRows, r, kc)) = make_uint4(0, 0, 0, 0);
    }
    tc05::fence_proxy_async_smem();
    __syncthreads();
    const uint32_t mask = SKY ? 0u : ((1u << p.log2_T) - 1u);

    if (warp < 8) {
        // =========================== EPILOGUE / COMPOSITING WARPS ===========================
        const int row = tid & (kRows - 1), half = tid >> 7;          // column half: 128*half .. +127
        const float *acc_row = p.acc + (size_t)blockIdx.x * 2 * kRows * kHidden + (size_t)row * kHidden;   // accumulator row
        uint32_t n = 0;                 // global step counter
        int loaded_img = -1;
        for (int it = 0;; it++) {
            const int work = fetch_work(it);
            if (work < 0) break;
            const int tile = RAYQ ? 0 : (ONE_STEP ? work : p.tile_list[work / wmult]);
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
                    const float *acc = acc_row + (g & 1u) * kRows * kHidden + half * 128;
                    // kBwd: LeakyReLU sign words of the forward activation A_{6-l} this layer's data gradient passes
                    // through (prefetched before the accumulator wait)
                    uint4 mw = make_uint4(0u, 0u, 0u, 0u);
                    if constexpr (BWD)
                        mw = __ldg(reinterpret_cast<const uint4 *>(p.tr.mask + ((step_id * kNumAct + (NACT - 1 - l)) * kRows + row) * 8 + half * 4));
                    if ((tid & 127) == 0) SDB_MARK(half, 1, n, l);
                    tc05::mbar_wait(&bars[B_ACC], (n * NH + l) & 1);
                    if ((tid & 127) == 0) SDB_MARK(half, 2, n, l);
                    if ((tid & 127) == 0) SDB_STAMP(n, l, 2 + 2 * half);
#pragma unroll 1
                    for (int c0 = 0; c0 < 128; c0 += 32) {
                        // a 32-column chunk in two 16-column halves (16 live accumulator registers instead of 32: the
                        // compositing state of the tile stays in registers next to them)
                        uint32_t rec[16];            // TRAIN / chain: bf16 (round-to-nearest) copy of the chunk for the record
                        uint32_t mword = 0;          // TRAIN: LeakyReLU sign bits of the chunk
                        (void)rec; (void)mword;
                        const uint32_t word = c0 == 0 ? mw.x : (c0 == 32 ? mw.y : (c0 == 64 ? mw.z : mw.w));
                        (void)word;
#pragma unroll
                        for (int hh = 0; hh < 2; hh++) {
                            float v[16];
                            acc_ld<16>(acc + c0 + 16 * hh, v);
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
                            // a 16-column K slab of the next layer's operand is complete (all 128 rows once the four quadrant
                            // warps of this half have arrived): the MMA issuer may start on it
                            tc05::fence_proxy_async_smem();
                            tc05::mbar_arrive(&bars[B_CHUNK + half * 8 + (c0 >> 4) + hh]);
                        }
                        // the training record is written AFTER the chunk has been handed to the MMA issuer (off the critical path)
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
                    tc05::mbar_arrive(&bars[B_EPIDONE + (g & 1u)]);        // accumulator buffer (g & 1) is free again
                    if ((tid & 127) == 0) SDB_STAMP(n, l, 3 + 2 * half);
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
                tc05::mbar_wait(&bars[B_OUTRDY], n & 1);
                if ((tid & 127) == 0) SDB_MARK(half, 4, n, NH);
                if ((tid & 127) == 0) SDB_STAMP(n, NH, 2 + 2 * half);
                if constexpr (SKYBWD) {
                    // last layer of the sky chain: dA1 [128 x 256] -> dZ1 = dA1 * LeakyReLU'(z1) -> bf16 record only
                    const uint4 mw = __ldg(reinterpret_cast<const uint4 *>(p.tr.mask + ((step_id * kNumAct + 0) * kRows + row) * 8 + half * 4));
#pragma unroll 1
                    for (int c0 = 0; c0 < 128; c0 += 32) {
                        float v[32];
                        acc_ld<32>(acc_row + (go & 1u) * kRows * kHidden + half * 128 + c0, v);
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
                    tc05::mbar_arrive(&bars[B_EPIDONE + (go & 1u)]);
                    if ((tid & 127) == 0) SDB_STAMP(n, NH, 3 + 2 * half);
                    continue;
                }
                float c[32];
                acc_ld<32>(acc_row + (go & 1u) * kRows * kHidden + half * (BWD ? 64 : 32), c);
                if constexpr (BWD) {
                    // d(hash-grid features) [128 rays x 128]: this half owns 64 columns -> fp32 record for the table backward
                    float c2[32];
                    acc_ld<32>(acc_row + (go & 1u) * kRows * kHidden + half * 64 + 32, c2);
                    tc05::mbar_arrive(&bars[B_EPIDONE + (go & 1u)]);
                    if ((tid & 127) == 0) SDB_STAMP(n, NH, 3 + 2 * half);
                    float *dst = p.tr.dx0 + slot * kFeat + half * 64;
#pragma unroll
                    for (int q = 0; q < 4; q++) st_global_v8f(dst + 8 * q, &c[8 * q]);
#pragma unroll
                    for (int q = 0; q < 4; q++) st_global_v8f(dst + 32 + 8 * q, &c2[8 * q]);
                    continue;
                }
                tc05::mbar_arrive(&bars[B_EPIDONE + (go & 1u)]);
                if ((tid & 127) == 0) SDB_STAMP(n, NH, 3 + 2 * half);
                if constexpr (SKY) {
#pragma unroll
                    for (int j = 0; j < 32; j++) outc[j] = c[j];
                } else if constexpr (RAYQ) {
                    // ---- compositing of ray slots (a10/a11): every row is its own ray at its own sample step ----
                    asm volatile("bar.sync 1, 256;" ::: "memory");
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
                        const float e = __fmul_rn(fmaxf(sigma, 0.0f), __fmul_rn(nd, p.dists_scale));      // mc_utils.py:155
                        const float a = 1.0f - expf(-e);
                        const float b = expf(-Eexcl);
                        w = a * b;
                        Eexcl = __fadd_rn(Eexcl, e);
                        Wsum += w;
                        {
                            const float pr = __fmul_rn(w, depth);
                            const float pe = __fmaf_rn(w, depth, -pr);
                            const float sn = __fadd_rn(Dsum, pr);
                            const float bv = __fsub_rn(sn, Dsum);
                            Dcomp = __fadd_rn(Dcomp, __fadd_rn(__fadd_rn(__fsub_rn(Dsum, __fsub_rn(sn, bv)), __fsub_rn(pr, bv)), pe));
                            Dsum = sn;
                        }
                        if (half == 0 && p.weights_out) p.weights_out[(long long)rq * S + s_ray] = w;
                        fin = (code & 0x200u) || (p.early_T > 0.0f && expf(-Eexcl) < p.early_T);
                    }
#pragma unroll
                    for (int j = 0; j < 32; j++) {
                        const float rgb = fminf(fmaxf(c[j], -1.0f), 1.0f) + 1.0f;                     // :407-408
                        outc[j] = fmaf(w, rgb, outc[j]);
                    }
                    if (act && fin) {
                        // ---- this slot's ray is finished: sky blend + output (scenedreamer.py:380-413) ----
                        const bool nosky = !(code & 0x800u) || (code & 0x1000u);
                        const float sky_w = 1.0f - Wsum;
                        const float4 *skp = reinterpret_cast<const float4 *>((nosky ? p.sky_avg : p.sky + (long long)rq * kOutC) + half * 32);
                        float4 *dst = reinterpret_cast<float4 *>(p.net_out + (long long)rq * kOutC + half * 32);
#pragma unroll
                        for (int q = 0; q < 8; q++) {
                            const float4 sk = __ldg(skp + q);
                            float4 o;
                            o.x = (outc[4 * q + 0] + sky_w * (fminf(fmaxf(sk.x, -1.0f), 1.0f) + 1.0f)) - 1.0f;
                            o.y = (outc[4 * q + 1] + sky_w * (fminf(fmaxf(sk.y, -1.0f), 1.0f) + 1.0f)) - 1.0f;
                            o.z = (outc[4 * q + 2] + sky_w * (fminf(fmaxf(sk.z, -1.0f), 1.0f) + 1.0f)) - 1.0f;
                            o.w = (outc[4 * q + 3] + sky_w * (fminf(fmaxf(sk.w, -1.0f), 1.0f) + 1.0f)) - 1.0f;
                            dst[q] = o;
                        }
                        if (half == 0) {
                            if (p.depth_out) p.depth_out[rq] = __fadd_rn(Dsum, Dcomp);
                            if (p.total_weight) p.total_weight[rq] = Wsum;
                        }
                        skip_ray = (code & 0x200u) ? -1 : rq;
                    }
                    // early finishes are reported to the gather role (it replaces the ray two steps on); natural ends it sees itself
                    if (half == 0) sDone[(s & 1) * kRows + row] = (act && fin && !(code & 0x200u)) ? rq + 1 : 0;
                    // is the CTA done?  every slot idle or finished AND the queue was already empty when this step was built
                    {
                        const bool idle = !act || fin;
                        const bool wall = __all_sync(0xffffffffu, idle);
                        if (lane == 0 && !wall) sVote[s & 1] = 1;
                        asm volatile("bar.sync 1, 256;" ::: "memory");
                        if (tid == 0) {
                            if (sVote[s & 1] == 0 && sExh[s & 3] != 0 && sStop[0] > s + 2) sStop[0] = s + 2;
                            sVote[s & 1] = 0;
                        }
                    }
                    tc05::mbar_arrive(&bars[B_COMP]);                      // compositing of step s is complete (done flags visible)
                } else {
                    // ---- compositing (a10/a11) ----
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                    const float sigma = (sSig[row] + sSig[kRows + row]) + sF[kFBsig];
                    const float e = __fmul_rn(fmaxf(sigma, 0.0f), __fmul_rn(sm.nd, p.dists_scale));   // mc_utils.py:155
                    const float a = 1.0f - expf(-e);
                    const float b = expf(-Eexcl);
                    float w = a * b;
                    Eexcl = __fadd_rn(Eexcl, e);
                    w = live ? w : 0.0f;                                                              // scenedreamer.py:376
                    Wsum += w;
                    {   // depth = sum w*t with t of several hundred voxels: 1e-3 absolute is ~16 ulp of the running sum, so the
                        // 24..64-term sum is carried compensated (exact product error + two-sum); costs 8 flops per sample
                        const float pr = __fmul_rn(w, sm.depth);
                        const float pe = __fmaf_rn(w, sm.depth, -pr);
                        const float sn = __fadd_rn(Dsum, pr);
                        const float bv = __fsub_rn(sn, Dsum);
                        Dcomp = __fadd_rn(Dcomp, __fadd_rn(__fadd_rn(__fsub_rn(Dsum, __fsub_rn(sn, bv)), __fsub_rn(pr, bv)), pe));
                        Dsum = sn;
                    }
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
                        asm volatile("bar.sync 1, 256;" ::: "memory");
                        if (tid == 0) {
                            if (sVote[s & 1] == 0 && sStop[buf] > S) sStop[buf] = s + 2;
                            sVote[s & 1] = 0;
                        }
                    }
#pragma unroll
                    for (int j = 0; j < 32; j++) {
                        const float rgb = fminf(fmaxf(c[j], -1.0f), 1.0f) + 1.0f;                     // :407-408
                        outc[j] = fmaf(w, rgb, outc[j]);
                    }
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
                // ---- finalize the tile (sky blend, scenedreamer.py:380-413) ----
                const bool sky_mask = flags & 2u;
                const bool nosky = (!sky_mask) || is_gnd;
                if constexpr (TRAIN) {
                    if (half == 0) p.tr.rayflags[(long long)work * kRows + row] = (live ? 1u : 0u) | (nosky ? 2u : 0u) | (valid ? 4u : 0u);
                }
                if (valid) {
                    const float sky_w = 1.0f - Wsum;
                    const float4 *skp = reinterpret_cast<const float4 *>((nosky ? p.sky_avg + (long long)tc.img * kOutC
                                                                                 : p.sky + ray * kOutC) + half * 32);
                    float4 *dst = reinterpret_cast<float4 *>(p.net_out + ray * kOutC + half * 32);
#pragma unroll
                    for (int q = 0; q < 8; q++) {
                        const float4 sk = __ldg(skp + q);
                        float4 o;
                        o.x = (outc[4 * q + 0] + sky_w * (fminf(fmaxf(sk.x, -1.0f), 1.0f) + 1.0f)) - 1.0f;
                        o.y = (outc[4 * q + 1] + sky_w * (fminf(fmaxf(sk.y, -1.0f), 1.0f) + 1.0f)) - 1.0f;
                        o.z = (outc[4 * q + 2] + sky_w * (fminf(fmaxf(sk.z, -1.0f), 1.0f) + 1.0f)) - 1.0f;
                        o.w = (outc[4 * q + 3] + sky_w * (fminf(fmaxf(sk.w, -1.0f), 1.0f) + 1.0f)) - 1.0f;
                        dst[q] = o;
                    }
                    if (half == 0) {
                        if (p.depth_out) p.depth_out[ray] = __fadd_rn(Dsum, Dcomp);
                        if (p.total_weight) p.total_weight[ray] = Wsum;
                    }
                }
                tc05::mbar_arrive(&bars[B_STFREE + buf]);
            }
        }
    } else if (warp < kGatherWarp0) {
      asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegsCtl));
      // =========================== MMA WARPGROUP ===========================
      // Layer l of a sample step: D[128 x N] = H[128 x K] * W_l^T, computed in 64-row x 32-column blocks (the sum over K in
      // registers), each written once to this CTA's fp32 accumulator buffer (g & 1) in global memory, where the epilogue reads
      // its rows.  Weights go through a 4-slot ring of 16 KB stages = up to 8 k16 slabs of one 32-column block; thread 0
      // issues the bulk copies up to 3 stages ahead of the MMAs.  Named barrier 3 is this warpgroup's (1: epilogue, 2: gather).
      const int t = tid - kMmaWarp0 * 32;
      constexpr uint32_t kSlot = 16384, kSlabB = 1024 * PARTS;       // ring slot; one k16 slab of a 32-column block
      uint32_t n = 0, q0 = 0;                                        // q0: ring stages of all earlier steps
      auto layer_stages = [&](int l) { return 2 * (layerN<MODE>(l) / 32) * ((layerK<MODE>(l) / 16 + 7) / 8); };
      for (int it = 0;; it++) {
          const int work = fetch_work(it);
          if (work < 0) break;
          const int tile = RAYQ ? 0 : (ONE_STEP ? work : p.tile_list[work / wmult]);
          const uint8_t *pack = p.pack + (long long)tile_coord(p, tile).img * p.pack_stride;
          int n_st = 0;
          for (int l = 0; l < NL; l++) n_st += layer_stages(l);
          // stage k of a step -> (layer, 32-column block, first slab, slabs); stages go (layer, row block, column block, slabs)
          auto issue = [&](int k) {
              int l = 0;
              while (k >= layer_stages(l)) { k -= layer_stages(l); l++; }
              const int N = layerN<MODE>(l), nK = layerK<MODE>(l) / 16, nsg = (nK + 7) / 8;
              const int blk = k / nsg, sg = k % nsg, cc = blk % (N / 32);
              const int kk0 = sg * 8;
              return make_int4(l, cc, kk0, min(8, nK - kk0));
          };
          for (int s = 0; s < SL; s++, n++) {
              if (ESTOP && s >= 2 && s >= sStop[it & 1]) break;
              int k = 0, k_issued = 0;
              auto produce = [&](int upto) {           // thread 0: stages k_issued .. upto - 1 of this step
                  for (; k_issued < upto && k_issued < n_st; k_issued++) {
                      const int4 d = issue(k_issued);
                      const int N = layerN<MODE>(d.x);
                      const uint32_t q = q0 + (uint32_t)k_issued, slot = q & 3u;
                      const uint8_t *w = pack + layerOff<MODE>(d.x, PARTS);
                      const uint32_t slabB = (uint32_t)N * 32u * PARTS;
                      tc05::mbar_arrive_expect_tx(&bars[B_WFULL + slot], (uint32_t)d.w * kSlabB);
                      for (int i = 0; i < d.w; i++)
#pragma unroll
                          for (int part = 0; part < PARTS; part++)
#pragma unroll
                              for (int kc = 0; kc < 2; kc++)
                                  tc05::bulk_g2s(sRing + slot * kSlot + i * kSlabB + part * 1024 + kc * 512,
                                                 w + (size_t)(d.z + i) * slabB + part * N * 32 + kc * N * 16 + d.y * 512, 512,
                                                 &bars[B_WFULL + slot]);
                  }
              };
              if (t == 0) produce(3);
#pragma unroll 1
              for (int l = 0; l < NL; l++) {
                  const uint32_t g = n * NL + l, buf = g & 1u;
                  if (t == 0) SDB_MARK(2, 1, n, l);
                  // accumulator buffer `buf` was last read by the epilogue of global layer g - 2
                  if (g >= 2) tc05::mbar_wait(&bars[B_EPIDONE + buf], ((g >> 1) - 1) & 1);
                  if (l == 0) {
                      tc05::mbar_wait(&bars[B_FEAT], n & 1);
                  } else {
                      const uint32_t cpar = (n * NH + l - 1) & 1;      // operand of this layer from the previous epilogue
                      for (int c = 0; c < 16; c++) tc05::mbar_wait(&bars[B_CHUNK + c], cpar);
                  }
                  if (t == 0) SDB_MARK(2, 2, n, l);
                  if (t == 0) SDB_STAMP(n, l, 0);
                  const int N = layerN<MODE>(l), nK = layerK<MODE>(l) / 16, nsg = (nK + 7) / 8;
                  float *dst = p.acc + ((size_t)blockIdx.x * 2 + buf) * kRows * kHidden;
#pragma unroll 1
                  for (int rb = 0; rb < 2; rb++) {
#pragma unroll 1
                      for (int cc = 0; cc < N / 32; cc++) {
                          float d[16], sum[16];
#pragma unroll 1
                          for (int sg = 0; sg < nsg; sg++, k++) {
                              if (t == 0) produce(k + 4);
                              const uint32_t q = q0 + (uint32_t)k, slot = q & 3u;
                              tc05::mbar_wait(&bars[B_WFULL + slot], (q >> 2) & 1u);
                              const uint32_t sb = tc05::smem_u32(sRing + slot * kSlot);
                              const int kk0 = sg * 8, ns = min(8, nK - kk0);
                              tc05::wgmma_fence();
#pragma unroll 1
                              for (int i = 0; i < ns; i++) {
                                  const uint32_t aoff = (uint32_t)(kk0 + i) * 2 * kLboA + rb * 1024;
                                  const uint64_t ah = tc05::make_smem_desc(tc05::smem_u32(sHhi) + aoff, kLboA, kSbo);
                                  const uint64_t bh = tc05::make_smem_desc(sb + i * kSlabB, 512, kSbo);
                                  tc05::wgmma_m64n32k16<BF16, 0, 0>(d, ah, bh, i > 0 ? 1u : 0u);
                                  if constexpr (X3) {
                                      const uint64_t al = tc05::make_smem_desc(tc05::smem_u32(sHlo) + aoff, kLboA, kSbo);
                                      tc05::wgmma_m64n32k16<BF16, 0, 0>(d, al, bh, 1u);
                                      tc05::wgmma_m64n32k16<BF16, 0, 0>(d, ah, bh + (1024 >> 4), 1u);
                                  }
                              }
                              tc05::wgmma_commit();
                              tc05::wgmma_wait<0>();
                              tc05::wgmma_fence_acc(d);
                              tc05::named_sync(3, 128);           // every warp is done with the slot: it may be refilled
                              // Every stage (<= 8 k16 slabs) starts a fresh tensor-core sum, added to the running sum in fp32
                              // with round-to-nearest: the tensor core's own accumulation does not round to nearest, and over a
                              // whole x3 layer (up to 51 chained MMAs) that moved the full-frame depth outside its parity bound.
#pragma unroll
                              for (int i = 0; i < 16; i++) sum[i] = sg == 0 ? d[i] : __fadd_rn(sum[i], d[i]);
                          }
#ifndef SDB_AB_NO_ACC
#pragma unroll
                          for (int i = 0; i < 16; i += 2)
                              *reinterpret_cast<float2 *>(dst + (size_t)(rb * 64 + tc05::frag_row(t, i)) * kHidden + cc * 32 +
                                                          tc05::frag_col(t, i)) = make_float2(sum[i], sum[i + 1]);
#endif
                      }
                  }
                  __threadfence_block();
                  tc05::named_sync(3, 128);
                  if (t == 0) SDB_STAMP(n, l, 1);
                  if (t == 0) {
                      if (l == NL - 1) {
                          tc05::mbar_arrive(&bars[B_OUTRDY]);
                          tc05::mbar_arrive(&bars[B_HFREE]);
                      } else {
                          tc05::mbar_arrive(&bars[B_ACC]);
                      }
                  }
              }
              q0 += (uint32_t)n_st;
          }
      }
    } else {
        // =========================== GATHER WARPS (layer-0 operand producers) ===========================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegsGather));
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
            const int tile = RAYQ ? 0 : (ONE_STEP ? work : p.tile_list[work / wmult]);
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
                const float o0 = __ldg(p.cam_ori + 0), o1 = __ldg(p.cam_ori + 1), o2 = __ldg(p.cam_ori + 2);
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
                                // per-ray sampling state (mc_utils.py:102-107, :141-143), as in the tile variant below
                                float accu = 0.0f, cum = 0.0f, entry0 = 0.0f, prev_exit = 0.0f;
                                uint32_t labs = 0;
                                int32_t idl = 0;
#pragma unroll
                                for (int j = 0; j < kMaxM; j++) {
                                    if (j < p.M) {
                                        const int32_t id = __ldg(p.voxel_id + (long long)rq * p.M + j);
                                        const float en = __ldg(p.depth2 + (long long)rq * p.M + j);
                                        const float ex = __ldg(p.depth2 + ((long long)p.H * p.W + rq) * p.M + j);
                                        float d = __fsub_rn(ex, en);
                                        if (d != d) d = 0.0f;
                                        accu = (j == 0) ? d : __fadd_rn(accu, d);
                                        st[(kStAccu + j) * kRows + row] = accu;
                                        if (j == 0) {
                                            entry0 = en;
                                            st[(kStHeads + 0) * kRows + row] = en;
                                        } else {
                                            const float dd = __fsub_rn(en, prev_exit);
                                            cum = (j == 1) ? dd : __fadd_rn(cum, dd);
                                            st[(kStHeads + j) * kRows + row] = __fadd_rn(cum, entry0);
                                        }
                                        prev_exit = ex;
                                        const int lid = (id >= 0 && id < p.n_lut) ? __ldg(p.lut + id) : 0;
                                        labs |= ((uint32_t)lid & 15u) << (4 * j);
                                        idl = id;
                                    }
                                }
                                st[kStTotal * kRows + row] = fminf(accu, p.sample_depth);
                                st[kStLab * kRows + row] = __uint_as_float(labs);
                                const float dx = __ldg(p.raydirs + (long long)rq * 3 + 0);
                                st[(kStDir + 0) * kRows + row] = dx;
                                st[(kStDir + 1) * kRows + row] = __ldg(p.raydirs + (long long)rq * 3 + 1);
                                st[(kStDir + 2) * kRows + row] = __ldg(p.raydirs + (long long)rq * 3 + 2);
                                // the ground test of the sky-leak logic looks at EVERY sample position (scenedreamer.py:380), also at
                                // those an early finish will skip; per-sample outputs of skipped samples: weight 0, depth as sampled
                                bool gnd = false;
                                for (int k = 0; k < S; k++) {
                                    const Sample sk = sample_at(p, st, row, k, sFrac, rq);
                                    gnd = gnd || (__fadd_rn(__fmul_rn(dx, sk.depth), o0) <= 1.0f);
                                    if (p.rdepth_out) p.rdepth_out[(long long)rq * S + k] = sk.depth;
                                    if (p.weights_out) p.weights_out[(long long)rq * S + k] = 0.0f;
                                }
                                code0 = (idl == 0 ? 0x800u : 0u) | (gnd ? 0x1000u : 0u);
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
                        const float d0 = st[(kStDir + 0) * kRows + row], d1 = st[(kStDir + 1) * kRows + row], d2 = st[(kStDir + 2) * kRows + row];
                        const float pw[3] = {__fadd_rn(__fmul_rn(d0, sm.depth), o0), __fadd_rn(__fmul_rn(d1, sm.depth), o1),
                                             __fadd_rn(__fmul_rn(d2, sm.depth), o2)};
                        oob = false;
#pragma unroll
                        for (int k = 0; k < 3; k++) {
                            const float nrm = __fsub_rn(__fmul_rn(__fdiv_rn(pw[k], p.vdim[k]), 2.0f), 1.0f);
                            x5[k] = __fmul_rn(__fadd_rn(nrm, 1.0f), 0.5f);
                            if (x5[k] < 0.0f || x5[k] > 1.0f) oob = true;       // gridencoder.cu:98-104
                        }
                    }
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        const int level = half + 2 * i;
                        float res[8];
                        if (oob) {
#pragma unroll
                            for (int c = 0; c < 8; c++) res[c] = 0.0f;
                        } else {
                            if constexpr (GU == 8) encode_level<RAW5D>(p.table + ((size_t)level << p.log2_T) * 8, mask, sScale[level], x5, res);
                            else encode_level_thin<GU>(p.table + ((size_t)level << p.log2_T) * 8, mask, sScale[level], x5, res);
                        }
                        split8<PREC>(res, fh[i], fl[i]);
                    }
                    const uint32_t label = (labs >> (4 * sm.idx)) & 15u;
                    uint32_t oh[4] = {0u, 0u, 0u, 0u};
                    {
                        const int k = (int)label - 8 * half;
                        if (k >= 0 && k < 8) oh[k >> 1] = one16<PREC>() << (16 * (k & 1));
                        if (half == 1) oh[3] |= one16<PREC>() << 16;             // column 143
                    }
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
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        const uint32_t off = tc05::chunk_off(kRows, row, half + 2 * i);
                        *reinterpret_cast<uint4 *>(sHhi + off) = fh[i];
                        if constexpr (X3) *reinterpret_cast<uint4 *>(sHlo + off) = fl[i];
                    }
                    {
                        const uint32_t off = tc05::chunk_off(kRows, row, kFeat / 8 + half);
                        *reinterpret_cast<uint4 *>(sHhi + off) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
                        if constexpr (X3) *reinterpret_cast<uint4 *>(sHlo + off) = make_uint4(0, 0, 0, 0);
                    }
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
                    float accu = 0.0f, cum = 0.0f, entry0 = 0.0f, prev_exit = 0.0f;
                    uint32_t labs = 0, flags = 0;
                    int32_t id0 = 0, idl = 0;
#pragma unroll
                    for (int j = 0; j < kMaxM; j++) {
                        if (j < p.M) {
                            float en = 0.0f, ex = 0.0f;
                            int32_t id = 0;
                            if (valid) {
                                id = __ldg(p.voxel_id + ray * p.M + j);
                                en = __ldg(p.depth2 + ((long long)tc.img * 2 + 0) * hw * p.M + pix * p.M + j);
                                ex = __ldg(p.depth2 + ((long long)tc.img * 2 + 1) * hw * p.M + pix * p.M + j);
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
                            int lid = (id >= 0 && id < p.n_lut) ? __ldg(p.lut + id) : 0;
                            labs |= ((uint32_t)lid & 15u) << (4 * j);
                            if (j == 0) id0 = id;
                            idl = id;
                        }
                    }
                    st[kStTotal * kRows + row] = fminf(accu, p.sample_depth);   // :107
                    flags = (valid && id0 != 0 ? 1u : 0u) | (idl == 0 ? 2u : 0u) | (valid ? 4u : 0u);
                    st[kStLab * kRows + row] = __uint_as_float(labs);
                    st[kStFlags * kRows + row] = __uint_as_float(flags);
#pragma unroll
                    for (int k = 0; k < 3; k++) st[(kStDir + k) * kRows + row] = valid ? __ldg(p.raydirs + ray * 3 + k) : 0.0f;
                }
                asm volatile("bar.sync 2, 256;" ::: "memory");
                if (half == 0) tc05::mbar_arrive(&bars[B_STRDY + buf]);
                const bool live = __float_as_uint(st[kStFlags * kRows + row]) & 1u;
                const uint32_t labs = __float_as_uint(st[kStLab * kRows + row]);
                const float d0 = st[(kStDir + 0) * kRows + row], d1 = st[(kStDir + 1) * kRows + row], d2 = st[(kStDir + 2) * kRows + row];
                const float o0 = __ldg(p.cam_ori + tc.img * 3 + 0), o1 = __ldg(p.cam_ori + tc.img * 3 + 1), o2 = __ldg(p.cam_ori + tc.img * 3 + 2);
                float x5[5];
                x5[3] = __fmul_rn(__fadd_rn(__ldg(p.genc + tc.img * 2 + 0), 1.0f), 0.5f);   // grid.py:144 on dims 3,4
                x5[4] = __fmul_rn(__fadd_rn(__ldg(p.genc + tc.img * 2 + 1), 1.0f), 0.5f);

                for (int s = 0; s < S; s++, n++) {
                    uint4 fh[8], fl[8];
                    const Sample sm = sample_at(p, st, row, s, sFrac, ray);
                    // world coordinate, normalisation and [0,1] mapping with the reference's operation order
                    // (scenedreamer.py:354, :299; grid.py:144): p = dir*t + ori; p / dim * 2 - 1; (x + 1) / 2
                    const float pw[3] = {__fadd_rn(__fmul_rn(d0, sm.depth), o0), __fadd_rn(__fmul_rn(d1, sm.depth), o1),
                                         __fadd_rn(__fmul_rn(d2, sm.depth), o2)};
                    bool oob = !live;
#pragma unroll
                    for (int k = 0; k < 3; k++) {
                        const float nrm = __fsub_rn(__fmul_rn(__fdiv_rn(pw[k], p.vdim[k]), 2.0f), 1.0f);
                        x5[k] = __fmul_rn(__fadd_rn(nrm, 1.0f), 0.5f);
                        if (x5[k] < 0.0f || x5[k] > 1.0f) oob = true;       // gridencoder.cu:98-104
                    }
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        const int level = half + 2 * i;
                        float res[8];
                        if (oob) {
#pragma unroll
                            for (int c = 0; c < 8; c++) res[c] = 0.0f;
                        } else {
                            encode_level<RAW5D>(p.table + ((size_t)level << p.log2_T) * 8, mask, sScale[level], x5, res);
                        }
                        split8<PREC>(res, fh[i], fl[i]);
                        if constexpr (TRAIN) {   // bf16 copy of the features: X0[slot][8*level ..] (operand of the fc_1 weight gradient)
                            const long long slot = ((long long)work * S + s) * kRows + row;
                            *reinterpret_cast<uint4 *>(rec_chunk(p.tr.x0, slot, kX0Cols / 8, level)) =
                                make_uint4(tc05::pack2<true>(res[0], res[1]), tc05::pack2<true>(res[2], res[3]),
                                           tc05::pack2<true>(res[4], res[5]), tc05::pack2<true>(res[6], res[7]));
                        }
                    }
                    if constexpr (TRAIN) {
                        const long long slot = ((long long)work * S + s) * kRows + row;
                        if (half == 0) p.tr.x3[slot] = make_float4(x5[0], x5[1], x5[2], oob ? -1.0f : 1.0f);
                    }
                    // K-extension of layer 0: one-hot label (columns 128..142) and the constant-1 bias column 143
                    // == the reference's fc_m_a(onehot) product and fc_1's bias (layers.py:102-105)
                    const uint32_t label = (labs >> (4 * sm.idx)) & 15u;
                    uint32_t oh[4] = {0u, 0u, 0u, 0u};
                    {
                        const int k = (int)label - 8 * half;                     // position inside this thread's 8-wide chunk
                        if (k >= 0 && k < 8) oh[k >> 1] = one16<PREC>() << (16 * (k & 1));
                        if (half == 1) oh[3] |= one16<PREC>() << 16;             // column 143
                    }
                    if constexpr (TRAIN) {   // X0 columns 128..143: one-hot label and the constant 1 (bf16)
                        const long long slot = ((long long)work * S + s) * kRows + row;
                        uint32_t ob[4] = {0u, 0u, 0u, 0u};
                        const int k = (int)label - 8 * half;
                        if (k >= 0 && k < 8) ob[k >> 1] = 0x3F80u << (16 * (k & 1));
                        if (half == 1) ob[3] |= 0x3F80u << 16;
                        *reinterpret_cast<uint4 *>(rec_chunk(p.tr.x0, slot, kX0Cols / 8, kFeat / 8 + half)) = make_uint4(ob[0], ob[1], ob[2], ob[3]);
                    }
                    if (gt == 0) SDB_MARK(4, 3, n, it);
                    if (n > 0) tc05::mbar_wait_backoff(&bars[B_HFREE], (n - 1) & 1);
                    if (gt == 0) SDB_MARK(4, 4, n, it);
                    if (ESTOP && s >= 2 && s >= sStop[buf]) break;           // the tile ended before this step: drop the features
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        const uint32_t off = tc05::chunk_off(kRows, row, half + 2 * i);
                        *reinterpret_cast<uint4 *>(sHhi + off) = fh[i];
                        if constexpr (X3) *reinterpret_cast<uint4 *>(sHlo + off) = fl[i];
                    }
                    {
                        const uint32_t off = tc05::chunk_off(kRows, row, kFeat / 8 + half);
                        *reinterpret_cast<uint4 *>(sHhi + off) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
                        if constexpr (X3) *reinterpret_cast<uint4 *>(sHlo + off) = make_uint4(0, 0, 0, 0);
                    }
                    tc05::fence_proxy_async_smem();
                    tc05::mbar_arrive(&bars[B_FEAT]);
                }
            }
        }
    }
}

// ---- pre-pass: live-tile list + outputs of sky-only tiles -----------------------------------------
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
    if (!valid) return;
    // sky-only ray: weights are zero, all samples sit at the camera origin (scenedreamer.py:350-354,376)
    const bool is_gnd = __ldg(p.cam_ori + tc.img * 3) <= 1.0f;
    const float4 *skp = reinterpret_cast<const float4 *>(is_gnd ? p.sky_avg + (long long)tc.img * kOutC : p.sky + ray * kOutC);
    float4 *dst = reinterpret_cast<float4 *>(p.net_out + ray * kOutC);
#pragma unroll
    for (int q = 0; q < kOutC / 4; q++) {
        const float4 sk = __ldg(skp + q);
        float4 o;
        o.x = (0.0f + 1.0f * (fminf(fmaxf(sk.x, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        o.y = (0.0f + 1.0f * (fminf(fmaxf(sk.y, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        o.z = (0.0f + 1.0f * (fminf(fmaxf(sk.z, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        o.w = (0.0f + 1.0f * (fminf(fmaxf(sk.w, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        dst[q] = o;
    }
    if (p.depth_out) p.depth_out[ray] = 0.0f;
    if (p.total_weight) p.total_weight[ray] = 0.0f;
    for (int s = 0; s < p.S; s++) {
        if (p.weights_out) p.weights_out[ray * p.S + s] = 0.0f;
        if (p.rdepth_out) p.rdepth_out[ray * p.S + s] = 0.0f;
    }
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
    if (!valid) return;
    // sky-only ray: weights are zero, all samples sit at the camera origin (scenedreamer.py:350-354,376)
    const bool is_gnd = __ldg(p.cam_ori + tc.img * 3) <= 1.0f;
    const float4 *skp = reinterpret_cast<const float4 *>(is_gnd ? p.sky_avg + (long long)tc.img * kOutC : p.sky + ray * kOutC);
    float4 *dst = reinterpret_cast<float4 *>(p.net_out + ray * kOutC);
#pragma unroll
    for (int q = 0; q < kOutC / 4; q++) {
        const float4 sk = __ldg(skp + q);
        float4 o;
        o.x = (0.0f + 1.0f * (fminf(fmaxf(sk.x, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        o.y = (0.0f + 1.0f * (fminf(fmaxf(sk.y, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        o.z = (0.0f + 1.0f * (fminf(fmaxf(sk.z, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        o.w = (0.0f + 1.0f * (fminf(fmaxf(sk.w, -1.0f), 1.0f) + 1.0f)) - 1.0f;
        dst[q] = o;
    }
    if (p.depth_out) p.depth_out[ray] = 0.0f;
    if (p.total_weight) p.total_weight[ray] = 0.0f;
    for (int s = 0; s < p.S; s++) {
        if (p.weights_out) p.weights_out[ray * p.S + s] = 0.0f;
        if (p.rdepth_out) p.rdepth_out[ray * p.S + s] = 0.0f;
    }
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
    for (int d = 0; d < 2; d++) {
        const float x = __fmul_rn(__fadd_rn(genc[d], 1.0f), 0.5f);
        const float pos = fmaf(x, scale, 0.5f);
        g[d] = (uint32_t)floorf(pos);
        f[d] = pos - (float)g[d];
    }
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const float *tl = table + ((size_t)level << log2_T) * 8;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int b3 = j & 1, b4 = j >> 1;
        const float w = (b3 ? f[0] : 1.0f - f[0]) * (b4 ? f[1] : 1.0f - f[1]);
        const uint32_t K = ((g[0] + b3) * kPrime3) ^ ((g[1] + b4) * kPrime4);
        float v[8];
        ld8(tl + (size_t)((e ^ K) & mask) * 8, v);
#pragma unroll
        for (int c = 0; c < 8; c++) acc[c] = fmaf(w, v[c], acc[c]);
    }
    float4 *o = reinterpret_cast<float4 *>(table3 + i * 8);
    o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// ---- weight packer ---------------------------------------------------------------------------------
// One thread per (layer, n, k) element of the K-extended weight matrices.
//   render: layer 0 [256 x 144]: cols 0..127 fc_1.weight, 128+lab emb[lab][n], 143 fc_1.bias;
//           layers 1..5 [256 x 272]: cols 0..255 W*alpha, 256 beta; colour [64 x 272]: W, 256 bias
//   sky:    layer 0 [256 x 48]: cols 0..32 fc1.weight, 47 bias (fc1.bias + fc_z_a(z)); layers 1..4, colour as above
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
        const int K = layerK<MODE>(l), N = layerN<MODE>(l);
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
            if (k < kHidden) v = wout[(long long)nn * kHidden + k];
            else if (k == kHidden) v = bout[nn];
        } else {
            if (k < kHidden) v = wh[((long long)(l - 1) * kHidden + nn) * kHidden + k];
            else if (k == kHidden) v = bh[(long long)(l - 1) * kHidden + nn];
        }
        const int kk = k >> 4, k16 = k & 15;
        const long long slab_off = (long long)(k16 >> 3) * N * 16 + (nn >> 3) * 128 + (nn & 7) * 16 + (k16 & 7) * 2;
        uint8_t *base = pack + layerOff<MODE>(l, PARTS) + (long long)kk * N * 32 * PARTS;
        if constexpr (PREC == 1) {
            const __nv_bfloat16 hi = __float2bfloat16_rn(v);
            const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
            *reinterpret_cast<__nv_bfloat16 *>(base + slab_off) = hi;
            *reinterpret_cast<__nv_bfloat16 *>(base + (long long)N * 32 + slab_off) = lo;
        } else if constexpr (PREC == 2) {
            const __half hi = __float2half_rn(v);
            const __half lo = __float2half_rn(v - __half2float(hi));
            *reinterpret_cast<__half *>(base + slab_off) = hi;
            *reinterpret_cast<__half *>(base + (long long)N * 32 + slab_off) = lo;
        } else {
            *reinterpret_cast<__half *>(base + slab_off) = __float2half_rn(v);
        }
        return;
    }
    if (SKY) return;
    const long long u = t - nW;
    if (u >= kFTotal) return;
    float *F = reinterpret_cast<float *>(pack + layerOff<MODE>(NL, PARTS));
    float v = 0.0f;
    if (u < kHidden) v = wsig[u];
    else if (u == kFBsig) v = bsig[0];
    F[u] = v;
}

template <bool SKY>
int launch_pack(const float *w0, const float *b0, const float *emb, int n_labels, const float *wh, const float *bh,
                const float *wsig, const float *bsig, const float *wout, const float *bout, int precision, void *pack,
                cudaStream_t st) {
    constexpr int MODE = SKY ? kSky : kRender;
    long long n = SKY ? 0 : kFTotal;
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

// Per-CTA fp32 accumulator buffers of the fused kernels ([grid][2][128][256], L2-resident), one per (device, stream): launches
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
        SDB_CUDA(cudaMalloc(&b.first, (size_t)grid * 2 * kRows * kHidden * sizeof(float)));
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
    const size_t smem = smem_map(PREC != 0).total;
    cudaFuncAttributes fa;
    SDB_CUDA(cudaFuncGetAttributes(&fa, mlp_kernel<PREC, RAW5D, MODE, TRAIN, RAYQ, GU>));
    if (fa.numRegs < kRegsLaunch) return SDB_EUNSUPPORTED;   // setmaxnreg pool would be too small: refuse rather than hang
    SDB_CUDA(cudaFuncSetAttribute(mlp_kernel<PREC, RAW5D, MODE, TRAIN, RAYQ, GU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mlp_kernel<PREC, RAW5D, MODE, TRAIN, RAYQ, GU><<<grid, kThreads, smem, st>>>(p);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

int launch_train_forward(const Params &p, int grid, cudaStream_t st) { return launch_mlp<2, false, kRender, true>(p, grid, st); }
int launch_bwd_chain(const Params &p, int grid, cudaStream_t st) { return launch_mlp<1, false, kBwd>(p, grid, st); }
int launch_sky_train_forward(const Params &p, int grid, cudaStream_t st) { return launch_mlp<2, false, kSky, true>(p, grid, st); }
int launch_sky_bwd_chain(const Params &p, int grid, cudaStream_t st) { return launch_mlp<1, false, kSkyBwd>(p, grid, st); }
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
        const int K = layerK<MODE>(l), N = layerN<MODE>(l);
        const int nn = (int)(r / K), k = (int)(r % K);
        float v;
        if (l == 0) v = wout[(long long)k * kHidden + nn];
        else if (MODE == kBwd && l == NL - 1) v = w1[(long long)k * kFeat + nn];
        else v = wh[((long long)((MODE == kBwd ? 5 : 4) - l) * kHidden + k) * kHidden + nn];
        const int kk = k >> 4, k16 = k & 15;
        const long long slab_off = (long long)(k16 >> 3) * N * 16 + (nn >> 3) * 128 + (nn & 7) * 16 + (k16 & 7) * 2;
        uint8_t *base = pack + layerOff<MODE>(l, PARTS) + (long long)kk * N * 32 * PARTS;
        const __nv_bfloat16 hi = __float2bfloat16_rn(v);
        const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
        *reinterpret_cast<__nv_bfloat16 *>(base + slab_off) = hi;
        *reinterpret_cast<__nv_bfloat16 *>(base + (long long)N * 32 + slab_off) = lo;
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
    if (d_record && (precision != 2 || n_img != 1)) return SDB_EUNSUPPORTED;
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
    return sky_forward_impl(d_raydirs, n_img, H, W, d_sky_pack, 0, 2, d_sky, d_sky_avg, d_workspace, d_record, stream);
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
