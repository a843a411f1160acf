// Shared definitions of the fused render engine (render_fused.cu) and the training-side kernels
// (render_train.cu): network shapes, the weight-pack layout, the shared-memory map, kernel
// parameters, ray sampling and hash-grid corner math.  Internal to libsdb200 (not part of the ABI).
#pragma once
#include <math.h>

#include "common.cuh"
#include "tc05.cuh"

namespace rf {

constexpr int kRows = 128, kTileW = 16, kTileH = 8;
constexpr int kHidden = 256, kFeat = 128, kOutC = 64, kLevels = 16;
constexpr int kKExt = 16;                       // extra K columns of the render network's layer 0: labels / fc_1 bias
constexpr int kMaxM = 8, kMaxS = 64, kMaxLabels = 15;
constexpr int kEpiThreads = 256, kGatherThreads = 256;
// warpgroup-aligned roles so that setmaxnreg can move registers between them (here: from the epilogue, the gather and the
// producer to the MMA warpgroup):
//   WG0-1 epilogue (warps 0-7), WG2 MMA (warps 8-11), WG3-4 gather (12-19), WG5 weight-ring producer (20-23)
constexpr int kMmaWarp0 = 8, kGatherWarp0 = 12, kProducerWarp0 = 20;
constexpr int kThreads = kEpiThreads + 128 + kGatherThreads + 128;   // 768
// setmaxnreg can only redistribute the registers the CTA was LAUNCHED with (768 threads x 80 = 61,440, the most ptxas
// grants a 768-thread __launch_bounds__; the allocator is a per-CTA pool -- USETMAXREG.TRY_ALLOC.CTAPOOL spins forever
// otherwise):
//   8 epilogue warps x 72 + 4 MMA warps x 112 + 8 gather warps x 96 + 4 producer warps x 32 = 61,440
// (the MMA warpgroup holds two 32-register accumulator sets of 64-column blocks and its loop state; at 96 that state spills
// inside the stage loop)
constexpr int kRegsLaunch = 80, kRegsEpi = 72, kRegsCtl = 112, kRegsGather = 96, kRegsProd = 32;
static_assert(8 * 32 * kRegsEpi + 4 * 32 * kRegsCtl + 8 * 32 * kRegsGather + 4 * 32 * kRegsProd <= kThreads * kRegsLaunch,
              "setmaxnreg budget exceeds the CTA's launch-time register allocation");
// a role's register count: released to / taken from the CTA's pool (no instruction when it is the launch count)
template <int R> __device__ __forceinline__ void set_maxnreg() {
    if constexpr (R < kRegsLaunch) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
    else if constexpr (R > kRegsLaunch) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
constexpr int kRingBytes = 65536;
constexpr uint32_t kLboA = kRows * 16, kSbo = 128;
constexpr int kHChunks = kHidden / 8;           // 32 16-byte k-chunks per row
constexpr int kHBytes = kHChunks * kRows * 16;  // 65,536 bytes per operand part
constexpr int kSkyK0 = 48;                      // PE(raydir) 33 + zeros + bias column 47
constexpr int kRenderK0 = kFeat + kKExt;        // 144

// Networks the tensor-core engine runs (MODE):
//   kRender: LightningMLP forward, 6 hidden layers + colour head (layers.py:92-126)
//   kSky   : SKYMLP forward, 5 hidden layers + colour head (gancraft_base.py:150-169)
//   kBwd   : data-gradient chain of LightningMLP: dC -> dA6 -> ... -> dA1 -> d(features); the B operands are
//            the TRANSPOSED forward weights (biases do not enter the data gradient)
//   kSkyBwd: data-gradient chain of SKYMLP: dSky -> dA5 -> ... -> dA1 (the PE input needs no gradient), so there are
//            4 operand-producing layers and the last layer's output (dA1 -> dZ1, N = 256) only goes to the record
constexpr int kRender = 0, kSky = 1, kBwd = 2, kSkyBwd = 3;
template <int MODE> struct Net {
    static constexpr bool ISBWD = MODE == kBwd || MODE == kSkyBwd;
    static constexpr int NH = MODE == kSky ? 5 : (MODE == kSkyBwd ? 4 : 6);   // layers whose epilogue feeds the next layer
    static constexpr int NL = NH + 1;
    static constexpr int K0 = MODE == kSky ? kSkyK0 : (ISBWD ? kOutC : kRenderK0);
    static constexpr int NOUT = MODE == kBwd ? kFeat : (MODE == kSkyBwd ? kHidden : kOutC);   // N of the last layer
    static constexpr int NACT = MODE == kSky || MODE == kSkyBwd ? 5 : 6;   // hidden activations of the forward network
    static constexpr bool TAIL = MODE == kRender || MODE == kBwd;          // the pack has the fp32 sigma head
    // fp32 biases of layers 1 .. NL-1 (forward networks), added to the accumulators at the write-out: entry (l - 1) * 256 + n
    static constexpr int NBIAS = ISBWD ? 0 : (NL - 2) * kHidden + NOUT;
};
// layers fed by hidden activations have K = 256; layer 0 carries its bias (and the label embedding) in K-extension columns
template <int MODE> __host__ __device__ constexpr int layerK(int l) { return l == 0 ? Net<MODE>::K0 : kHidden; }
template <int MODE> __host__ __device__ constexpr int layerN(int l) { return l == Net<MODE>::NL - 1 ? Net<MODE>::NOUT : kHidden; }
template <int MODE> __host__ __device__ constexpr int64_t layerOff(int l, int parts) {
    int64_t o = 0;
    for (int j = 0; j < l; j++) o += (int64_t)layerK<MODE>(j) * layerN<MODE>(j) * 2 * parts;
    return o;
}
// fp32 tail of the render / backward packs: sigma head
constexpr int kFWsig = 0, kFBsig = 256, kFTotal = 264;
// the pack: the 16-bit layers, then the sigma head (TAIL), then the bias table (NBIAS floats, the last bytes of the pack)
template <int MODE> __host__ __device__ constexpr int64_t biasOff(int parts) {
    return layerOff<MODE>(Net<MODE>::NL, parts) + (Net<MODE>::TAIL ? (int64_t)kFTotal * 4 : 0);
}
template <int MODE> __host__ __device__ constexpr int64_t packBytes(int parts) {
    return biasOff<MODE>(parts) + (int64_t)Net<MODE>::NBIAS * 4;
}
// Byte offset of weight element (output n, input k), 16-bit part `part` (hi / lo), inside one layer of the pack, for a layer
// of nK k16 slabs and `parts` parts.  The layer is stored in the order the MMA warpgroup streams it:
//   [64-column block n/64][k16 slab k/16][part][k-chunk (k/8)%2][64 outputs][8 k]
// so one k16 slab of a 64-column block is a 2 KB-per-part wgmma B operand (K-major, no swizzle, LBO 1024), and a ring stage
// (consecutive slabs of one block) is ONE contiguous range that a single bulk copy fetches.
__host__ __device__ constexpr int64_t wpack_off(int nK, int parts, int n, int k, int part) {
    return ((((int64_t)(n >> 6) * nK + (k >> 4)) * parts + part) * 2 + ((k >> 3) & 1)) * 1024 + (n & 63) * 16 + (k & 7) * 2;
}
static_assert(kHidden % 64 == 0 && kOutC % 64 == 0 && kFeat % 64 == 0, "every layer is whole 64-column blocks");

// Ring stages of one 64-column block of a layer with nK k16 slabs, `sps` slabs per ring slot.  The block's sum over K is two
// numerics groups -- slabs 0..7 and slabs 8..nK-1, each a fresh tensor-core sum -- and a stage never straddles them.
__host__ __device__ constexpr int group0_stages(int nK, int sps) { return ((nK < 8 ? nK : 8) + sps - 1) / sps; }
__host__ __device__ constexpr int block_stages(int nK, int sps) {
    return group0_stages(nK, sps) + ((nK > 8 ? nK - 8 : 0) + sps - 1) / sps;
}
// first slab and slab count of stage js of a block
__host__ __device__ constexpr int stage_slab0(int nK, int sps, int js) {
    return js < group0_stages(nK, sps) ? js * sps : 8 + (js - group0_stages(nK, sps)) * sps;
}
__host__ __device__ constexpr int stage_slabs(int nK, int sps, int js) {
    const int end = js < group0_stages(nK, sps) ? (nK < 8 ? nK : 8) : nK, left = end - stage_slab0(nK, sps, js);
    return left < sps ? left : sps;
}

// ring stages of one sample step of network MODE: per layer and row block, the stages of the layer's 64-column blocks
template <int MODE> __host__ __device__ constexpr int step_stages(int sps) {
    int n = 0;
    for (int l = 0; l < Net<MODE>::NL; l++) n += 2 * (layerN<MODE>(l) / 64) * block_stages(layerK<MODE>(l) / 16, sps);
    return n;
}
constexpr int kMaxStepStages = 192;   // the render network at x3 (4 slabs per stage)
static_assert(step_stages<kRender>(4) <= kMaxStepStages && step_stages<kSky>(4) <= kMaxStepStages &&
              step_stages<kBwd>(4) <= kMaxStepStages && step_stages<kSkyBwd>(4) <= kMaxStepStages &&
              step_stages<kRender>(8) <= kMaxStepStages && step_stages<kSky>(8) <= kMaxStepStages,
              "stage table of one sample step");
// a layer is whole [64 x 16] blocks of 16-bit parts, so every stage starts and ends on a 2 KB boundary of the pack, and an entry
// of the table holds the stage's offset and size in 2 KB units in 16 bits each
static_assert(64 * 16 * 2 == 2048, "stage table entries count 2 KB units");
static_assert((layerOff<kRender>(Net<kRender>::NL, 2) >> 11) < 65536 && (layerOff<kBwd>(Net<kBwd>::NL, 2) >> 11) < 65536 &&
              (layerOff<kSky>(Net<kSky>::NL, 2) >> 11) < 65536 && (layerOff<kSkyBwd>(Net<kSkyBwd>::NL, 2) >> 11) < 65536,
              "stage table offsets fit 16 bits");

__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}\n" : "=r"(pred));
    return pred != 0;
}

// ---- shared memory map ---------------------------------------------------------------------------
struct Smem {
    uint32_t h_hi, h_lo, ring, fsec, bias, scales, frac, sig, state, bars, stop, sched, walk, total;
};
__host__ __device__ constexpr Smem smem_map() {
    Smem m{};
    uint32_t o = 0;
    m.h_hi = o; o += kHBytes;
    m.h_lo = o; o += kHBytes;                   // fp16 (!x3): no lo operand, the lo half of blocks staged there (hand_plan)
    m.ring = o; o += kRingBytes;
    m.fsec = o; o += kFTotal * 4;
    m.bias = o; o += Net<kRender>::NBIAS * 4;   // the largest bias table (read by the MMA warpgroup)
    m.scales = o; o += kLevels * 4;
    m.frac = o; o += ((kMaxS + 1) * 4 + 15) / 16 * 16;
    m.sig = o; o += 2 * kRows * 4;
    m.state = o; o += 2 * (2 * kMaxM + 6) * kRows * 4;
    m.bars = o; o += 40 * 8;
    m.stop = o; o += 32;                         // early termination: int stop_step[2] (per tile buffer), int vote[2], int voted[2]
    m.sched = o; o += 32;                        // dynamic tile scheduler: int work[4] (ring), int published
    m.walk = o; o += kMaxStepStages * 4;         // the weight stages of one sample step (read by the producer)
    m.total = o;
    return m;
}
// per-buffer ray state: float arrays of kRows each
constexpr int kStAccu = 0;                   // [kMaxM]
constexpr int kStHeads = kMaxM;              // [kMaxM]
constexpr int kStTotal = 2 * kMaxM;          // 1
constexpr int kStDir = 2 * kMaxM + 1;        // 3
constexpr int kStLab = 2 * kMaxM + 4;        // 1 (uint32: 4 bits per slot)
constexpr int kStFlags = 2 * kMaxM + 5;      // 1 (uint32: bit0 live, bit1 sky_mask, bit2 valid)
constexpr int kStFloats = 2 * kMaxM + 6;

// barrier indices.  The MMA warpgroup and the epilogue hand a layer over per 64-row block rb (B_OPND, B_ACC, B_OUTRDY: + rb;
// B_EPIDONE: + accumulator buffer * 2 + rb), so that one row block's epilogue runs while the other's MMAs do.  Ring slot i is
// loaded (B_WFULL + i, the producer's bulk copy) and free again (B_WEMPTY + i, one arrival per MMA warp).
enum { B_WFULL = 0, B_FEAT = 4, B_HFREE, B_OPND, B_ACC = B_OPND + 2, B_OUTRDY = B_ACC + 2, B_EPIDONE = B_OUTRDY + 2,
       B_STRDY = B_EPIDONE + 4, B_STFREE = B_STRDY + 2, B_COMP = B_STFREE + 2, B_WEMPTY = B_COMP + 1, B_COUNT = B_WEMPTY + 4 };
constexpr int kBarSlots = 40;
static_assert(B_COUNT <= kBarSlots, "barrier table");

// ---- training-side record of one forward pass (all DEVICE pointers; see sdb_train_layout in sdb200.h) ----
// A "slot" is one (work item, sample step, tile row): slot = (work * S + s) * 128 + row, where `work` is the
// position of the ray tile in the live-tile list of the forward launch.  Every slot of a live tile is written
// (rows outside the image / sky-only rays included), so the backward GEMMs may run over [0, n_live*S*128).
constexpr int kX0Cols = kRenderK0;           // 144: features | one-hot label | 1
constexpr int kActCols = kHidden + 16;       // 272: activations | 1 | 0 x 15 (the 1 makes the wgrad GEMM emit the bias grad; 544 B rows stay 32 B aligned)
constexpr int kNumAct = 6;
// The bf16 arrays of the record (x0, act, dz, dc16) are kept as MMA-READY TILES, not row-major: an array of C columns is
//   [work item = slot / 128][chunk = column / 8][row = slot % 128][8 columns]      (16 B per (row, chunk), 2 KB per chunk)
// so that (a) a warp of 32 consecutive rows writes 512 contiguous bytes per store instruction and (b) one item of an
// array is a contiguous range that the weight-gradient kernel (wgrad.cu) bulk-copies into shared memory, where it is a
// canonical MN-major wgmma operand whose reduction dimension is the samples.
__host__ __device__ __forceinline__ uint16_t *rec_chunk(uint16_t *base, long long slot, int n_chunks, int chunk) {
    return base + ((((slot >> 7) * n_chunks + chunk) << 10) + ((slot & 127) << 3));
}
static_assert(kRows == 128, "rec_chunk assumes 128-row work items");

struct TrainBuf {
    long long slot_cap;        // slots the buffers were sized for (n_tiles * S * 128)
    float4 *x3;                // [slots] (x, y, z in [0,1], w = +1 inside / -1 skip in the table backward)
    uint16_t *x0;              // tiled [slots x 144] bf16 (render) / [slots x 48] bf16 (sky: PE(raydir) | 0 | 1)
    uint16_t *act;             // [6] x tiled [slot_cap x 272] bf16: A1..A6
    uint32_t *mask;            // [steps][6][128][8]: bit j of word q = (A[., 32q + j] > 0)
    float *sig, *nds;          // [slots] sigma (pre-relu), new_dists * dists_scale
    float *c;                  // [slots][64] colour head output (pre-clamp)
    uint32_t *rayflags;        // [n_live*128]: bit0 live, bit1 nosky, bit2 valid
    int32_t *tile_work;        // [n_tiles]: position in the live list or -1
    // backward chain
    const float *dc;           // [slots][64] fp32 (render) / [R][64] fp32 in RAY order (sky: dL/dsky)
    uint16_t *dc16;            // sky only: tiled [slots x 64] bf16 copy of dL/dsky written by the chain's operand producer
    const float *dsig;         // [slots]
    uint16_t *dz;              // [6] x tiled [slot_cap x 256] bf16: dZ1..dZ6
    float *dx0;                // [slots][128]
};

struct Params {
    int n_img, H, W, M, S;
    const int32_t *voxel_id;
    const float *depth2, *raydirs, *cam_ori, *genc;
    float vdim[3];
    float sample_depth, dists_scale;
    float early_T;                 // > 0: a ray tile stops once every live ray's transmittance is below this (inference only)
    const float *fractions, *uniforms;
    const int32_t *lut;
    int n_lut;
    const float *table;
    int raw5d;
    int log2_T;
    float level_S;
    int base_res;
    const uint8_t *pack;
    long long pack_stride;
    const float *sky, *sky_avg;
    float *net_out, *depth_out, *total_weight, *weights_out, *rdepth_out;
    const int32_t *tile_list;      // [n_live] (render) / nullptr (sky: all tiles)
    const int32_t *n_live;
    int32_t *steps_done;           // optional counter (workspace word 1): sample steps actually executed, summed over tiles
    int32_t *work_counter;         // optional (workspace word 2, zeroed per launch): dynamic tile scheduling across the persistent CTAs
    int work_mult;                 // > 1: every live tile is work_mult independent work items (the gradient chain: one per sample step)
    int n_tiles;
    int tiles_x, tiles_y;
    // sky mode
    float *sky_out;                // [R, 64]
    float *sky_partial;            // [n_tiles, 64] per-tile column sums (deterministic mean)
    int32_t *debug;                // optional host-mapped progress buffer (diagnostics), else nullptr
    TrainBuf tr;                   // training record (TRAIN forward writes it, the kBwd chain reads it)
    float *acc;                    // [grid][2] fp32 accumulator buffers of 128 x 128 (acc_off), set by the launcher
    const int32_t *view;           // kBwd over one image of a multi-view record: {first live-list position, live tiles} (device)
};

// ---- layer hand-off: the order of a row block's column blocks, and where each finished block goes ----
// Block c of a layer is output columns 64c .. 64c+63.  Operand region r of the shared-memory operand buffer is K slabs
// 4r .. 4r+3 (columns 64r .. 64r+63); a layer reads a slab in numerics group 0 (slabs 0..7) or group 1 (slabs 8..nK-1).  A
// finished block is STAGED as fp32 in a region of its own rows that no MMA of the layer reads any more, or goes to the per-CTA
// accumulator buffer in L2 (acc_off).  In a hidden layer the region is the block's own (c): the epilogue turns it into the
// next layer's operand in place.  The last layer's output only goes to the epilogue, so it may sit in any dead region that
// the gather does not write -- the gather writes the next step's layer-0 operand (columns 0 .. K0-1) as soon as B_HFREE fires.
// bit 0: group 0 of layer l reads a slab of region r, bit 1: group 1 does
template <int MODE> __host__ __device__ constexpr int region_readers(int l, int r) {
    const int nK = layerK<MODE>(l) / 16, s0 = 4 * r, g0e = nK < 8 ? nK : 8;
    return (s0 < g0e ? 1 : 0) | (s0 < nK && s0 + 4 > 8 ? 2 : 0);
}
// walk, byte p = the p-th column block the MMA warpgroup computes: bits 0-1 the block c, then the flags below and the region
// (bits 4-5) it is staged in.  src, nibble c: 0 = block c is in the L2 buffer (at column block c & 1), r + 1 = staged in region r.
enum { kHStaged = 4, kHDelayed = 8, kHBarrier = 64, kHFirst = 128 };
// kHDelayed: the region is read by the NEXT block's group 0 only; the block stays in its accumulator set until that group has
//            retired, and the next block's group 1 is issued into the set after the store
// kHBarrier: an MMA of this layer read the region since the warpgroup last met, so it meets (named barrier 3) before the store
// kHFirst:   the row block's first staged store
struct HandPlan { uint32_t walk, src; };
template <int MODE> __host__ __device__ constexpr HandPlan hand_plan(int l) {
    const bool last = l == Net<MODE>::NL - 1;
    const int ncb = layerN<MODE>(l) / 64, L = ncb - 1;
    // order: blocks whose own region group 1 reads first (they cannot be staged), then those whose region no MMA of the layer
    // reads, then those only group 0 reads: a hidden layer walks 2, 3, 0, 1.  The last layer walks 0, 1, ...
    int order[4] = {0, 1, 2, 3}, n = 0;
    if (!last)
        for (int cat = 2; cat < 5; cat++)                       // categories 2, 0, 1
            for (int c = 0; c < ncb; c++)
                if ((region_readers<MODE>(l, c) & 2 ? 2 : region_readers<MODE>(l, c)) == cat % 3) order[n++] = c;
    const int r_min = last ? (Net<MODE>::K0 + 63) / 64 : 0;    // the last layer: regions clear of the gather's columns
    int dst[4] = {-1, -1, -1, -1}, used = 0;
    bool del[4] = {false, false, false, false};
    for (int p = 0; p < ncb; p++) {
        for (int pass = 0; pass < 2 && dst[p] < 0; pass++)     // pass 0: dead once the block is done; pass 1: delayed
            for (int r = last ? 3 : order[p]; r >= (last ? r_min : order[p]); r--) {
                const int rd = region_readers<MODE>(l, r);
                const bool dead = pass == 0 ? (p == L || rd == 0) : (p == L - 1 && rd == 1);
                if (!(used >> r & 1) && dead) { dst[p] = r; del[p] = pass == 1; used |= 1 << r; break; }
            }
    }
    // when the last reader of each region retires, in the order W(p) = 3p (block p's groups), staged store of block p: 3p + 1,
    // or 3p + 2 with block p + 1's group 0 retired just before
    HandPlan h{0u, 0u};
    int met = -1;
    for (int p = 0; p < ncb; p++) {
        uint32_t b = (uint32_t)order[p];
        if (dst[p] >= 0) {
            const int rd = region_readers<MODE>(l, dst[p]);
            const int t_read = rd == 0 ? -1 : ((rd & 2) || L == 0 || !del[L - 1] ? 3 * L : 3 * L - 1);
            b |= kHStaged | (del[p] ? kHDelayed : 0u) | ((uint32_t)dst[p] << 4) | (h.src == 0 ? kHFirst : 0u);
            if (t_read > met) { b |= kHBarrier; met = 3 * p + (del[p] ? 2 : 1); }
            h.src |= (uint32_t)(dst[p] + 1) << (4 * order[p]);
        }
        h.walk |= b << (8 * p);
    }
    return h;
}
template <int MODE> __host__ __device__ constexpr bool hand_all_staged(int l) {
    for (int c = 0; c < layerN<MODE>(l) / 64; c++)
        if ((hand_plan<MODE>(l).src >> (4 * c) & 15u) == 0) return false;
    return true;
}
// every mode: at most two blocks of a layer pass through L2, in different column blocks of the buffer; a hidden layer stages a
// block in its own region; and layer 0 stages a block (its first staged store is where the MMA warpgroup waits until the
// epilogue has read the previous step's last layer)
template <int MODE> __host__ __device__ constexpr bool hand_plan_ok() {
    for (int l = 0; l < Net<MODE>::NL; l++) {
        const HandPlan h = hand_plan<MODE>(l);
        int l2 = 0;
        for (int c = 0; c < layerN<MODE>(l) / 64; c++) {
            const uint32_t src = h.src >> (4 * c) & 15u;
            if (src == 0) {
                if (l2 >> (c & 1) & 1) return false;
                l2 |= 1 << (c & 1);
            } else if (l < Net<MODE>::NL - 1 && src != (uint32_t)c + 1) {
                return false;
            }
        }
        if (l == 0 && h.src == 0) return false;
    }
    return true;
}
static_assert(hand_plan_ok<kRender>() && hand_plan_ok<kSky>() && hand_plan_ok<kBwd>() && hand_plan_ok<kSkyBwd>(), "hand-off plan");
static_assert(hand_plan<kRender>(1).walk == 0x15cc0302u && hand_plan<kRender>(1).src == 0x21u, "hidden layer: 2, 3, 0, 1");

// Element (row, col) of one fp32 accumulator buffer: the column blocks of a 128 x 256 layer output that are not staged, at most
// two per layer, block c at column block c & 1.  The buffer is 4 blocks of 64 rows x 64 columns, 16 KB each (row block rb,
// column block c: block rb * 2 + (c & 1)), and a block is stored
//   [row group r / 16 (4)][column chunk c / 4 (16)][row r % 16 (16)][4 floats]      (r, c inside the block)
// so that one MMA warp's 16 rows of a block (its part of the wgmma accumulator fragment) are one contiguous 4 KB range, a warp's
// 8-byte fragment stores of one (j, h) pair fill two whole 128-byte lines (8 rows of two 4-column chunks), and the 32
// consecutive rows that an epilogue warp reads of one 4-column chunk are two 256-byte runs: 4 lines per 128-bit warp load.
// In a row-major buffer the same store touched 8 lines and the same load 32.
constexpr int kAccCols = 128;
__host__ __device__ __forceinline__ constexpr uint32_t acc_off(uint32_t row, uint32_t col) {
    return (((row >> 6) * (kAccCols / 64) + ((col >> 6) & 1u)) << 12) + (((row >> 4) & 3u) << 10) + (((col >> 2) & 15u) << 6) +
           ((row & 15u) << 2) + (col & 3u);
}
static_assert(acc_off(kRows - 1, kHidden - 1) == kRows * kAccCols - 1 && acc_off(16, 0) - acc_off(0, 0) == 1024,
              "accumulator buffer layout");

// Columns col .. col + NV - 1 of one row of a block staged in the operand buffer (col a multiple of 8): the MMA warpgroup
// stores floats 0-3 of 8-column chunk j in the hi part's 16-byte slot of (row, j) and floats 4-7 in the lo part's slot.  The
// epilogue thread that owns the row reads both and writes its 16-bit operand back into the same two slots.
template <int NV>
__device__ __forceinline__ void stg_ld(const uint8_t *sHhi, const uint8_t *sHlo, int row, int col, float (&v)[NV]) {
    static_assert(NV % 8 == 0, "whole 8-column chunks");
#pragma unroll
    for (int i = 0; i < NV; i += 8) {
        const uint32_t off = tc05::chunk_off(kRows, row, (col + i) >> 3);
        const float4 a = *reinterpret_cast<const float4 *>(sHhi + off), b = *reinterpret_cast<const float4 *>(sHlo + off);
        v[i] = a.x; v[i + 1] = a.y; v[i + 2] = a.z; v[i + 3] = a.w;
        v[i + 4] = b.x; v[i + 5] = b.y; v[i + 6] = b.z; v[i + 7] = b.w;
    }
}

// Columns col .. col + NV - 1 of one row of an accumulator buffer (col a multiple of NV, so they lie in one 64-column block).
// Written by the MMA warpgroup of the same CTA; read at L2 (.cg), since every line a warp load touches is used whole by that
// one instruction and keeping it in L1 would buy nothing.
// SDB_AB_NO_ACC (diagnostics build only, results are wrong): the accumulator buffer is neither written nor read, so that
// the kernel time with and without that traffic can be compared on the same work (bench.py --no-early-stop).
template <int NV>
__device__ __forceinline__ void acc_ld(const float *buf, int row, int col, float (&v)[NV]) {
    static_assert(NV % 4 == 0 && NV <= 64 && 64 % NV == 0, "one 64-column block, whole float4s");
#ifdef SDB_AB_NO_ACC
#pragma unroll
    for (int i = 0; i < NV; i++) v[i] = __int_as_float((int)(reinterpret_cast<uintptr_t>(buf) & 1));   // 0.0f, not a constant
    (void)row; (void)col;
    return;
#endif
    const float *src = buf + acc_off(row, col);
#pragma unroll
    for (int i = 0; i < NV; i += 4) {
        const float4 a = __ldcg(reinterpret_cast<const float4 *>(src + acc_off(0, i)));   // the next 4-column chunk
        v[i] = a.x; v[i + 1] = a.y; v[i + 2] = a.z; v[i + 3] = a.w;
    }
}

// progress markers (CTA 0 only): debug[role*4 + {0,1,2}] = {marker, step, layer/stage}
#define SDB_MARK(role, marker, a, b)                                              \
    do {                                                                          \
        if (p.debug != nullptr && blockIdx.x == 0) {                              \
            volatile int32_t *d__ = p.debug + (role) * 4;                         \
            d__[0] = (marker); d__[1] = (int32_t)(a); d__[2] = (int32_t)(b);      \
        }                                                                         \
    } while (0)

// timeline of CTA 0 (diagnostics, tools/render_timeline.py; library built with SDB_NVCC_EXTRA=-DSDB_TIMELINE): with debug[60] == kTraceMagic, sample steps
// debug[61] .. debug[61]+kTraceSteps-1 of the CTA record clock() stamps, debug[64 + ((n - first) * 8 + layer) * 8 + slot]:
//   slot 2 rb    MMA warpgroup, row block rb: the inputs are ready (buffer free, operand rows written)
//   slot 2 rb + 1  MMA warpgroup, row block rb: the accumulators are written
//   slot 4 + 2 rb  epilogue of row block rb: accumulators seen        slot 5 + 2 rb: the next layer's operand rows handed over
//   layer row 7 = the gather role preparing step n: 0 compositing of step n-2 seen, 1 slots refilled, 2 features gathered, 3 operand buffer free
// and the MMA warpgroup's row-block time (slot 2 rb -> slot 2 rb + 1) split into cycles spent in kSplit* (thread 0's clock):
//   debug[kSplitBase + (((n - first) * 8 + layer) * 2 + rb) * 8 + k]
// full-barrier waits, wgmma issue, wait_group, then what follows wait_group: the row-block hand-over barrier, ring-slot
// releases (each warp's empty-barrier arrive), the block's sums and bias adds, its accumulator-buffer stores;
// and the producer's empty-barrier waits of step n (cycles): debug[kProdBase + n - first]
constexpr int32_t kTraceMagic = 0x7131;
constexpr int kTraceSteps = 6, kSplitBase = 512, kProdBase = kSplitBase + kTraceSteps * 8 * 2 * 8;
enum { kSplitFull = 0, kSplitIssue, kSplitWait, kSplitBarrier, kSplitRelease, kSplitReduce, kSplitStore, kSplitN };
#ifndef SDB_TIMELINE
#define SDB_STAMP(n_, layer, slot) do { } while (0)      // compiled out: the stamps cost the epilogue role registers (spills)
struct TSplit {
    __device__ __forceinline__ void start() {}
    __device__ __forceinline__ void lap(int) {}
};
#define SDB_STAMP_SPLIT(n_, layer, rb, ts) do { } while (0)
#define SDB_STAMP_PROD(n_, cycles) do { } while (0)
#define SDB_CLOCK() 0u
#else
#define SDB_CLOCK() ((uint32_t)clock())
struct TSplit {                                   // cycles since the last lap, charged to category k
    uint32_t acc[kSplitN], t;
    __device__ __forceinline__ void start() {
        for (int k = 0; k < kSplitN; k++) acc[k] = 0;
        t = (uint32_t)clock();
    }
    __device__ __forceinline__ void lap(int k) { const uint32_t c = (uint32_t)clock(); acc[k] += c - t; t = c; }
};
#define SDB_STAMP_SPLIT(n_, layer, rb, ts)                                                                         \
    do {                                                                                                           \
        if (p.debug != nullptr && blockIdx.x == 0 && p.debug[60] == kTraceMagic) {                                 \
            const int rel__ = (int)(n_) - p.debug[61];                                                             \
            if (rel__ >= 0 && rel__ < kTraceSteps)                                                                 \
                for (int k__ = 0; k__ < kSplitN; k__++) p.debug[kSplitBase + ((rel__ * 8 + (layer)) * 2 + (rb)) * 8 + k__] = (int32_t)(ts).acc[k__]; \
        }                                                                                                          \
    } while (0)
#define SDB_STAMP_PROD(n_, cycles)                                                                                 \
    do {                                                                                                           \
        if (p.debug != nullptr && blockIdx.x == 0 && p.debug[60] == kTraceMagic) {                                 \
            const int rel__ = (int)(n_) - p.debug[61];                                                             \
            if (rel__ >= 0 && rel__ < kTraceSteps) p.debug[kProdBase + rel__] = (int32_t)(cycles);                 \
        }                                                                                                          \
    } while (0)
#define SDB_STAMP(n_, layer, slot)                                                                                 \
    do {                                                                                                           \
        if (p.debug != nullptr && blockIdx.x == 0 && p.debug[60] == kTraceMagic) {                                 \
            const int rel__ = (int)(n_) - p.debug[61];                                                             \
            if (rel__ >= 0 && rel__ < kTraceSteps) p.debug[64 + (rel__ * 8 + (layer)) * 8 + (slot)] = (int32_t)clock(); \
        }                                                                                                          \
    } while (0)
#endif

__device__ __constant__ uint32_t kPrime1 = 2654435761u, kPrime2 = 805459861u, kPrime3 = 3674653429u, kPrime4 = 2097192037u;

struct TileCoord { int img, y0, x0; };
__device__ __forceinline__ TileCoord tile_coord(const Params &p, int tile) {
    const int per_img = p.tiles_x * p.tiles_y;
    TileCoord t;
    t.img = tile / per_img;
    const int r = tile - t.img * per_img;
    t.y0 = (r / p.tiles_x) * kTileH;
    t.x0 = (r % p.tiles_x) * kTileW;
    return t;
}

// a thread's 32 contiguous bytes as two 128-bit global stores (`p` 32-byte aligned)
__device__ __forceinline__ void st_global_v8(void *p, uint4 a, uint4 b) {
    reinterpret_cast<uint4 *>(p)[0] = a;
    reinterpret_cast<uint4 *>(p)[1] = b;
}
__device__ __forceinline__ void st_global_v8f(float *p, const float *v) {
    reinterpret_cast<float4 *>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4 *>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}

__device__ __forceinline__ void ld8(const float *g, float (&v)[8]) {
    const float4 a = __ldg(reinterpret_cast<const float4 *>(g));
    const float4 b = __ldg(reinterpret_cast<const float4 *>(g) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// cell g and interpolation fraction f of coordinate x on a hash-grid level of resolution `scale` (gridencoder.cu:133-140);
// pos = x*scale + 0.5 is one FFMA in the reference's device code
__device__ __forceinline__ void grid_cell(float x, float scale, uint32_t &g, float &f) {
    const float pos = fmaf(x, scale, 0.5f);
    g = (uint32_t)floorf(pos);
    f = pos - (float)g;
}

// table row and trilinear weight of corner i (bit d set: the upper neighbour on dim d) of the 3-D cell (g, f)
__device__ __forceinline__ uint32_t corner3(uint32_t mask, const uint32_t (&g)[3], const float (&f)[3], uint32_t i, float &w) {
    const uint32_t b0 = i & 1, b1 = (i >> 1) & 1, b2 = (i >> 2) & 1;
    w = b0 ? f[0] : 1.0f - f[0];
    w *= b1 ? f[1] : 1.0f - f[1];
    w *= b2 ? f[2] : 1.0f - f[2];
    return ((g[0] + b0) ^ ((g[1] + b1) * kPrime1) ^ ((g[2] + b2) * kPrime2)) & mask;
}

// corner j (bit 0: upper neighbour on dim 3, bit 1: on dim 4) of the cell (g, f) of the two constant encoder dims: its hash
// key (a 5-D corner's row is the 3-D corner's row ^ key) and its weight factors on dims 3 and 4
struct GencCorner { uint32_t key; float w3, w4; };
__device__ __forceinline__ GencCorner genc_corner(const uint32_t (&g)[2], const float (&f)[2], uint32_t j) {
    const uint32_t b3 = j & 1, b4 = j >> 1;
    return {((g[0] + b3) * kPrime3) ^ ((g[1] + b4) * kPrime4), b3 ? f[0] : 1.0f - f[0], b4 ? f[1] : 1.0f - f[1]};
}

// the 8 corner (weight, row) pairs of a point on one level of the PRE-BLENDED 3-D table -- the corners the forward
// gather (encode_level in render_fused.cu) reads, for the table backward
struct Corners3 { float w[8]; uint32_t idx[8]; };
__device__ __forceinline__ Corners3 corners3(uint32_t mask, float scale, const float (&x)[3]) {
    float f[3];
    uint32_t g[3];
#pragma unroll
    for (int d = 0; d < 3; d++) grid_cell(x[d], scale, g[d], f[d]);
    Corners3 c;
#pragma unroll
    for (int i = 0; i < 8; i++) c.idx[i] = corner3(mask, g, f, i, c.w[i]);
    return c;
}

// record of a sky training forward (slot = tile * 128 + row over ALL tiles of the frame) and workspace of its backward
struct SkyRecordLayout { size_t x0, act, mask, total; };
static inline size_t rf_align_up(size_t v) { return (v + 255) / 256 * 256; }
static inline SkyRecordLayout sky_record_layout(long long n_tiles) {
    const size_t cap = (size_t)n_tiles * kRows;
    SkyRecordLayout r{};
    size_t o = 0;
    r.x0 = o; o = rf_align_up(o + cap * kSkyK0 * 2);
    r.act = o; o = rf_align_up(o + (size_t)Net<kSky>::NACT * cap * kActCols * 2);
    r.mask = o; o = rf_align_up(o + (size_t)n_tiles * kNumAct * kRows * 8 * 4);
    r.total = o;
    return r;
}
struct SkyBwdLayout { size_t dc16, dz, total; };
static inline SkyBwdLayout sky_bwd_layout(long long n_tiles) {
    const size_t cap = (size_t)n_tiles * kRows;
    SkyBwdLayout b{};
    size_t o = 0;
    b.dc16 = o; o = rf_align_up(o + cap * kOutC * 2);
    b.dz = o; o = rf_align_up(o + (size_t)Net<kSky>::NACT * cap * kHidden * 2);
    b.total = o;
    return b;
}

// launchers implemented in render_fused.cu, used by render_train.cu
int launch_train_forward(const Params &p, int precision, int grid, cudaStream_t st);     // mlp_kernel<fp16 x1 | x3, table3, kRender, TRAIN>
int launch_bwd_chain(const Params &p, int grid, cudaStream_t st);         // mlp_kernel<bf16x3, -, kBwd>
int launch_sky_train_forward(const Params &p, int grid, cudaStream_t st); // mlp_kernel<fp16x3, -, kSky, TRAIN>
int launch_sky_bwd_chain(const Params &p, int grid, cudaStream_t st);     // mlp_kernel<bf16x3, -, kSkyBwd>
int launch_prepass(const Params &p, int32_t *ws, cudaStream_t st);        // zeroes the counter, fills tile list (+ tile_work)
int launch_train_prepass(const Params &p, int32_t *hdr, int32_t *tile_list, cudaStream_t st);   // live tiles grouped by image
int params_from_abi(const sdb_render_params *sp, Params &p);        // validate + translate the ABI struct
extern int32_t *g_debug_buffer;

}  // namespace rf
