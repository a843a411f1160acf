// Shared definitions of the fused render engine (render_fused.cu) and the training-side kernels
// (render_train.cu): network shapes, the static weight-ring schedule, the shared-memory map, kernel
// parameters, ray sampling and hash-grid corner math.  Internal to libsdb200 (not part of the ABI).
#pragma once
#include <math.h>

#include "common.cuh"
#include "tc05.cuh"

namespace rf {

constexpr int kRows = 128, kTileW = 16, kTileH = 8;
constexpr int kHidden = 256, kFeat = 128, kOutC = 64, kLevels = 16;
constexpr int kKExt = 16;                       // extra K columns: labels / bias
constexpr int kKH = kHidden + kKExt;            // 272: K of every forward layer fed by hidden activations
constexpr int kMaxM = 8, kMaxS = 64, kMaxLabels = 15;
constexpr int kEpiThreads = 256, kGatherThreads = 256;
// warpgroup-aligned roles so that setmaxnreg can move registers from the control group to the gather group:
//   WG0-1 epilogue (warps 0-7), WG2 MMA + weight loads (warps 8-11), WG3-4 gather (12-19)
constexpr int kMmaWarp0 = 8, kGatherWarp0 = 12;
constexpr int kThreads = kEpiThreads + 128 + kGatherThreads;   // 640
// setmaxnreg can only redistribute the registers the CTA was LAUNCHED with (640 threads x 96 = 61,440; the
// allocator is a per-CTA pool -- USETMAXREG.TRY_ALLOC.CTAPOOL spins forever otherwise):
//   8 epilogue warps x 96 + 4 control warps x 48 + 8 gather warps x 120 = 61,440
constexpr int kRegsLaunch = 96, kRegsCtl = 48, kRegsGather = 120;
static_assert(8 * 32 * kRegsLaunch + 4 * 32 * kRegsCtl + 8 * 32 * kRegsGather <= kThreads * kRegsLaunch,
              "setmaxnreg budget exceeds the CTA's launch-time register allocation");
constexpr int kRingBytes = 65536;
constexpr uint32_t kLboA = kRows * 16, kSbo = 128;
constexpr int kHChunks = kKH / 8;               // 34 16-byte k-chunks per row
constexpr int kHBytes = kHChunks * kRows * 16;  // 69,632 bytes per operand part
constexpr int kSkyK0 = 48;                      // PE(raydir) 33 + zeros + bias column 47
constexpr int kRenderK0 = kFeat + kKExt;        // 144

// Networks the tensor-core engine runs (MODE):
//   kRender: LightningMLP forward, 6 hidden layers + colour head (layers.py:92-126)
//   kSky   : SKYMLP forward, 5 hidden layers + colour head (gancraft_base.py:150-169)
//   kBwd   : data-gradient chain of LightningMLP: dC -> dA6 -> ... -> dA1 -> d(features); the B operands are
//            the TRANSPOSED forward weights, there is no K extension (biases do not enter the data gradient)
//   kSkyBwd: data-gradient chain of SKYMLP: dSky -> dA5 -> ... -> dA1 (the PE input needs no gradient), so there are
//            4 operand-producing layers and the last layer's output (dA1 -> dZ1, N = 256) only goes to the record
constexpr int kRender = 0, kSky = 1, kBwd = 2, kSkyBwd = 3;
template <int MODE> struct Net {
    static constexpr bool ISBWD = MODE == kBwd || MODE == kSkyBwd;
    static constexpr int NH = MODE == kSky ? 5 : (MODE == kSkyBwd ? 4 : 6);   // layers whose epilogue feeds the next layer
    static constexpr int NL = NH + 1;
    static constexpr int K0 = MODE == kSky ? kSkyK0 : (ISBWD ? kOutC : kRenderK0);
    static constexpr bool EXT = !ISBWD;                     // hidden operands carry the 16-column K extension
    static constexpr int KH = EXT ? kKH : kHidden;          // K of the layers fed by hidden activations
    static constexpr int NOUT = MODE == kBwd ? kFeat : (MODE == kSkyBwd ? kHidden : kOutC);   // N of the last layer
    static constexpr int NACT = MODE == kSky || MODE == kSkyBwd ? 5 : 6;   // hidden activations of the forward network
    static constexpr bool TAIL = MODE == kRender || MODE == kBwd;          // the pack ends with the fp32 sigma head
};
template <int MODE> __host__ __device__ constexpr int layerK(int l) { return l == 0 ? Net<MODE>::K0 : Net<MODE>::KH; }
template <int MODE> __host__ __device__ constexpr int layerN(int l) { return l == Net<MODE>::NL - 1 ? Net<MODE>::NOUT : kHidden; }
template <int MODE> __host__ __device__ constexpr int64_t layerOff(int l, int parts) {
    int64_t o = 0;
    for (int j = 0; j < l; j++) o += (int64_t)layerK<MODE>(j) * layerN<MODE>(j) * 2 * parts;
    return o;
}
// fp32 tail of the render / backward packs: sigma head
constexpr int kFWsig = 0, kFBsig = 256, kFTotal = 264;
template <int MODE> __host__ __device__ constexpr int64_t packBytes(int parts) {
    return layerOff<MODE>(Net<MODE>::NL, parts) + (Net<MODE>::TAIL ? (int64_t)kFTotal * 4 : 0);
}
// Weight-ring schedule.  A ring stage holds KS consecutive k16 slabs (KS = 1 for the x3 modes, 2 for the
// single-pass mode so that a stage is 16 KB either way).  Layers fed by hidden activations consume the K
// extension first (no dependency; forward networks only), then the 32-column chunks in the order the two
// epilogue halves produce them.  Loader and MMA issuer walk the same list.
template <int KS, int MODE> __host__ __device__ constexpr int num_stages(int l) {
    return l == 0 ? (Net<MODE>::K0 / 16 + KS - 1) / KS : (Net<MODE>::EXT ? 1 : 0) + 16 / KS;   // [extension +] 8 chunks x (2 / KS)
}
// The epilogue hands the next layer's operand over in 16-column pieces = one k16 slab each: slabs 0..7 come from the
// epilogue half that owns columns 0..127, slabs 8..15 from the other half, both halves advance together.  Consumption
// order: KS = 1 (x3 modes, one slab per ring stage): 0,8,1,9,...,7,15; KS = 2 (single-pass mode, two slabs per stage):
// (0,1),(8,9),(2,3),(10,11),...
template <int KS> __host__ __device__ constexpr int hidden_stage_slab(int i) {
    return KS == 1 ? (i >> 1) + (i & 1) * 8 : ((i >> 1) * 2 + (i & 1) * 8);
}
template <int KS, int MODE> __host__ __device__ constexpr int stage_kk(int l, int j) {
    if (l == 0) return j * KS;
    if (Net<MODE>::EXT && j == 0) return 16;
    return hidden_stage_slab<KS>(j - (Net<MODE>::EXT ? 1 : 0));
}
template <int KS, int MODE> __host__ __device__ constexpr int stage_cnt(int l, int j) {
    if (l == 0) { const int nk = Net<MODE>::K0 / 16; return (j * KS + KS <= nk) ? KS : nk - j * KS; }
    return (Net<MODE>::EXT && j == 0) ? 1 : KS;
}
// slab barrier to wait on before stage j of a hidden-fed layer (-1: none): the LAST slab of the stage (a half's threads
// arrive on its slab barriers in order, so that one implies the earlier ones)
template <int KS, int MODE> __host__ __device__ constexpr int stage_chunk_wait(int l, int j) {
    if (l == 0 || (Net<MODE>::EXT && j == 0)) return -1;
    return hidden_stage_slab<KS>(j - (Net<MODE>::EXT ? 1 : 0)) + KS - 1;
}

// Static schedule: the number of ring stages per sample step is padded to a multiple of the ring depth (4),
// so the ring slot of every stage is a compile-time constant and its mbarrier parity depends only on the
// step parity -- the issue loops become straight-line code with immediate addresses.
template <int KS, int MODE> __host__ __device__ constexpr int stage_index(int l, int j) {
    int i = j;
    for (int k = 0; k < l; k++) i += num_stages<KS, MODE>(k);
    return i;
}
template <int KS, int MODE> __host__ __device__ constexpr int stages_per_step() { return stage_index<KS, MODE>(Net<MODE>::NL, 0); }
template <int KS, int MODE> __host__ __device__ constexpr int stages_per_step_padded() { return (stages_per_step<KS, MODE>() + 3) / 4 * 4; }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}\n" : "=r"(pred));
    return pred != 0;
}

// ---- shared memory map ---------------------------------------------------------------------------
struct Smem {
    uint32_t h_hi, h_lo, ring, fsec, scales, frac, sig, state, bars, stop, sched, total;
};
__host__ __device__ constexpr Smem smem_map(bool x3) {
    Smem m{};
    uint32_t o = 0;
    m.h_hi = o; o += kHBytes;
    m.h_lo = o; if (x3) o += kHBytes;
    m.ring = o; o += kRingBytes;
    m.fsec = o; o += kFTotal * 4;
    m.scales = o; o += kLevels * 4;
    m.frac = o; o += ((kMaxS + 1) * 4 + 15) / 16 * 16;
    m.sig = o; o += 2 * kRows * 4;
    m.state = o; o += 2 * (2 * kMaxM + 6) * kRows * 4;
    m.bars = o; o += 40 * 8;
    m.stop = o; o += 16;                         // early termination: int stop_step[2] (per tile buffer), int vote[2]
    m.sched = o; o += 32;                        // dynamic tile scheduler: int work[4] (ring), int published
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

// barrier indices
enum { B_WFULL = 0, B_WEMPTY = 4, B_FEAT = 8, B_HFREE, B_CHUNK, B_ACC = B_CHUNK + 16, B_OUTRDY, B_EPIDONE,
       B_STRDY = B_EPIDONE + 2, B_STFREE = B_STRDY + 2, B_COMP = B_STFREE + 2, B_COUNT = B_COMP + 1 };
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
    float *acc;                    // [grid][2][128][256] fp32 accumulator buffers, set by the launcher
};

// NV consecutive fp32 accumulators of one row (written by the MMA warpgroup of the same CTA: plain loads, not the
// non-coherent path)
// SDB_AB_NO_ACC (diagnostics build only, results are wrong): the accumulator buffer is neither written nor read, so that
// the kernel time with and without that traffic can be compared on the same work (bench.py --no-early-stop).
template <int NV>
__device__ __forceinline__ void acc_ld(const float *src, float (&v)[NV]) {
#ifdef SDB_AB_NO_ACC
#pragma unroll
    for (int i = 0; i < NV; i++) v[i] = __int_as_float((int)(reinterpret_cast<uintptr_t>(src) & 1));   // 0.0f, not a constant
    return;
#endif
#pragma unroll
    for (int i = 0; i < NV; i += 4) {
        const float4 a = *reinterpret_cast<const float4 *>(src + i);
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
//   slot 0 MMA warpgroup: the layer's inputs are ready (buffer free, operand written)   1 MMA warpgroup: the layer's accumulators are written
//   slot 2/4 epilogue half 0/1: accumulator of the layer complete          3/5 epilogue half 0/1: last slab handed over
//   layer row 7 = the gather role preparing step n: 0 compositing of step n-2 seen, 1 slots refilled, 2 features gathered, 3 operand buffer free
constexpr int32_t kTraceMagic = 0x7131;
constexpr int kTraceSteps = 6;
#ifndef SDB_TIMELINE
#define SDB_STAMP(n_, layer, slot) do { } while (0)      // compiled out: the stamps cost the epilogue role registers (spills)
#else
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

// cell + interpolation fractions of a point on one level of the PRE-BLENDED 3-D table, and the 8 corner
// (weight, row) pairs -- the arithmetic of encode_level<false> in render_fused.cu, shared with the table backward
struct Corners3 { float w[8]; uint32_t idx[8]; };
__device__ __forceinline__ Corners3 corners3(uint32_t mask, float scale, const float (&x)[3]) {
    float f[3];
    uint32_t g[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        const float pos = fmaf(x[d], scale, 0.5f);
        const float fl = floorf(pos);
        g[d] = (uint32_t)fl;
        f[d] = pos - (float)g[d];
    }
    const uint32_t h0[2] = {g[0], g[0] + 1u};
    const uint32_t h1[2] = {g[1] * kPrime1, (g[1] + 1u) * kPrime1};
    const uint32_t h2[2] = {g[2] * kPrime2, (g[2] + 1u) * kPrime2};
    Corners3 c;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int b0 = i & 1, b1 = (i >> 1) & 1, b2 = (i >> 2) & 1;
        float w = b0 ? f[0] : 1.0f - f[0];
        w *= b1 ? f[1] : 1.0f - f[1];
        w *= b2 ? f[2] : 1.0f - f[2];
        c.w[i] = w;
        c.idx[i] = (h0[b0] ^ h1[b1] ^ h2[b2]) & mask;
    }
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
int launch_train_forward(const Params &p, int grid, cudaStream_t st);     // mlp_kernel<fp16x3, table3, kRender, TRAIN>
int launch_bwd_chain(const Params &p, int grid, cudaStream_t st);         // mlp_kernel<bf16x3, -, kBwd>
int launch_sky_train_forward(const Params &p, int grid, cudaStream_t st); // mlp_kernel<fp16x3, -, kSky, TRAIN>
int launch_sky_bwd_chain(const Params &p, int grid, cudaStream_t st);     // mlp_kernel<bf16x3, -, kSkyBwd>
int launch_prepass(const Params &p, int32_t *ws, cudaStream_t st);        // zeroes the counter, fills tile list (+ tile_work)
int params_from_abi(const sdb_render_params *sp, Params &p);        // validate + translate the ABI struct
extern int32_t *g_debug_buffer;

}  // namespace rf
