// RenderCNN + tanh on the Hopper tensor cores (sm_90a, wgmma): the step right after the per-pixel path.
// Behavioural contract: imaginaire/generators/gancraft_base.py:172-225 (RenderCNN.forward: conv1 1x1 64->256, two residual
// blocks of two 3x3 convolutions with a style-dependent affine modulation, a residual block of two 1x1 convolutions, conv4
// 1x1 256->3; LeakyReLU 0.2 throughout) and :588-603 (`_forward_global`: NHWC -> NCHW, denoiser, tanh).
//
// The reference runs it per 158x158 tile because the unfused per-pixel stage cannot hold a frame (scenedreamer.py:600-628);
// its receptive radius is 4 px < pad/2, so evaluating it ONCE on the whole padded frame is the same function of the same
// pixels (DESIGN.md section 1, "Tiling equivalence").  Every layer is one launch of ONE implicit-GEMM kernel:
//
//   * activations live in HBM as fp16 hi/lo planes in the operand layout  [plane][row + 1][8-channel chunk][x + 1][8]
//     (16 B per pixel and chunk, a zero border of one pixel): a 128-pixel row segment of one chunk WITH its halo is one
//     contiguous 2080-byte range, fetched by one 1-D bulk copy (TMA engine) straight into the K-major, no-swizzle
//     canonical layout of a wgmma operand (rows = pixels, 16 B apart).  A tap (dy, dx) of a 3x3 convolution is the same
//     shared-memory buffer read through another row buffer (dy) and a start address shifted by dx * 16 bytes
//     (operand form checked by sdb_tc_selftest variant 2) -- no im2col, nothing is gathered;
//   * a CTA owns a tile of 2 image rows x 128 pixels; warpgroup o keeps the fp32 accumulators of row o in registers,
//     [128 pixels x 128 channels] per pass, two passes per tile.  Every 16 KB weight stage (one tap x 32 input channels x
//     one fp16 plane, streamed through a 4-stage ring from L2) feeds 8-16 MMAs of each warpgroup; input channels go by
//     in double-buffered slabs of 32 (4 row buffers x 4 chunks x hi/lo = 65 KB);
//   * fp32-grade arithmetic: fp16 hi/lo split of activations and weights, 3 MMAs per product, fp32 accumulation
//     (precision 2, the parity mode, like the per-pixel MLP) or one fp16 pass (precision 0 -- the class of the reference's
//     own default, cuDNN TF32 convolutions);
//   * epilogue on the accumulator fragments (two channels of a pixel per element pair): bias / residual + style
//     modulation / LeakyReLU, split, 4-byte stores; the last layer folds conv4 (256 -> 3) and tanh in.
// Roles: warps 0-7 MMA + epilogue (two warpgroups), warp 8 activation loader, warp 9 weight loader.
// Bound: tensor pipe (5.0 MFLOP per pixel; the activations make one HBM round trip per layer: 0.3 GB of 1.2 TFLOP).
#include "common.cuh"
#include "tc05.cuh"

namespace cnn {

constexpr int kCh = 256;                       // hidden channels
constexpr int kInCh = 64;                      // per-pixel feature channels (final_feat_dim)
constexpr int kSeg = 128;                      // pixels per row segment = M of one MMA
constexpr int kSegH = kSeg + 2;                // with the one-pixel halo
constexpr int kTileRows = 2;                   // image rows per tile (two accumulators)
constexpr uint32_t kChunkRow = kSegH * 16;     // 2080 B: one 8-channel chunk of one haloed row segment
constexpr int kSlabChunks = 4;                 // 32 input channels per slab
constexpr uint32_t kWStage = 256 * 32 * 2;     // 16 KB: [4 chunks][256 out][8] fp16 of one (slab, tap, plane)
constexpr int kWStages = 4;
constexpr int kThreads = 320;
constexpr int kPasses = 2;                     // output-channel halves per tile (accumulator registers)

enum { EPI_BIAS_LRELU = 0, EPI_RES_MOD_LRELU = 1, EPI_RES_BIAS_LRELU_RGB = 2 };

struct LayerParams {
    const uint8_t *in;         // activation tensor, `planes` planes of [Hp][in_chunks][Wp][16 B]
    const uint8_t *res;        // residual input (256 channels) or nullptr
    uint8_t *out;              // output activation tensor (256 channels) or nullptr (last layer)
    const uint8_t *wpack;      // [slab][tap][plane][4][256][8] fp16
    const float *bias;         // [256] or nullptr
    const float *mod_w, *mod_b;   // [256] each (EPI_RES_MOD_LRELU)
    const float *w4, *b4;      // [3][256], [3] (EPI_RES_BIAS_LRELU_RGB)
    float *rgb, *rgb_raw;      // [3][H][W] tanh(.) and pre-tanh (last layer; rgb_raw may be nullptr)
    int H, W, Hp, Wp;
    int in_chunks;             // 8 (conv1) or 32
    int taps;                  // 1 or 9
    int planes;                // 1 (fp16 x1) or 2 (fp16 x3)
    int epi;
    int tiles_x, tiles_y;
};

__host__ __device__ inline size_t plane_bytes(int Hp, int chunks, int Wp) { return (size_t)Hp * chunks * Wp * 16; }

__device__ __forceinline__ float lrelu(float v) { return v > 0.0f ? v : 0.2f * v; }

// 16-bit hi/lo split of 8 consecutive channels (fp16, or bf16 for the training path)
template <bool BF16>
__device__ __forceinline__ void split8(const float (&v)[8], uint4 &hi, uint4 &lo) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        h[i] = tc05::pack2<BF16>(v[2 * i], v[2 * i + 1]);
        const float2 back = tc05::unpack2<BF16>(h[i]);
        l[i] = tc05::pack2<BF16>(v[2 * i] - back.x, v[2 * i + 1] - back.y);
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

template <bool BF16>
__device__ __forceinline__ void unpack8(uint4 u, float (&v)[8]) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const float2 f = tc05::unpack2<BF16>(w[i]);
        v[2 * i] = f.x;
        v[2 * i + 1] = f.y;
    }
}

struct Smem {
    uint32_t slab[2], wring, bars, consts, total;
    uint32_t slab_bytes;
};
__host__ __device__ inline Smem smem_map(int taps, int planes) {
    Smem m{};
    const int rows_in = taps == 9 ? 4 : 2;
    m.slab_bytes = (uint32_t)rows_in * planes * kSlabChunks * kChunkRow;
    uint32_t o = 0;
    m.slab[0] = o; o += (m.slab_bytes + 1023u) & ~1023u;
    m.slab[1] = o; o += (m.slab_bytes + 1023u) & ~1023u;
    m.wring = o; o += kWStages * kWStage;
    m.consts = o; o += 6 * kCh * 4 + 64;            // bias | mod_w | mod_b | w4[3][256] | b4
    m.bars = o; o += 16 * 8;
    m.total = o;
    return m;
}
enum { B_SLAB_FULL = 0, B_SLAB_EMPTY = 2, B_W_FULL = 4, B_W_EMPTY = 8 };

// 16-bit split of a channel pair: hi at `dst`, and (X3) lo = v - hi one plane further
template <bool X3, bool BF16>
__device__ __forceinline__ void store_split2(uint8_t *dst, size_t plane, float v0, float v1) {
    const uint32_t hi = tc05::pack2<BF16>(v0, v1);
    *reinterpret_cast<uint32_t *>(dst) = hi;
    if (X3) {
        const float2 back = tc05::unpack2<BF16>(hi);
        *reinterpret_cast<uint32_t *>(dst + plane) = tc05::pack2<BF16>(v0 - back.x, v1 - back.y);
    }
}
// hi + lo (X3) of the channel pair at `src`
template <bool X3, bool BF16>
__device__ __forceinline__ float2 load_pair(const uint8_t *src, size_t plane) {
    float2 r = tc05::unpack2<BF16>(*reinterpret_cast<const uint32_t *>(src));
    if (X3) {
        const float2 l = tc05::unpack2<BF16>(*reinterpret_cast<const uint32_t *>(src + plane));
        r.x += l.x;
        r.y += l.y;
    }
    return r;
}

__device__ __forceinline__ void init_barriers(uint64_t *bars) {
    // the two epilogue warpgroups both read every slab and weight stage: one arrival each frees it
    for (int i = 0; i < 2; i++) { tc05::mbar_init(&bars[B_SLAB_FULL + i], 1); tc05::mbar_init(&bars[B_SLAB_EMPTY + i], 2); }
    for (int i = 0; i < kWStages; i++) { tc05::mbar_init(&bars[B_W_FULL + i], 1); tc05::mbar_init(&bars[B_W_EMPTY + i], 2); }
    tc05::fence_mbar_init();
}

// Every tile is computed in kPasses passes over the input channels, one per 128-wide half of the output channels
// (accumulators of a [128 pixel x 128 channel] half: 128 registers per thread of a warpgroup).
// ---------------- activation loader (warp 8): one slab = rows_in rows x P planes x 4 chunks, 2080 B each ----------------
template <bool X3>
__device__ __forceinline__ void load_slabs(const LayerParams &p, uint8_t *smem, const Smem &sm, uint64_t *bars, int lane,
                                           int n_slabs, int n_tiles, int rows_in, int row_base, size_t in_plane) {
    constexpr int P = X3 ? 2 : 1;
    uint32_t cnt = 0;
    const int n_copies = rows_in * P * kSlabChunks;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int y0 = (tile / p.tiles_x) * kTileRows, x0 = (tile % p.tiles_x) * kSeg;
        for (int pass = 0; pass < kPasses; pass++) {
            for (int s = 0; s < n_slabs; s++, cnt++) {
                const uint32_t buf = cnt & 1u, use = cnt >> 1;
                if (use > 0) tc05::mbar_wait_backoff(&bars[B_SLAB_EMPTY + buf], (use - 1) & 1u, 64);
                if (lane == 0) tc05::mbar_arrive_expect_tx(&bars[B_SLAB_FULL + buf], (uint32_t)n_copies * kChunkRow);
                __syncwarp();
                for (int i = lane; i < n_copies; i += 32) {
                    const int c = i % kSlabChunks, pl = (i / kSlabChunks) % P, r = i / (kSlabChunks * P);
                    const uint8_t *src = p.in + (size_t)pl * in_plane +
                                         (((size_t)(y0 + row_base + r) * p.in_chunks + s * kSlabChunks + c) * p.Wp + x0) * 16;
                    tc05::bulk_g2s(smem + sm.slab[buf] + (uint32_t)i * kChunkRow, src, kChunkRow, &bars[B_SLAB_FULL + buf]);
                }
            }
        }
    }
}

// ---------------- weight loader (warp 9): 16 KB stages in (slab, tap, plane) order, the same for every tile and pass ----------------
template <bool X3>
__device__ __forceinline__ void load_weights(const LayerParams &p, uint8_t *smem, const Smem &sm, uint64_t *bars, int lane,
                                             int n_slabs, int n_tiles, int taps) {
    constexpr int P = X3 ? 2 : 1;
    if (lane == 0) {
        uint32_t cnt = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            const int n_stages = n_slabs * taps * P;
            for (int pass = 0; pass < kPasses; pass++) {
                for (int g = 0; g < n_stages; g++, cnt++) {
                    const uint32_t st = cnt % kWStages, use = cnt / kWStages;
                    if (use > 0) tc05::mbar_wait_backoff(&bars[B_W_EMPTY + st], (use - 1) & 1u, 32);
                    tc05::mbar_arrive_expect_tx(&bars[B_W_FULL + st], kWStage);
                    tc05::bulk_g2s(smem + sm.wring + st * kWStage, p.wpack + (size_t)g * kWStage, kWStage, &bars[B_W_FULL + st]);
                }
            }
        }
    }
}

// ---------------- MMA main loop of one pass: warpgroup o (thread t of it) accumulates image row y0 + o ----------------
// acc[rb][nh]: pixels 64 rb .., output channels 128 pass + 64 nh ..
template <bool X3, bool BF16>
__device__ __forceinline__ void mma_pass(float (&acc)[2][2][32], const LayerParams &p, uint8_t *smem, const Smem &sm, uint64_t *bars,
                                         int o, int t, int pass, int taps, int n_slabs, uint32_t &scnt, uint32_t &wcnt) {
    constexpr int P = X3 ? 2 : 1;
#pragma unroll
    for (int i = 0; i < 128; i++) (&acc[0][0][0])[i] = 0.0f;
    for (int s = 0; s < n_slabs; s++, scnt++) {
        const uint32_t buf = scnt & 1u;
        tc05::mbar_wait(&bars[B_SLAB_FULL + buf], (scnt >> 1) & 1u);
        const uint32_t slab = tc05::smem_u32(smem + sm.slab[buf]);
        for (int tp = 0; tp < taps; tp++) {
            const int dy = taps == 9 ? tp / 3 : 0, dx = taps == 9 ? tp % 3 : 1;
#pragma unroll
            for (int pw = 0; pw < P; pw++, wcnt++) {
                const uint32_t st = wcnt % kWStages;
                tc05::mbar_wait(&bars[B_W_FULL + st], (wcnt / kWStages) & 1u);
                const uint32_t wbase = tc05::smem_u32(smem + sm.wring + st * kWStage) + (uint32_t)pass * 128u * 16u;
                // products with this weight plane: W_hi meets A_hi and (x3) A_lo; W_lo meets A_hi only
                const int n_pa = (X3 && pw == 0) ? 2 : 1;
                tc05::wgmma_fence();
                for (int pa = 0; pa < n_pa; pa++) {
#pragma unroll
                    for (int k16 = 0; k16 < 2; k16++) {
                        const uint32_t a_addr = slab + (uint32_t)(((o + dy) * P + pa) * kSlabChunks + 2 * k16) * kChunkRow + dx * 16;
#pragma unroll
                        for (int rb = 0; rb < 2; rb++) {
                            const uint64_t da = tc05::make_smem_desc(a_addr + rb * 1024u, kChunkRow, 128);
#pragma unroll
                            for (int nh = 0; nh < 2; nh++) {
                                const uint64_t db = tc05::make_smem_desc(wbase + (uint32_t)(2 * k16) * 4096u + nh * 1024u, 4096u, 128);
                                tc05::wgmma_m64n64k16<BF16, 0, 0>(acc[rb][nh], da, db, 1u);
                            }
                        }
                    }
                }
                tc05::wgmma_commit();
                tc05::wgmma_wait<0>();
#pragma unroll
                for (int rb = 0; rb < 2; rb++)
#pragma unroll
                    for (int nh = 0; nh < 2; nh++) tc05::wgmma_fence_acc(acc[rb][nh]);
                tc05::named_sync(1 + o, 128);
                if (t == 0) tc05::mbar_arrive(&bars[B_W_EMPTY + st]);
            }
        }
        if (t == 0) tc05::mbar_arrive(&bars[B_SLAB_EMPTY + buf]);
    }
}

// Forward layer.  <X3, fp16, false>: inference (precisions 2 and 0).  REC: a training forward, which also records the
// pre-modulation sum u of a modulated layer in the planes right before its output (the record layout, RecLayout):
// <true, bf16> the bf16 x3 path, <false, fp16 / bf16> the one-pass paths of autocast.
template <bool X3, bool BF16, bool REC>
__global__ void __launch_bounds__(kThreads, 1)
conv_kernel(const LayerParams p)
{
    constexpr int P = X3 ? 2 : 1;
    extern __shared__ __align__(1024) uint8_t smem[];
    const Smem sm = smem_map(p.taps, P);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + sm.bars);
    float *sBias = reinterpret_cast<float *>(smem + sm.consts);
    float *sModW = sBias + kCh, *sModB = sModW + kCh, *sW4 = sModB + kCh, *sB4 = sW4 + 3 * kCh;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int taps = p.taps, n_slabs = p.in_chunks / kSlabChunks;
    const int rows_in = taps == 9 ? 4 : 2, row_base = taps == 9 ? 0 : 1;
    const int n_tiles = p.tiles_x * p.tiles_y;

    for (int i = tid; i < kCh; i += kThreads) {
        sBias[i] = p.bias ? p.bias[i] : 0.0f;
        sModW[i] = p.mod_w ? p.mod_w[i] + 1.0f : 1.0f;          // modulate(): x * (w + 1) + b  (gancraft_base.py:196-199)
        sModB[i] = p.mod_b ? p.mod_b[i] : 0.0f;
    }
    if (p.w4) {
        for (int i = tid; i < 3 * kCh; i += kThreads) sW4[i] = p.w4[i];
        if (tid < 3) sB4[tid] = p.b4[tid];
    }
    if (tid == 0) init_barriers(bars);
    __syncthreads();
    const size_t in_plane = plane_bytes(p.Hp, p.in_chunks, p.Wp);

    if (warp == 8) {
        load_slabs<X3>(p, smem, sm, bars, lane, n_slabs, n_tiles, rows_in, row_base, in_plane);
    } else if (warp == 9) {
        load_weights<X3>(p, smem, sm, bars, lane, n_slabs, n_tiles, taps);
    } else {
        // ---------------- MMA + epilogue: warpgroup o = warps 4o .. 4o + 3 owns image row y0 + o ----------------
        const int o = warp >> 2, t = tid & 127;
        const size_t out_plane = plane_bytes(p.Hp, kCh / 8, p.Wp);
        uint32_t scnt = 0, wcnt = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            const int y = (tile / p.tiles_x) * kTileRows + o, x0 = (tile % p.tiles_x) * kSeg;
            // rgb partial sums of the 4 pixels this thread holds fragments of: [row block][+8][channel]
            float rgb[2][2][3];
#pragma unroll
            for (int i = 0; i < 12; i++) (&rgb[0][0][0])[i] = 0.0f;
#pragma unroll 1
            for (int pass = 0; pass < kPasses; pass++) {
                float acc[2][2][32];
                mma_pass<X3, BF16>(acc, p, smem, sm, bars, o, t, pass, taps, n_slabs, scnt, wcnt);
                // ---- epilogue of this channel half, on the accumulator fragments: element (pixel, c, c + 1) per pair ----
#pragma unroll
                for (int rb = 0; rb < 2; rb++) {
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const int px = rb * 64 + tc05::frag_row(t, 2 * h), x = x0 + px;
                        const bool valid = y < p.H && x < p.W;
                        const size_t pix = (((size_t)(y + 1) * (kCh / 8)) * p.Wp + (x + 1)) * 16;
#pragma unroll
                        for (int nh = 0; nh < 2; nh++) {
#pragma unroll
                            for (int j = 0; j < 8; j++) {
                                const int ch = pass * 128 + nh * 64 + tc05::frag_col(t, 4 * j);
                                float v0 = acc[rb][nh][4 * j + 2 * h], v1 = acc[rb][nh][4 * j + 2 * h + 1];
                                const size_t off = pix + (size_t)(ch >> 3) * p.Wp * 16 + (ch & 7) * 2;
                                if (p.epi != EPI_BIAS_LRELU) {
                                    const float2 r = load_pair<X3, BF16>(p.res + off, out_plane);
                                    v0 = r.x + v0;                                            // y + conv(...)
                                    v1 = r.y + v1;
                                }
                                if (p.epi == EPI_RES_MOD_LRELU) {
                                    if (REC && valid) store_split2<X3, BF16>(p.out - P * out_plane + off, out_plane, v0, v1);   // u: the record's planes before y
                                    v0 = lrelu(fmaf(v0, sModW[ch], sModB[ch]));
                                    v1 = lrelu(fmaf(v1, sModW[ch + 1], sModB[ch + 1]));
                                } else if (p.epi == EPI_RES_BIAS_LRELU_RGB) {
                                    v0 = lrelu(v0 + sBias[ch]);
                                    v1 = lrelu(v1 + sBias[ch + 1]);
#pragma unroll
                                    for (int k = 0; k < 3; k++)
                                        rgb[rb][h][k] = fmaf(v1, sW4[k * kCh + ch + 1], fmaf(v0, sW4[k * kCh + ch], rgb[rb][h][k]));
                                } else {
                                    v0 = lrelu(v0 + sBias[ch]);
                                    v1 = lrelu(v1 + sBias[ch + 1]);
                                }
                                if (p.out != nullptr && valid) store_split2<X3, BF16>(p.out + off, out_plane, v0, v1);
                            }
                        }
                    }
                }
            }
            if (p.epi == EPI_RES_BIAS_LRELU_RGB) {
                // the 4 threads of a quad hold the same pixels: sum their channel partials, one of them writes
#pragma unroll
                for (int rb = 0; rb < 2; rb++)
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const int x = x0 + rb * 64 + tc05::frag_row(t, 2 * h);
#pragma unroll
                        for (int k = 0; k < 3; k++) {
                            float v = rgb[rb][h][k];
                            v += __shfl_xor_sync(0xffffffffu, v, 1);
                            v += __shfl_xor_sync(0xffffffffu, v, 2);
                            if ((lane & 3) == 0 && y < p.H && x < p.W) {
                                const float raw = v + sB4[k];
                                const size_t idx = ((size_t)k * p.H + y) * p.W + x;
                                p.rgb[idx] = tanhf(raw);
                                if (p.rgb_raw) p.rgb_raw[idx] = raw;
                            }
                        }
                    }
            }
        }
    }
}

// ================================================ training (bf16 x3) ================================================
//
// Forward contract, per pixel, sigma = LeakyReLU(0.2), m0..m3 = the four 256-wide chunks of fc_z_cond(z):
//   p1  = conv1(x) + b1                 y1 = sigma(p1)
//   p2a = conv2a(y1) + b2a              t1 = sigma(p2a)
//   u2  = y1 + conv2b(t1)               y2 = sigma(u2 (1 + m0) + m1)
//   p3a = conv3a(y2) + b3a              t2 = sigma(p3a)
//   u3  = y2 + conv3b(t2)               y3 = sigma(u3 (1 + m2) + m3)
//   p4a = conv4a(y3) + b4a              t3 = sigma(p4a)
//   p4b = y3 + conv4b(t3) + b4b         y4 = sigma(p4b)
//   raw = conv4(y4) + b4                rgb = tanh(raw)
// The training forward is conv_kernel<true, bf16> over a RECORD that keeps every layer output (x, y1, t1, y2, t2, y3, t3,
// y4) and the pre-modulation sums u2, u3 in plane pairs of their own (u is stored, not recovered from y: dividing by 1 + m
// is ill-conditioned when m ~ -1), plus rgb.  bf16, not fp16: gradients of a mean loss fall below fp16's normal range,
// the weight-gradient GEMM needs both operands in one type, and a small positive activation must keep its sign.
//
// Backward, from G_rgb and/or G_raw: g_raw = G_raw + G_rgb (1 - rgb^2), then the chain in reverse.  sigma' is 1 or 0.2 by
// the sign of the stored output (nn.LeakyReLU(inplace=True) differentiates through its result); a residual sends its
// gradient to both branches; a modulation gives dm_odd = sum g_s, dm_even = sum g_s u, g_u = g_s (1 + m_even); a conv gives
// dW = sum_pix g (x) shifted input, db = sum_pix g and the data gradient, the transposed convolution (3x3: in / out channels
// swapped, taps flipped) -- the same engine as the forward (load_slabs / load_weights / mma_pass) with a backward pack:
//   head_bwd_kernel   tanh', conv4^T, sigma'(y4)                      -> g_p4b        (dW4, db4, db4b)
//   conv4b^T          sigma'(t3)                                      -> g_p4a        (db4a)
//   conv4a^T          + g_p4b, sigma'(y3), modulation (m2, m3)        -> g_u3         (dm3, dm2)
//   conv3b^T          sigma'(t2)                                      -> g_p3a        (db3a)
//   conv3a^T          + g_u3, sigma'(y2), modulation (m0, m1)         -> g_u2         (dm1, dm0)
//   conv2b^T          sigma'(t1)                                      -> g_p2a        (db2a)
//   conv2a^T          + g_u2, sigma'(y1)                              -> g_p1         (db1)
//   conv1^T           fp32 NHWC                                       -> dL/dnet_out
// and after each data step the weight gradient of that layer (conv_wgrad_kernel).  Gradients are bf16 hi/lo plane pairs
// in the activation layout, zero outside the frame.  Every product is bf16 x3 (hi hi + lo hi + hi lo), fp32 accumulation.
//
// One-pass training (X3 = false; precision 0 = fp16, 3 = bf16): the class of autocast's own convolutions.  The same record
// order and layout with ONE 16-bit plane per activation in the forward's type, single gradient planes in that type, one
// product per MMA step, fp32 accumulation and the same fp32 epilogue arithmetic everywhere.

// Backward of tanh, conv4 (256 -> 3) and the last LeakyReLU, per pixel; block (., c) owns 8-channel chunk c.  Each of the
// 32 chunk rows recomputes g_raw from G_rgb, G_raw and rgb (36 B per pixel): those planes are at most 20 MB at 570 x 990 and
// stay in L2, so the re-reads cost L2 bandwidth next to the 1 KB of y4 read and 1 KB of g_p4b written per pixel.
struct HeadParams {
    const uint8_t *y4;          // record planes of y4
    const float *rgb;           // record [3][H][W]
    const float *g_rgb, *g_raw; // [3][H][W] each, either may be nullptr
    const float *w4;            // [3][256]
    uint8_t *out;               // g_p4b planes
    float *dw4, *db4, *db4b;    // [3][256], [3], [256] (each may be nullptr)
    int H, W, Hp, Wp;
};

template <bool X3, bool BF16>
__global__ void __launch_bounds__(256)
head_bwd_kernel(const HeadParams h)
{
    __shared__ float red[8][35];
    const int c = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t plane = plane_bytes(h.Hp, kCh / 8, h.Wp);
    const long long HW = (long long)h.H * h.W;
    float w[3][8], part[35];                               // part: dW4 [3][8] | db4b [8] | db4 [3]
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
        for (int j = 0; j < 8; j++) w[k][j] = h.w4[k * kCh + 8 * c + j];
#pragma unroll
    for (int i = 0; i < 35; i++) part[i] = 0.0f;
    for (long long pix = blockIdx.x * 256LL + tid; pix < HW; pix += gridDim.x * 256LL) {
        const int y = (int)(pix / h.W), x = (int)(pix % h.W);
        float gr[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            float g = h.g_raw ? h.g_raw[k * HW + pix] : 0.0f;
            if (h.g_rgb) {
                const float r = h.rgb[k * HW + pix];
                g = fmaf(h.g_rgb[k * HW + pix], 1.0f - r * r, g);
            }
            gr[k] = g;
            part[32 + k] += g;
        }
        const size_t off = ((((size_t)(y + 1) * (kCh / 8)) + c) * h.Wp + (x + 1)) * 16;
        float yh[8], yl[8], g[8];
        unpack8<BF16>(*reinterpret_cast<const uint4 *>(h.y4 + off), yh);
        if (X3) unpack8<BF16>(*reinterpret_cast<const uint4 *>(h.y4 + plane + off), yl);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float gy = fmaf(w[2][j], gr[2], fmaf(w[1][j], gr[1], w[0][j] * gr[0]));
            g[j] = yh[j] > 0.0f ? gy : 0.2f * gy;
            part[24 + j] += g[j];
#pragma unroll
            for (int k = 0; k < 3; k++) part[8 * k + j] = fmaf(gr[k], X3 ? yh[j] + yl[j] : yh[j], part[8 * k + j]);
        }
        uint4 hi, lo;
        split8<BF16>(g, hi, lo);
        *reinterpret_cast<uint4 *>(h.out + off) = hi;
        if (X3) *reinterpret_cast<uint4 *>(h.out + plane + off) = lo;
    }
#pragma unroll
    for (int i = 0; i < 35; i++) {
        float v = part[i];
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
        if (lane == 0) red[warp][i] = v;
    }
    __syncthreads();
    if (tid < 35) {
        float v = 0.0f;
        for (int i = 0; i < 8; i++) v += red[i][tid];
        if (tid < 24) {
            if (h.dw4) atomicAdd(h.dw4 + (tid / 8) * kCh + 8 * c + tid % 8, v);
        } else if (tid < 32) {
            if (h.db4b) atomicAdd(h.db4b + 8 * c + tid - 24, v);
        } else if (c == 0 && h.db4) {
            atomicAdd(h.db4 + tid - 32, v);
        }
    }
}

// Data gradient of one conv layer: the forward engine over gradient planes with a backward pack, and the epilogue
//   v = (res + conv^T(in)) * sigma'(sign);  sum1 += v;  [modulated: sum2 += v u;  v *= 1 + m_even]  -> out planes / dx
struct BwdParams {
    LayerParams l;              // in: gradient planes; res: residual gradient planes or nullptr; out: output gradient planes;
                                // wpack: backward pack of the layer; mod_w: m_even of a modulated layer or nullptr
    const uint8_t *sign;        // record planes whose sign selects sigma' (nullptr: identity)
    const uint8_t *mod_u;       // record planes of u (modulated layers) or nullptr
    float *sum1, *sum2;         // [256] channel sums of v (bias gradient or dm_odd) and of v u (dm_even), or nullptr
    float *dx;                  // conv1^T: dL/dnet_out [H][W][64] fp32 instead of `out`
};

template <bool X3, bool BF16>
__global__ void __launch_bounds__(kThreads, 1)
conv_bwd_kernel(const BwdParams q)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    const LayerParams &p = q.l;
    const Smem sm = smem_map(p.taps, X3 ? 2 : 1);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + sm.bars);
    float *sScale = reinterpret_cast<float *>(smem + sm.consts), *sSum1 = sScale + kCh, *sSum2 = sSum1 + kCh;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int taps = p.taps, n_slabs = p.in_chunks / kSlabChunks;
    const int n_tiles = p.tiles_x * p.tiles_y;
    for (int i = tid; i < kCh; i += kThreads) {
        sScale[i] = p.mod_w ? p.mod_w[i] + 1.0f : 1.0f;
        sSum1[i] = 0.0f;
        sSum2[i] = 0.0f;
    }
    if (tid == 0) init_barriers(bars);
    __syncthreads();

    if (warp == 8) {
        load_slabs<X3>(p, smem, sm, bars, lane, n_slabs, n_tiles, taps == 9 ? 4 : 2, taps == 9 ? 0 : 1,
                       plane_bytes(p.Hp, p.in_chunks, p.Wp));
    } else if (warp == 9) {
        load_weights<X3>(p, smem, sm, bars, lane, n_slabs, n_tiles, taps);
    } else {
        const int o = warp >> 2, t = tid & 127;
        const size_t plane = plane_bytes(p.Hp, kCh / 8, p.Wp);
        uint32_t scnt = 0, wcnt = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            const int y = (tile / p.tiles_x) * kTileRows + o, x0 = (tile % p.tiles_x) * kSeg;
#pragma unroll 1
            for (int pass = 0; pass < kPasses; pass++) {
                float acc[2][2][32];
                mma_pass<X3, BF16>(acc, p, smem, sm, bars, o, t, pass, taps, n_slabs, scnt, wcnt);
#pragma unroll
                for (int nh = 0; nh < 2; nh++) {
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const int ch = pass * 128 + nh * 64 + tc05::frag_col(t, 4 * j);
                        float s1[2] = {0.0f, 0.0f}, s2[2] = {0.0f, 0.0f};
#pragma unroll
                        for (int rb = 0; rb < 2; rb++) {
#pragma unroll
                            for (int h = 0; h < 2; h++) {
                                const int x = x0 + rb * 64 + tc05::frag_row(t, 2 * h);
                                if (y >= p.H || x >= p.W) continue;
                                const size_t off = ((((size_t)(y + 1) * (kCh / 8)) + (ch >> 3)) * p.Wp + (x + 1)) * 16 + (ch & 7) * 2;
                                float v0 = acc[rb][nh][4 * j + 2 * h], v1 = acc[rb][nh][4 * j + 2 * h + 1];
                                if (p.res) {
                                    const float2 r = load_pair<X3, BF16>(p.res + off, plane);
                                    v0 += r.x;
                                    v1 += r.y;
                                }
                                if (q.sign) {
                                    const float2 sg = tc05::unpack2<BF16>(*reinterpret_cast<const uint32_t *>(q.sign + off));
                                    v0 = sg.x > 0.0f ? v0 : 0.2f * v0;
                                    v1 = sg.y > 0.0f ? v1 : 0.2f * v1;
                                }
                                s1[0] += v0;
                                s1[1] += v1;
                                if (q.mod_u) {
                                    const float2 u = load_pair<X3, BF16>(q.mod_u + off, plane);
                                    s2[0] = fmaf(v0, u.x, s2[0]);
                                    s2[1] = fmaf(v1, u.y, s2[1]);
                                    v0 *= sScale[ch];
                                    v1 *= sScale[ch + 1];
                                }
                                if (q.dx) {
                                    if (ch < kInCh) *reinterpret_cast<float2 *>(q.dx + ((size_t)y * p.W + x) * kInCh + ch) = make_float2(v0, v1);
                                } else {
                                    store_split2<X3, BF16>(p.out + off, plane, v0, v1);
                                }
                            }
                        }
                        if (q.sum1 || q.sum2) {
                            // lanes l, l ^ 4, .., l ^ 28 hold the same two channels (other pixels)
#pragma unroll
                            for (int m = 4; m < 32; m <<= 1)
#pragma unroll
                                for (int e = 0; e < 2; e++) {
                                    s1[e] += __shfl_xor_sync(0xffffffffu, s1[e], m);
                                    s2[e] += __shfl_xor_sync(0xffffffffu, s2[e], m);
                                }
                            if (lane < 4) {
                                atomicAdd(&sSum1[ch], s1[0]);
                                atomicAdd(&sSum1[ch + 1], s1[1]);
                                atomicAdd(&sSum2[ch], s2[0]);
                                atomicAdd(&sSum2[ch + 1], s2[1]);
                            }
                        }
                    }
                }
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < kCh; i += kThreads) {
        if (q.sum1) atomicAdd(q.sum1 + i, sSum1[i]);
        if (q.sum2) atomicAdd(q.sum2 + i, sSum2[i]);
    }
}

// Weight gradient of one conv layer, dW[n][ci][tap] = sum_pix g[pix][n] in[pix + tap offset][ci], on the tensor cores.
// Jobs are (tap, 128 output channels); pixels are the reduction dimension, in items of one 64-pixel row segment, split
// over CTAs.  Both operands are MN-major straight from the planes: one 8-channel chunk of an item is 64 pixels 16 B apart
// (K-adjacent core matrices +128 B, MN-adjacent chunks +1 KB); the tap's dx is a 16 B start shift of the input copy, its
// dy another input row.  fp32 accumulators [128 x cin] stay in two warpgroups' registers for the whole reduction and
// are added to the zeroed gradient with red.add.  Warp 8 issues the bulk copies into a ring of stages: two of 96 KB for
// bf16 x3 (plane pairs), four of 48 KB for one pass (single planes), whose one product per stage hides less of a copy.
constexpr int kWgSeg = 64;
constexpr uint32_t kWgChunk = kWgSeg * 16;               // 1 KB
constexpr int kWgThreads = 288;
template <bool X3> struct WgRing {
    static constexpr uint32_t P = X3 ? 2 : 1;
    static constexpr uint32_t GBytes = P * 16 * kWgChunk;    // gradient: P planes x 128 output channels
    static constexpr uint32_t XBytes = P * 32 * kWgChunk;    // input: P planes x up to 256 channels
    static constexpr uint32_t Stage = GBytes + XBytes;       // 96 KB (x3) or 48 KB
    static constexpr int LogStages = X3 ? 1 : 2;
    static constexpr int Stages = 1 << LogStages;
    static constexpr uint32_t Smem = Stages * Stage + 16 * Stages;
};

struct WgradParams {
    const uint8_t *g, *in;      // gradient planes (256 channels), input record planes (in_chunks chunks)
    float *dw;                  // [256][cin][taps] (PyTorch layout), zeroed
    int in_chunks, taps, H, Hp, Wp, segs, nsplit;
};

template <int NQ, bool X3, bool BF16>                    // NQ: 64-channel column blocks of the input: 1 (conv1) or 4
__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad_kernel(const WgradParams p)
{
    using R = WgRing<X3>;
    constexpr int S = R::Stages, LS = R::LogStages;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + S * R::Stage);      // full[S], empty[S]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int job = blockIdx.x / p.nsplit, split = blockIdx.x % p.nsplit;
    const int tap = job >> 1, n0 = (job & 1) * 128;
    const int dy = p.taps == 9 ? tap / 3 : 1, dx = p.taps == 9 ? tap % 3 : 1;
    const long long n_items = (long long)p.H * p.segs;
    const long long my_items = split < n_items ? (n_items - split + p.nsplit - 1) / p.nsplit : 0;
    if (tid == 0) {
        for (int s = 0; s < S; s++) { tc05::mbar_init(&bars[s], 1); tc05::mbar_init(&bars[S + s], 2); }
        tc05::fence_mbar_init();
    }
    __syncthreads();
    if (my_items == 0) return;
    if (warp == 8) {
        const size_t gplane = plane_bytes(p.Hp, kCh / 8, p.Wp), xplane = plane_bytes(p.Hp, p.in_chunks, p.Wp);
        const int n_gcopies = (int)R::P * 16, n_copies = n_gcopies + (int)R::P * p.in_chunks;
        for (long long n = 0; n < my_items; n++) {
            const int s = (int)(n & (S - 1));
            if (n >= S) tc05::mbar_wait_backoff(&bars[S + s], (uint32_t)(((n >> LS) - 1) & 1), 64);
            const long long item = split + n * p.nsplit;
            const int y = (int)(item / p.segs), x0 = (int)(item % p.segs) * kWgSeg;
            if (lane == 0) tc05::mbar_arrive_expect_tx(&bars[s], (uint32_t)n_copies * kWgChunk);
            __syncwarp();
            for (int i = lane; i < n_copies; i += 32) {
                const uint8_t *src;
                uint32_t dst;
                if (i < n_gcopies) {
                    const int pl = i >> 4, c = i & 15;
                    src = p.g + pl * gplane + ((((size_t)(y + 1) * (kCh / 8)) + (n0 >> 3) + c) * p.Wp + x0 + 1) * 16;
                    dst = (uint32_t)(pl * 16 + c) * kWgChunk;
                } else {
                    const int pl = (i - n_gcopies) / p.in_chunks, c = (i - n_gcopies) % p.in_chunks;
                    src = p.in + pl * xplane + ((((size_t)(y + dy) * p.in_chunks) + c) * p.Wp + x0 + dx) * 16;
                    dst = R::GBytes + (uint32_t)(pl * 32 + c) * kWgChunk;
                }
                tc05::bulk_g2s(smem + s * R::Stage + dst, src, kWgChunk, &bars[s]);
            }
        }
        return;
    }
    const int wg = warp >> 2, t = tid & 127;
    float acc[NQ][32];
#pragma unroll
    for (int i = 0; i < NQ * 32; i++) (&acc[0][0])[i] = 0.0f;
    for (long long n = 0; n < my_items; n++) {
        const int s = (int)(n & (S - 1));
        tc05::mbar_wait(&bars[s], (uint32_t)((n >> LS) & 1));
        const uint32_t sG = tc05::smem_u32(smem + s * R::Stage), sX = sG + R::GBytes;
        tc05::wgmma_fence();
#pragma unroll
        for (int pr = 0; pr < (X3 ? 3 : 1); pr++) {         // x3: g_hi in_hi, g_lo in_hi, g_hi in_lo
            const uint32_t ga = pr == 1 ? 1u : 0u, xb = pr == 2 ? 1u : 0u;
#pragma unroll 1
            for (int kk = 0; kk < kWgSeg / 16; kk++) {
                const uint64_t da = tc05::make_smem_desc(sG + (ga * 16 + wg * 8) * kWgChunk + kk * 256, 128, kWgChunk);
#pragma unroll
                for (int q = 0; q < NQ; q++)
                    tc05::wgmma_m64n64k16<BF16, 1, 1>(acc[q], da, tc05::make_smem_desc(sX + (xb * 32 + 8 * q) * kWgChunk + kk * 256, 128, kWgChunk), 1u);
            }
        }
        tc05::wgmma_commit();
        tc05::wgmma_wait<0>();
#pragma unroll
        for (int q = 0; q < NQ; q++) tc05::wgmma_fence_acc(acc[q]);
        tc05::named_sync(1 + wg, 128);
        if (t == 0) tc05::mbar_arrive(&bars[S + s]);
    }
    const int cin = p.in_chunks * 8;
#pragma unroll
    for (int q = 0; q < NQ; q++) {
#pragma unroll
        for (int i = 0; i < 32; i++) {
            const int n = n0 + wg * 64 + tc05::frag_row(t, i), ci = 64 * q + tc05::frag_col(t, i);
            atomicAdd(p.dw + ((size_t)n * cin + ci) * p.taps + tap, acc[q][i]);
        }
    }
}

// per-pixel features fp32 [H][W][64] (NHWC, the fused kernel's net_out) -> operand planes [P][Hp][8][Wp][8] (fp16 / bf16)
template <bool BF16>
__global__ void __launch_bounds__(256)
pack_input_kernel(const float *__restrict__ net_out, uint8_t *__restrict__ act, int H, int W, int Hp, int Wp, int planes)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long n = (long long)H * W * (kInCh / 8);
    if (i >= n) return;
    const int c = (int)(i % (kInCh / 8));
    const long long pix = i / (kInCh / 8);
    const int x = (int)(pix % W), y = (int)(pix / W);
    const float4 a = __ldg(reinterpret_cast<const float4 *>(net_out + pix * kInCh + c * 8));
    const float4 b = __ldg(reinterpret_cast<const float4 *>(net_out + pix * kInCh + c * 8) + 1);
    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint4 hi, lo;
    split8<BF16>(v, hi, lo);
    const size_t off = ((((size_t)(y + 1) * (kInCh / 8)) + c) * Wp + (x + 1)) * 16;
    *reinterpret_cast<uint4 *>(act + off) = hi;
    if (planes == 2) *reinterpret_cast<uint4 *>(act + plane_bytes(Hp, kInCh / 8, Wp) + off) = lo;
}

// conv weight fp32 [256][cin][taps] (PyTorch [out][in][kh][kw]) -> [slab][tap][plane][chunk 4][n 256][8] (fp16 / bf16).
// T: the data-gradient pack of a forward weight [cin][n_src][taps]: element (n, ci, t) = w[ci][n][taps - 1 - t] (in / out
// channels swapped, taps flipped), zero for n >= n_src (conv1^T has 64 real output channels of the engine's 256).
template <bool BF16, bool T>
__global__ void __launch_bounds__(256)
pack_weight_kernel(const float *__restrict__ w, uint8_t *__restrict__ pack, int cin, int taps, int planes, int n_src)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long n = (long long)kCh * cin * taps;
    if (i >= n) return;
    const int t = (int)(i % taps);
    const int ci = (int)((i / taps) % cin);
    const int no = (int)(i / ((long long)taps * cin));
    const float v = !T ? w[i] : no < n_src ? w[((size_t)ci * n_src + no) * taps + (taps - 1 - t)] : 0.0f;
    uint16_t hi, lo;
    if constexpr (BF16) {
        const __nv_bfloat16 h = __float2bfloat16_rn(v), l = __float2bfloat16_rn(v - __bfloat162float(h));
        hi = *reinterpret_cast<const uint16_t *>(&h);
        lo = *reinterpret_cast<const uint16_t *>(&l);
    } else {
        const __half h = __float2half_rn(v), l = __float2half_rn(v - __half2float(h));
        hi = *reinterpret_cast<const uint16_t *>(&h);
        lo = *reinterpret_cast<const uint16_t *>(&l);
    }
    const int s = ci / 32, c = (ci % 32) / 8, j = ci % 8;
    const size_t stage = ((size_t)s * taps + t) * planes;
    const size_t inner = ((size_t)c * 256 + no) * 8 + j;
    reinterpret_cast<uint16_t *>(pack + stage * kWStage)[inner] = hi;
    if (planes == 2) reinterpret_cast<uint16_t *>(pack + (stage + 1) * kWStage)[inner] = lo;
}

struct PackLayout { size_t w[7], f32, total; };
// fp32 tail: b1 | b2a | b3a | b4a | b4b | w4 [3][256] | b4 [3] (+pad)
constexpr int kF32Floats = 5 * kCh + 3 * kCh + 4;
constexpr int kTaps[7] = {1, 9, 9, 9, 9, 1, 1};          // conv1, conv2a, conv2b, conv3a, conv3b, conv4a, conv4b
static PackLayout pack_layout(int planes) {
    PackLayout l{};
    const int cin[7] = {kInCh, kCh, kCh, kCh, kCh, kCh, kCh};
    size_t o = 0;
    for (int i = 0; i < 7; i++) { l.w[i] = o; o += (size_t)(cin[i] / 32) * kTaps[i] * planes * kWStage; }
    l.f32 = o; o += (size_t)kF32Floats * 4;
    l.total = (o + 255) / 256 * 256;
    return l;
}
// data-gradient pack: the 7 transposed layers, 256 input channels each (conv1^T: 256 -> 64, padded to 256), in the
// training path's planes (2: bf16 x3, 1: one pass)
static PackLayout bwd_pack_layout(int planes) {
    PackLayout l{};
    size_t o = 0;
    for (int i = 0; i < 7; i++) { l.w[i] = o; o += (size_t)(kCh / 32) * kTaps[i] * planes * kWStage; }
    l.f32 = o;
    l.total = o;
    return l;
}

static void padded_dims(int H, int W, int &Hp, int &Wp) {
    Hp = H + 4;                                              // one zero row above, (up to) three below: tiles are 2 rows tall
    Wp = ((W + kSeg - 1) / kSeg) * kSeg + 2;
}

struct WsLayout { size_t a0, y, t, y2, total; };
static WsLayout ws_layout(int H, int W, int planes, int &Hp, int &Wp) {
    padded_dims(H, W, Hp, Wp);
    WsLayout l{};
    size_t o = 0;
    l.a0 = o; o += (plane_bytes(Hp, kInCh / 8, Wp) * planes + 255) / 256 * 256;
    const size_t big = (plane_bytes(Hp, kCh / 8, Wp) * planes + 255) / 256 * 256;
    l.y = o; o += big;
    l.t = o; o += big;
    l.y2 = o; o += big;
    l.total = o;
    return l;
}

// Training record of one view: `planes` 16-bit planes per activation (bf16 pairs for x3, one plane in the forward's type for
// one pass) with zero borders, each u directly before the y it modulates into (conv_kernel<., ., true> finds u at out -
// planes), then rgb [3][H][W] fp32.
struct RecLayout { size_t x, y1, t1, u2, y2, t2, u3, y3, t3, y4, rgb, total; };
static RecLayout rec_layout(int H, int W, int planes, int &Hp, int &Wp) {
    padded_dims(H, W, Hp, Wp);
    RecLayout l{};
    size_t o = 0;
    l.x = o; o += (plane_bytes(Hp, kInCh / 8, Wp) * planes + 255) / 256 * 256;
    const size_t big = plane_bytes(Hp, kCh / 8, Wp) * planes;     // a multiple of 512 B
    size_t *pairs[9] = {&l.y1, &l.t1, &l.u2, &l.y2, &l.t2, &l.u3, &l.y3, &l.t3, &l.y4};
    for (int i = 0; i < 9; i++) { *pairs[i] = o; o += big; }
    l.rgb = o; o += ((size_t)3 * H * W * 4 + 255) / 256 * 256;
    l.total = o;
    return l;
}

// Backward workspace: three gradient tensors of `planes` planes in rotation
static size_t bwd_ws_bytes(int H, int W, int planes, int &Hp, int &Wp) {
    padded_dims(H, W, Hp, Wp);
    return 3 * plane_bytes(Hp, kCh / 8, Wp) * planes;
}

// one forward layer table entry: byte offsets into the activation buffer (NONE = absent)
struct FwdLayer { size_t in, res, out; int in_chunks, epi; const float *bias, *mw, *mb; };
constexpr size_t NONE = (size_t)-1;

template <bool X3, bool BF16, bool REC>
static int launch_forward_layers(const FwdLayer (&layers)[7], uint8_t *buf, const uint8_t *pack, const PackLayout &pl,
                                 LayerParams base, float *d_rgb, float *d_rgb_raw, cudaStream_t st)
{
    const float *f = reinterpret_cast<const float *>(pack + pl.f32);
    const int n_tiles = base.tiles_x * base.tiles_y;
    const int grid = n_tiles < sdb_num_sms() ? n_tiles : sdb_num_sms();
    for (int i = 0; i < 7; i++) {
        LayerParams p = base;
        const FwdLayer &l = layers[i];
        p.in = buf + l.in;
        p.res = l.res == NONE ? nullptr : buf + l.res;
        p.out = l.out == NONE ? nullptr : buf + l.out;
        p.wpack = pack + pl.w[i];
        p.bias = l.bias; p.mod_w = l.mw; p.mod_b = l.mb;
        p.in_chunks = l.in_chunks; p.taps = kTaps[i]; p.epi = l.epi;
        if (l.epi == EPI_RES_BIAS_LRELU_RGB) { p.w4 = f + 5 * kCh; p.b4 = f + 8 * kCh; p.rgb = d_rgb; p.rgb_raw = d_rgb_raw; }
        const uint32_t smem = smem_map(p.taps, X3 ? 2 : 1).total;
        SDB_CUDA(cudaFuncSetAttribute(conv_kernel<X3, BF16, REC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        conv_kernel<X3, BF16, REC><<<grid, kThreads, smem, st>>>(p);
        SDB_CHECK_LAUNCH();
    }
    return SDB_OK;
}

static LayerParams frame_params(int H, int W, int Hp, int Wp, int planes) {
    LayerParams base{};
    base.H = H; base.W = W; base.Hp = Hp; base.Wp = Wp; base.planes = planes;
    base.tiles_x = (W + kSeg - 1) / kSeg; base.tiles_y = (H + kTileRows - 1) / kTileRows;
    return base;
}

// pack precisions: 0 = fp16 x1, 1 = bf16 x3, 2 = fp16 x3, 3 = bf16 x1 (the one-pass bf16 training path only)
static int pack_planes(int precision) { return precision == 0 || precision == 3 ? 1 : 2; }

}  // namespace cnn

extern "C" int64_t sdb_cnn_pack_bytes_ex(int32_t precision) {
    if (precision < 0 || precision > 3) return 0;
    return (int64_t)cnn::pack_layout(cnn::pack_planes(precision)).total;
}

extern "C" int64_t sdb_cnn_pack_bytes(int32_t precision) {
    if (precision < 0 || precision > 2) return 0;
    return sdb_cnn_pack_bytes_ex(precision);
}

// Device fp32 tensors with the reference's state-dict shapes (denoiser.*): conv1 [256,64,1,1] + [256]; conv2a / conv3a
// [256,256,3,3] + [256]; conv2b / conv3b [256,256,3,3] (no bias); conv4a / conv4b [256,256,1,1] + [256]; conv4 [3,256,1,1] + [3].
extern "C" int sdb_cnn_pack_ex(const float *d_w1, const float *d_b1, const float *d_w2a, const float *d_b2a, const float *d_w2b,
                               const float *d_w3a, const float *d_b3a, const float *d_w3b, const float *d_w4a, const float *d_b4a,
                               const float *d_w4b, const float *d_b4b, const float *d_w4, const float *d_b4, int32_t precision,
                               void *d_pack, void *stream)
{
    using namespace cnn;
    if (!d_w1 || !d_b1 || !d_w2a || !d_b2a || !d_w2b || !d_w3a || !d_b3a || !d_w3b || !d_w4a || !d_b4a || !d_w4b || !d_b4b || !d_w4 ||
        !d_b4 || !d_pack)
        return SDB_EINVAL;
    if (precision < 0 || precision > 3) return SDB_EUNSUPPORTED;
    const int planes = pack_planes(precision);
    const bool bf16 = precision == 1 || precision == 3;
    const PackLayout l = pack_layout(planes);
    cudaStream_t st = (cudaStream_t)stream;
    const float *ws[7] = {d_w1, d_w2a, d_w2b, d_w3a, d_w3b, d_w4a, d_w4b};
    const int cin[7] = {kInCh, kCh, kCh, kCh, kCh, kCh, kCh};
    for (int i = 0; i < 7; i++) {
        const long long n = (long long)kCh * cin[i] * kTaps[i];
        const unsigned blocks = (unsigned)((n + 255) / 256);
        uint8_t *dst = (uint8_t *)d_pack + l.w[i];
        if (bf16) pack_weight_kernel<true, false><<<blocks, 256, 0, st>>>(ws[i], dst, cin[i], kTaps[i], planes, kCh);
        else pack_weight_kernel<false, false><<<blocks, 256, 0, st>>>(ws[i], dst, cin[i], kTaps[i], planes, kCh);
        SDB_CHECK_LAUNCH();
    }
    float *f = reinterpret_cast<float *>((uint8_t *)d_pack + l.f32);
    const float *bs[5] = {d_b1, d_b2a, d_b3a, d_b4a, d_b4b};
    for (int i = 0; i < 5; i++) SDB_CUDA(cudaMemcpyAsync(f + i * kCh, bs[i], kCh * 4, cudaMemcpyDeviceToDevice, st));
    SDB_CUDA(cudaMemcpyAsync(f + 5 * kCh, d_w4, 3 * kCh * 4, cudaMemcpyDeviceToDevice, st));
    SDB_CUDA(cudaMemcpyAsync(f + 8 * kCh, d_b4, 3 * 4, cudaMemcpyDeviceToDevice, st));
    return SDB_OK;
}

extern "C" int sdb_cnn_pack(const float *d_w1, const float *d_b1, const float *d_w2a, const float *d_b2a, const float *d_w2b,
                            const float *d_w3a, const float *d_b3a, const float *d_w3b, const float *d_w4a, const float *d_b4a,
                            const float *d_w4b, const float *d_b4b, const float *d_w4, const float *d_b4, int32_t precision,
                            void *d_pack, void *stream)
{
    if (!d_w1 || !d_b1 || !d_w2a || !d_b2a || !d_w2b || !d_w3a || !d_b3a || !d_w3b || !d_w4a || !d_b4a || !d_w4b || !d_b4b || !d_w4 ||
        !d_b4 || !d_pack)
        return SDB_EINVAL;
    if (precision < 0 || precision > 2) return SDB_EUNSUPPORTED;
    return sdb_cnn_pack_ex(d_w1, d_b1, d_w2a, d_b2a, d_w2b, d_w3a, d_b3a, d_w3b, d_w4a, d_b4a, d_w4b, d_b4b, d_w4, d_b4, precision,
                           d_pack, stream);
}

extern "C" int64_t sdb_cnn_workspace_bytes(int32_t H, int32_t W, int32_t precision) {
    if (H <= 0 || W <= 0 || (precision != 0 && precision != 2)) return 0;
    int Hp, Wp;
    return (int64_t)cnn::ws_layout(H, W, precision == 2 ? 2 : 1, Hp, Wp).total;
}

// d_net_out [H][W][64] fp32 -> d_rgb [3][H][W] = tanh(RenderCNN(net_out, style)), d_rgb_raw (optional) the pre-tanh image.
// d_mod [4][256]: the four chunks of fc_z_cond(z) (gancraft_base.py:208-209): w, b of block 2, w, b of block 3.
// d_workspace: sdb_cnn_workspace_bytes(); its activation planes carry a ZERO border that the kernels never write:
// pass workspace_ready = 0 on the first call for a given (workspace, H, W, precision) -- the call then clears it -- and 1 afterwards.
extern "C" int sdb_cnn_forward(const float *d_net_out, int32_t H, int32_t W, const void *d_pack, const float *d_mod,
                               int32_t precision, float *d_rgb, float *d_rgb_raw, void *d_workspace, int32_t workspace_ready,
                               void *stream)
{
    using namespace cnn;
    if (!d_net_out || !d_pack || !d_mod || !d_rgb || !d_workspace || H <= 0 || W <= 0) return SDB_EINVAL;
    if (precision != 0 && precision != 2) return SDB_EUNSUPPORTED;
    const int planes = precision == 2 ? 2 : 1;
    cudaStream_t st = (cudaStream_t)stream;
    int Hp, Wp;
    const WsLayout wl = ws_layout(H, W, planes, Hp, Wp);
    const PackLayout pl = pack_layout(planes);
    uint8_t *ws = (uint8_t *)d_workspace;
    const uint8_t *pack = (const uint8_t *)d_pack;
    const float *f = reinterpret_cast<const float *>(pack + pl.f32);
    if (!workspace_ready) SDB_CUDA(cudaMemsetAsync(ws, 0, wl.total, st));
    {
        const long long n = (long long)H * W * (kInCh / 8);
        pack_input_kernel<false><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_net_out, ws + wl.a0, H, W, Hp, Wp, planes);
        SDB_CHECK_LAUNCH();
    }
    const FwdLayer layers[7] = {
        {wl.a0, NONE, wl.y, kInCh / 8, EPI_BIAS_LRELU, f + 0 * kCh, nullptr, nullptr},                        // conv1
        {wl.y, NONE, wl.t, kCh / 8, EPI_BIAS_LRELU, f + 1 * kCh, nullptr, nullptr},                           // conv2a
        {wl.t, wl.y, wl.y2, kCh / 8, EPI_RES_MOD_LRELU, nullptr, d_mod + 0 * kCh, d_mod + 1 * kCh},           // conv2b + modulate
        {wl.y2, NONE, wl.t, kCh / 8, EPI_BIAS_LRELU, f + 2 * kCh, nullptr, nullptr},                          // conv3a
        {wl.t, wl.y2, wl.y, kCh / 8, EPI_RES_MOD_LRELU, nullptr, d_mod + 2 * kCh, d_mod + 3 * kCh},           // conv3b + modulate
        {wl.y, NONE, wl.t, kCh / 8, EPI_BIAS_LRELU, f + 3 * kCh, nullptr, nullptr},                           // conv4a
        {wl.t, wl.y, NONE, kCh / 8, EPI_RES_BIAS_LRELU_RGB, f + 4 * kCh, nullptr, nullptr},                   // conv4b, conv4, tanh
    };
    const LayerParams base = frame_params(H, W, Hp, Wp, planes);
    if (planes == 2) return launch_forward_layers<true, false, false>(layers, ws, pack, pl, base, d_rgb, d_rgb_raw, st);
    return launch_forward_layers<false, false, false>(layers, ws, pack, pl, base, d_rgb, d_rgb_raw, st);
}

// ---------------------------------------------- training (include/sdb200.h, f1 under autograd) ----------------------------------------------
// Training precisions: 0 = fp16 x1, 1 = bf16 x3, 3 = bf16 x1; pack, record, backward pack and workspace of one training pass
// all come from the same precision.  The entries without _ex are precision 1.
static bool train_precision_ok(int32_t precision) { return precision == 0 || precision == 1 || precision == 3; }

extern "C" int64_t sdb_cnn_train_record_bytes_ex(int32_t H, int32_t W, int32_t precision) {
    if (H <= 0 || W <= 0 || !train_precision_ok(precision)) return 0;
    int Hp, Wp;
    return (int64_t)cnn::rec_layout(H, W, cnn::pack_planes(precision), Hp, Wp).total;
}

extern "C" int64_t sdb_cnn_train_record_bytes(int32_t H, int32_t W) { return sdb_cnn_train_record_bytes_ex(H, W, 1); }

// Diagnostics: Hp, Wp, then the byte offsets of the record's x, y1, t1, u2, y2, t2, u3, y3, t3, y4 planes and of rgb, then
// the record size -- 14 int64 in all.  An activation is `planes` 16-bit planes of [Hp][channels / 8][Wp][8] (bf16 [hi, lo]
// at precision 1, one plane of the forward's type at 0 and 3); pixel (y, x) sits at row y + 1, column x + 1.
extern "C" int sdb_cnn_debug_record_layout_ex(int32_t H, int32_t W, int32_t precision, int64_t *out)
{
    if (!out || H <= 0 || W <= 0) return SDB_EINVAL;
    if (!train_precision_ok(precision)) return SDB_EUNSUPPORTED;
    int Hp, Wp;
    const cnn::RecLayout r = cnn::rec_layout(H, W, cnn::pack_planes(precision), Hp, Wp);
    const size_t v[14] = {(size_t)Hp, (size_t)Wp, r.x, r.y1, r.t1, r.u2, r.y2, r.t2, r.u3, r.y3, r.t3, r.y4, r.rgb, r.total};
    for (int i = 0; i < 14; i++) out[i] = (int64_t)v[i];
    return SDB_OK;
}

extern "C" int sdb_cnn_debug_record_layout(int32_t H, int32_t W, int64_t *out) { return sdb_cnn_debug_record_layout_ex(H, W, 1, out); }

extern "C" int sdb_cnn_train_forward_ex(const float *d_net_out, int32_t H, int32_t W, const void *d_pack, const float *d_mod,
                                        int32_t precision, float *d_rgb, float *d_rgb_raw, void *d_record, void *stream)
{
    using namespace cnn;
    if (!d_net_out || !d_pack || !d_mod || !d_rgb || !d_record || H <= 0 || W <= 0) return SDB_EINVAL;
    if (!train_precision_ok(precision)) return SDB_EUNSUPPORTED;
    const int planes = pack_planes(precision);
    cudaStream_t st = (cudaStream_t)stream;
    int Hp, Wp;
    const RecLayout r = rec_layout(H, W, planes, Hp, Wp);
    const PackLayout pl = pack_layout(planes);
    uint8_t *rec = (uint8_t *)d_record;
    const uint8_t *pack = (const uint8_t *)d_pack;
    const float *f = reinterpret_cast<const float *>(pack + pl.f32);
    SDB_CUDA(cudaMemsetAsync(rec, 0, r.rgb, st));                     // the zero borders (and the area past the frame)
    {
        const long long n = (long long)H * W * (kInCh / 8);
        if (precision == 0) pack_input_kernel<false><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_net_out, rec + r.x, H, W, Hp, Wp, planes);
        else pack_input_kernel<true><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_net_out, rec + r.x, H, W, Hp, Wp, planes);
        SDB_CHECK_LAUNCH();
    }
    const FwdLayer layers[7] = {
        {r.x, NONE, r.y1, kInCh / 8, EPI_BIAS_LRELU, f + 0 * kCh, nullptr, nullptr},                          // conv1
        {r.y1, NONE, r.t1, kCh / 8, EPI_BIAS_LRELU, f + 1 * kCh, nullptr, nullptr},                           // conv2a
        {r.t1, r.y1, r.y2, kCh / 8, EPI_RES_MOD_LRELU, nullptr, d_mod + 0 * kCh, d_mod + 1 * kCh},            // conv2b + modulate (u2)
        {r.y2, NONE, r.t2, kCh / 8, EPI_BIAS_LRELU, f + 2 * kCh, nullptr, nullptr},                           // conv3a
        {r.t2, r.y2, r.y3, kCh / 8, EPI_RES_MOD_LRELU, nullptr, d_mod + 2 * kCh, d_mod + 3 * kCh},            // conv3b + modulate (u3)
        {r.y3, NONE, r.t3, kCh / 8, EPI_BIAS_LRELU, f + 3 * kCh, nullptr, nullptr},                           // conv4a
        {r.t3, r.y3, r.y4, kCh / 8, EPI_RES_BIAS_LRELU_RGB, f + 4 * kCh, nullptr, nullptr},                   // conv4b (y4), conv4, tanh
    };
    const LayerParams base = frame_params(H, W, Hp, Wp, planes);
    int rc;
    if (precision == 1) rc = launch_forward_layers<true, true, true>(layers, rec, pack, pl, base, d_rgb, d_rgb_raw, st);
    else if (precision == 3) rc = launch_forward_layers<false, true, true>(layers, rec, pack, pl, base, d_rgb, d_rgb_raw, st);
    else rc = launch_forward_layers<false, false, true>(layers, rec, pack, pl, base, d_rgb, d_rgb_raw, st);
    if (rc != SDB_OK) return rc;
    SDB_CUDA(cudaMemcpyAsync(rec + r.rgb, d_rgb, (size_t)3 * H * W * 4, cudaMemcpyDeviceToDevice, st));
    return SDB_OK;
}

extern "C" int sdb_cnn_train_forward(const float *d_net_out, int32_t H, int32_t W, const void *d_pack, const float *d_mod,
                                     float *d_rgb, float *d_rgb_raw, void *d_record, void *stream)
{
    return sdb_cnn_train_forward_ex(d_net_out, H, W, d_pack, d_mod, 1, d_rgb, d_rgb_raw, d_record, stream);
}

extern "C" int64_t sdb_cnn_backward_pack_bytes_ex(int32_t precision) {
    if (!train_precision_ok(precision)) return 0;
    return (int64_t)cnn::bwd_pack_layout(cnn::pack_planes(precision)).total;
}

extern "C" int64_t sdb_cnn_backward_pack_bytes(void) { return sdb_cnn_backward_pack_bytes_ex(1); }

extern "C" int sdb_cnn_pack_backward_ex(const float *d_w1, const float *d_w2a, const float *d_w2b, const float *d_w3a,
                                        const float *d_w3b, const float *d_w4a, const float *d_w4b, int32_t precision, void *d_pack,
                                        void *stream)
{
    using namespace cnn;
    if (!d_w1 || !d_w2a || !d_w2b || !d_w3a || !d_w3b || !d_w4a || !d_w4b || !d_pack) return SDB_EINVAL;
    if (!train_precision_ok(precision)) return SDB_EUNSUPPORTED;
    const int planes = pack_planes(precision);
    const PackLayout l = bwd_pack_layout(planes);
    cudaStream_t st = (cudaStream_t)stream;
    const float *ws[7] = {d_w1, d_w2a, d_w2b, d_w3a, d_w3b, d_w4a, d_w4b};
    for (int i = 0; i < 7; i++) {
        const long long n = (long long)kCh * kCh * kTaps[i];
        const unsigned blocks = (unsigned)((n + 255) / 256);
        uint8_t *dst = (uint8_t *)d_pack + l.w[i];
        if (precision == 0) pack_weight_kernel<false, true><<<blocks, 256, 0, st>>>(ws[i], dst, kCh, kTaps[i], planes, i == 0 ? kInCh : kCh);
        else pack_weight_kernel<true, true><<<blocks, 256, 0, st>>>(ws[i], dst, kCh, kTaps[i], planes, i == 0 ? kInCh : kCh);
        SDB_CHECK_LAUNCH();
    }
    return SDB_OK;
}

extern "C" int sdb_cnn_pack_backward(const float *d_w1, const float *d_w2a, const float *d_w2b, const float *d_w3a,
                                     const float *d_w3b, const float *d_w4a, const float *d_w4b, void *d_pack, void *stream)
{
    return sdb_cnn_pack_backward_ex(d_w1, d_w2a, d_w2b, d_w3a, d_w3b, d_w4a, d_w4b, 1, d_pack, stream);
}

extern "C" int64_t sdb_cnn_backward_workspace_bytes_ex(int32_t H, int32_t W, int32_t precision) {
    if (H <= 0 || W <= 0 || !train_precision_ok(precision)) return 0;
    int Hp, Wp;
    return (int64_t)cnn::bwd_ws_bytes(H, W, cnn::pack_planes(precision), Hp, Wp);
}

extern "C" int64_t sdb_cnn_backward_workspace_bytes(int32_t H, int32_t W) { return sdb_cnn_backward_workspace_bytes_ex(H, W, 1); }

namespace cnn {

struct BwdStep { int layer; int gin, gres, gout; size_t sign, u, x; const float *mw; float *s1, *s2, *dw; int x_chunks; };

// the data and weight gradient steps of the conv layers, from the last to the first (see sdb_cnn_backward_ex)
template <bool X3, bool BF16>
static int launch_backward_layers(const BwdStep (&steps)[7], const uint8_t *rec, const uint8_t *bpack, const PackLayout &bl,
                                  uint8_t *const (&G)[3], const LayerParams &base, float *d_grad_net_out, cudaStream_t st)
{
    using R = WgRing<X3>;
    const int n_tiles = base.tiles_x * base.tiles_y, sms = sdb_num_sms();
    const int grid = n_tiles < sms ? n_tiles : sms;
    for (int i = 0; i < 7; i++) {
        const BwdStep &s = steps[i];
        if (s.layer > 0 || d_grad_net_out) {
            BwdParams q{};
            q.l = base;
            q.l.in = G[s.gin];
            q.l.res = s.gres < 0 ? nullptr : G[s.gres];
            q.l.out = s.gout < 0 ? nullptr : G[s.gout];
            q.l.wpack = bpack + bl.w[s.layer];
            q.l.mod_w = s.mw;
            q.l.in_chunks = kCh / 8;
            q.l.taps = kTaps[s.layer];
            q.sign = s.sign == NONE ? nullptr : rec + s.sign;
            q.mod_u = s.u == NONE ? nullptr : rec + s.u;
            q.sum1 = s.s1; q.sum2 = s.s2;
            q.dx = s.layer == 0 ? d_grad_net_out : nullptr;
            const uint32_t smem = smem_map(q.l.taps, X3 ? 2 : 1).total;
            SDB_CUDA(cudaFuncSetAttribute(conv_bwd_kernel<X3, BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            conv_bwd_kernel<X3, BF16><<<grid, kThreads, smem, st>>>(q);
            SDB_CHECK_LAUNCH();
        }
        if (s.dw) {
            WgradParams w{};
            w.g = G[s.gin];
            w.in = rec + s.x;
            w.dw = s.dw;
            w.in_chunks = s.x_chunks;
            w.taps = kTaps[s.layer];
            w.H = base.H; w.Hp = base.Hp; w.Wp = base.Wp; w.segs = (base.Wp - 2) / kWgSeg;
            const int jobs = 2 * w.taps;
            const long long n_items = (long long)base.H * w.segs;
            long long ns = (2LL * sms + jobs - 1) / jobs;
            if (ns > n_items) ns = n_items;
            w.nsplit = (int)ns;
            if (w.in_chunks == kInCh / 8) {
                SDB_CUDA(cudaFuncSetAttribute(conv_wgrad_kernel<1, X3, BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)R::Smem));
                conv_wgrad_kernel<1, X3, BF16><<<(unsigned)(jobs * w.nsplit), kWgThreads, R::Smem, st>>>(w);
            } else {
                SDB_CUDA(cudaFuncSetAttribute(conv_wgrad_kernel<4, X3, BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)R::Smem));
                conv_wgrad_kernel<4, X3, BF16><<<(unsigned)(jobs * w.nsplit), kWgThreads, R::Smem, st>>>(w);
            }
            SDB_CHECK_LAUNCH();
        }
    }
    return SDB_OK;
}

}  // namespace cnn

extern "C" int sdb_cnn_backward_ex(int32_t H, int32_t W, int32_t precision, const void *d_record, const float *d_grad_rgb,
                                   const float *d_grad_rgb_raw, const void *d_bwd_pack, const void *d_pack, const float *d_mod,
                                   const sdb_cnn_grads *g, void *d_workspace, void *stream)
{
    using namespace cnn;
    if (!d_record || (!d_grad_rgb && !d_grad_rgb_raw) || !d_bwd_pack || !d_pack || !d_mod || !g || !d_workspace || H <= 0 || W <= 0)
        return SDB_EINVAL;
    if (!train_precision_ok(precision)) return SDB_EUNSUPPORTED;
    const int planes = pack_planes(precision);
    cudaStream_t st = (cudaStream_t)stream;
    int Hp, Wp;
    const RecLayout r = rec_layout(H, W, planes, Hp, Wp);
    const size_t gbytes = plane_bytes(Hp, kCh / 8, Wp) * planes;
    const PackLayout bl = bwd_pack_layout(planes), pl = pack_layout(planes);
    const uint8_t *rec = (const uint8_t *)d_record, *bpack = (const uint8_t *)d_bwd_pack;
    const float *f = reinterpret_cast<const float *>((const uint8_t *)d_pack + pl.f32);
    uint8_t *const G[3] = {(uint8_t *)d_workspace, (uint8_t *)d_workspace + gbytes, (uint8_t *)d_workspace + 2 * gbytes};
    SDB_CUDA(cudaMemsetAsync(d_workspace, 0, 3 * gbytes, st));
    float *zeroed[16] = {g->d_grad_mod, g->d_grad_w1, g->d_grad_b1, g->d_grad_w2a, g->d_grad_b2a, g->d_grad_w2b, g->d_grad_w3a,
                         g->d_grad_b3a, g->d_grad_w3b, g->d_grad_w4a, g->d_grad_b4a, g->d_grad_w4b, g->d_grad_b4b, g->d_grad_w4, g->d_grad_b4, nullptr};
    const size_t zbytes[15] = {4 * kCh, (size_t)kCh * kInCh, kCh, (size_t)kCh * kCh * 9, kCh, (size_t)kCh * kCh * 9, (size_t)kCh * kCh * 9,
                               kCh, (size_t)kCh * kCh * 9, (size_t)kCh * kCh, kCh, (size_t)kCh * kCh, kCh, 3 * kCh, 3};
    for (int i = 0; i < 15; i++)
        if (zeroed[i]) SDB_CUDA(cudaMemsetAsync(zeroed[i], 0, zbytes[i] * 4, st));
    float *dm = g->d_grad_mod;

    {   // tanh', conv4^T, sigma'(y4) -> g_p4b in G[0]
        HeadParams h{};
        h.y4 = rec + r.y4; h.rgb = reinterpret_cast<const float *>(rec + r.rgb); h.g_rgb = d_grad_rgb; h.g_raw = d_grad_rgb_raw;
        h.w4 = f + 5 * kCh; h.out = G[0]; h.dw4 = g->d_grad_w4; h.db4 = g->d_grad_b4; h.db4b = g->d_grad_b4b;
        h.H = H; h.W = W; h.Hp = Hp; h.Wp = Wp;
        const long long HW = (long long)H * W;
        long long bx = (HW + 255) / 256;
        if (bx > sdb_num_sms()) bx = sdb_num_sms();                                      // x 32 chunks: 32 blocks of 256 per SM
        const dim3 grid((unsigned)bx, kCh / 8);
        if (precision == 1) head_bwd_kernel<true, true><<<grid, 256, 0, st>>>(h);
        else if (precision == 3) head_bwd_kernel<false, true><<<grid, 256, 0, st>>>(h);
        else head_bwd_kernel<false, false><<<grid, 256, 0, st>>>(h);
        SDB_CHECK_LAUNCH();
    }
    // the conv layers from the last to the first: data gradient, then the layer's weight gradient, which reads the gradient at
    // the layer's output (the input of its data step, G[gin]) and the layer's input from the record (x)
    const int N_ = -1;
    const BwdStep steps[7] = {
        {6, 0, N_, 1, r.t3, NONE, r.t3, nullptr, g->d_grad_b4a, nullptr, g->d_grad_w4b, kCh / 8},                      // conv4b^T -> g_p4a
        {5, 1, 0, 2, r.y3, r.u3, r.y3, d_mod + 2 * kCh, dm ? dm + 3 * kCh : nullptr, dm ? dm + 2 * kCh : nullptr, g->d_grad_w4a, kCh / 8},   // conv4a^T -> g_u3
        {4, 2, N_, 0, r.t2, NONE, r.t2, nullptr, g->d_grad_b3a, nullptr, g->d_grad_w3b, kCh / 8},                      // conv3b^T -> g_p3a
        {3, 0, 2, 1, r.y2, r.u2, r.y2, d_mod + 0 * kCh, dm ? dm + 1 * kCh : nullptr, dm ? dm + 0 * kCh : nullptr, g->d_grad_w3a, kCh / 8},   // conv3a^T -> g_u2
        {2, 1, N_, 2, r.t1, NONE, r.t1, nullptr, g->d_grad_b2a, nullptr, g->d_grad_w2b, kCh / 8},                      // conv2b^T -> g_p2a
        {1, 2, 1, 0, r.y1, NONE, r.y1, nullptr, g->d_grad_b1, nullptr, g->d_grad_w2a, kCh / 8},                        // conv2a^T -> g_p1
        {0, 0, N_, N_, NONE, NONE, r.x, nullptr, nullptr, nullptr, g->d_grad_w1, kInCh / 8},                          // conv1^T -> dL/dnet_out
    };
    const LayerParams base = frame_params(H, W, Hp, Wp, planes);
    if (precision == 1) return launch_backward_layers<true, true>(steps, rec, bpack, bl, G, base, g->d_grad_net_out, st);
    if (precision == 3) return launch_backward_layers<false, true>(steps, rec, bpack, bl, G, base, g->d_grad_net_out, st);
    return launch_backward_layers<false, false>(steps, rec, bpack, bl, G, base, g->d_grad_net_out, st);
}

extern "C" int sdb_cnn_backward(int32_t H, int32_t W, const void *d_record, const float *d_grad_rgb, const float *d_grad_rgb_raw,
                                const void *d_bwd_pack, const void *d_pack, const float *d_mod, const sdb_cnn_grads *g,
                                void *d_workspace, void *stream)
{
    return sdb_cnn_backward_ex(H, W, 1, d_record, d_grad_rgb, d_grad_rgb_raw, d_bwd_pack, d_pack, d_mod, g, d_workspace, stream);
}
