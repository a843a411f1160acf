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
constexpr int kEpiThreads = 256;

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

__device__ __forceinline__ void split8h(const float (&v)[8], uint4 &hi, uint4 &lo) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const __half2 hh = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
        const float2 back = __half22float2(hh);
        const __half2 ll = __floats2half2_rn(v[2 * i] - back.x, v[2 * i + 1] - back.y);
        h[i] = *reinterpret_cast<const uint32_t *>(&hh);
        l[i] = *reinterpret_cast<const uint32_t *>(&ll);
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

__device__ __forceinline__ void unpack8h(uint4 u, float (&v)[8]) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&w[i]));
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

template <bool X3>
__global__ void __launch_bounds__(kThreads, 1)
conv_kernel(const LayerParams p)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr int P = X3 ? 2 : 1;
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
    if (tid == 0) {
        // the two epilogue warpgroups both read every slab and weight stage: one arrival each frees it
        for (int i = 0; i < 2; i++) { tc05::mbar_init(&bars[B_SLAB_FULL + i], 1); tc05::mbar_init(&bars[B_SLAB_EMPTY + i], 2); }
        for (int i = 0; i < kWStages; i++) { tc05::mbar_init(&bars[B_W_FULL + i], 1); tc05::mbar_init(&bars[B_W_EMPTY + i], 2); }
        tc05::fence_mbar_init();
    }
    __syncthreads();
    const size_t in_plane = plane_bytes(p.Hp, p.in_chunks, p.Wp);

    // Every tile is computed in kPasses passes over the input channels, one per 128-wide half of the output channels
    // (accumulators of a [128 pixel x 128 channel] half: 128 registers per thread of a warpgroup).
    if (warp == 8) {
        // ---------------- activation loader: one slab = rows_in rows x P planes x 4 chunks, 2080 B each ----------------
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
    } else if (warp == 9) {
        // ---------------- weight loader: 16 KB stages in (slab, tap, plane) order, the same for every tile and pass ----------------
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
                // acc[rb][nh]: pixels 64 rb .., output channels 128 pass + 64 nh ..
                float acc[2][2][32];
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
                                            tc05::wgmma_m64n64k16<false, 0, 0>(acc[rb][nh], da, db, 1u);
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
                                    float2 r = __half22float2(*reinterpret_cast<const __half2 *>(p.res + off));
                                    if (X3) {
                                        const float2 l = __half22float2(*reinterpret_cast<const __half2 *>(p.res + out_plane + off));
                                        r.x += l.x;
                                        r.y += l.y;
                                    }
                                    v0 = r.x + v0;                                            // y + conv(...)
                                    v1 = r.y + v1;
                                }
                                if (p.epi == EPI_RES_MOD_LRELU) {
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
                                if (p.out != nullptr && valid) {
                                    const __half2 hi = __floats2half2_rn(v0, v1);
                                    *reinterpret_cast<__half2 *>(p.out + off) = hi;
                                    if (X3) {
                                        const float2 back = __half22float2(hi);
                                        *reinterpret_cast<__half2 *>(p.out + out_plane + off) = __floats2half2_rn(v0 - back.x, v1 - back.y);
                                    }
                                }
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

// per-pixel features fp32 [H][W][64] (NHWC, the fused kernel's net_out) -> operand planes [P][Hp][8][Wp][8] fp16
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
    split8h(v, hi, lo);
    const size_t off = ((((size_t)(y + 1) * (kInCh / 8)) + c) * Wp + (x + 1)) * 16;
    *reinterpret_cast<uint4 *>(act + off) = hi;
    if (planes == 2) *reinterpret_cast<uint4 *>(act + plane_bytes(Hp, kInCh / 8, Wp) + off) = lo;
}

// conv weight fp32 [256][cin][taps] (PyTorch [out][in][kh][kw]) -> [slab][tap][plane][chunk 4][n 256][8] fp16
__global__ void __launch_bounds__(256)
pack_weight_kernel(const float *__restrict__ w, uint8_t *__restrict__ pack, int cin, int taps, int planes)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long n = (long long)kCh * cin * taps;
    if (i >= n) return;
    const int t = (int)(i % taps);
    const int ci = (int)((i / taps) % cin);
    const int no = (int)(i / ((long long)taps * cin));
    const float v = w[i];
    const __half hi = __float2half_rn(v);
    const __half lo = __float2half_rn(v - __half2float(hi));
    const int s = ci / 32, c = (ci % 32) / 8, j = ci % 8;
    const size_t stage = ((size_t)s * taps + t) * planes;
    const size_t inner = ((size_t)c * 256 + no) * 8 + j;
    reinterpret_cast<__half *>(pack + stage * kWStage)[inner] = hi;
    if (planes == 2) reinterpret_cast<__half *>(pack + (stage + 1) * kWStage)[inner] = lo;
}

struct PackLayout { size_t w[7], f32, total; };
// fp32 tail: b1 | b2a | b3a | b4a | b4b | w4 [3][256] | b4 [3] (+pad)
constexpr int kF32Floats = 5 * kCh + 3 * kCh + 4;
static PackLayout pack_layout(int planes) {
    PackLayout l{};
    const int cin[7] = {kInCh, kCh, kCh, kCh, kCh, kCh, kCh}, taps[7] = {1, 9, 9, 9, 9, 1, 1};
    size_t o = 0;
    for (int i = 0; i < 7; i++) { l.w[i] = o; o += (size_t)(cin[i] / 32) * taps[i] * planes * kWStage; }
    l.f32 = o; o += (size_t)kF32Floats * 4;
    l.total = (o + 255) / 256 * 256;
    return l;
}

struct WsLayout { size_t a0, y, t, y2, total; };
static WsLayout ws_layout(int H, int W, int planes, int &Hp, int &Wp) {
    Hp = H + 4;                                              // one zero row above, (up to) three below: tiles are 2 rows tall
    Wp = ((W + kSeg - 1) / kSeg) * kSeg + 2;
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

}  // namespace cnn

extern "C" int64_t sdb_cnn_pack_bytes(int32_t precision) {
    if (precision != 0 && precision != 2) return 0;
    return (int64_t)cnn::pack_layout(precision == 2 ? 2 : 1).total;
}

// Device fp32 tensors with the reference's state-dict shapes (denoiser.*): conv1 [256,64,1,1] + [256]; conv2a / conv3a
// [256,256,3,3] + [256]; conv2b / conv3b [256,256,3,3] (no bias); conv4a / conv4b [256,256,1,1] + [256]; conv4 [3,256,1,1] + [3].
extern "C" int sdb_cnn_pack(const float *d_w1, const float *d_b1, const float *d_w2a, const float *d_b2a, const float *d_w2b,
                            const float *d_w3a, const float *d_b3a, const float *d_w3b, const float *d_w4a, const float *d_b4a,
                            const float *d_w4b, const float *d_b4b, const float *d_w4, const float *d_b4, int32_t precision,
                            void *d_pack, void *stream)
{
    using namespace cnn;
    if (!d_w1 || !d_b1 || !d_w2a || !d_b2a || !d_w2b || !d_w3a || !d_b3a || !d_w3b || !d_w4a || !d_b4a || !d_w4b || !d_b4b || !d_w4 ||
        !d_b4 || !d_pack)
        return SDB_EINVAL;
    if (precision != 0 && precision != 2) return SDB_EUNSUPPORTED;
    const int planes = precision == 2 ? 2 : 1;
    const PackLayout l = pack_layout(planes);
    cudaStream_t st = (cudaStream_t)stream;
    const float *ws[7] = {d_w1, d_w2a, d_w2b, d_w3a, d_w3b, d_w4a, d_w4b};
    const int cin[7] = {kInCh, kCh, kCh, kCh, kCh, kCh, kCh}, taps[7] = {1, 9, 9, 9, 9, 1, 1};
    for (int i = 0; i < 7; i++) {
        const long long n = (long long)kCh * cin[i] * taps[i];
        pack_weight_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws[i], (uint8_t *)d_pack + l.w[i], cin[i], taps[i], planes);
        SDB_CHECK_LAUNCH();
    }
    float *f = reinterpret_cast<float *>((uint8_t *)d_pack + l.f32);
    const float *bs[5] = {d_b1, d_b2a, d_b3a, d_b4a, d_b4b};
    for (int i = 0; i < 5; i++) SDB_CUDA(cudaMemcpyAsync(f + i * kCh, bs[i], kCh * 4, cudaMemcpyDeviceToDevice, st));
    SDB_CUDA(cudaMemcpyAsync(f + 5 * kCh, d_w4, 3 * kCh * 4, cudaMemcpyDeviceToDevice, st));
    SDB_CUDA(cudaMemcpyAsync(f + 8 * kCh, d_b4, 3 * 4, cudaMemcpyDeviceToDevice, st));
    return SDB_OK;
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
        pack_input_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_net_out, ws + wl.a0, H, W, Hp, Wp, planes);
        SDB_CHECK_LAUNCH();
    }
    LayerParams base{};
    base.H = H; base.W = W; base.Hp = Hp; base.Wp = Wp; base.planes = planes;
    base.tiles_x = (W + kSeg - 1) / kSeg; base.tiles_y = (H + kTileRows - 1) / kTileRows;
    const int n_tiles = base.tiles_x * base.tiles_y;
    const int grid = n_tiles < sdb_num_sms() ? n_tiles : sdb_num_sms();
    struct L { size_t in, res, out; int wi, in_chunks, taps, epi; const float *bias, *mw, *mb; };
    const size_t NONE = (size_t)-1;
    const L layers[7] = {
        {wl.a0, NONE, wl.y, 0, kInCh / 8, 1, EPI_BIAS_LRELU, f + 0 * kCh, nullptr, nullptr},                        // conv1
        {wl.y, NONE, wl.t, 1, kCh / 8, 9, EPI_BIAS_LRELU, f + 1 * kCh, nullptr, nullptr},                           // conv2a
        {wl.t, wl.y, wl.y2, 2, kCh / 8, 9, EPI_RES_MOD_LRELU, nullptr, d_mod + 0 * kCh, d_mod + 1 * kCh},           // conv2b + modulate
        {wl.y2, NONE, wl.t, 3, kCh / 8, 9, EPI_BIAS_LRELU, f + 2 * kCh, nullptr, nullptr},                          // conv3a
        {wl.t, wl.y2, wl.y, 4, kCh / 8, 9, EPI_RES_MOD_LRELU, nullptr, d_mod + 2 * kCh, d_mod + 3 * kCh},           // conv3b + modulate
        {wl.y, NONE, wl.t, 5, kCh / 8, 1, EPI_BIAS_LRELU, f + 3 * kCh, nullptr, nullptr},                           // conv4a
        {wl.t, wl.y, NONE, 6, kCh / 8, 1, EPI_RES_BIAS_LRELU_RGB, f + 4 * kCh, nullptr, nullptr},                   // conv4b, conv4, tanh
    };
    for (int i = 0; i < 7; i++) {
        LayerParams p = base;
        const L &l = layers[i];
        p.in = ws + l.in;
        p.res = l.res == NONE ? nullptr : ws + l.res;
        p.out = l.out == NONE ? nullptr : ws + l.out;
        p.wpack = pack + pl.w[l.wi];
        p.bias = l.bias; p.mod_w = l.mw; p.mod_b = l.mb;
        p.in_chunks = l.in_chunks; p.taps = l.taps; p.epi = l.epi;
        if (l.epi == EPI_RES_BIAS_LRELU_RGB) { p.w4 = f + 5 * kCh; p.b4 = f + 8 * kCh; p.rgb = d_rgb; p.rgb_raw = d_rgb_raw; }
        const uint32_t smem = smem_map(p.taps, planes).total;
        if (planes == 2) {
            SDB_CUDA(cudaFuncSetAttribute(conv_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            conv_kernel<true><<<grid, kThreads, smem, st>>>(p);
        } else {
            SDB_CUDA(cudaFuncSetAttribute(conv_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            conv_kernel<false><<<grid, kThreads, smem, st>>>(p);
        }
        SDB_CHECK_LAUNCH();
    }
    return SDB_OK;
}
