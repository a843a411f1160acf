// f3: building the voxel world of a scene from its bird's-eye-view maps ON THE DEVICE.
// Behavioural contract: PCGVoxelGenerator.next_world (imaginaire/model_utils/pcg_gen.py:83-174):
//   world[h, x, z] = label(x, z) for h = hq(x, z) and for clip(hq + 1 .. hq + 16, 0, 255)        (:119-125, surface shell, hollow below)
//   trees: voxel models pasted at height hq + 16 in iteration order, only where the world is still 0 (:132-151);
//          a model voxel that is 0 leaves the cell open for a later tree
//   heightmap[x, z] = topmost non-zero h (0 for an empty column) (:160-163); gnd = min, sky = max + 1 (:164-165)
//   voxel_t = world[gnd:sky] (:173)
// The reference does this with 17 CPU scatter passes over a 1-4 GB tensor, a Python loop over every tree, and a 1-4 GB
// host->device copy.  Here the full-height volume only ever exists in HBM:
//   columns_kernel   one thread per (x, z) column writes its shell (the volume is zero-filled by a memset);
//   trees_kernel     one CTA per tree instance; the sequential "first tree wins" rule becomes an atomicMin on a key
//                    (sequence index << 10 | block id) -- order-independent, hence deterministic and identical to the loop;
//   heightmap_kernel one thread per column scans down from the top; block-level min / max -> gnd, sky;
//   truncate_kernel  copies world[gnd:sky] into the caller's tensor, decoding tree keys to block ids on the way.
// Bound: HBM (one memset, one sweep for the height map, one for the copy).
#include "common.cuh"

namespace {
constexpr int kTreeShift = 10;                  // block ids are < 1024 (Minecraft ids < 680)
constexpr int kShell = 16;                      // pad_num, pcg_gen.py:123

__global__ void __launch_bounds__(256)
columns_kernel(const int32_t *__restrict__ hq, const int32_t *__restrict__ label, int32_t *__restrict__ world, int X, int Z, int SH)
{
    const long long i = blockIdx.x * 256ll + threadIdx.x;
    if (i >= (long long)X * Z) return;
    const int h = hq[i], lab = label[i];
    const long long plane = (long long)X * Z;
    for (int k = 0; k <= kShell; k++) {
        int y = h + k;
        y = y < 0 ? 0 : (y > SH - 1 ? SH - 1 : y);             // torch.clip(h + k, 0, sample_height - 1)
        world[(long long)y * plane + i] = lab;
    }
}

// tree instance t: anchor (h, x, z) = inst[4t .. 4t+2], model = inst[4t+3]; model m: dims mdim[3m..], voxels at moff[m]
__global__ void __launch_bounds__(128)
trees_kernel(const int32_t *__restrict__ inst, int n_inst, const int32_t *__restrict__ models, const int32_t *__restrict__ mdim,
             const long long *__restrict__ moff, int32_t *__restrict__ world, int X, int Z, int SH)
{
    const int t = blockIdx.x;
    if (t >= n_inst) return;
    const int h0 = inst[4 * t], x0 = inst[4 * t + 1], z0 = inst[4 * t + 2], m = inst[4 * t + 3];
    const int dh = mdim[3 * m], dx = mdim[3 * m + 1], dz = mdim[3 * m + 2];
    const int32_t *vox = models + moff[m];
    const long long plane = (long long)X * Z;
    for (int i = threadIdx.x; i < dh * dx * dz; i += blockDim.x) {
        const int v = vox[i];
        if (v == 0) continue;                                   // writes 0 into a cell that is 0: leaves it open (pcg_gen.py:148-151)
        const int a = i / (dx * dz), b = (i / dz) % dx, c = i % dz;
        const int y = h0 + a, x = x0 + b, z = z0 + c;
        if (y >= SH || x >= X || z >= Z) continue;               // python slicing clips at the array end
        int32_t *cell = world + (long long)y * plane + (long long)x * Z + z;
        const int32_t key = ((t + 1) << kTreeShift) | v;
        int32_t old = *cell;
        while (old == 0 || (old >= (1 << kTreeShift) && old > key)) {   // empty, or claimed by a LATER tree
            const int32_t seen = atomicCAS(cell, old, key);
            if (seen == old) break;
            old = seen;
        }
    }
}

__global__ void __launch_bounds__(256)
heightmap_kernel(const int32_t *__restrict__ world, long long *__restrict__ heightmap, int *__restrict__ minmax, int X, int Z, int SH)
{
    __shared__ int smin[8], smax[8];
    const long long i = blockIdx.x * 256ll + threadIdx.x;
    const long long plane = (long long)X * Z;
    int top = 0;
    bool in = i < plane;
    if (in) {
        for (int y = SH - 1; y >= 0; y--)
            if (world[(long long)y * plane + i] != 0) { top = y; break; }
        heightmap[i] = top;
    }
    int lo = in ? top : 0x7fffffff, hi = in ? top : -1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    if ((threadIdx.x & 31) == 0) { smin[threadIdx.x >> 5] = lo; smax[threadIdx.x >> 5] = hi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; w++) { lo = min(lo, smin[w]); hi = max(hi, smax[w]); }
        lo = min(lo, smin[0]); hi = max(hi, smax[0]);
        atomicMin(&minmax[0], lo);
        atomicMax(&minmax[1], hi);
    }
}

__global__ void __launch_bounds__(256)
truncate_kernel(const int32_t *__restrict__ world, int32_t *__restrict__ out, long long n, long long first)
{
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += stride) {
        const int32_t v = world[first + i];
        out[i] = v >= (1 << kTreeShift) ? (v & ((1 << kTreeShift) - 1)) : v;
    }
}
}  // namespace

// Stage 1: fills d_world [SH, X, Z] (caller-owned scratch), the height map [X, Z] (int64, like the reference's) and
// d_minmax[2] = {gnd_level, topmost height}.  d_hq / d_label: int32 [X, Z] quantised height index and block id of the column;
// trees: d_inst int32 [n_inst, 4] = (h, x, z, model) in the reference's iteration order, d_models / d_mdim [n_models, 3] /
// d_moff int64 [n_models] the concatenated voxel models.
extern "C" int sdb_world_build(const int32_t *d_hq, const int32_t *d_label, int32_t X, int32_t Z, int32_t SH, const int32_t *d_inst,
                               int32_t n_inst, const int32_t *d_models, const int32_t *d_mdim, const int64_t *d_moff,
                               int32_t *d_world, int64_t *d_heightmap, int32_t *d_minmax, void *stream)
{
    if (!d_hq || !d_label || !d_world || !d_heightmap || !d_minmax || X <= 0 || Z <= 0 || SH <= 0 || n_inst < 0) return SDB_EINVAL;
    if (n_inst > 0 && (!d_inst || !d_models || !d_mdim || !d_moff)) return SDB_EINVAL;
    if (n_inst >= (1 << (31 - kTreeShift)) - 1) return SDB_EUNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    const long long plane = (long long)X * Z;
    SDB_CUDA(cudaMemsetAsync(d_world, 0, (size_t)plane * SH * 4, st));
    const int32_t init[2] = {0x7fffffff, -1};
    SDB_CUDA(cudaMemcpyAsync(d_minmax, init, 8, cudaMemcpyHostToDevice, st));
    const unsigned cb = (unsigned)((plane + 255) / 256);
    columns_kernel<<<cb, 256, 0, st>>>(d_hq, d_label, d_world, X, Z, SH);
    SDB_CHECK_LAUNCH();
    if (n_inst > 0) {
        trees_kernel<<<n_inst, 128, 0, st>>>(d_inst, n_inst, d_models, d_mdim, (const long long *)d_moff, d_world, X, Z, SH);
        SDB_CHECK_LAUNCH();
    }
    heightmap_kernel<<<cb, 256, 0, st>>>(d_world, (long long *)d_heightmap, d_minmax, X, Z, SH);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

// Stage 2 (after the caller has read d_minmax and allocated the result): d_voxel_t [sky - gnd, X, Z] = world[gnd:sky].
extern "C" int sdb_world_truncate(const int32_t *d_world, int32_t X, int32_t Z, int32_t gnd, int32_t sky, int32_t *d_voxel_t, void *stream)
{
    if (!d_world || !d_voxel_t || X <= 0 || Z <= 0 || gnd < 0 || sky <= gnd) return SDB_EINVAL;
    const long long plane = (long long)X * Z, n = plane * (sky - gnd);
    const long long want = (n + 255) / 256, cap = (long long)sdb_num_sms() * 32;
    truncate_kernel<<<(int)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(d_world, d_voxel_t, n, plane * gnd);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}
