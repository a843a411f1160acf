/*
 * oracle.c -- CPU restatement of the SceneDreamer render hot path's native ops.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under scenedreamer_b200/ may import, link or call this
 * file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs use it, and only as the checker / the CPU baseline.
 *
 * Each function restates (does not copy) the algorithm of one reference CUDA kernel, in plain
 * scalar C, in float32 with the same operation order, so results can be compared bit-for-bit
 * (integer / index buffers) or to ~1 ulp (float buffers).  Citations are relative to
 * /root/reference/.
 *
 * Build: see oracle/Makefile (gcc -O2 -mfma -ffp-contract=off -fopenmp).  -ffp-contract=off
 * plus explicit fmaf() reproduces exactly the FMA contraction nvcc applied to the reference
 * device code (verified from the SASS of oracle/_ref/ref_voxlib: FMUL,FFMA,FFMA for the ray
 * direction, FFMA x3 for the squared length); host-side camera math in the reference is
 * compiled by g++ for baseline x86-64, i.e. without contraction.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

/* ------------------------------------------------------------------------------------------
 * Camera frame, host side.
 * Follows imaginaire/model_utils/gancraft/voxlib/ray_voxel_intersection.cu:279-284 and the
 * helpers in voxlib_common.h:26-31 (cross), :47-74 (normalize).  Plain float mul/add, sqrtf
 * and division, no contraction (host code).
 * ------------------------------------------------------------------------------------------ */
static void host_normalize3(float *r, const float *a) {
    float len = 0.0f;
    for (int i = 0; i < 3; i++) len += a[i] * a[i];
    len = sqrtf(len);
    for (int i = 0; i < 3; i++) r[i] = a[i] / len;
}
static void host_cross3(float *r, const float *a, const float *b) {
    r[0] = a[1] * b[2] - a[2] * b[1];
    r[1] = a[2] * b[0] - a[0] * b[2];
    r[2] = a[0] * b[1] - a[1] * b[0];
}
void sdo_camera_frame(const float *cam_dir, const float *cam_up, float *fwd, float *side, float *up) {
    float t[3];
    host_normalize3(fwd, cam_dir);
    host_cross3(t, fwd, cam_up);
    host_normalize3(side, t);
    host_cross3(t, side, fwd);
    host_normalize3(up, t);
}

/* ------------------------------------------------------------------------------------------
 * Ray / voxel intersection (perspective camera): Amanatides-Woo DDA.
 * Follows ray_voxel_intersection.cu:52-235 (kernel) with the launch-side parameter packing of
 * :253-325.  Outputs use the reference layouts:
 *   out_voxel_id [H, W, M]      int32   (reference shape [H,W,M,1])
 *   out_depth    [2, H, W, M]   float   (entry t, exit t; NaN when the slot is unfilled)
 *   out_raydirs  [H, W, 3]      float
 * steps_out (optional, [H,W] int32) = number of voxel reads the ray performed; used only to
 * state the DDA's algorithmic bytes.
 * ------------------------------------------------------------------------------------------ */
static inline float axis_t_init(int cell, float o, float d) {
    /* ray_voxel_intersection.cu:95-106 */
    if (d > 0) return ((float)(cell + 1) - o) / d;
    if (d < 0) return ((float)cell - o) / d;
    return HUGE_VALF;
}

void sdo_ray_voxel_intersection_perspective(
    const int32_t *voxel, const int64_t dims[3], const int64_t strides[3],
    const float cam_ori[3], const float cam_dir[3], const float cam_up[3],
    float cam_f, const float cam_c[2], const int img_dims[2], int max_samples,
    int32_t *out_voxel_id, float *out_depth, float *out_raydirs, int32_t *steps_out)
{
    float fwd[3], side[3], up[3];
    sdo_camera_frame(cam_dir, cam_up, fwd, side, up);
    const int H = img_dims[0], W = img_dims[1], M = max_samples;
    const int64_t plane = (int64_t)H * W * M;
    const int d0 = (int)dims[0], d1 = (int)dims[1], d2 = (int)dims[2];

#pragma omp parallel for schedule(dynamic, 4)
    for (int i = 0; i < H; i++) {
        for (int j = 0; j < W; j++) {
            const int64_t pix = (int64_t)i * W + j;
            /* :71-78 -- device code: FADD, FADD, then per component FMUL, FFMA, FFMA */
            const float n0 = cam_c[0] - (float)i;
            const float n1 = (float)j - cam_c[1];
            float rd[3];
            for (int k = 0; k < 3; k++)
                rd[k] = fmaf(fwd[k], cam_f, fmaf(up[k], n0, side[k] * n1));
            float len = fmaf(rd[2], rd[2], fmaf(rd[1], rd[1], fmaf(rd[0], rd[0], 0.0f)));
            len = sqrtf(len);
            for (int k = 0; k < 3; k++) rd[k] = rd[k] / len;
            out_raydirs[pix * 3 + 0] = rd[0];
            out_raydirs[pix * 3 + 1] = rd[1];
            out_raydirs[pix * 3 + 2] = rd[2];

            int cell[3];
            float at[3];
            for (int k = 0; k < 3; k++) {
                cell[k] = (int)floorf(cam_ori[k]);              /* :90-92 */
                at[k] = axis_t_init(cell[k], cam_ori[k], rd[k]);
            }
            const int dim[3] = {d0, d1, d2};
            int quit = 0;
            int32_t nread = 0;
            for (int s = 0; s < M; s++) {
                float t = NAN, t2 = NAN;
                int32_t id = 0;
                while (!quit) {
                    /* :143-190 -- tie rule: axis0 if <= both, else axis1 if <= axis2, else axis2 */
                    int a;
                    if (at[0] <= at[1] && at[0] <= at[2]) a = 0;
                    else if (at[1] <= at[2]) a = 1;
                    else a = 2;
                    const float tnow = at[a];
                    if (rd[a] > 0) {
                        cell[a] += 1;
                        if (cell[a] >= dim[a]) quit = 1;
                        at[a] = ((float)(cell[a] + 1) - cam_ori[a]) / rd[a];
                    } else {
                        cell[a] -= 1;
                        if (cell[a] < 0) quit = 1;
                        at[a] = ((float)cell[a] - cam_ori[a]) / rd[a];
                    }
                    if (quit) break;
                    /* :198-200 */
                    if (cell[0] < 0 || cell[0] >= d0 || cell[1] < 0 || cell[1] >= d1 ||
                        cell[2] < 0 || cell[2] >= d2)
                        continue;
                    nread++;
                    const int32_t v = voxel[cell[0] * strides[0] + cell[1] * strides[1] + cell[2] * strides[2]];
                    if (v == 0) continue;
                    id = v;
                    t = tnow;
                    if (at[0] <= at[1] && at[0] <= at[2]) t2 = at[0];   /* :222-228 */
                    else if (at[1] <= at[2]) t2 = at[1];
                    else t2 = at[2];
                    break;
                }
                out_depth[pix * M + s] = t;
                out_depth[plane + pix * M + s] = t2;
                out_voxel_id[pix * M + s] = id;
            }
            if (steps_out) steps_out[pix] = nread;
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * Multi-resolution hash / tiled grid encoding.
 * Follows gridencoder/src/gridencoder.cu:35-51 (fast_hash), :54-72 (get_grid_index),
 * :75-224 (kernel_grid), :227-314 (kernel_grid_backward), :317-343 (kernel_input_backward).
 * float32 only (the SceneDreamer path never enables autocast for the encoder's caller).
 * ------------------------------------------------------------------------------------------ */
#define SDO_MAX_D 5
static const uint32_t SDO_PRIMES[7] = {1u, 2654435761u, 805459861u, 3674653429u,
                                       2097192037u, 1434869437u, 2165219737u};

static inline uint32_t grid_index(uint32_t D, uint32_t C, uint32_t gridtype, int align_corners,
                                  uint32_t hashmap_size, uint32_t resolution, const uint32_t *pg) {
    uint32_t stride = 1, index = 0;
    for (uint32_t d = 0; d < D && stride <= hashmap_size; d++) {
        index += pg[d] * stride;
        stride *= align_corners ? resolution : (resolution + 1);
    }
    if (gridtype == 0 && stride > hashmap_size) {
        uint32_t h = 0;
        for (uint32_t d = 0; d < D; d++) h ^= pg[d] * SDO_PRIMES[d];
        index = h;
    }
    return (index % hashmap_size) * C;
}

/* outputs: [L, B, C] (level-major, like the reference buffer); dy_dx: [B, L, D, C] or NULL */
void sdo_grid_encode_forward(const float *inputs, const float *embeddings, const int32_t *offsets,
                             float *outputs, uint32_t B, uint32_t D, uint32_t C, uint32_t L,
                             float S, uint32_t H, int calc_grad_inputs, float *dy_dx,
                             uint32_t gridtype, int align_corners, const float *level_scales)
{
#pragma omp parallel for schedule(static)
    for (int64_t bl = 0; bl < (int64_t)B * L; bl++) {
        const uint32_t level = (uint32_t)(bl / B);
        const uint32_t b = (uint32_t)(bl % B);
        const float *grid = embeddings + (size_t)(uint32_t)offsets[level] * C;
        const float *x = inputs + (size_t)b * D;
        float *out = outputs + ((size_t)level * B + b) * C;
        float *dd = calc_grad_inputs ? dy_dx + ((size_t)b * L + level) * D * C : NULL;

        int oob = 0;
        for (uint32_t d = 0; d < D; d++)
            if (x[d] < 0 || x[d] > 1) oob = 1;
        if (oob) {
            for (uint32_t c = 0; c < C; c++) out[c] = 0;
            if (dd) memset(dd, 0, sizeof(float) * D * C);
            continue;
        }
        const uint32_t hashmap_size = (uint32_t)(offsets[level + 1] - offsets[level]);
        /* level_scales (optional) overrides exp2f(): CUDA's exp2f may differ from libm's by 1 ulp,
           which moves samples by ~1e-4 cells at the finest level; tests pass device-computed values */
        const float scale = level_scales ? level_scales[level] : exp2f((float)level * S) * (float)H - 1.0f;
        const uint32_t resolution = (uint32_t)ceilf(scale) + 1;

        float pos[SDO_MAX_D];
        uint32_t pg[SDO_MAX_D];
        for (uint32_t d = 0; d < D; d++) {
            /* device code contracts x*scale + 0.5f into one FFMA */
            pos[d] = fmaf(x[d], scale, align_corners ? 0.0f : 0.5f);
            pg[d] = (uint32_t)floorf(pos[d]);
            pos[d] -= (float)pg[d];
        }
        float res[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (uint32_t idx = 0; idx < (1u << D); idx++) {
            float w = 1;
            uint32_t pl[SDO_MAX_D];
            for (uint32_t d = 0; d < D; d++) {
                if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                else { w *= pos[d]; pl[d] = pg[d] + 1; }
            }
            const uint32_t index = grid_index(D, C, gridtype, align_corners, hashmap_size, resolution, pl);
            for (uint32_t c = 0; c < C; c++) res[c] = fmaf(w, grid[index + c], res[c]);
        }
        for (uint32_t c = 0; c < C; c++) out[c] = res[c];

        if (dd) {
            for (uint32_t gd = 0; gd < D; gd++) {
                float rg[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                for (uint32_t idx = 0; idx < (1u << (D - 1)); idx++) {
                    float w = scale;
                    uint32_t pl[SDO_MAX_D];
                    for (uint32_t nd = 0; nd < D - 1; nd++) {
                        const uint32_t d = (nd >= gd) ? (nd + 1) : nd;
                        if ((idx & (1u << nd)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                        else { w *= pos[d]; pl[d] = pg[d] + 1; }
                    }
                    pl[gd] = pg[gd];
                    const uint32_t il = grid_index(D, C, gridtype, align_corners, hashmap_size, resolution, pl);
                    pl[gd] = pg[gd] + 1;
                    const uint32_t ir = grid_index(D, C, gridtype, align_corners, hashmap_size, resolution, pl);
                    for (uint32_t c = 0; c < C; c++) rg[c] = fmaf(w, grid[ir + c] - grid[il + c], rg[c]);
                }
                for (uint32_t c = 0; c < C; c++) dd[gd * C + c] = rg[c];
            }
        }
    }
}

/* grad: [L,B,C]; grad_embeddings pre-zeroed [sum T, C]; grad_inputs [B,D] (written iff calc) */
void sdo_grid_encode_backward(const float *grad, const float *inputs, const float *embeddings,
                              const int32_t *offsets, float *grad_embeddings, uint32_t B, uint32_t D,
                              uint32_t C, uint32_t L, float S, uint32_t H, int calc_grad_inputs,
                              const float *dy_dx, float *grad_inputs, uint32_t gridtype, int align_corners,
                              const float *level_scales)
{
    (void)embeddings;
    /* levels write disjoint slices of grad_embeddings -> parallel over levels is race-free */
#pragma omp parallel for schedule(dynamic, 1)
    for (int level = 0; level < (int)L; level++) {
        float *gg = grad_embeddings + (size_t)(uint32_t)offsets[level] * C;
        const uint32_t hashmap_size = (uint32_t)(offsets[level + 1] - offsets[level]);
        const float scale = level_scales ? level_scales[level] : exp2f((float)level * S) * (float)H - 1.0f;
        const uint32_t resolution = (uint32_t)ceilf(scale) + 1;
        for (uint32_t b = 0; b < B; b++) {
            const float *x = inputs + (size_t)b * D;
            const float *g = grad + ((size_t)level * B + b) * C;
            int oob = 0;
            for (uint32_t d = 0; d < D; d++)
                if (x[d] < 0 || x[d] > 1) oob = 1;
            if (oob) continue;
            float pos[SDO_MAX_D];
            uint32_t pg[SDO_MAX_D];
            for (uint32_t d = 0; d < D; d++) {
                pos[d] = fmaf(x[d], scale, align_corners ? 0.0f : 0.5f);
                pg[d] = (uint32_t)floorf(pos[d]);
                pos[d] -= (float)pg[d];
            }
            for (uint32_t idx = 0; idx < (1u << D); idx++) {
                float w = 1;
                uint32_t pl[SDO_MAX_D];
                for (uint32_t d = 0; d < D; d++) {
                    if ((idx & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                const uint32_t index = grid_index(D, C, gridtype, align_corners, hashmap_size, resolution, pl);
                for (uint32_t c = 0; c < C; c++) gg[index + c] += w * g[c];
            }
        }
    }
    if (calc_grad_inputs) {
#pragma omp parallel for schedule(static)
        for (int64_t t = 0; t < (int64_t)B * D; t++) {
            const uint32_t b = (uint32_t)(t / D), d = (uint32_t)(t % D);
            const float *dd = dy_dx + (size_t)b * L * D * C;
            float r = 0;
            for (uint32_t l = 0; l < L; l++)
                for (uint32_t c = 0; c < C; c++)
                    r = fmaf(grad[((size_t)l * B + b) * C + c], dd[(l * D + d) * C + c], r);
            grad_inputs[t] = r;
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * Positional encoding along one dimension.
 * Follows voxlib/positional_encoding_kernel.cu:40-75 (forward), :77-118 (backward) and the
 * pure-PyTorch statement in voxlib/positional_encoding.py:45-54.
 * in [pre, post]; out [pre, stride, post] with stride = 2*ndeg (+1 if incl_orig):
 * channel blocks ordered sin_0, cos_0, sin_1, cos_1, ..., (orig).
 * ------------------------------------------------------------------------------------------ */
void sdo_positional_encoding(const float *in, float *out, int64_t pre, int64_t post, int ndeg, int incl_orig)
{
    const int stride = 2 * ndeg + (incl_orig ? 1 : 0);
#pragma omp parallel for schedule(static)
    for (int64_t e = 0; e < pre; e++) {
        for (int64_t f = 0; f < post; f++) {
            const float x = in[e * post + f];
            for (int i = 0; i < ndeg; i++) {
                const float rad = x * 3.14159265358979323846f * exp2f((float)i);
                out[(e * stride + 2 * i) * post + f] = sinf(rad);
                out[(e * stride + 2 * i + 1) * post + f] = cosf(rad);
            }
            if (incl_orig) out[(e * stride + stride - 1) * post + f] = x;
        }
    }
}

void sdo_positional_encoding_backward(const float *out_grad, const float *out, float *in_grad,
                                      int64_t pre, int64_t post, int ndeg, int incl_orig)
{
    const int stride = 2 * ndeg + (incl_orig ? 1 : 0);
#pragma omp parallel for schedule(static)
    for (int64_t e = 0; e < pre; e++) {
        for (int64_t f = 0; f < post; f++) {
            float g = 0.0f;
            for (int i = 0; i < ndeg; i++) {
                float gt = out_grad[(e * stride + 2 * i) * post + f] * out[(e * stride + 2 * i + 1) * post + f];
                gt -= out_grad[(e * stride + 2 * i + 1) * post + f] * out[(e * stride + 2 * i) * post + f];
                g += gt * 3.14159265358979323846f * exp2f((float)i);
            }
            if (incl_orig) g += out_grad[(e * stride + stride - 1) * post + f];
            in_grad[e * post + f] = g;
        }
    }
}

int sdo_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
