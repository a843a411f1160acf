// f2: the Adam step of the hash table in ONE pass.
// Behavioural contract: torch.optim.Adam as the reference builds it for `hash_encoder.embeddings`
// (imaginaire/utils/trainer.py:297-323 with configs/scenedreamer_train.yaml:36-61: lr 1e-4, eps 1e-7, betas (0, 0.999), no
// weight decay, no amsgrad), i.e. per element, with t the step count after the increment:
//     m = beta1 m + (1 - beta1) g ;  v = beta2 v + (1 - beta2) g^2
//     p = p - (lr / (1 - beta1^t)) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
// The table has 67 M entries of which a training view touches a few per cent: the reference's optimiser makes ~10 passes
// over four 268 MB arrays.  Here: one kernel, one pass; g is read once; with beta1 == 0 (the reference's setting) an entry
// whose gradient is exactly zero needs neither p nor m read: m := g = 0, p unchanged (the update is 0 / (..) = 0), only v
// decays -- bit for bit what the dense formula gives.  Result state (p, exp_avg, exp_avg_sq) is what torch's Adam would hold,
// so checkpoints stay interchangeable.  Bound: HBM, 12 B (beta1 == 0) to 28 B per entry.
#include "common.cuh"

namespace {

// omb1 / omb2 = (1 - beta) evaluated in double on the host and then narrowed, like torch's Python-float scalars
// (1.0f - 0.999f differs from float(1 - 0.999) by 1.3e-5 relative)
__device__ __forceinline__ float adam_one(float &p, float g, float &m, float &v, float b1, float b2, float omb1, float omb2,
                                          float step_size, float bc2_sqrt, float eps) {
    // exp_avg.lerp_(grad, 1 - beta1) with ATen's formula: w < 0.5 ? m + w (g - m) : g - (g - m)(1 - w)
    {
        const float diff = g - m;
        m = (fabsf(omb1) < 0.5f) ? __fmaf_rn(omb1, diff, m) : g - diff * (1.0f - omb1);
    }
    v = __fmaf_rn(b2, v, (omb2 * g) * g);                        // mul_(beta2).addcmul_(g, g, value = 1 - beta2)
    const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), bc2_sqrt), eps);   // (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps)
    p = __fmaf_rn(-step_size, __fdiv_rn(m, denom), p);           // addcdiv_(m, denom, value = -step_size)
    return p;
}

template <bool B1ZERO>
__global__ void __launch_bounds__(256)
adam_table_kernel(float4 *__restrict__ p, const float4 *__restrict__ g, float4 *__restrict__ m, float4 *__restrict__ v,
                  long long n4, float b1, float b2, float omb1, float omb2, float step_size, float bc2_sqrt, float eps)
{
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 gg = __ldg(g + i);
        float4 vv = v[i];
        if (B1ZERO && gg.x == 0.0f && gg.y == 0.0f && gg.z == 0.0f && gg.w == 0.0f) {
            // untouched entries: m = g = 0, p -= lr * 0 / (..) = p, v decays
            vv.x *= b2; vv.y *= b2; vv.z *= b2; vv.w *= b2;
            v[i] = vv;
            m[i] = gg;
            continue;
        }
        float4 pp = p[i];
        float4 mm = B1ZERO ? make_float4(0.0f, 0.0f, 0.0f, 0.0f) : m[i];
        adam_one(pp.x, gg.x, mm.x, vv.x, b1, b2, omb1, omb2, step_size, bc2_sqrt, eps);
        adam_one(pp.y, gg.y, mm.y, vv.y, b1, b2, omb1, omb2, step_size, bc2_sqrt, eps);
        adam_one(pp.z, gg.z, mm.z, vv.z, b1, b2, omb1, omb2, step_size, bc2_sqrt, eps);
        adam_one(pp.w, gg.w, mm.w, vv.w, b1, b2, omb1, omb2, step_size, bc2_sqrt, eps);
        p[i] = pp;
        m[i] = mm;
        v[i] = vv;
    }
}
}  // namespace

// n must be a multiple of 4 and the arrays 16-byte aligned (the table is [rows, 8] fp32).  `step` = the step count AFTER the
// increment (1 on the first call), exactly torch's state['step'].
extern "C" int sdb_adam_step(float *d_param, const float *d_grad, float *d_exp_avg, float *d_exp_avg_sq, int64_t n, double lr,
                             double beta1d, double beta2d, double epsd, int64_t step, void *stream)
{
    if (!d_param || !d_grad || !d_exp_avg || !d_exp_avg_sq || n <= 0 || (n & 3) || step < 1) return SDB_EINVAL;
    if (((uintptr_t)d_param | (uintptr_t)d_grad | (uintptr_t)d_exp_avg | (uintptr_t)d_exp_avg_sq) & 15) return SDB_EINVAL;
    // scalar bookkeeping in double like torch's Python floats (torch/optim/adam.py: _single_tensor_adam), narrowed last
    const double bc1 = 1.0 - pow(beta1d, (double)step), bc2 = 1.0 - pow(beta2d, (double)step);
    const float step_size = (float)(lr / bc1), bc2_sqrt = (float)sqrt(bc2);
    const float beta1 = (float)beta1d, beta2 = (float)beta2d, eps = (float)epsd;
    const float omb1 = (float)(1.0 - beta1d), omb2 = (float)(1.0 - beta2d);
    const long long n4 = n / 4;
    const long long want = (n4 + 255) / 256, cap = (long long)sdb_num_sms() * 16;
    const int grid = (int)(want < cap ? want : cap);
    if (beta1d == 0.0)
        adam_table_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>((float4 *)d_param, (const float4 *)d_grad, (float4 *)d_exp_avg,
                                                                       (float4 *)d_exp_avg_sq, n4, beta1, beta2, omb1, omb2, step_size, bc2_sqrt, eps);
    else
        adam_table_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>((float4 *)d_param, (const float4 *)d_grad, (float4 *)d_exp_avg,
                                                                        (float4 *)d_exp_avg_sq, n4, beta1, beta2, omb1, omb2, step_size, bc2_sqrt, eps);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}
