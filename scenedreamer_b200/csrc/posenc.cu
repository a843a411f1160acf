// a9: positional encoding along one dimension, forward + backward, sm_90a.
//
// Behavioural contract = voxlib.positional_encoding / positional_encoding_backward of the reference
// (voxlib/positional_encoding_kernel.cu:40-75 forward, :77-118 backward, :125-285 wrappers):
// in viewed as [pre, post] -> out [pre, stride, post] with channel blocks sin_0, cos_0, ...,
// sin_{n-1}, cos_{n-1}, (orig); rad = x * pi * 2^i.
// Purely bandwidth bound (1 read, stride writes): one thread per input element, `post` is the
// fastest-varying index so every one of the `stride` stores of a warp is a coalesced row.
#include "common.cuh"

namespace {

constexpr float kPi = 3.14159265358979323846f;

__global__ void __launch_bounds__(256)
pe_forward_kernel(float *__restrict__ out, const float *__restrict__ in, long long pre, long long post, int ndeg,
                  bool incl_orig)
{
    const long long n = pre * post;
    const int stride = 2 * ndeg + (incl_orig ? 1 : 0);
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n;
         t += (long long)gridDim.x * blockDim.x) {
        const long long e = t / post, f = t - e * post;
        const float x = in[t];
        float *o = out + e * stride * post + f;
        for (int i = 0; i < ndeg; i++) {
            const float rad = x * kPi * exp2f((float)i);
            float s, c;
            sincosf(rad, &s, &c);
            o[(2 * i) * post] = s;
            o[(2 * i + 1) * post] = c;
        }
        if (incl_orig) o[(long long)(stride - 1) * post] = x;
    }
}

__global__ void __launch_bounds__(256)
pe_backward_kernel(float *__restrict__ in_grad, const float *__restrict__ out_grad, const float *__restrict__ outp,
                   long long pre, long long post, int ndeg, bool incl_orig)
{
    const long long n = pre * post;
    const int stride = 2 * ndeg + (incl_orig ? 1 : 0);
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n;
         t += (long long)gridDim.x * blockDim.x) {
        const long long e = t / post, f = t - e * post;
        const float *og = out_grad + e * stride * post + f;
        const float *o = outp + e * stride * post + f;
        float g = 0.0f;
        for (int i = 0; i < ndeg; i++) {
            float gt = og[(2 * i) * post] * o[(2 * i + 1) * post];
            gt -= og[(2 * i + 1) * post] * o[(2 * i) * post];
            g += gt * kPi * exp2f((float)i);
        }
        if (incl_orig) g += og[(long long)(stride - 1) * post];
        in_grad[t] = g;
    }
}

int pe_grid(long long n) {
    long long blocks = (n + 255) / 256;
    const long long cap = (long long)sdb_num_sms() * 16;
    return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

}  // namespace

extern "C" int sdb_positional_encoding(const float *d_in, float *d_out, int64_t pre, int64_t post,
                                       int32_t ndegrees, int incl_orig, void *stream)
{
    if (!d_in || !d_out || pre < 0 || post <= 0 || ndegrees < 0) return SDB_EINVAL;
    if (pre == 0) return SDB_OK;
    pe_forward_kernel<<<pe_grid(pre * post), 256, 0, (cudaStream_t)stream>>>(d_out, d_in, pre, post, ndegrees,
                                                                             incl_orig != 0);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}

extern "C" int sdb_positional_encoding_backward(const float *d_out_grad, const float *d_out, float *d_in_grad,
                                                int64_t pre, int64_t post, int32_t ndegrees, int incl_orig,
                                                void *stream)
{
    if (!d_out_grad || !d_out || !d_in_grad || pre < 0 || post <= 0 || ndegrees < 0) return SDB_EINVAL;
    if (pre == 0) return SDB_OK;
    pe_backward_kernel<<<pe_grid(pre * post), 256, 0, (cudaStream_t)stream>>>(d_in_grad, d_out_grad, d_out, pre,
                                                                              post, ndegrees, incl_orig != 0);
    SDB_CHECK_LAUNCH();
    return SDB_OK;
}
