// Loss, metric and optimiser kernels for the training loop (robosat/losses.py, robosat/metrics.py,
// torch.optim.Adam as used by robosat/tools/train.py:81,188). All HBM-bound integer / elementwise work:
// one pass per tensor where the algorithm allows, warp-shuffle reductions, one atomic per block.

#include <cuda_fp16.h>
#include <math.h>

#include "../../include/rsb200.h"
#include "rsb_host.h"

namespace rsb {

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// A label outside [0, C) (a stray palette index in a label PNG) must never become an index: weight[t] and logits[t * HW] would read
// out of bounds. Such a pixel is left out of every sum and gets a zero gradient, as if the image did not contain it. `rs train`
// rejects these labels on the host (tools/train.py: check_mask_range), so this is the second line of defence, not the report.
__device__ __forceinline__ bool target_in_range(int64_t t, int C) { return t >= 0 && t < static_cast<int64_t>(C); }

// =================================================================================================
// CrossEntropyLoss2d (losses.py:24-25): NLLLoss(weight)(log_softmax(x, dim=1), t), reduction = weighted mean
// =================================================================================================
__global__ void ce_reduce_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets,
                                 const float* __restrict__ weight, double* __restrict__ scratch, int N, int C, int64_t HW) {
    const int64_t total = static_cast<int64_t>(N) * HW;
    double num = 0.0, den = 0.0;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        if (!target_in_range(targets[i], C)) continue;
        const int64_t n = i / HW, pix = i % HW;
        const float* l = logits + n * C * HW + pix;
        float m = l[0];
        for (int c = 1; c < C; ++c) m = fmaxf(m, l[c * HW]);
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += expf(l[c * HW] - m);
        const int t = static_cast<int>(targets[i]);
        const float logp = (l[static_cast<int64_t>(t) * HW] - m) - logf(s);
        const float w = weight ? weight[t] : 1.0f;
        num += static_cast<double>(-logp * w);
        den += static_cast<double>(w);
    }
    num = warp_sum(num);
    den = warp_sum(den);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&scratch[0], num);
        atomicAdd(&scratch[1], den);
    }
}

__global__ void ce_finish_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets,
                                 const float* __restrict__ weight, const double* __restrict__ scratch,
                                 float* __restrict__ loss_out, float* __restrict__ grad, int N, int C, int64_t HW) {
    const double den = scratch[1];
    if (blockIdx.x == 0 && threadIdx.x == 0) *loss_out = static_cast<float>(scratch[0] / den);
    if (!grad) return;
    const float inv_den = static_cast<float>(1.0 / den);
    const int64_t total = static_cast<int64_t>(N) * HW;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t n = i / HW, pix = i % HW;
        const float* l = logits + n * C * HW + pix;
        float* g = grad + n * C * HW + pix;
        if (!target_in_range(targets[i], C)) {
            for (int c = 0; c < C; ++c) g[c * HW] = 0.0f;
            continue;
        }
        float m = l[0];
        for (int c = 1; c < C; ++c) m = fmaxf(m, l[c * HW]);
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += expf(l[c * HW] - m);
        const int t = static_cast<int>(targets[i]);
        const float w = (weight ? weight[t] : 1.0f) * inv_den;
        for (int c = 0; c < C; ++c) {
            const float p = expf(l[c * HW] - m) / s;
            g[c * HW] = w * (p - (c == t ? 1.0f : 0.0f));
        }
    }
}

// =================================================================================================
// FocalLoss2d (losses.py:49-50): NLLLoss(weight)((1 - softmax)^gamma * log_softmax, t), weighted mean.
// d/dx_c of f = (1-p_t)^gamma * log p_t  is  (delta_tc - p_c) * [(1-p_t)^gamma - gamma (1-p_t)^(gamma-1) p_t log p_t]
// =================================================================================================
__global__ void focal_reduce_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets, const float* __restrict__ weight,
                                    double* __restrict__ scratch, float gamma, int N, int C, int64_t HW) {
    const int64_t total = static_cast<int64_t>(N) * HW;
    double num = 0.0, den = 0.0;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        if (!target_in_range(targets[i], C)) continue;
        const int64_t n = i / HW, pix = i % HW;
        const float* l = logits + n * C * HW + pix;
        float m = l[0];
        for (int c = 1; c < C; ++c) m = fmaxf(m, l[c * HW]);
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += expf(l[c * HW] - m);
        const int t = static_cast<int>(targets[i]);
        const float logp = (l[static_cast<int64_t>(t) * HW] - m) - logf(s);
        const float pt = expf(l[static_cast<int64_t>(t) * HW] - m) / s;
        const float w = weight ? weight[t] : 1.0f;
        num += static_cast<double>(-powf(1.0f - pt, gamma) * logp * w);
        den += static_cast<double>(w);
    }
    num = warp_sum(num);
    den = warp_sum(den);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&scratch[0], num);
        atomicAdd(&scratch[1], den);
    }
}

__global__ void focal_finish_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets, const float* __restrict__ weight,
                                    const double* __restrict__ scratch, float* __restrict__ loss_out, float* __restrict__ grad, float gamma,
                                    int N, int C, int64_t HW) {
    const double den = scratch[1];
    if (blockIdx.x == 0 && threadIdx.x == 0) *loss_out = static_cast<float>(scratch[0] / den);
    if (!grad) return;
    const float inv_den = static_cast<float>(1.0 / den);
    const int64_t total = static_cast<int64_t>(N) * HW;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t n = i / HW, pix = i % HW;
        const float* l = logits + n * C * HW + pix;
        float* g = grad + n * C * HW + pix;
        if (!target_in_range(targets[i], C)) {
            for (int c = 0; c < C; ++c) g[c * HW] = 0.0f;
            continue;
        }
        float m = l[0];
        for (int c = 1; c < C; ++c) m = fmaxf(m, l[c * HW]);
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += expf(l[c * HW] - m);
        const int t = static_cast<int>(targets[i]);
        const float logp = (l[static_cast<int64_t>(t) * HW] - m) - logf(s);
        const float pt = expf(l[static_cast<int64_t>(t) * HW] - m) / s;
        const float q = 1.0f - pt;
        // gamma == 0: the penalty is the constant 1 and its derivative term is zero, as in torch's pow backward (exponent 0
        // gives a zero gradient). Evaluated, it would be 0 * powf(0, -1) = 0 * inf = NaN wherever softmax saturates to p_t = 1.
        // q == 0 (softmax saturated at the target, so log p_t == 0 too): the term's limit is 0 for every gamma > 0, since
        // q^(gamma-1) log p_t ~ -q^gamma. Evaluated for gamma < 1 it is inf * 0 = NaN.
        const float dpen = (gamma == 0.0f || q == 0.0f) ? 0.0f : gamma * powf(q, gamma - 1.0f) * pt * logp;
        const float k = powf(q, gamma) - dpen;
        const float w = -(weight ? weight[t] : 1.0f) * inv_den * k;
        for (int c = 0; c < C; ++c) {
            const float p = expf(l[c * HW] - m) / s;
            g[c * HW] = w * ((c == t ? 1.0f : 0.0f) - p);
        }
    }
}

// =================================================================================================
// mIoULoss2d (losses.py:71-83): miou = 1 - mean_{c,n}( sum_hw softs*masks / sum_hw (softs + masks - softs*masks) ),
// returned value = max(miou, weighted cross entropy): both are computed on the device and the larger one selects
// which gradient the final pass writes (the reference's Python max() picks one of the two tensors).
// sums[(n*C + c)*2 + {0,1}] = {intersection, union}; scratch[0..1] = CE numerator / denominator
// =================================================================================================
__global__ void miou_reduce_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets, const float* __restrict__ weight,
                                   double* __restrict__ sums, double* __restrict__ scratch, int C, int64_t HW) {
    const int n = blockIdx.y;
    extern __shared__ double sh[];  // [C][2]
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) sh[i] = 0.0;
    __syncthreads();
    double num = 0.0, den = 0.0;
    for (int64_t pix = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; pix < HW; pix += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        if (!target_in_range(targets[static_cast<int64_t>(n) * HW + pix], C)) continue;  // in neither the soft IoU sums nor the cross entropy
        const float* l = logits + static_cast<int64_t>(n) * C * HW + pix;
        float m = l[0];
        for (int c = 1; c < C; ++c) m = fmaxf(m, l[c * HW]);
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += expf(l[c * HW] - m);
        const int t = static_cast<int>(targets[static_cast<int64_t>(n) * HW + pix]);
        for (int c = 0; c < C; ++c) {
            const float p = expf(l[c * HW] - m) / s;
            if (c == t) {
                atomicAdd(&sh[2 * c], static_cast<double>(p));   // inters: softs * masks
                atomicAdd(&sh[2 * c + 1], 1.0);                  // unions: softs + 1 - softs
            } else {
                atomicAdd(&sh[2 * c + 1], static_cast<double>(p));
            }
        }
        const float logp = (l[static_cast<int64_t>(t) * HW] - m) - logf(s);
        const float w = weight ? weight[t] : 1.0f;
        num += static_cast<double>(-logp * w);
        den += static_cast<double>(w);
    }
    num = warp_sum(num);
    den = warp_sum(den);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&scratch[0], num);
        atomicAdd(&scratch[1], den);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) atomicAdd(&sums[static_cast<int64_t>(n) * C * 2 + i], sh[i]);
}

__global__ void miou_select_kernel(const double* __restrict__ sums, double* __restrict__ scratch, float* __restrict__ loss_out, int N, int C) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        // (inters.sum / unions.sum).mean() in fp32 like the reference
        float acc = 0.f;
        for (int i = 0; i < N * C; ++i) acc += static_cast<float>(sums[2 * i]) / static_cast<float>(sums[2 * i + 1]);
        const float miou = 1.0f - acc / static_cast<float>(N * C);
        const float ce = static_cast<float>(scratch[0] / scratch[1]);
        // Python's max(miou, ce) returns ce only when ce > miou
        scratch[2] = ce > miou ? 0.0 : 1.0;
        *loss_out = ce > miou ? ce : miou;
    }
}

__global__ void miou_grad_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets, const float* __restrict__ weight,
                                 const double* __restrict__ sums, const double* __restrict__ scratch, float* __restrict__ grad, int N, int C,
                                 int64_t HW) {
    const bool use_miou = scratch[2] > 0.5;
    const float inv_den = static_cast<float>(1.0 / scratch[1]);
    const float inv_cn = 1.0f / static_cast<float>(N * C);
    const int64_t total = static_cast<int64_t>(N) * HW;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t n = i / HW, pix = i % HW;
        const float* l = logits + n * C * HW + pix;
        float* g = grad + n * C * HW + pix;
        if (!target_in_range(targets[i], C)) {
            for (int c = 0; c < C; ++c) g[c * HW] = 0.0f;
            continue;
        }
        float m = l[0];
        for (int c = 1; c < C; ++c) m = fmaxf(m, l[c * HW]);
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += expf(l[c * HW] - m);
        const int t = static_cast<int>(targets[i]);
        if (!use_miou) {
            const float w = (weight ? weight[t] : 1.0f) * inv_den;
            for (int c = 0; c < C; ++c) g[c * HW] = w * (expf(l[c * HW] - m) / s - (c == t ? 1.0f : 0.0f));
        } else {
            // d miou / d s_c = -(1/CN) * [ m_c / U - I (1 - m_c) / U^2 ];  dx_k = s_k (ds_k - sum_c ds_c s_c)
            // I / U^2 as (I / U) / U, like torch's div backward: the union of a class that is absent from the image and has
            // subnormal probabilities is so small that U * U underflows to 0, and 0 / 0 would put NaN into the whole image
            float dot = 0.f;
            for (int c = 0; c < C; ++c) {
                const float I = static_cast<float>(sums[(n * C + c) * 2]), U = static_cast<float>(sums[(n * C + c) * 2 + 1]);
                const float ds = -inv_cn * (c == t ? 1.0f / U : -(I / U) / U);
                dot += ds * (expf(l[c * HW] - m) / s);
            }
            for (int c = 0; c < C; ++c) {
                const float I = static_cast<float>(sums[(n * C + c) * 2]), U = static_cast<float>(sums[(n * C + c) * 2 + 1]);
                const float ds = -inv_cn * (c == t ? 1.0f / U : -(I / U) / U);
                const float p = expf(l[c * HW] - m) / s;
                g[c * HW] = p * (ds - dot);
            }
        }
    }
}

// =================================================================================================
// Metrics.add (metrics.py:27-41) over a batch
// =================================================================================================
__global__ void metrics_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets,
                               unsigned long long* __restrict__ counts, int N, int C, int64_t HW) {
    const int64_t total = static_cast<int64_t>(N) * HW;
    unsigned long long tn = 0, fn = 0, fp = 0, tp = 0;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t n = i / HW, pix = i % HW;
        const float* l = logits + n * C * HW + pix;
        int m = 0;
        float best = l[0];
        for (int c = 1; c < C; ++c) {
            const float v = l[c * HW];
            if (v > best) {  // first maximum wins, like torch.argmax
                best = v;
                m = c;
            }
        }
        const int64_t a = targets[i];
        // confusion = float(m) / float(a): NaN (0/0) -> tn, inf (m>0, a=0) -> fn, 0 (m=0, a>0) -> fp, 1 (m==a>0) -> tp
        if (a == 0) {
            if (m == 0) ++tn; else ++fn;
        } else {
            const float q = static_cast<float>(m) / static_cast<float>(a);
            if (q == 0.0f) ++fp;
            else if (q == 1.0f) ++tp;
        }
    }
    tn = warp_sum_u64(tn);
    fn = warp_sum_u64(fn);
    fp = warp_sum_u64(fp);
    tp = warp_sum_u64(tp);
    if ((threadIdx.x & 31) == 0) {
        if (tn) atomicAdd(&counts[0], tn);
        if (fn) atomicAdd(&counts[1], fn);
        if (fp) atomicAdd(&counts[2], fp);
        if (tp) atomicAdd(&counts[3], tp);
    }
}

// =================================================================================================
// Adam (torch.optim.Adam single-tensor step, amsgrad=False, weight_decay=0, maximize=False)
// =================================================================================================
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            int64_t n, float beta1, float beta2, float one_minus_beta1, float one_minus_beta2, float step_size,
                            float bc2_sqrt, float eps) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float gi = g[i];
        float mi = m[i], vi = v[i];
        mi = mi + one_minus_beta1 * (gi - mi);            // exp_avg.lerp_(grad, 1 - beta1)
        vi = vi * beta2 + one_minus_beta2 * (gi * gi);    // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
        const float denom = sqrtf(vi) / bc2_sqrt + eps;   // (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps)
        p[i] = p[i] - step_size * (mi / denom);           // param.addcdiv_(exp_avg, denom, value=-step_size)
        m[i] = mi;
        v[i] = vi;
    }
}

// Guarded variant (mixed-precision training): activation gradients are fp16 under a loss scale, so one overflowing batch puts
// inf / NaN into the flat gradient arena -- and from there, permanently, into exp_avg, exp_avg_sq and the weights. The guard is
// three launches on the same stream and no host synchronisation:
//   state[0]  this step's "gradients are not finite" flag (set by grad_finite_kernel)
//   state[1]  number of skipped steps so far (bias corrections use step - skipped, like a GradScaler-wrapped torch.optim.Adam)
//   state[2]  flag of the most recent finished step (what the host polls, asynchronously, to adapt the loss scale)
//   state[3]  steps seen
__global__ void grad_finite_kernel(const float* __restrict__ g, int64_t n, int32_t* __restrict__ state) {
    bool bad = false;
    const int64_t n4 = (reinterpret_cast<uintptr_t>(g) & 15) ? 0 : n / 4;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float4 x = reinterpret_cast<const float4*>(g)[i];
        bad |= !(fabsf(x.x) <= 3.402823466e38f) | !(fabsf(x.y) <= 3.402823466e38f) | !(fabsf(x.z) <= 3.402823466e38f) | !(fabsf(x.w) <= 3.402823466e38f);
    }
    for (int64_t i = 4 * n4 + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float x = g[i];
        bad |= !(fabsf(x) <= 3.402823466e38f);  // inf or NaN
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(&state[0], 1);
}

__global__ void adam_guarded_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, int64_t n,
                                    float beta1, float beta2, float one_minus_beta1, float one_minus_beta2, float lr, float step_size_host,
                                    float bc2_sqrt_host, float eps, int step, const int32_t* __restrict__ state) {
    if (state[0]) return;  // skip the whole update: parameters and both moments stay untouched
    float step_size = step_size_host, bc2_sqrt = bc2_sqrt_host;
    if (state[1] > 0) {  // earlier steps were skipped: bias corrections count the steps actually taken
        const int eff = step - state[1];
        step_size = static_cast<float>(static_cast<double>(lr) / (1.0 - pow(static_cast<double>(beta1), eff)));
        bc2_sqrt = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(beta2), eff)));
    }
    // four parameters per thread and iteration through 16-byte loads / stores (the arenas are 256-byte aligned torch allocations);
    // per element the arithmetic is exactly adam_kernel's
    auto upd = [&](float& pi, float gi, float& mi, float& vi) {
        mi = mi + one_minus_beta1 * (gi - mi);
        vi = vi * beta2 + one_minus_beta2 * (gi * gi);
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        pi = pi - step_size * (mi / denom);
    };
    const int64_t n4 = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) ? 0 : n / 4;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        float4 p4 = reinterpret_cast<float4*>(p)[i], m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i];
        const float4 g4 = reinterpret_cast<const float4*>(g)[i];
        upd(p4.x, g4.x, m4.x, v4.x);
        upd(p4.y, g4.y, m4.y, v4.y);
        upd(p4.z, g4.z, m4.z, v4.z);
        upd(p4.w, g4.w, m4.w, v4.w);
        reinterpret_cast<float4*>(p)[i] = p4;
        reinterpret_cast<float4*>(m)[i] = m4;
        reinterpret_cast<float4*>(v)[i] = v4;
    }
    for (int64_t i = 4 * n4 + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        float pi = p[i], mi = m[i], vi = v[i];
        upd(pi, g[i], mi, vi);
        p[i] = pi;
        m[i] = mi;
        v[i] = vi;
    }
}

__global__ void adam_guard_bookkeep_kernel(int32_t* state) {
    state[2] = state[0];
    if (state[0]) state[1] += 1;
    state[3] += 1;
    state[0] = 0;
}

// =================================================================================================
// LovaszLoss2d (losses.py:96-119): per image a descending sort of P = C*H*W margin errors, then the
// Jaccard-gradient weights from two cumulative sums and dot(relu(errors_sorted), J).
//
// Pipeline per call (all images at once, segment = image):
//   keys    e = 1 - (2*onehot - 1) * x  -> order-preserving uint32 key (inverted for descending), payload = index
//   sort    4 passes of a stable 8-bit LSD radix sort: per-tile digit histogram -> per-image exclusive scan over
//           (digit, tile) -> stable scatter (warp match_any ranking on top of per-warp digit counters)
//   scan    positives-per-tile -> per-image exclusive scan -> per element: cumsum, J_k, J_{k-1}, loss term, gradient
// cumsums are integers < 2^24 held exactly in fp32, so J matches the reference's fp32 arithmetic bit for bit;
// only the final dot product is accumulated differently (double).
// =================================================================================================
static constexpr int kSortThreads = 256;
static constexpr int kSortItems = 16;
static constexpr int kSortTile = kSortThreads * kSortItems;  // 4096 keys per block
static constexpr int kSortWarps = kSortThreads / 32;

__device__ __forceinline__ uint32_t desc_key(float e) {
    uint32_t b = __float_as_uint(e);
    b ^= (b >> 31) ? 0xFFFFFFFFu : 0x80000000u;  // ascending-orderable
    return ~b;                                    // ascending sort of ~key == descending sort of e
}
__device__ __forceinline__ float key_to_float(uint32_t k) {
    uint32_t b = ~k;
    b ^= (b >> 31) ? 0x80000000u : 0xFFFFFFFFu;
    return __uint_as_float(b);
}

__global__ void lovasz_keys_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets,
                                   uint32_t* __restrict__ keys, uint32_t* __restrict__ idx, int C, int64_t HW, int64_t P, int64_t Pp) {
    const int64_t n = blockIdx.y;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < Pp; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        uint32_t k = 0xFFFFFFFFu;  // padding sorts last
        if (i < P) {
            const int64_t c = i / HW, pix = i % HW;
            const float sign = (targets[n * HW + pix] == c) ? 1.0f : -1.0f;  // mask * 2 - 1
            const float e = 1.0f - sign * logits[n * P + i];                // max_margin_errors
            k = desc_key(e);
        }
        keys[n * Pp + i] = k;
        idx[n * Pp + i] = static_cast<uint32_t>(i);
    }
}

// per-tile digit histogram: hist[image][digit][tile]
__global__ void radix_hist_kernel(const uint32_t* __restrict__ keys, uint32_t* __restrict__ hist, int shift, int64_t Pp, int tiles) {
    __shared__ uint32_t sh[256];
    const int n = blockIdx.y, tile = blockIdx.x;
    sh[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t* k = keys + n * Pp + static_cast<int64_t>(tile) * kSortTile;
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) atomicAdd(&sh[(k[j * kSortThreads + threadIdx.x] >> shift) & 255u], 1u);
    __syncthreads();
    hist[(static_cast<int64_t>(n) * 256 + threadIdx.x) * tiles + tile] = sh[threadIdx.x];
}

// per-image exclusive scan over the 256*tiles counters (digit-major): one block per image
__global__ void radix_scan_kernel(uint32_t* __restrict__ hist, int tiles) {
    __shared__ uint32_t warp_tot[32];
    __shared__ uint32_t carry_s;
    uint32_t* h = hist + static_cast<int64_t>(blockIdx.x) * 256 * tiles;
    const int total = 256 * tiles;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < total; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const uint32_t v = i < total ? h[i] : 0;
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((threadIdx.x & 31) >= o) incl += t;
        }
        if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = incl;
        __syncthreads();
        if (threadIdx.x < 32) {
            const uint32_t w = threadIdx.x < (blockDim.x >> 5) ? warp_tot[threadIdx.x] : 0;
            uint32_t wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
                if (threadIdx.x >= o) wi += t;
            }
            warp_tot[threadIdx.x] = wi - w;  // exclusive prefix of warp totals
        }
        __syncthreads();
        const uint32_t carry = carry_s;
        if (i < total) h[i] = carry + warp_tot[threadIdx.x >> 5] + incl - v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry_s = carry + warp_tot[threadIdx.x >> 5] + incl;
        __syncthreads();
    }
}

// stable scatter of one tile: warp w owns the contiguous 512-key slice [w*512, w*512+512) of the tile
__global__ void radix_scatter_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ idx_in,
                                     uint32_t* __restrict__ keys_out, uint32_t* __restrict__ idx_out,
                                     const uint32_t* __restrict__ hist, int shift, int64_t Pp, int tiles) {
    __shared__ uint32_t cnt[kSortWarps][256];
    const int n = blockIdx.y, tile = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < kSortWarps * 256; i += blockDim.x) (&cnt[0][0])[i] = 0;
    __syncthreads();
    const int64_t base = n * Pp + static_cast<int64_t>(tile) * kSortTile + warp * (32 * kSortItems);
    uint32_t k[kSortItems], v[kSortItems];
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        k[j] = keys_in[base + j * 32 + lane];
        v[j] = idx_in[base + j * 32 + lane];
    }
    // per-warp digit counts
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        const uint32_t d = (k[j] >> shift) & 255u;
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        if (lane == (__ffs(peers) - 1)) cnt[warp][d] += __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    // turn counts into absolute output offsets: global base of (digit, tile) + earlier warps of this tile
    {
        const int d = threadIdx.x;  // 256 threads, one digit each
        uint32_t run = hist[(static_cast<int64_t>(n) * 256 + d) * tiles + tile];
#pragma unroll
        for (int w = 0; w < kSortWarps; ++w) {
            const uint32_t c = cnt[w][d];
            cnt[w][d] = run;
            run += c;
        }
    }
    __syncthreads();
    const int64_t obase = n * Pp;
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        const uint32_t d = (k[j] >> shift) & 255u;
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
        const uint32_t off = cnt[warp][d] + rank;
        __syncwarp();
        if (lane == (__ffs(peers) - 1)) cnt[warp][d] += __popc(peers);
        __syncwarp();
        keys_out[obase + off] = k[j];
        idx_out[obase + off] = v[j];
    }
}

// positives (label 1) per tile of the sorted order
__global__ void lovasz_tilepos_kernel(const uint32_t* __restrict__ idx, const int64_t* __restrict__ targets, uint32_t* __restrict__ tilepos,
                                      int64_t HW, int64_t P, int64_t Pp, int tiles) {
    __shared__ int sh[kSortWarps];
    const int n = blockIdx.y, tile = blockIdx.x;
    int c = 0;
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        const int64_t kpos = static_cast<int64_t>(tile) * kSortTile + j * kSortThreads + threadIdx.x;
        if (kpos < P) {
            const uint32_t i = idx[n * Pp + kpos];
            c += (targets[n * HW + (i % HW)] == static_cast<int64_t>(i / HW)) ? 1 : 0;
        }
    }
    c = warp_sum_i(c);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < kSortWarps; ++w) t += sh[w];
        tilepos[n * tiles + tile] = t;
    }
}

// exclusive scan of tilepos per image (tiles is small: P / 4096) and G = total positives
__global__ void lovasz_tilescan_kernel(uint32_t* __restrict__ tilepos, uint32_t* __restrict__ gts, int tiles) {
    if (threadIdx.x == 0) {
        uint32_t* t = tilepos + static_cast<int64_t>(blockIdx.x) * tiles;
        uint32_t run = 0;
        for (int i = 0; i < tiles; ++i) {
            const uint32_t v = t[i];
            t[i] = run;
            run += v;
        }
        gts[blockIdx.x] = run;
    }
}

__global__ void lovasz_final_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ idx,
                                    const int64_t* __restrict__ targets, const uint32_t* __restrict__ tilepos,
                                    const uint32_t* __restrict__ gts, double* __restrict__ loss_acc, float* __restrict__ grad,
                                    int64_t HW, int64_t P, int64_t Pp, int tiles, float inv_n) {
    // thread t owns the 16 consecutive sorted positions [tile*4096 + t*16, +16) so its local scan is sequential
    __shared__ int warp_tot[kSortWarps];
    const int n = blockIdx.y, tile = blockIdx.x;
    const int64_t k0 = static_cast<int64_t>(tile) * kSortTile + static_cast<int64_t>(threadIdx.x) * kSortItems;
    uint32_t id[kSortItems];
    int lab[kSortItems];
    int local = 0;
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        const int64_t kpos = k0 + j;
        lab[j] = 0;
        id[j] = 0;
        if (kpos < P) {
            id[j] = idx[n * Pp + kpos];
            lab[j] = (targets[n * HW + (id[j] % HW)] == static_cast<int64_t>(id[j] / HW)) ? 1 : 0;
        }
        local += lab[j];
    }
    // block exclusive scan of `local`
    int incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((threadIdx.x & 31) >= o) incl += t;
    }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = incl;
    __syncthreads();
    int wprefix = 0;
    for (int w = 0; w < (threadIdx.x >> 5); ++w) wprefix += warp_tot[w];
    int cs = static_cast<int>(tilepos[n * tiles + tile]) + wprefix + incl - local;  // positives strictly before k0
    const float G = static_cast<float>(gts[n]);
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        const int64_t kpos = k0 + j;
        if (kpos < P) {
            // J_{k-1} from the counts before this element, J_k including it (losses.py:109-115)
            float jprev = 0.0f;
            if (kpos > 0) {
                const float inter_p = G - static_cast<float>(cs);
                const float union_p = G + static_cast<float>(kpos - cs);
                jprev = 1.0f - inter_p / union_p;
            }
            cs += lab[j];
            const float inter = G - static_cast<float>(cs);
            const float uni = G + static_cast<float>(kpos + 1 - cs);
            const float jk = 1.0f - inter / uni;
            const float w = jk - jprev;
            const float e = key_to_float(keys[n * Pp + kpos]);
            if (e > 0.0f) {
                acc += static_cast<double>(e * w);
                if (grad) grad[n * P + id[j]] = (lab[j] ? -1.0f : 1.0f) * w * inv_n;  // -(2*mask-1) * J / N
            } else if (grad) {
                grad[n * P + id[j]] = 0.0f;
            }
        }
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0 && acc != 0.0) atomicAdd(&loss_acc[0], acc);
}

__global__ void lovasz_loss_out_kernel(const double* __restrict__ loss_acc, float* __restrict__ loss_out, float inv_n) {
    *loss_out = static_cast<float>(loss_acc[0] * static_cast<double>(inv_n));
}

static inline unsigned blocks_for(int64_t total, int block, int cap = 132 * 16) {
    int64_t b = (total + block - 1) / block;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return static_cast<unsigned>(b);
}

static inline int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

struct LovaszWs {
    int64_t Pp;
    int tiles;
    int64_t off_keys[2], off_idx[2], off_hist, off_tilepos, off_gts, off_loss, total;
};

static LovaszWs lovasz_layout(int N, int C, int64_t HW) {
    LovaszWs w;
    const int64_t P = static_cast<int64_t>(C) * HW;
    w.Pp = align_up(P, kSortTile);
    w.tiles = static_cast<int>(w.Pp / kSortTile);
    int64_t o = 0;
    for (int i = 0; i < 2; ++i) {
        w.off_keys[i] = o;
        o += align_up(4 * w.Pp * N, 256);
    }
    for (int i = 0; i < 2; ++i) {
        w.off_idx[i] = o;
        o += align_up(4 * w.Pp * N, 256);
    }
    w.off_hist = o;
    o += align_up(4LL * 256 * w.tiles * N, 256);
    w.off_tilepos = o;
    o += align_up(4LL * w.tiles * N, 256);
    w.off_gts = o;
    o += align_up(4LL * N, 256);
    w.off_loss = o;
    o += 256;
    w.total = o;
    return w;
}

}  // namespace rsb

using namespace rsb;

extern "C" int rsb_cross_entropy(const float* logits, const int64_t* targets, const float* weight, float* loss_out, float* grad,
                                 double* scratch, int32_t N, int32_t C, int32_t HW, void* stream) {
    if (!logits || !targets || !loss_out || !scratch || N <= 0 || C <= 0 || HW <= 0) return set_error(RSB_E_INVALID, "cross_entropy: bad arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(scratch, 0, 2 * sizeof(double), st);
    if (e != cudaSuccess) return set_cuda_error(e, "cross_entropy memset");
    const int64_t total = static_cast<int64_t>(N) * HW;
    ce_reduce_kernel<<<blocks_for(total, 256), 256, 0, st>>>(logits, targets, weight, scratch, N, C, HW);
    ce_finish_kernel<<<grad ? blocks_for(total, 256) : 1, 256, 0, st>>>(logits, targets, weight, scratch, loss_out, grad, N, C, HW);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "cross_entropy launch");
}

extern "C" int rsb_focal(const float* logits, const int64_t* targets, const float* weight, float gamma, float* loss_out, float* grad,
                         double* scratch, int32_t N, int32_t C, int32_t HW, void* stream) {
    if (!logits || !targets || !loss_out || !scratch || N <= 0 || C <= 0 || HW <= 0) return set_error(RSB_E_INVALID, "focal: bad arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(scratch, 0, 2 * sizeof(double), st);
    if (e != cudaSuccess) return set_cuda_error(e, "focal memset");
    const int64_t total = static_cast<int64_t>(N) * HW;
    focal_reduce_kernel<<<blocks_for(total, 256), 256, 0, st>>>(logits, targets, weight, scratch, gamma, N, C, HW);
    focal_finish_kernel<<<grad ? blocks_for(total, 256) : 1, 256, 0, st>>>(logits, targets, weight, scratch, loss_out, grad, gamma, N, C, HW);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "focal launch");
}

extern "C" int64_t rsb_miou_scratch_doubles(int32_t N, int32_t C) { return (N <= 0 || C <= 0) ? 0 : 4 + 2LL * N * C; }

extern "C" int rsb_miou(const float* logits, const int64_t* targets, const float* weight, float* loss_out, float* grad, double* scratch,
                        int32_t N, int32_t C, int32_t HW, void* stream) {
    if (!logits || !targets || !loss_out || !scratch || N <= 0 || C <= 0 || C > 64 || HW <= 0) return set_error(RSB_E_INVALID, "miou: bad arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemsetAsync(scratch, 0, (4 + 2LL * N * C) * sizeof(double), st);
    if (e != cudaSuccess) return set_cuda_error(e, "miou memset");
    double* sums = scratch + 4;
    miou_reduce_kernel<<<dim3(blocks_for(HW, 256, 64), N), 256, 2 * C * sizeof(double), st>>>(logits, targets, weight, sums, scratch, C, HW);
    miou_select_kernel<<<1, 32, 0, st>>>(sums, scratch, loss_out, N, C);
    if (grad) miou_grad_kernel<<<blocks_for(static_cast<int64_t>(N) * HW, 256), 256, 0, st>>>(logits, targets, weight, sums, scratch, grad, N, C, HW);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "miou launch");
}

extern "C" int rsb_metrics_count(const float* logits, const int64_t* targets, int64_t* counts, int32_t N, int32_t C, int32_t HW, void* stream) {
    if (!logits || !targets || !counts || N <= 0 || C <= 0 || HW <= 0) return set_error(RSB_E_INVALID, "metrics: bad arguments");
    const int64_t total = static_cast<int64_t>(N) * HW;
    metrics_kernel<<<blocks_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        logits, targets, reinterpret_cast<unsigned long long*>(counts), N, C, HW);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "metrics launch");
}

extern "C" int rsb_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float b1,
                             float b2, float eps, int32_t step, void* stream) {
    if (!param || !grad || !exp_avg || !exp_avg_sq || n <= 0 || step < 1) return set_error(RSB_E_INVALID, "adam: bad arguments");
    // torch computes the bias corrections in Python doubles and casts the scalars to the tensor dtype
    const double bc1 = 1.0 - pow(static_cast<double>(b1), step);
    const double bc2 = 1.0 - pow(static_cast<double>(b2), step);
    const float step_size = static_cast<float>(static_cast<double>(lr) / bc1);
    const float bc2_sqrt = static_cast<float>(sqrt(bc2));
    const float omb1 = static_cast<float>(1.0 - static_cast<double>(b1));
    const float omb2 = static_cast<float>(1.0 - static_cast<double>(b2));
    adam_kernel<<<blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(param, grad, exp_avg, exp_avg_sq, n, b1, b2, omb1, omb2,
                                                                                 step_size, bc2_sqrt, eps);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "adam launch");
}

extern "C" int rsb_adam_step_guarded(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float b1,
                                     float b2, float eps, int32_t step, int32_t* guard_state, void* stream) {
    if (!param || !grad || !exp_avg || !exp_avg_sq || n <= 0 || step < 1 || !guard_state) return set_error(RSB_E_INVALID, "adam_guarded: bad arguments");
    const double bc1 = 1.0 - pow(static_cast<double>(b1), step);
    const double bc2 = 1.0 - pow(static_cast<double>(b2), step);
    const float step_size = static_cast<float>(static_cast<double>(lr) / bc1);
    const float bc2_sqrt = static_cast<float>(sqrt(bc2));
    const float omb1 = static_cast<float>(1.0 - static_cast<double>(b1));
    const float omb2 = static_cast<float>(1.0 - static_cast<double>(b2));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    grad_finite_kernel<<<blocks_for(n, 256), 256, 0, st>>>(grad, n, guard_state);
    adam_guarded_kernel<<<blocks_for(n, 256), 256, 0, st>>>(param, grad, exp_avg, exp_avg_sq, n, b1, b2, omb1, omb2, lr, step_size, bc2_sqrt, eps, step,
                                                            guard_state);
    adam_guard_bookkeep_kernel<<<1, 1, 0, st>>>(guard_state);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "adam_guarded launch");
}

extern "C" int64_t rsb_lovasz_workspace_bytes(int32_t N, int32_t C, int32_t HW) {
    if (N <= 0 || C <= 0 || HW <= 0) return 0;
    return lovasz_layout(N, C, HW).total;
}

extern "C" int rsb_lovasz(const float* logits, const int64_t* targets, float* loss_out, float* grad, void* workspace,
                          int64_t workspace_bytes, int32_t N, int32_t C, int32_t HW, void* stream) {
    if (!logits || !targets || !loss_out || !workspace || N <= 0 || C <= 0 || HW <= 0) return set_error(RSB_E_INVALID, "lovasz: bad arguments");
    const LovaszWs w = lovasz_layout(N, C, HW);
    if (workspace_bytes < w.total) return set_error(RSB_E_INVALID, "lovasz: workspace too small (%lld < %lld)", (long long)workspace_bytes, (long long)w.total);
    if (static_cast<int64_t>(C) * HW >= (1LL << 24)) return set_error(RSB_E_INVALID, "lovasz: C*H*W must stay below 2^24 for exact fp32 cumulative sums");
    if (reinterpret_cast<uintptr_t>(workspace) & 255) return set_error(RSB_E_INVALID, "lovasz: workspace must be 256-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    uint32_t* keys[2] = {reinterpret_cast<uint32_t*>(ws + w.off_keys[0]), reinterpret_cast<uint32_t*>(ws + w.off_keys[1])};
    uint32_t* idx[2] = {reinterpret_cast<uint32_t*>(ws + w.off_idx[0]), reinterpret_cast<uint32_t*>(ws + w.off_idx[1])};
    uint32_t* hist = reinterpret_cast<uint32_t*>(ws + w.off_hist);
    uint32_t* tilepos = reinterpret_cast<uint32_t*>(ws + w.off_tilepos);
    uint32_t* gts = reinterpret_cast<uint32_t*>(ws + w.off_gts);
    double* loss_acc = reinterpret_cast<double*>(ws + w.off_loss);
    const int64_t P = static_cast<int64_t>(C) * HW;

    cudaError_t e = cudaMemsetAsync(loss_acc, 0, sizeof(double), st);
    if (e != cudaSuccess) return set_cuda_error(e, "lovasz memset");
    const dim3 tile_grid(w.tiles, N);
    lovasz_keys_kernel<<<dim3(blocks_for(w.Pp, 256, 1024), N), 256, 0, st>>>(logits, targets, keys[0], idx[0], C, HW, P, w.Pp);
    int cur = 0;
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 8 * pass;
        radix_hist_kernel<<<tile_grid, kSortThreads, 0, st>>>(keys[cur], hist, shift, w.Pp, w.tiles);
        radix_scan_kernel<<<N, 1024, 0, st>>>(hist, w.tiles);
        radix_scatter_kernel<<<tile_grid, kSortThreads, 0, st>>>(keys[cur], idx[cur], keys[cur ^ 1], idx[cur ^ 1], hist, shift, w.Pp, w.tiles);
        cur ^= 1;
    }
    lovasz_tilepos_kernel<<<tile_grid, kSortThreads, 0, st>>>(idx[cur], targets, tilepos, HW, P, w.Pp, w.tiles);
    lovasz_tilescan_kernel<<<N, 32, 0, st>>>(tilepos, gts, w.tiles);
    const float inv_n = 1.0f / static_cast<float>(N);
    lovasz_final_kernel<<<tile_grid, kSortThreads, 0, st>>>(keys[cur], idx[cur], targets, tilepos, gts, loss_acc, grad, HW, P, w.Pp, w.tiles, inv_n);
    lovasz_loss_out_kernel<<<1, 1, 0, st>>>(loss_acc, loss_out, inv_n);
    e = cudaGetLastError();
    return e == cudaSuccess ? RSB_OK : set_cuda_error(e, "lovasz launch");
}
