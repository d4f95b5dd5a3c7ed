// b2cnn_train.cu -- one training step of MyCNN on the device (SURVEY.md section 8, row f4):
//   optimizer.zero_grad(); output = model(input, age); loss = criterion(output, target); loss.backward(); optimizer.step()
// (bin/utils.py:200-208 with criterion = nn.BCEWithLogitsLoss(pos_weight=...), bin/explore_torch.ipynb:3204, optionally
// without the class weight, and torch.optim.Adam, bin/explore_torch.ipynb:3205) for the layer stack of bin/models.py:22-36 in
// train() mode:
//
//   c1 = conv1(x)            y1 = tanh(c1)   p1 = maxpool(y1)   d1 = dropout(p1)          models.py:23-25
//   c2 = conv2(d1)           y2 = tanh(c2)   p2 = maxpool(y2)   f  = dropout(p2)          models.py:26-28
//   f.view(-1, MAGICNUM) -> 2-layer LSTM over the BATCH axis (an unbatched sequence of B steps) models.py:29-30
//   z = out(h1) * relu(age * coef + 1)                                                    models.py:31-34
//   loss = mean_b( max(z,0) - z y + log(1 + exp(-|z|)) )
//
// Dropout cannot share torch's Philox stream, so the two masks are INPUTS (already scaled by 1/(1-p), or NULL = no
// dropout); everything else is bit-for-bit the same graph, differentiated by hand:
//   train_conv_fwd   per window: c1, p1, c2, f (kept for the backward pass)
//   train_lstm_fwd   one CTA scans the batch axis, keeps gate activations / cell / hidden states, logits, loss
//   train_lstm_bwd   BPTT over the batch axis: gradients of the head and of every recurrent matrix, d(gates of layer 0)
//   train_wih0_grad  dW_ih_l0 = d(gates0)^T x f            train_dfeat   d f = d(gates0) x W_ih_l0
//   train_conv_bwd   per window: dropout / pool (argmax routing, first maximum like ATen) / tanh / conv2 / conv1 backward
//   train_dx         d x (the input gradient), gather form: one thread per input sample
//   train_adam       torch.optim.Adam (no amsgrad, weight_decay 0) on the packed parameter blob
// The head of the two LSTM kernels is a template parameter (Head): the fused step's BCE, BCE with pos_weight, or logits
// only, with d loss / d z supplied by the caller (b2cnn_train_forward / b2cnn_train_backward, driven by torch autograd).
// These are launch-latency kernels for the training shape [B,10,120] (44 k MAC per window); they take any geometry the
// forward path takes (all intermediates live in the caller's workspace), but are not tuned for the stretched windows.
#include <cfloat>
#include <cstring>

#include "b2cnn_internal.cuh"

namespace b2cnn {

struct TrainDims {
    int C, K1, K2, PK, PS, W, L1, P1, L2, L;
    float age_coef;
};

// offsets (floats) of the tensors inside the packed parameter blob (include/b2cnn.h: b2cnn_weight_count)
struct BlobOff {
    int64_t w1, b1, w2, b2, wih0, whh0, bih0, bhh0, wih1, whh1, bih1, bhh1, wo, bo, total;
};
static BlobOff blob_offsets(const TrainDims &d) {
    BlobOff o;
    int64_t p = 0;
    o.w1 = p; p += (int64_t)kCMid * d.C * d.K1;
    o.b1 = p; p += kCMid;
    o.w2 = p; p += kCMid * d.K2;
    o.b2 = p; p += 1;
    o.wih0 = p; p += (int64_t)kGates * d.L;
    o.whh0 = p; p += kGates * kHidden;
    o.bih0 = p; p += kGates;
    o.bhh0 = p; p += kGates;
    o.wih1 = p; p += kGates * kHidden;
    o.whh1 = p; p += kGates * kHidden;
    o.bih1 = p; p += kGates;
    o.bhh1 = p; p += kGates;
    o.wo = p; p += kHidden;
    o.bo = p; p += 1;
    o.total = p;
    return o;
}

// workspace layout (floats)
struct TrainWs {
    int64_t c1, p1, c2, f, acts, cs, hs, lin, z, da0, dfeat, dc2, dd1, dc1, total;
};
static TrainWs train_ws(const TrainDims &d, int64_t B) {
    TrainWs w;
    int64_t p = 0;
    auto take = [&](int64_t n) { int64_t at = p; p += (n + 63) / 64 * 64; return at; };
    w.c1 = take(B * kCMid * d.L1);
    w.p1 = take(B * kCMid * d.P1);
    w.c2 = take(B * d.L2);
    w.f = take(B * d.L);
    w.acts = take(B * 2 * kGates);      // [t][layer][i f g o] post-activation
    w.cs = take(B * 2 * kHidden);       // [t][layer] cell state
    w.hs = take(B * 2 * kHidden);       // [t][layer] hidden state
    w.lin = take(B);                    // out(h1) before the age scale (d age needs it)
    w.z = take(B);
    w.da0 = take(B * kGates);           // d loss / d (layer-0 gate pre-activations)
    w.dfeat = take(B * d.L);
    w.dc2 = take(B * d.L2);
    w.dd1 = take(B * kCMid * d.P1);
    w.dc1 = take(B * kCMid * d.L1);
    w.total = p;
    return w;
}

__device__ __forceinline__ float sigmoidf_(float v) { return 1.0f / (1.0f + expf(-v)); }
// d tanh(v) / dv = 1 - tanh(v)^2 = 4t / (1 + t)^2 with t = exp(-2|v|), from the pre-activation: 1 - y*y of a float y
// near +-1 cancels to a few ulps of 1 (relative error ~1 at |v| ~ 8), this form has no cancellation.  NaN stays NaN,
// +-inf gives 0 like 1 - tanh(+-inf)^2.
__device__ __forceinline__ float dtanhf_(float v) {
    const float t = expf(-2.f * fabsf(v)), u = 1.f + t;
    return 4.f * t / (u * u);
}

// What follows the logits z.  kHeadLogits: no loss in the forward kernel, d loss / d z read from the caller's array in the
// backward kernel.  kHeadBce: BCEWithLogitsLoss (mean).  kHeadBcePw: BCEWithLogitsLoss(pos_weight=pw) (mean).
enum Head : int { kHeadLogits = 0, kHeadBce = 1, kHeadBcePw = 2 };

// ------------------------------------------------------------------------------------------------------------------
// forward, convolutional part: one CTA per window
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
train_conv_fwd(const float *__restrict__ x, const float *__restrict__ prm, BlobOff o, TrainDims d, const float *__restrict__ mask1,
               const float *__restrict__ mask2, float *__restrict__ c1, float *__restrict__ p1, float *__restrict__ c2,
               float *__restrict__ f) {
    const int b = blockIdx.x, tid = threadIdx.x;
    const float *xb = x + (int64_t)b * d.C * d.W;
    float *c1b = c1 + (int64_t)b * kCMid * d.L1, *p1b = p1 + (int64_t)b * kCMid * d.P1;
    float *c2b = c2 + (int64_t)b * d.L2, *fb = f + (int64_t)b * d.L;
    // conv1: same summation order as the inference kernels (channels outer, taps inner, fmaf chain from the bias)
    for (int e = tid; e < kCMid * d.L1; e += blockDim.x) {
        const int oc = e / d.L1, t = e % d.L1;
        float acc = prm[o.b1 + oc];
        for (int c = 0; c < d.C; ++c)
            for (int k = 0; k < d.K1; ++k) acc = fmaf(prm[o.w1 + ((int64_t)oc * d.C + c) * d.K1 + k], xb[(int64_t)c * d.W + t + k], acc);
        c1b[e] = acc;
    }
    __syncthreads();
    for (int e = tid; e < kCMid * d.P1; e += blockDim.x) {
        const int oc = e / d.P1, i = e % d.P1;
        float m = c1b[oc * d.L1 + d.PS * i];
        for (int j = 1; j < d.PK; ++j) m = max_nan(m, c1b[oc * d.L1 + d.PS * i + j]);
        p1b[e] = tanhf(m);                  // pooling before tanh: tanh is monotone, and a NaN in the window wins either way
    }
    __syncthreads();
    for (int t = tid; t < d.L2; t += blockDim.x) {
        float acc = prm[o.b2];
        for (int oc = 0; oc < kCMid; ++oc)
            for (int k = 0; k < d.K2; ++k) {
                const int64_t at = (int64_t)oc * d.P1 + t + k;
                const float dv = p1b[at] * (mask1 ? mask1[(int64_t)b * kCMid * d.P1 + at] : 1.0f);
                acc = fmaf(prm[o.w2 + oc * d.K2 + k], dv, acc);
            }
        c2b[t] = acc;
    }
    __syncthreads();
    for (int i = tid; i < d.L; i += blockDim.x) {
        float m = c2b[d.PS * i];
        for (int j = 1; j < d.PK; ++j) m = max_nan(m, c2b[d.PS * i + j]);
        fb[i] = tanhf(m) * (mask2 ? mask2[(int64_t)b * d.L + i] : 1.0f);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// LSTM forward over the batch axis with everything the backward pass needs kept; logits and loss.
// One CTA of 64 threads: thread r owns gate row r of every matrix.  sequence == 0: every step starts from the zero state
// (independent windows).  HEAD == kHeadLogits: target and loss_out are not used.
// ------------------------------------------------------------------------------------------------------------------
template <int HEAD>
__global__ void __launch_bounds__(64)
train_lstm_fwd(const float *__restrict__ f, const float *__restrict__ prm, BlobOff o, TrainDims d, int64_t B, int sequence,
               const float *__restrict__ age, const float *__restrict__ target, float pos_weight, float *__restrict__ acts,
               float *__restrict__ cs, float *__restrict__ hs, float *__restrict__ lin, float *__restrict__ z,
               float *__restrict__ loss_out) {
    __shared__ float g[kGates], h0[kHidden], c0[kHidden], h1[kHidden], c1s[kHidden];
    const int r = threadIdx.x;
    if (r < kHidden) { h0[r] = c0[r] = h1[r] = c1s[r] = 0.f; }
    float loss = 0.f;
    __syncthreads();
    for (int64_t t = 0; t < B; ++t) {
        if (!sequence) {
            if (r < kHidden) { h0[r] = c0[r] = h1[r] = c1s[r] = 0.f; }
            __syncthreads();
        }
        // ---- layer 0: g = (W_ih f_t + b_ih) + (W_hh h_{t-1} + b_hh)
        {
            const float *ft = f + t * d.L;
            const float *wr = prm + o.wih0 + (int64_t)r * d.L;
            float a = 0.f;
            for (int p = 0; p < d.L; ++p) a = fmaf(wr[p], ft[p], a);
            float rr = 0.f;
            for (int k = 0; k < kHidden; ++k) rr = fmaf(prm[o.whh0 + r * kHidden + k], h0[k], rr);
            g[r] = (a + prm[o.bih0 + r]) + (rr + prm[o.bhh0 + r]);
        }
        __syncthreads();
        const int q = r >> 4;                                   // gate order i, f, g, o
        float av = q == 2 ? tanhf(g[r]) : sigmoidf_(g[r]);
        acts[(t * 2 + 0) * kGates + r] = av;
        __syncthreads();
        g[r] = av;
        __syncthreads();
        if (r < kHidden) {
            const float cn = g[kHidden + r] * c0[r] + g[r] * g[2 * kHidden + r];
            c0[r] = cn;
            h0[r] = g[3 * kHidden + r] * tanhf(cn);
            cs[(t * 2 + 0) * kHidden + r] = cn;
            hs[(t * 2 + 0) * kHidden + r] = h0[r];
        }
        __syncthreads();
        // ---- layer 1
        {
            float a = 0.f, rr = 0.f;
            for (int k = 0; k < kHidden; ++k) {
                a = fmaf(prm[o.wih1 + r * kHidden + k], h0[k], a);
                rr = fmaf(prm[o.whh1 + r * kHidden + k], h1[k], rr);
            }
            av = (a + prm[o.bih1 + r]) + (rr + prm[o.bhh1 + r]);
            av = q == 2 ? tanhf(av) : sigmoidf_(av);
        }
        acts[(t * 2 + 1) * kGates + r] = av;
        __syncthreads();
        g[r] = av;
        __syncthreads();
        if (r < kHidden) {
            const float cn = g[kHidden + r] * c1s[r] + g[r] * g[2 * kHidden + r];
            c1s[r] = cn;
            h1[r] = g[3 * kHidden + r] * tanhf(cn);
            cs[(t * 2 + 1) * kHidden + r] = cn;
            hs[(t * 2 + 1) * kHidden + r] = h1[r];
        }
        __syncthreads();
        if (r == 0) {
            float y = 0.f;
            for (int k = 0; k < kHidden; ++k) y = fmaf(prm[o.wo + k], h1[k], y);
            y += prm[o.bo];
            lin[t] = y;
            float s = __fadd_rn(__fmul_rn(age[t], d.age_coef), 1.0f);
            s = (s > 0.f || s != s) ? s : 0.f;
            y *= s;
            z[t] = y;
            if constexpr (HEAD == kHeadBce) {
                const float yt = target[t];
                loss += fmaxf(y, 0.f) - y * yt + log1pf(expf(-fabsf(y)));   // BCEWithLogitsLoss, the stable form ATen uses
            } else if constexpr (HEAD == kHeadBcePw) {
                const float yt = target[t], lw = 1.f + (pos_weight - 1.f) * yt;
                loss += (1.f - yt) * y + lw * (log1pf(expf(-fabsf(y))) + fmaxf(-y, 0.f));   // ATen's pos_weight form
            }
        }
        __syncthreads();
    }
    if (HEAD != kHeadLogits && r == 0) *loss_out = loss / (float)B;
}

// ------------------------------------------------------------------------------------------------------------------
// BPTT over the batch axis.  64 threads: thread r owns gate row r.  Gradients of the recurrent matrices, biases and of
// the head are accumulated in registers / shared memory and written once; d(gates of layer 0) goes to da0[t][64].
// HEAD == kHeadLogits: d loss / d z is dz_in[t] and, when dage != NULL, d loss / d age goes to dage[t] (torch's relu
// backward: zero where relu(age * coef + 1) is not positive); otherwise dz comes from z and target, dage is not written.
// ------------------------------------------------------------------------------------------------------------------
template <int HEAD>
__global__ void __launch_bounds__(64)
train_lstm_bwd(const float *__restrict__ prm, BlobOff o, TrainDims d, int64_t B, int sequence, const float *__restrict__ age,
               const float *__restrict__ target, float pos_weight, const float *__restrict__ dz_in, const float *__restrict__ acts,
               const float *__restrict__ cs, const float *__restrict__ hs, const float *__restrict__ lin, const float *__restrict__ z,
               float *__restrict__ da0, float *__restrict__ grad, float *__restrict__ dage) {
    __shared__ float da[kGates], dh0c[kHidden], dc0c[kHidden], dh1c[kHidden], dc1c[kHidden], dh0ext[kHidden], dh1ext[kHidden];
    const int r = threadIdx.x, u = r & 15, q = r >> 4;
    float gWhh0[kHidden], gWih1[kHidden], gWhh1[kHidden];
#pragma unroll
    for (int k = 0; k < kHidden; ++k) gWhh0[k] = gWih1[k] = gWhh1[k] = 0.f;
    float gb0 = 0.f, gb1 = 0.f, gwo = 0.f, gbo = 0.f;
    if (r < kHidden) dh0c[r] = dc0c[r] = dh1c[r] = dc1c[r] = 0.f;
    __syncthreads();
    for (int64_t t = B - 1; t >= 0; --t) {
        if (!sequence) {
            if (r < kHidden) dh0c[r] = dc0c[r] = dh1c[r] = dc1c[r] = 0.f;
            __syncthreads();
        }
        const bool first = !sequence || t == 0;               // no previous step: h_{t-1} = c_{t-1} = 0
        // ---- head: z = (wo . h1 + bo) * s
        float s = __fadd_rn(__fmul_rn(age[t], d.age_coef), 1.0f);
        s = (s > 0.f || s != s) ? s : 0.f;
        float dz;
        if constexpr (HEAD == kHeadBce) {
            dz = (sigmoidf_(z[t]) - target[t]) / (float)B;
        } else if constexpr (HEAD == kHeadBcePw) {
            const float yt = target[t], lw = 1.f + (pos_weight - 1.f) * yt;
            dz = ((1.f - yt) - lw * sigmoidf_(-z[t])) / (float)B;
        } else {
            dz = dz_in[t];
            if (dage && r == 0) dage[t] = s > 0.f ? dz * lin[t] * d.age_coef : 0.f;
        }
        const float dlin = dz * s;
        if (r < kHidden) {
            gwo += dlin * hs[(t * 2 + 1) * kHidden + r];
            dh1ext[r] = dlin * prm[o.wo + r];
        }
        if (r == 0) gbo += dlin;
        __syncthreads();
        // ---- layer 1
        {
            const float *a = acts + (t * 2 + 1) * kGates;
            const float ct = cs[(t * 2 + 1) * kHidden + u];
            const float cprev = first ? 0.f : cs[((t - 1) * 2 + 1) * kHidden + u];
            const float tc = tanhf(ct);
            const float dh = dh1ext[u] + dh1c[u];
            const float dc = dc1c[u] + dh * a[3 * kHidden + u] * (1.f - tc * tc);
            float v;
            if (q == 0) v = dc * a[2 * kHidden + u] * a[u] * (1.f - a[u]);                                   // i
            else if (q == 1) v = dc * cprev * a[kHidden + u] * (1.f - a[kHidden + u]);                       // f
            else if (q == 2) v = dc * a[u] * (1.f - a[2 * kHidden + u] * a[2 * kHidden + u]);               // g
            else v = dh * tc * a[3 * kHidden + u] * (1.f - a[3 * kHidden + u]);                             // o
            __syncthreads();                                   // every thread has read dh1c / dc1c of this step
            da[r] = v;
            if (q == 0) dc1c[u] = dc * a[kHidden + u];         // carried to step t-1: dc * f
            gb1 += v;
#pragma unroll
            for (int k = 0; k < kHidden; ++k) {
                gWih1[k] += v * hs[(t * 2 + 0) * kHidden + k];                      // layer-1 input = h0_t
                gWhh1[k] += v * (first ? 0.f : hs[((t - 1) * 2 + 1) * kHidden + k]);  // v * 0: a NaN v still counts
            }
        }
        __syncthreads();
        if (r < kHidden) {
            float e0 = 0.f, e1 = 0.f;
            for (int rr = 0; rr < kGates; ++rr) {
                e0 = fmaf(prm[o.wih1 + rr * kHidden + r], da[rr], e0);   // -> d h0_t
                e1 = fmaf(prm[o.whh1 + rr * kHidden + r], da[rr], e1);   // -> d h1_{t-1}
            }
            dh0ext[r] = e0;
            dh1c[r] = e1;
        }
        __syncthreads();
        // ---- layer 0
        {
            const float *a = acts + (t * 2 + 0) * kGates;
            const float ct = cs[(t * 2 + 0) * kHidden + u];
            const float cprev = first ? 0.f : cs[((t - 1) * 2 + 0) * kHidden + u];
            const float tc = tanhf(ct);
            const float dh = dh0ext[u] + dh0c[u];
            const float dc = dc0c[u] + dh * a[3 * kHidden + u] * (1.f - tc * tc);
            float v;
            if (q == 0) v = dc * a[2 * kHidden + u] * a[u] * (1.f - a[u]);
            else if (q == 1) v = dc * cprev * a[kHidden + u] * (1.f - a[kHidden + u]);
            else if (q == 2) v = dc * a[u] * (1.f - a[2 * kHidden + u] * a[2 * kHidden + u]);
            else v = dh * tc * a[3 * kHidden + u] * (1.f - a[3 * kHidden + u]);
            __syncthreads();
            da[r] = v;
            da0[t * kGates + r] = v;
            if (q == 0) dc0c[u] = dc * a[kHidden + u];
            gb0 += v;
#pragma unroll
            for (int k = 0; k < kHidden; ++k) gWhh0[k] += v * (first ? 0.f : hs[((t - 1) * 2 + 0) * kHidden + k]);
        }
        __syncthreads();
        if (r < kHidden) {
            float e = 0.f;
            for (int rr = 0; rr < kGates; ++rr) e = fmaf(prm[o.whh0 + rr * kHidden + r], da[rr], e);
            dh0c[r] = e;
        }
        __syncthreads();
    }
#pragma unroll
    for (int k = 0; k < kHidden; ++k) {
        grad[o.whh0 + r * kHidden + k] = gWhh0[k];
        grad[o.wih1 + r * kHidden + k] = gWih1[k];
        grad[o.whh1 + r * kHidden + k] = gWhh1[k];
    }
    grad[o.bih0 + r] = gb0; grad[o.bhh0 + r] = gb0;
    grad[o.bih1 + r] = gb1; grad[o.bhh1 + r] = gb1;
    if (r < kHidden) grad[o.wo + r] = gwo;
    if (r == 0) grad[o.bo] = gbo;
}

// dW_ih_l0[g][p] = sum_t da0[t][g] f[t][p]
__global__ void train_wih0_grad(const float *__restrict__ da0, const float *__restrict__ f, int64_t B, int L, float *__restrict__ gw) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)kGates * L) return;
    const int g = (int)(e / L), p = (int)(e % L);
    float a = 0.f;
    for (int64_t t = 0; t < B; ++t) a = fmaf(da0[t * kGates + g], f[t * L + p], a);
    gw[e] = a;
}
// d f[t][p] = sum_g da0[t][g] W_ih_l0[g][p]
__global__ void train_dfeat(const float *__restrict__ da0, const float *__restrict__ wih0, int64_t B, int L, float *__restrict__ dfeat) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= B * L) return;
    const int64_t t = e / L;
    const int p = (int)(e % L);
    float a = 0.f;
    for (int g = 0; g < kGates; ++g) a = fmaf(da0[t * kGates + g], wih0[(int64_t)g * L + p], a);
    dfeat[e] = a;
}

// first maximum of a pooling window, like ATen's max_pool1d ((v > m) || isnan(v) replaces).  This is the first maximum
// of the pre-activation; the reference pools after tanh and takes the first maximum there.  The two differ only where
// tanhf maps distinct pre-activations to one float: this choice is the one exact arithmetic makes.
__device__ __forceinline__ int pool_argmax(const float *v, int start, int pk) {
    int best = start;
    float m = v[start];
    for (int j = 1; j < pk; ++j) {
        const float c = v[start + j];
        if (c > m || c != c) { m = c; best = start + j; }
    }
    return best;
}

// ------------------------------------------------------------------------------------------------------------------
// backward, convolutional part: one CTA per window; conv weight gradients are reduced per CTA and added atomically
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
train_conv_bwd(const float *__restrict__ x, const float *__restrict__ prm, BlobOff o, TrainDims d, const float *__restrict__ mask1,
               const float *__restrict__ mask2, const float *__restrict__ c1, const float *__restrict__ p1,
               const float *__restrict__ c2, const float *__restrict__ dfeat, float *__restrict__ dc2, float *__restrict__ dd1,
               float *__restrict__ dc1, float *__restrict__ grad) {
    const int b = blockIdx.x, tid = threadIdx.x;
    const float *xb = x + (int64_t)b * d.C * d.W;
    const float *c1b = c1 + (int64_t)b * kCMid * d.L1, *p1b = p1 + (int64_t)b * kCMid * d.P1, *c2b = c2 + (int64_t)b * d.L2;
    const float *dfb = dfeat + (int64_t)b * d.L;
    float *dc2b = dc2 + (int64_t)b * d.L2, *dd1b = dd1 + (int64_t)b * kCMid * d.P1, *dc1b = dc1 + (int64_t)b * kCMid * d.L1;
    __shared__ float red[256];
    // ---- dropout 2 + pool 2 + tanh: gather form -- position t collects from the (overlapping) windows whose maximum it is
    for (int t = tid; t < d.L2; t += blockDim.x) {
        float a = 0.f;
        int i_lo = (t - d.PK + d.PS) / d.PS;                   // ceil((t - PK + 1) / PS)
        if (t - d.PK + 1 <= 0) i_lo = 0;
        for (int i = i_lo; i <= t / d.PS && i < d.L; ++i)
            if (pool_argmax(c2b, d.PS * i, d.PK) == t) a += dfb[i] * (mask2 ? mask2[(int64_t)b * d.L + i] : 1.0f);
        dc2b[t] = a * dtanhf_(c2b[t]);
    }
    __syncthreads();
    // ---- conv2: weight / bias gradients (block reduction, one atomic per value and CTA), d d1
    for (int e = 0; e < kCMid * d.K2 + 1; ++e) {
        float part = 0.f;
        if (e < kCMid * d.K2) {
            const int oc = e / d.K2, k = e % d.K2;
            for (int t = tid; t < d.L2; t += blockDim.x) {
                const int64_t at = (int64_t)oc * d.P1 + t + k;
                part = fmaf(dc2b[t], p1b[at] * (mask1 ? mask1[(int64_t)b * kCMid * d.P1 + at] : 1.0f), part);
            }
        } else {
            for (int t = tid; t < d.L2; t += blockDim.x) part += dc2b[t];
        }
        red[tid] = part;
        __syncthreads();
        for (int sft = 128; sft > 0; sft >>= 1) {
            if (tid < sft) red[tid] += red[tid + sft];
            __syncthreads();
        }
        if (tid == 0) atomicAdd(grad + (e < kCMid * d.K2 ? o.w2 + e : o.b2), red[0]);
        __syncthreads();
    }
    for (int e = tid; e < kCMid * d.P1; e += blockDim.x) {
        const int oc = e / d.P1, uu = e % d.P1;
        float a = 0.f;
        for (int k = 0; k < d.K2; ++k) {
            const int t = uu - k;
            if (t >= 0 && t < d.L2) a = fmaf(prm[o.w2 + oc * d.K2 + k], dc2b[t], a);
        }
        dd1b[e] = a * (mask1 ? mask1[(int64_t)b * kCMid * d.P1 + e] : 1.0f);     // through dropout 1: d p1
    }
    __syncthreads();
    // ---- pool 1 + tanh
    for (int e = tid; e < kCMid * d.L1; e += blockDim.x) {
        const int oc = e / d.L1, t = e % d.L1;
        const float *row = c1b + oc * d.L1;
        float a = 0.f;
        int i_lo = (t - d.PK + d.PS) / d.PS;
        if (t - d.PK + 1 <= 0) i_lo = 0;
        for (int i = i_lo; i <= t / d.PS && i < d.P1; ++i)
            if (pool_argmax(row, d.PS * i, d.PK) == t) a += dd1b[oc * d.P1 + i];
        dc1b[e] = a * dtanhf_(row[t]);
    }
    __syncthreads();
    // ---- conv1: one thread per weight, a dot product over the positions
    for (int e = tid; e < kCMid * d.C * d.K1 + kCMid; e += blockDim.x) {
        float a = 0.f;
        if (e < kCMid * d.C * d.K1) {
            const int oc = e / (d.C * d.K1), c = (e / d.K1) % d.C, k = e % d.K1;
            const float *dr = dc1b + oc * d.L1, *xr = xb + (int64_t)c * d.W + k;
            for (int t = 0; t < d.L1; ++t) a = fmaf(dr[t], xr[t], a);
            atomicAdd(grad + o.w1 + e, a);
        } else {
            const int oc = e - kCMid * d.C * d.K1;
            const float *dr = dc1b + oc * d.L1;
            for (int t = 0; t < d.L1; ++t) a += dr[t];
            atomicAdd(grad + o.b1 + oc, a);
        }
    }
}

// d x[b][c][t] = sum_oc sum_k w1[oc][c][k] * dc1[b][oc][t-k] over the valid t-k in [0, L1): conv1's input gradient in
// gather form, one thread per input sample (no atomics)
__global__ void train_dx(const float *__restrict__ dc1, const float *__restrict__ prm, BlobOff o, TrainDims d, int64_t B,
                         float *__restrict__ dx) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= B * d.C * d.W) return;
    const int t = (int)(e % d.W), c = (int)((e / d.W) % d.C);
    const int64_t b = e / ((int64_t)d.C * d.W);
    const int k_lo = max(0, t - (d.L1 - 1)), k_hi = min(d.K1 - 1, t);
    float a = 0.f;
    for (int oc = 0; oc < kCMid; ++oc) {
        const float *wr = prm + o.w1 + ((int64_t)oc * d.C + c) * d.K1;
        const float *dr = dc1 + (b * kCMid + oc) * d.L1 + t;
        for (int k = k_lo; k <= k_hi; ++k) a = fmaf(wr[k], dr[-k], a);
    }
    dx[e] = a;
}

// torch.optim.Adam, single-tensor form: exp_avg.lerp_(grad, 1-b1); exp_avg_sq = b2*v + (1-b2) g^2;
// denom = sqrt(v) / sqrt(1 - b2^t) + eps; param -= (lr / (1 - b1^t)) * m / denom
__global__ void train_adam(float *__restrict__ prm, float *__restrict__ m, float *__restrict__ v, const float *__restrict__ grad, int64_t n,
                           float lr, float b1, float b2, float eps, float bc1, float bc2_sqrt) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const float g = grad[e];
    const float mm = m[e] + (g - m[e]) * (1.f - b1);
    const float vv = b2 * v[e] + (1.f - b2) * g * g;
    m[e] = mm; v[e] = vv;
    const float denom = sqrtf(vv) / bc2_sqrt + eps;
    prm[e] = prm[e] - (lr / bc1) * (mm / denom);
}

static bool train_dims(const b2cnn_config &c, TrainDims &d, const char **err) {
    d.C = c.in_channels; d.K1 = c.k1; d.K2 = c.k2; d.PK = c.pool_k; d.PS = c.pool_s; d.W = c.window; d.age_coef = c.age_coef;
    if (c.c_mid != kCMid || c.hidden != kHidden || c.layers != 2) { *err = "training: c_mid / hidden / layers must be 4 / 16 / 2"; return false; }
    if (c.act != B2CNN_ACT_TANH || (c.flags & B2CNN_FLAG_AFFINE)) { *err = "training: tanh activations without affine only (bin/models.py:23,26)"; return false; }
    if (d.C < 1 || d.K1 < 1 || d.K2 < 1 || d.PK < 1 || d.PS < 1 || d.W < 1) { *err = "training: bad geometry"; return false; }
    d.L1 = d.W - d.K1 + 1;
    if (d.L1 < d.PK) { *err = "training: window too short"; return false; }
    d.P1 = (d.L1 - d.PK) / d.PS + 1;
    d.L2 = d.P1 - d.K2 + 1;
    if (d.L2 < d.PK) { *err = "training: window too short"; return false; }
    d.L = (d.L2 - d.PK) / d.PS + 1;
    if (d.L != c.lstm_input) { *err = "training: L_out(window) != lstm_input (x.view(-1, MAGICNUM) would straddle windows)"; return false; }
    return true;
}

int64_t train_workspace_bytes(const b2cnn_config *cfg, int64_t B) {
    TrainDims d;
    const char *err = "";
    if (!cfg || B < 1 || !train_dims(*cfg, d, &err)) return -1;
    return train_ws(d, B).total * (int64_t)sizeof(float);
}

// Sets cfg->device current for the launches of one call (when it is >= 0) and restores the caller's device afterwards.
struct DeviceScope {
    int prev = -1;
    bool ok = true;
    explicit DeviceScope(int device) {
        if (device >= 0) ok = cudaGetDevice(&prev) == cudaSuccess && cudaSetDevice(device) == cudaSuccess;
    }
    ~DeviceScope() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// everything after d(head): d W_ih_l0, d f, the convolutional backward into `grads` (zeroed by the caller: conv weight
// gradients are added atomically) and, when dx != NULL, the input gradient
static void launch_backward_tail(const TrainDims &d, const BlobOff &o, const TrainWs &w, float *ws, const float *params,
                                 const float *x, int64_t B, const float *mask1, const float *mask2, float *grads, float *dx,
                                 cudaStream_t st) {
    const int64_t n1 = (int64_t)kGates * d.L, n2 = B * d.L;
    train_wih0_grad<<<(unsigned)((n1 + 255) / 256), 256, 0, st>>>(ws + w.da0, ws + w.f, B, d.L, grads + o.wih0);
    train_dfeat<<<(unsigned)((n2 + 255) / 256), 256, 0, st>>>(ws + w.da0, params + o.wih0, B, d.L, ws + w.dfeat);
    train_conv_bwd<<<(unsigned)B, 256, 0, st>>>(x, params, o, d, mask1, mask2, ws + w.c1, ws + w.p1, ws + w.c2, ws + w.dfeat, ws + w.dc2,
                                               ws + w.dd1, ws + w.dc1, grads);
    if (dx) {
        const int64_t n = B * d.C * d.W;
        train_dx<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws + w.dc1, params, o, d, B, dx);
    }
}

int train_step(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step, float lr, float beta1,
               float beta2, float eps, int apply_update, const float *x, int64_t B, const float *age, const float *target,
               int weighted, float pos_weight, int sequence, const float *mask1, const float *mask2, float *loss_out, void *workspace,
               int64_t ws_bytes, cudaStream_t st, const char **err) {
    TrainDims d;
    if (!cfg || !train_dims(*cfg, d, err)) return B2CNN_EINVAL;
    if (!params || !grads || !x || !age || !target || !loss_out || !workspace || B < 1 || step < 1) { *err = "training: null argument / bad step"; return B2CNN_EINVAL; }
    if (apply_update && (!adam_m || !adam_v)) { *err = "training: Adam state missing"; return B2CNN_EINVAL; }
    if (weighted && !(pos_weight > 0.f && pos_weight <= FLT_MAX)) { *err = "training: pos_weight must be positive and finite"; return B2CNN_EINVAL; }
    const TrainWs w = train_ws(d, B);
    if (ws_bytes < w.total * (int64_t)sizeof(float)) { *err = "training: workspace smaller than b2cnn_train_workspace_bytes()"; return B2CNN_ESTATE; }
    const BlobOff o = blob_offsets(d);
    float *ws = reinterpret_cast<float *>(workspace);
    if (cudaMemsetAsync(grads, 0, sizeof(float) * o.total, st) != cudaSuccess) { *err = "memset grads"; return B2CNN_ECUDA; }
    train_conv_fwd<<<(unsigned)B, 256, 0, st>>>(x, params, o, d, mask1, mask2, ws + w.c1, ws + w.p1, ws + w.c2, ws + w.f);
    if (weighted) {
        train_lstm_fwd<kHeadBcePw><<<1, 64, 0, st>>>(ws + w.f, params, o, d, B, sequence, age, target, pos_weight, ws + w.acts, ws + w.cs,
                                                     ws + w.hs, ws + w.lin, ws + w.z, loss_out);
        train_lstm_bwd<kHeadBcePw><<<1, 64, 0, st>>>(params, o, d, B, sequence, age, target, pos_weight, nullptr, ws + w.acts, ws + w.cs,
                                                     ws + w.hs, ws + w.lin, ws + w.z, ws + w.da0, grads, nullptr);
    } else {
        train_lstm_fwd<kHeadBce><<<1, 64, 0, st>>>(ws + w.f, params, o, d, B, sequence, age, target, 1.f, ws + w.acts, ws + w.cs,
                                                   ws + w.hs, ws + w.lin, ws + w.z, loss_out);
        train_lstm_bwd<kHeadBce><<<1, 64, 0, st>>>(params, o, d, B, sequence, age, target, 1.f, nullptr, ws + w.acts, ws + w.cs,
                                                   ws + w.hs, ws + w.lin, ws + w.z, ws + w.da0, grads, nullptr);
    }
    launch_backward_tail(d, o, w, ws, params, x, B, mask1, mask2, grads, nullptr, st);
    if (apply_update) {
        const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
        train_adam<<<(unsigned)((o.total + 255) / 256), 256, 0, st>>>(params, adam_m, adam_v, grads, o.total, lr, beta1, beta2, eps, bc1, sqrtf(bc2));
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

// the checks b2cnn_train_forward and b2cnn_train_backward share; no CUDA call
static int autograd_args(const b2cnn_config *cfg, int64_t B, int mode, int64_t ws_bytes, bool ptrs_ok, TrainDims &d, TrainWs &w,
                         const char **err) {
    if (!cfg || !train_dims(*cfg, d, err)) return B2CNN_EINVAL;
    if (mode != B2CNN_MODE_INDEPENDENT && mode != B2CNN_MODE_SEQUENCE) { *err = "training: bad mode"; return B2CNN_EINVAL; }
    if (!ptrs_ok || B < 1) { *err = "training: null argument / bad batch"; return B2CNN_EINVAL; }
    w = train_ws(d, B);
    if (ws_bytes < w.total * (int64_t)sizeof(float)) { *err = "training: workspace smaller than b2cnn_train_workspace_bytes()"; return B2CNN_ESTATE; }
    return B2CNN_OK;
}

int train_forward(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age, int mode, const float *mask1,
                  const float *mask2, float *z_out, void *workspace, int64_t ws_bytes, cudaStream_t st, const char **err) {
    TrainDims d;
    TrainWs w;
    const int rc = autograd_args(cfg, B, mode, ws_bytes, params && x && age && z_out && workspace, d, w, err);
    if (rc != B2CNN_OK) return rc;
    DeviceScope dev(cfg->device);
    if (!dev.ok) { *err = "cudaSetDevice"; return B2CNN_ECUDA; }
    const BlobOff o = blob_offsets(d);
    const int sequence = mode == B2CNN_MODE_SEQUENCE ? 1 : 0;
    float *ws = reinterpret_cast<float *>(workspace);
    train_conv_fwd<<<(unsigned)B, 256, 0, st>>>(x, params, o, d, mask1, mask2, ws + w.c1, ws + w.p1, ws + w.c2, ws + w.f);
    train_lstm_fwd<kHeadLogits><<<1, 64, 0, st>>>(ws + w.f, params, o, d, B, sequence, age, nullptr, 1.f, ws + w.acts, ws + w.cs,
                                                  ws + w.hs, ws + w.lin, z_out, nullptr);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

int train_backward(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age, int mode,
                   const float *mask1, const float *mask2, const float *dz, float *grads, float *dx, float *dage, void *workspace,
                   int64_t ws_bytes, cudaStream_t st, const char **err) {
    TrainDims d;
    TrainWs w;
    const int rc = autograd_args(cfg, B, mode, ws_bytes, params && x && age && dz && grads && workspace, d, w, err);
    if (rc != B2CNN_OK) return rc;
    DeviceScope dev(cfg->device);
    if (!dev.ok) { *err = "cudaSetDevice"; return B2CNN_ECUDA; }
    const BlobOff o = blob_offsets(d);
    const int sequence = mode == B2CNN_MODE_SEQUENCE ? 1 : 0;
    float *ws = reinterpret_cast<float *>(workspace);
    if (cudaMemsetAsync(grads, 0, sizeof(float) * o.total, st) != cudaSuccess) { *err = "memset grads"; return B2CNN_ECUDA; }
    train_lstm_bwd<kHeadLogits><<<1, 64, 0, st>>>(params, o, d, B, sequence, age, nullptr, 1.f, dz, ws + w.acts, ws + w.cs, ws + w.hs,
                                                  ws + w.lin, nullptr, ws + w.da0, grads, dage);
    launch_backward_tail(d, o, w, ws, params, x, B, mask1, mask2, grads, dx, st);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

}  // namespace b2cnn
