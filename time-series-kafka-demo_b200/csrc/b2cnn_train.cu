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
// dropout); everything else is bit-for-bit the same graph, differentiated by hand.  The conv layers work on position
// tiles of kT = 128 final features of one window (a window with fewer features, such as the training shape [B,10,120]
// with L = 25, is one tile; the waveform window [B,3,75000] has L = 18745, 147 tiles):
//   train_conv_fwd         grid (position tiles x B): a CTA stages its tile's x span in shared memory, runs conv_tile()
//                          there and writes only f
//   train_pre0_partial     layer-0 pre-activations f . W_ih_l0^T as a split-K GEMM over slices of kPre0Slice positions;
//                          with more than one slice train_sum_chunks adds the partials in slice order
//   train_lstm_fwd         scans the batch axis from those pre-activations, keeps gate activations / cell / hidden
//                          states, logits, loss; one CTA, or with seq_lengths (the _seq entry points) one CTA per group
//                          of consecutive sequences, each sequence from the zero state
//   train_lstm_bwd         BPTT over the batch axis (over each CTA's sequences): gradients of the head and of every
//                          recurrent matrix, d(gates of layer 0) = da0
//   train_head_reduce      with more than one scan CTA: sums the CTAs' head-gradient and loss rows in CTA (= sequence)
//                          order
//   train_wih0_grad        dW_ih_l0 = da0^T f with f read once: a thread owns a position and all 64 gate rows, the batch
//                          is split into chunks, and train_sum_chunks adds the chunk partials in chunk order
//   train_dfeat            d f = da0 W_ih_l0 with a thread's 64 W_ih_l0 values in registers
//   train_dfeat_fold       (whole recordings only) d f of each recording feature = the sum of its covering windows' d f
//   train_conv_bwd         grid (position tiles x groups of windows): recomputes c1 / d1 / c2 with conv_tile(), back-
//                          propagates the gradients of ITS OWN features through its receptive span in shared memory
//                          (dropout / pool with first-maximum routing like ATen / tanh / conv2 / conv1), keeps the conv
//                          weight-gradient partials of its windows and adds d x into a zeroed array
//   train_conv_grad_reduce sums the per-CTA partials in a fixed order (no atomic on a parameter gradient: gradients
//                          repeat bit for bit)
//   train_adam             torch.optim.Adam (no amsgrad, weight_decay 0) on the packed parameter blob
// Candidate heads on one frozen front end (the train_heads_* entry points, train_heads_step at the end of this file):
// the conv forward once, the *_heads kernels (projection and dW_ih_l0 two heads per CTA, Adam per head) and the scan
// kernels with one grid row per head; no d f and no conv backward.
// The head of the two LSTM kernels is a template parameter (Head): the fused step's BCE, BCE with pos_weight, or logits
// only, with d loss / d z supplied by the caller (b2cnn_train_forward / b2cnn_train_backward, driven by torch autograd).
// Everything below f is linear in d f, so the sum over tiles of what each tile back-propagates from its own features is
// the full gradient; no halo is exchanged and dc1 / dd1 / dc2 never reach global memory.  A window's values depend on
// its geometry alone; the batch sets only the order in which conv-gradient partials and dW_ih_l0's chunks are added.
//
// Whole recordings (the _record entry points and the *_record kernels, whose bodies are the window kernels' with
// REC = true): the rows of the scans are the counted windows of
// B recordings [B][C][N].  The conv kernels run over each recording's geometry (a "window" of N samples, L_N features,
// one grid row per recording), the projection and dW_ih_l0 read window w of recording b as features [w S/F, w S/F + L)
// of the recording's row, and train_dfeat_fold sums the windows' d f onto the recording before the conv backward.  A
// tile that no counted window reaches does no conv work, and the conv backward zeroes every staged sample that no counted
// window reads, so NaN / inf there cannot reach a gradient.
#include <cfloat>
#include <cstring>
#include <optional>
#include <vector>

#include "b2cnn_internal.cuh"

namespace b2cnn {

// workspace layout (floats)
struct TrainWs {
    int64_t f, pre0, acts, cs, hs, lin, z, da0, dfeat, part, off, dfw, roff, total;
};

constexpr int kT = 128;             // final features per tile
constexpr int kThreads = 256;       // threads of a conv tile's CTA
constexpr int kWin = 8;             // at most this many windows per CTA of the conv backward (one partial row per CTA)
constexpr int kBwdCtas = 1024;      // the conv backward puts several windows in a CTA only beyond this many CTAs
constexpr int kPre0Slice = 1024;    // positions per split-K slice of the pre-activation GEMM
constexpr int kWihChunks = 16;      // at most this many batch chunks in dW_ih_l0
constexpr int kRowBatch = 64;       // da0 rows staged per pass of train_dfeat / train_wih0_grad
constexpr int kSeqCtas = 256;       // at most this many CTAs scan the sequences of a batch (one partial row per CTA)

// The head's gradients (blob entries [o.whh0, o.bo], contiguous) and, after them, a loss sum: one scan CTA's partial row
__host__ __device__ inline int64_t head_row_len(const BlobOff &o) { return o.bo + 1 - o.whh0 + 1; }

// float offsets of a conv tile's buffers in dynamic shared memory; xp / pp are the row pitches of x and d1 / dd1
struct TileSmem {
    int w1, b1, w2, b2, x, xp, c1, d1, pp, c2, df, dc2, dd1, dc1, g, total;
};
// The largest tile: min(kT, L) features plus the few positions the last tile takes on beyond its last pooling window.
__host__ __device__ inline TileSmem tile_smem(const Dims &d, bool backward) {
    const int T = d.L < kT ? d.L : kT;
    const int n2 = d.PS * (T - 1) + d.PK + d.PS - 1, np1 = n2 + d.K2 - 1, n1 = d.PS * (np1 - 1) + d.PK + d.PS - 1, nx = n1 + d.K1 - 1;
    TileSmem s;
    int p = 0;
    auto take = [&](int n) { int at = p; p += (n + 3) / 4 * 4; return at; };
    s.w1 = take(kCMid * d.C * d.K1);      // [c][k][oc]
    s.b1 = take(kCMid);
    s.w2 = take(kCMid * d.K2);
    s.b2 = take(1);
    s.xp = (nx + 3) / 4 * 4;
    s.x = take(d.C * s.xp);
    s.c1 = take(kCMid * n1);              // [position][oc]
    s.pp = (np1 + 3) / 4 * 4;
    s.d1 = take(kCMid * s.pp);            // tanh(pool(c1)) * mask1
    s.c2 = take(n2);
    s.df = s.dc2 = s.dd1 = s.dc1 = s.g = 0;
    if (backward) {
        s.df = take(T);
        s.dc2 = take(n2);
        s.dd1 = take(kCMid * s.pp);
        s.dc1 = take(kCMid * n1);         // [position][oc]
        s.g = take((int)blob_offsets(d).wih0);   // the conv parameters' gradient sums
    }
    s.total = p;
    return s;
}

// The grids and the workspace of a shape; read by every entry point and by the workspace query.
struct TrainPlan {
    TrainWs w;
    int tiles, slices, wih_chunk, wih_chunks, win, groups, n_conv;
    int64_t part_rows;                  // per-CTA conv weight-gradient partials
    size_t smem_fwd, smem_bwd;
    int seq_per, seq_ctas;              // sequences per scan CTA, scan CTAs
};

// n_seq: the number of sequences of a _seq call, 0 for the calls that take a mode (their layout has no offsets region).
// rd: a _record call's recording geometry, whose n_rec recordings the conv kernels run over; B is then the number of
// counted windows (the scans' rows), and the layout gains the per-window d f [B][L] and the row offsets [n_rec + 1].
// heads: 0 for the calls that train one whole model; K >= 1 for a b2cnn_train_heads_* call, whose layout is f once and
// K copies of every per-row region ([K][B][...], head-major), with no d f and no conv-gradient partials.
static TrainPlan train_plan(const Dims &d, int64_t B, int64_t n_seq = 0, const Dims *rd = nullptr, int64_t n_rec = 0, int heads = 0) {
    TrainPlan pl{};
    const int64_t K = heads > 0 ? heads : 1;
    const Dims &cd = rd ? *rd : d;                      // the conv kernels' geometry and rows
    const int64_t cb = rd ? n_rec : B;
    // consecutive sequences per scan CTA: ceil(n_seq / kSeqCtas), from (B, n_seq) alone, never the device
    pl.seq_per = n_seq > kSeqCtas ? (int)((n_seq + kSeqCtas - 1) / kSeqCtas) : 1;
    pl.seq_ctas = n_seq > 0 ? (int)((n_seq + pl.seq_per - 1) / pl.seq_per) : 1;
    pl.tiles = (cd.L + kT - 1) / kT;
    pl.slices = (d.L + kPre0Slice - 1) / kPre0Slice;
    pl.wih_chunk = (int)((B + kWihChunks - 1) / kWihChunks);
    pl.wih_chunks = (int)((B + pl.wih_chunk - 1) / pl.wih_chunk);
    // windows per conv-backward CTA: ceil(B x tiles / kBwdCtas) within [1, kWin], from the shape alone, never the device
    const int64_t bt = cb * pl.tiles, win = (bt + kBwdCtas - 1) / kBwdCtas;
    pl.win = (int)(win < 1 ? 1 : win > kWin ? kWin : win);
    pl.groups = (int)((cb + pl.win - 1) / pl.win);
    pl.n_conv = (int)blob_offsets(d).wih0;
    pl.part_rows = (int64_t)pl.tiles * pl.groups;
    pl.smem_fwd = sizeof(float) * tile_smem(cd, false).total;
    pl.smem_bwd = sizeof(float) * tile_smem(cd, true).total;
    TrainWs &w = pl.w;
    int64_t p = 0;
    auto take = [&](int64_t n) { int64_t at = p; p += (n + 63) / 64 * 64; return at; };
    w.f = take(cb * cd.L);
    w.pre0 = take(K * B * kGates);      // f . W_ih_l0^T
    w.acts = take(K * B * 2 * kGates);  // [t][layer][i f g o] post-activation
    w.cs = take(K * B * 2 * kHidden);   // [t][layer] cell state
    w.hs = take(K * B * 2 * kHidden);   // [t][layer] hidden state
    w.lin = take(K * B);                // out(h1) before the age scale (d age needs it)
    w.z = take(K * B);
    w.da0 = take(K * B * kGates);       // d loss / d (layer-0 gate pre-activations)
    w.dfeat = take(heads ? 0 : cb * cd.L);
    // one region for the partial sums of three reductions that never overlap in time
    int64_t part = (int64_t)pl.slices * K * B * kGates;
    if ((int64_t)pl.wih_chunks * K * kGates * d.L > part) part = (int64_t)pl.wih_chunks * K * kGates * d.L;
    if (!heads && pl.part_rows * pl.n_conv > part) part = pl.part_rows * pl.n_conv;
    // the scan CTAs' head rows: written by the LSTM kernels and summed before any other reduction uses the region
    if (pl.seq_ctas > 1 && K * pl.seq_ctas * head_row_len(blob_offsets(d)) > part) part = K * pl.seq_ctas * head_row_len(blob_offsets(d));
    w.part = take(part);
    w.off = n_seq > 0 ? take(2 * (n_seq + 1)) : 0;     // int64 sequence offsets [n_seq + 1], copied in by every _seq call
    w.dfw = rd && !heads ? take(B * d.L) : 0;          // the windows' d f, folded into dfeat
    w.roff = rd ? take(2 * (n_rec + 1)) : 0;           // int64 row offsets of the recordings, copied in by every _record call
    w.total = p;
    return pl;
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

// The sequences of a batch.  off == nullptr: one sequence of all B rows (with sequence == 0: B sequences of one row),
// scanned by one CTA.  Otherwise sequence s is rows [off[s], off[s + 1]) and CTA c scans sequences [c per, min(n, (c + 1)
// per)) in order, each from the zero state.  rows == nullptr: the (only) CTA writes the head's gradients into grad and the
// mean loss into loss_out; otherwise CTA c writes row c of rows [CTAs][head_row_len(o)] (its gradients of blob entries
// [o.whh0, o.bo], then its loss sum), which train_head_reduce adds up.
struct SeqSpan {
    const int64_t *off;
    int64_t n;
    int per;
    float *rows;
};

// The rows of a _record call: recording b holds rows [roff[b], roff[b + 1]) (its counted windows, in order); window w of
// it starts at sample w S, i.e. at feature w sf (sf = S / F) of the recording's L_N = LN features, and holds Lw of them.
struct RecRows {
    const int64_t *roff;
    int64_t nrec;
    int S, sf, W, Lw, LN;
};
// the recording of row m: the last b with roff[b] <= m (a recording without windows never matches)
__device__ __forceinline__ int64_t rec_row_base(const RecRows &r, int64_t m) {
    int64_t lo = 0, hi = r.nrec - 1;
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (r.roff[mid] <= m) lo = mid; else hi = mid - 1;
    }
    return lo * r.LN + (m - r.roff[lo]) * r.sf;          // where the window's features start in f [nrec][LN]
}
// the windows [lo, hi] of a recording with n counted windows whose features include recording feature p (empty: lo > hi)
__device__ __forceinline__ int64_t rec_first_window(const RecRows &r, int p) { return p >= r.Lw ? (p - r.Lw) / r.sf + 1 : 0; }
__device__ __forceinline__ int64_t rec_last_window(const RecRows &r, int64_t n, int p) { return min(n - 1, (int64_t)(p / r.sf)); }
// does a counted window hold one of the features [i0, i0 + nf)?
__device__ __forceinline__ bool rec_covers(const RecRows &r, int64_t n, int i0, int nf) {
    return rec_first_window(r, i0) <= rec_last_window(r, n, i0 + nf - 1);
}
// does a counted window read sample s? (the last window starting at or before s is the one that can)
__device__ __forceinline__ bool rec_reads(const RecRows &r, int64_t n, int s) {
    const int64_t w = min(n - 1, (int64_t)(s / r.S));
    return w >= 0 && s < w * r.S + r.W;
}

// The heads the scans train: blockIdx.y = h reads head h's blob prm[h] and writes its gradients to grad[h].  The calls
// that train one model launch gridDim.y = 1 with their blob at h = 0; a b2cnn_train_heads_* call launches one grid row
// per head, and head h's per-row regions lie at h B rows into each region of the workspace.
constexpr int kMaxHeads = B2CNN_SLIDE_MAX_HEADS;
struct ScanHeads {
    const float *prm[kMaxHeads];
    float *grad[kMaxHeads];
};
// a b2cnn_train_heads_* call's blobs, Adam state and learning rates (host arrays copied into the kernel parameters)
struct AdamHeads {
    float *prm[kMaxHeads], *m[kMaxHeads], *v[kMaxHeads];
    const float *grad[kMaxHeads];
    float lr[kMaxHeads];
};

// The LSTM state of each recording of a _record_state call (RecordArgs), [nrec][64] = h0 | c0 | h1 | c1; every pointer
// null for every other call.  A scan's sequence is a recording with windows, found from its first row in roff.
struct ScanState {
    const float *in;
    float *out;
    const float *d_out;
    float *d_in;
    const int64_t *roff;
    int64_t nrec;
};
// the recording whose rows start at row m: the last b with roff[b] <= m
__device__ __forceinline__ int64_t scan_recording(const ScanState &ss, int64_t m) {
    int64_t lo = 0, hi = ss.nrec - 1;
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (ss.roff[mid] <= m) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ------------------------------------------------------------------------------------------------------------------
// LSTM forward over the batch axis with everything the backward pass needs kept; logits and loss.
// A CTA of 64 threads per group of sequences (SeqSpan): thread r owns gate row r of every matrix; W_ih_l0 f_t was
// computed before the scan (pre0[t][r]).  sequence == 0: every step starts from the zero state (independent windows).
// A sequence starts from the zero state, or from its recording's row of ss.in, and with ss.out its final state is
// stored there (STATE == false: ss is ignored, and the kernel compiles to the scan without it).  HEAD == kHeadLogits:
// target and loss_out are not used.  blockIdx.y: the head (ScanHeads), whose mean loss goes to loss_out[blockIdx.y].
// ------------------------------------------------------------------------------------------------------------------
template <int HEAD, bool STATE>
__device__ __forceinline__ void
lstm_fwd_body(const float *__restrict__ pre0, const float *__restrict__ prm, BlobOff o, Dims d, int64_t B, int sequence, SeqSpan sq,
              const float *__restrict__ age, const float *__restrict__ target, float pos_weight, float *__restrict__ acts,
              float *__restrict__ cs, float *__restrict__ hs, float *__restrict__ lin, float *__restrict__ z,
              float *__restrict__ loss_out, ScanState ss) {
    if constexpr (!STATE) ss = ScanState{};
    __shared__ float g[kGates], h0[kHidden], c0[kHidden], h1[kHidden], c1s[kHidden];
    const int r = threadIdx.x;
    // this CTA's sequences [s0, s1); one sequence of all B rows without offsets
    const int64_t s0 = sq.off ? (int64_t)blockIdx.x * sq.per : 0, s1 = sq.off ? min(sq.n, s0 + sq.per) : 1;
    float loss = 0.f;
    for (int64_t sid = s0; sid < s1; ++sid) {            // the body is the single-sequence scan, over rows [t0, t1)
    const int64_t t0 = sq.off ? sq.off[sid] : 0, t1 = sq.off ? sq.off[sid + 1] : B;
    const int64_t rec = ss.in || ss.out ? scan_recording(ss, t0) : 0;
    if (r < kHidden) {
        if (ss.in) {
            const float *si = ss.in + rec * kGates;
            h0[r] = si[r]; c0[r] = si[kHidden + r]; h1[r] = si[2 * kHidden + r]; c1s[r] = si[3 * kHidden + r];
        } else {
            h0[r] = c0[r] = h1[r] = c1s[r] = 0.f;
        }
    }
    __syncthreads();
    for (int64_t t = t0; t < t1; ++t) {
        if (!sequence) {
            if (r < kHidden) { h0[r] = c0[r] = h1[r] = c1s[r] = 0.f; }
            __syncthreads();
        }
        // ---- layer 0: g = (W_ih f_t + b_ih) + (W_hh h_{t-1} + b_hh)
        {
            const float a = pre0[t * kGates + r];
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
    if (ss.out && r < kHidden) {                          // each thread stores the units it wrote last
        float *so = ss.out + rec * kGates;
        so[r] = h0[r]; so[kHidden + r] = c0[r]; so[2 * kHidden + r] = h1[r]; so[3 * kHidden + r] = c1s[r];
    }
    }
    if (HEAD != kHeadLogits && r == 0) {
        if (sq.rows) sq.rows[blockIdx.x * head_row_len(o) + head_row_len(o) - 1] = loss;
        else *loss_out = loss / (float)B;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// BPTT over the batch axis (over each CTA's sequences, SeqSpan).  64 threads: thread r owns gate row r.  Gradients of
// the recurrent matrices, biases and of the head are accumulated in registers / shared memory and written once (into
// grad, or as the CTA's row of sq.rows); d(gates of layer 0) goes to da0[t][64].
// HEAD == kHeadLogits: d loss / d z is dz_in[t] and, when dage != NULL, d loss / d age goes to dage[t] (torch's relu
// backward: zero where relu(age * coef + 1) is not positive); otherwise dz comes from z and target, dage is not written.
// With ss.in, a sequence's first step reads its recording's initial state (h_{t-1}, c_{t-1}) there instead of zeros;
// with ss.d_out, the carried d h / d c start from the gradient arriving at the final state instead of zeros; with
// ss.d_in, the carries after the first step -- d loss / d (initial state) -- are stored there (STATE == false: as for
// train_lstm_fwd).  blockIdx.y: the head, as in train_lstm_fwd (dz_in and dage belong to gridDim.y = 1 launches).
// ------------------------------------------------------------------------------------------------------------------
template <int HEAD, bool STATE>
__device__ __forceinline__ void
lstm_bwd_body(const float *__restrict__ prm, BlobOff o, Dims d, int64_t B, int sequence, SeqSpan sq, const float *__restrict__ age,
              const float *__restrict__ target, float pos_weight, const float *__restrict__ dz_in, const float *__restrict__ acts,
              const float *__restrict__ cs, const float *__restrict__ hs, const float *__restrict__ lin, const float *__restrict__ z,
              float *__restrict__ da0, float *__restrict__ grad, float *__restrict__ dage, ScanState ss) {
    if constexpr (!STATE) ss = ScanState{};
    __shared__ float da[kGates], dh0c[kHidden], dc0c[kHidden], dh1c[kHidden], dc1c[kHidden], dh0ext[kHidden], dh1ext[kHidden];
    const int r = threadIdx.x, u = r & 15, q = r >> 4;
    // this CTA's sequences [s0, s1), walked last to first; one sequence of all B rows without offsets
    const int64_t s0 = sq.off ? (int64_t)blockIdx.x * sq.per : 0, s1 = sq.off ? min(sq.n, s0 + sq.per) : 1;
    float gWhh0[kHidden], gWih1[kHidden], gWhh1[kHidden];
#pragma unroll
    for (int k = 0; k < kHidden; ++k) gWhh0[k] = gWih1[k] = gWhh1[k] = 0.f;
    float gb0 = 0.f, gb1 = 0.f, gwo = 0.f, gbo = 0.f;
    for (int64_t sid = s1 - 1; sid >= s0; --sid) {       // the body is the single-sequence walk, over rows [t0, t1)
    const int64_t t0 = sq.off ? sq.off[sid] : 0, t1 = sq.off ? sq.off[sid + 1] : B;
    const int64_t rec = ss.in || ss.d_out || ss.d_in ? scan_recording(ss, t0) : 0;
    const float *const sin = ss.in ? ss.in + rec * kGates : nullptr;      // h0 | c0 | h1 | c1 before step t0
    if (r < kHidden) {
        if (ss.d_out) {
            const float *g = ss.d_out + rec * kGates;
            dh0c[r] = g[r]; dc0c[r] = g[kHidden + r]; dh1c[r] = g[2 * kHidden + r]; dc1c[r] = g[3 * kHidden + r];
        } else {
            dh0c[r] = dc0c[r] = dh1c[r] = dc1c[r] = 0.f;
        }
    }
    __syncthreads();
    for (int64_t t = t1 - 1; t >= t0; --t) {
        if (!sequence) {
            if (r < kHidden) dh0c[r] = dc0c[r] = dh1c[r] = dc1c[r] = 0.f;
            __syncthreads();
        }
        const bool first = !sequence || t == t0;              // no previous step: h_{t-1}, c_{t-1} = 0 or from sin
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
            const float cprev = first ? (sin ? sin[3 * kHidden + u] : 0.f) : cs[((t - 1) * 2 + 1) * kHidden + u];
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
                gWhh1[k] += v * (first ? (sin ? sin[2 * kHidden + k] : 0.f) : hs[((t - 1) * 2 + 1) * kHidden + k]);  // v * 0: a NaN v still counts
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
            const float cprev = first ? (sin ? sin[kHidden + u] : 0.f) : cs[((t - 1) * 2 + 0) * kHidden + u];
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
            for (int k = 0; k < kHidden; ++k) gWhh0[k] += v * (first ? (sin ? sin[k] : 0.f) : hs[((t - 1) * 2 + 0) * kHidden + k]);
        }
        __syncthreads();
        if (r < kHidden) {
            float e = 0.f;
            for (int rr = 0; rr < kGates; ++rr) e = fmaf(prm[o.whh0 + rr * kHidden + r], da[rr], e);
            dh0c[r] = e;
        }
        __syncthreads();
    }
    if (ss.d_in && r < kHidden) {                         // the carries after the first step: d (h0, c0, h1, c1)
        float *g = ss.d_in + rec * kGates;
        g[r] = dh0c[r]; g[kHidden + r] = dc0c[r]; g[2 * kHidden + r] = dh1c[r]; g[3 * kHidden + r] = dc1c[r];
    }
    }
    // blob entry e of the head goes to grad[e], or to entry e - o.whh0 of this CTA's row
    float *const gout = sq.rows ? sq.rows + blockIdx.x * head_row_len(o) : grad;
    const int64_t base = sq.rows ? o.whh0 : 0;
#pragma unroll
    for (int k = 0; k < kHidden; ++k) {
        gout[o.whh0 - base + r * kHidden + k] = gWhh0[k];
        gout[o.wih1 - base + r * kHidden + k] = gWih1[k];
        gout[o.whh1 - base + r * kHidden + k] = gWhh1[k];
    }
    gout[o.bih0 - base + r] = gb0; gout[o.bhh0 - base + r] = gb0;
    gout[o.bih1 - base + r] = gb1; gout[o.bhh1 - base + r] = gb1;
    if (r < kHidden) gout[o.wo - base + r] = gwo;
    if (r == 0) gout[o.bo - base] = gbo;
}

// The scans of head blockIdx.y: its blob and gradients from hd, its rows of every per-row region at blockIdx.y B, its
// loss at loss_out[blockIdx.y] and its CTAs' head rows after the previous head's.  The bodies take the pointers as
// __restrict__ arguments, so the weights' loads are hoisted out of the scan as in a kernel of one model.
template <int HEAD, bool STATE>
__global__ void __launch_bounds__(64)
train_lstm_fwd(const float *__restrict__ pre0, const __grid_constant__ ScanHeads hd, BlobOff o, Dims d, int64_t B, int sequence, SeqSpan sq,
               const float *__restrict__ age, const float *__restrict__ target, float pos_weight, float *__restrict__ acts,
               float *__restrict__ cs, float *__restrict__ hs, float *__restrict__ lin, float *__restrict__ z,
               float *__restrict__ loss_out, ScanState ss) {
    const int64_t hb = (int64_t)blockIdx.y * B;
    if (sq.rows) sq.rows += (int64_t)blockIdx.y * gridDim.x * head_row_len(o);
    lstm_fwd_body<HEAD, STATE>(pre0 + hb * kGates, hd.prm[blockIdx.y], o, d, B, sequence, sq, age, target, pos_weight, acts + hb * 2 * kGates,
                               cs + hb * 2 * kHidden, hs + hb * 2 * kHidden, lin + hb, z + hb, loss_out ? loss_out + blockIdx.y : nullptr, ss);
}
template <int HEAD, bool STATE>
__global__ void __launch_bounds__(64, 1)   // the 48 gradient sums stay in registers: no spill
train_lstm_bwd(const __grid_constant__ ScanHeads hd, BlobOff o, Dims d, int64_t B, int sequence, SeqSpan sq, const float *__restrict__ age,
               const float *__restrict__ target, float pos_weight, const float *__restrict__ dz_in, const float *__restrict__ acts,
               const float *__restrict__ cs, const float *__restrict__ hs, const float *__restrict__ lin, const float *__restrict__ z,
               float *__restrict__ da0, float *__restrict__ dage, ScanState ss) {
    const int64_t hb = (int64_t)blockIdx.y * B;
    if (sq.rows) sq.rows += (int64_t)blockIdx.y * gridDim.x * head_row_len(o);
    lstm_bwd_body<HEAD, STATE>(hd.prm[blockIdx.y], o, d, B, sequence, sq, age, target, pos_weight, dz_in, acts + hb * 2 * kGates,
                               cs + hb * 2 * kHidden, hs + hb * 2 * kHidden, lin + hb, z + hb, da0 + hb * kGates, hd.grad[blockIdx.y], dage, ss);
}

// grad[o.whh0 + e] = the sum of rows[c][e] over the scan CTAs c in order, i.e. in sequence order (no atomic: gradients
// repeat bit for bit); the rows' last column is the loss sum, and loss_out (when not NULL) gets that sum / B.
// blockIdx.y: the head, whose rows follow the previous head's and whose gradients go to hd.grad[blockIdx.y]
__global__ void __launch_bounds__(256)
train_head_reduce(const float *__restrict__ rows, int n_rows, BlobOff o, int64_t B, const __grid_constant__ ScanHeads hd, float *__restrict__ loss_out) {
    const int64_t len = head_row_len(o), e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= len) return;
    rows += (int64_t)blockIdx.y * n_rows * len;
    float a = rows[e];
    for (int c = 1; c < n_rows; ++c) a += rows[c * len + e];
    if (e < len - 1) hd.grad[blockIdx.y][o.whh0 + e] = a;
    else if (loss_out) loss_out[blockIdx.y] = a / (float)B;
}

// ------------------------------------------------------------------------------------------------------------------
// Position tiles.
// Tile `tile` of a window owns final features [i0, i0 + nf).  Their receptive span starts at c2 / p1 position
// s2 = PS i0 and at c1 / x position s1 = PS s2 and holds n2 / np1 / n1 / nx positions of c2 / p1 / c1 / x.  The last tile
// also takes the positions after the last pooling window (a geometry may leave a few): they get no gradient, but a NaN
// there reaches d tanh and so the conv gradients, as in the reference.
// ------------------------------------------------------------------------------------------------------------------
struct Tile {
    int i0, nf, s2, s1, n2, np1, n1, nx;
};
__device__ __forceinline__ Tile tile_of(const Dims &d, int tile) {
    Tile t;
    t.i0 = tile * kT;
    t.nf = min(kT, d.L - t.i0);
    t.s2 = d.PS * t.i0;
    t.s1 = d.PS * t.s2;
    const bool last = t.i0 + t.nf == d.L;
    t.n2 = last ? d.L2 - t.s2 : d.PS * (t.nf - 1) + d.PK;
    t.np1 = last ? d.P1 - t.s2 : t.n2 + d.K2 - 1;
    t.n1 = last ? d.L1 - t.s1 : d.PS * (t.np1 - 1) + d.PK;
    t.nx = last ? d.W - t.s1 : t.n1 + d.K1 - 1;
    return t;
}

// conv weights into shared memory; conv1's as [c][k][oc], so one 16-byte load feeds the four output channels of a tap
__device__ __forceinline__ void tile_stage_weights(const float *__restrict__ prm, const BlobOff &o, const Dims &d, const TileSmem &s,
                                                   float *sm, int tid) {
    const int ck = d.C * d.K1;
    for (int e = tid; e < kCMid * ck; e += kThreads) sm[s.w1 + (e % ck) * kCMid + e / ck] = prm[o.w1 + e];
    if (tid < kCMid) sm[s.b1 + tid] = prm[o.b1 + tid];
    for (int e = tid; e < kCMid * d.K2; e += kThreads) sm[s.w2 + e] = prm[o.w2 + e];
    if (tid == 0) sm[s.b2] = prm[o.b2];
}

// One tile of one window, everything in shared memory: x span -> c1 -> pool -> tanh -> mask1 (d1) -> c2.  Every sum in
// the inference kernels' order (an fmaf chain from the bias, channels outer, taps inner), so a value does not depend on
// the tile that computes it.  Pooling comes before tanh: tanh is monotone, and a NaN in the window wins either way.
// xb / m1b: the window's x [C][W] and its mask1 [4][P1] (or NULL).  Ends with a barrier.
// ZERO: xb is a recording with n counted windows (rr), and a sample none of them reads is staged as 0.
template <bool ZERO = false>
__device__ __forceinline__ void conv_tile(const float *__restrict__ xb, const float *__restrict__ m1b, const Dims &d, const Tile &t,
                                          const TileSmem &s, float *sm, int tid, const RecRows *rr = nullptr, int64_t n = 0) {
    for (int c = 0; c < d.C; ++c)
        for (int j = tid; j < t.nx; j += kThreads) {
            float v = xb[(int64_t)c * d.W + t.s1 + j];
            if constexpr (ZERO) v = rec_reads(*rr, n, t.s1 + j) ? v : 0.f;
            sm[s.x + c * s.xp + j] = v;
        }
    __syncthreads();
    for (int j = tid; j < t.n1; j += kThreads) {
        float4 acc = *reinterpret_cast<const float4 *>(sm + s.b1);
        for (int c = 0; c < d.C; ++c) {
            const float *xr = sm + s.x + c * s.xp + j;
            const float4 *wr = reinterpret_cast<const float4 *>(sm + s.w1) + c * d.K1;
            for (int k = 0; k < d.K1; ++k) {
                const float4 w = wr[k];
                const float xv = xr[k];
                acc.x = fmaf(w.x, xv, acc.x); acc.y = fmaf(w.y, xv, acc.y); acc.z = fmaf(w.z, xv, acc.z); acc.w = fmaf(w.w, xv, acc.w);
            }
        }
        *reinterpret_cast<float4 *>(sm + s.c1 + 4 * j) = acc;
    }
    __syncthreads();
    for (int e = tid; e < kCMid * t.np1; e += kThreads) {
        const int oc = e / t.np1, i = e % t.np1;
        const float *col = sm + s.c1 + oc;
        float m = col[4 * d.PS * i];
        for (int j = 1; j < d.PK; ++j) m = max_nan(m, col[4 * (d.PS * i + j)]);
        sm[s.d1 + oc * s.pp + i] = tanhf(m) * (m1b ? m1b[(int64_t)oc * d.P1 + t.s2 + i] : 1.0f);
    }
    __syncthreads();
    for (int j = tid; j < t.n2; j += kThreads) {
        float acc = sm[s.b2];
        for (int oc = 0; oc < kCMid; ++oc)
            for (int k = 0; k < d.K2; ++k) acc = fmaf(sm[s.w2 + oc * d.K2 + k], sm[s.d1 + oc * s.pp + j + k], acc);
        sm[s.c2 + j] = acc;
    }
    __syncthreads();
}

// grid: B x tiles CTAs, window-major.  REC: d is a recording's geometry, and a tile that no counted window of it reaches
// writes nothing (f there is never read)
template <bool REC>
__device__ __forceinline__ void train_conv_fwd_body(const float *__restrict__ x, const float *__restrict__ prm, BlobOff o, Dims d, int tiles,
               const float *__restrict__ mask1, const float *__restrict__ mask2, float *__restrict__ f, const RecRows &rr) {
    extern __shared__ __align__(16) float sm[];
    const TileSmem s = tile_smem(d, false);
    const int tid = threadIdx.x;
    const int64_t b = blockIdx.x / tiles;
    const Tile t = tile_of(d, blockIdx.x % tiles);
    if constexpr (REC) {
        if (!rec_covers(rr, rr.roff[b + 1] - rr.roff[b], t.i0, t.nf)) return;
    }
    tile_stage_weights(prm, o, d, s, sm, tid);
    conv_tile(x + b * d.C * d.W, mask1 ? mask1 + b * kCMid * d.P1 : nullptr, d, t, s, sm, tid);
    for (int i = tid; i < t.nf; i += kThreads) {
        float m = sm[s.c2 + d.PS * i];
        for (int j = 1; j < d.PK; ++j) m = max_nan(m, sm[s.c2 + d.PS * i + j]);
        f[b * d.L + t.i0 + i] = tanhf(m) * (mask2 ? mask2[b * d.L + t.i0 + i] : 1.0f);
    }
}
__global__ void __launch_bounds__(kThreads)
train_conv_fwd(const float *__restrict__ x, const float *__restrict__ prm, BlobOff o, Dims d, int tiles,
               const float *__restrict__ mask1, const float *__restrict__ mask2, float *__restrict__ f) {
    train_conv_fwd_body<false>(x, prm, o, d, tiles, mask1, mask2, f, RecRows{});
}
__global__ void __launch_bounds__(kThreads)
train_conv_fwd_record(const float *__restrict__ x, const float *__restrict__ prm, BlobOff o, Dims d, int tiles,
               const float *__restrict__ mask1, const float *__restrict__ mask2, float *__restrict__ f, RecRows rr) {
    train_conv_fwd_body<true>(x, prm, o, d, tiles, mask1, mask2, f, rr);
}

// pre0 partial[slice][b][g] = sum over the slice's positions of f[b][p] W_ih_l0[g][p]: 64 windows x 64 gates per CTA,
// K chunks of 32, a 4 x 4 register tile per thread (the tiling of the inference projection, reading W_ih_l0 as stored)
// REC: row b is a window of a recording (rr), read in place from the recording's feature row.
// HP heads per CTA: the f tile is staged once for all of them, head h multiplies it by its own W_ih_l0 wih0[h] into its
// own accumulators (in the order of HP = 1) and writes partial[slice][b][g] at part[h] + slice pstride 64 (pstride = B
// for one head; K B for K heads' partials laid out [slice][K][B][64])
constexpr int kGemmK = 32, kGemmStride = 68;
template <bool REC, int HP>
__device__ __forceinline__ void train_pre0_partial_body(const float *__restrict__ f, const float *const (&wih0)[HP], int64_t B, int64_t pstride,
                                                        int L, float *const (&part)[HP], const RecRows &rr) {
    __shared__ __align__(16) float Fs[kGemmK][kGemmStride];
    __shared__ __align__(16) float Ws[HP][kGemmK][kGemmStride];
    const int tid = threadIdx.x, tm = tid >> 4, tn = tid & 15;
    const int64_t b0 = (int64_t)blockIdx.x * 64;
    const int kbeg = blockIdx.y * kPre0Slice, kend = min(L, kbeg + kPre0Slice);
    [[maybe_unused]] __shared__ int64_t row_at[REC ? 64 : 1];
    if constexpr (REC) {
        if (tid < 64 && b0 + tid < B) row_at[tid] = rec_row_base(rr, b0 + tid);
        __syncthreads();
    }
    float acc[HP][4][4];
#pragma unroll
    for (int h = 0; h < HP; ++h)
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[h][i][j] = 0.f;
    for (int k0 = kbeg; k0 < kend; k0 += kGemmK) {
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            const int e = tid + it * 256, m = e >> 5, kk = e & 31, k = k0 + kk;
            if constexpr (REC) Fs[kk][m] = (b0 + m < B && k < kend) ? f[row_at[m] + k] : 0.f;
            else Fs[kk][m] = (b0 + m < B && k < kend) ? f[(b0 + m) * L + k] : 0.f;
#pragma unroll
            for (int h = 0; h < HP; ++h) Ws[h][kk][m] = k < kend ? wih0[h][(int64_t)m * L + k] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kGemmK; ++kk) {
            const float4 a = *reinterpret_cast<const float4 *>(&Fs[kk][4 * tm]);
            const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int h = 0; h < HP; ++h) {
                const float4 w = *reinterpret_cast<const float4 *>(&Ws[h][kk][4 * tn]);
                const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[h][i][j] = fmaf(av[i], wv[j], acc[h][i][j]);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int h = 0; h < HP; ++h)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t b = b0 + 4 * tm + i;
            if (b < B)
                *reinterpret_cast<float4 *>(part[h] + ((int64_t)blockIdx.y * pstride + b) * kGates + 4 * tn) =
                    make_float4(acc[h][i][0], acc[h][i][1], acc[h][i][2], acc[h][i][3]);
        }
}
__global__ void __launch_bounds__(256)
train_pre0_partial(const float *__restrict__ f, const float *__restrict__ wih0, int64_t B, int L, float *__restrict__ part) {
    const float *const w[1] = {wih0};
    float *const p[1] = {part};
    train_pre0_partial_body<false, 1>(f, w, B, B, L, p, RecRows{});
}
__global__ void __launch_bounds__(256)
train_pre0_partial_record(const float *__restrict__ f, const float *__restrict__ wih0, int64_t B, int L, float *__restrict__ part, RecRows rr) {
    const float *const w[1] = {wih0};
    float *const p[1] = {part};
    train_pre0_partial_body<true, 1>(f, w, B, B, L, p, rr);
}
// The K heads of a b2cnn_train_heads_* call, kPre0Heads per CTA on gridDim.z: CTA z projects heads 2z and 2z + 1 into
// their slots of part [slice][K][B][64].  With an odd K the last CTA's second head is its first again: it computes the
// same partials twice and stores the same bits to the same place.
constexpr int kPre0Heads = 2;
template <bool REC>
__global__ void __launch_bounds__(256)
train_pre0_partial_heads(const float *__restrict__ f, const __grid_constant__ ScanHeads hd, int n_heads, BlobOff o, int64_t B, int L, float *__restrict__ part, RecRows rr) {
    const float *w[kPre0Heads];
    float *p[kPre0Heads];
#pragma unroll
    for (int i = 0; i < kPre0Heads; ++i) {
        const int h = min((int)blockIdx.z * kPre0Heads + i, n_heads - 1);
        w[i] = hd.prm[h] + o.wih0;
        p[i] = part + (int64_t)h * B * kGates;
    }
    train_pre0_partial_body<REC, kPre0Heads>(f, w, B, (int64_t)n_heads * B, L, p, rr);
}

// out[e] = part[0][e] + part[1][e] + ... in that order (split-K slices of pre0, batch chunks of dW_ih_l0)
__global__ void train_sum_chunks(const float *__restrict__ part, int n_chunks, int64_t n, float *__restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    float a = part[e];
    for (int c = 1; c < n_chunks; ++c) a += part[(int64_t)c * n + e];
    out[e] = a;
}

// dW_ih_l0 partial[chunk][g][p] = sum over the chunk's windows t (ascending) of da0[t][g] f[t][p].  Thread = position p
// with the 64 gate rows' sums in registers, so f is read once; grid (position tiles of 128, batch chunks).  REC: window t
// is read in place from its recording's feature row (rr).  HP heads per CTA: f is read once per position for all of
// them, head h's sums (in the order of HP = 1) come from its own da0[h] and go to part[h].
template <bool REC, int HP>
__device__ __forceinline__ void train_wih0_grad_body(const float *const (&da0)[HP], const float *__restrict__ f, int64_t B, int L, int chunk,
                                                     float *const (&part)[HP], const RecRows &rr) {
    __shared__ __align__(16) float sda[HP][kRowBatch * kGates];
    [[maybe_unused]] __shared__ int64_t row_at[REC ? kRowBatch : 1];
    const int p = blockIdx.x * 128 + threadIdx.x;
    const int64_t t0 = (int64_t)blockIdx.y * chunk, t1 = min(B, t0 + chunk);
    float acc[HP][kGates];
#pragma unroll
    for (int h = 0; h < HP; ++h)
#pragma unroll
        for (int g = 0; g < kGates; ++g) acc[h][g] = 0.f;
    for (int64_t tb = t0; tb < t1; tb += kRowBatch) {
        const int rows = (int)min((int64_t)kRowBatch, t1 - tb);
        __syncthreads();
        for (int e = threadIdx.x; e < rows * kGates; e += 128)
#pragma unroll
            for (int h = 0; h < HP; ++h) sda[h][e] = da0[h][tb * kGates + e];
        if constexpr (REC) {
            if (threadIdx.x < rows) row_at[threadIdx.x] = rec_row_base(rr, tb + threadIdx.x);
        }
        __syncthreads();
        if (p < L)
            for (int r = 0; r < rows; ++r) {
                float fv;
                if constexpr (REC) fv = f[row_at[r] + p];
                else fv = f[(tb + r) * L + p];
#pragma unroll
                for (int h = 0; h < HP; ++h)
#pragma unroll
                    for (int g4 = 0; g4 < kGates / 4; ++g4) {
                        const float4 a = *reinterpret_cast<const float4 *>(sda[h] + r * kGates + 4 * g4);
                        acc[h][4 * g4 + 0] = fmaf(a.x, fv, acc[h][4 * g4 + 0]); acc[h][4 * g4 + 1] = fmaf(a.y, fv, acc[h][4 * g4 + 1]);
                        acc[h][4 * g4 + 2] = fmaf(a.z, fv, acc[h][4 * g4 + 2]); acc[h][4 * g4 + 3] = fmaf(a.w, fv, acc[h][4 * g4 + 3]);
                    }
            }
    }
    if (p < L)
#pragma unroll
        for (int h = 0; h < HP; ++h)
#pragma unroll
            for (int g = 0; g < kGates; ++g) part[h][((int64_t)blockIdx.y * kGates + g) * L + p] = acc[h][g];
}
__global__ void __launch_bounds__(128)
train_wih0_grad(const float *__restrict__ da0, const float *__restrict__ f, int64_t B, int L, int chunk, float *__restrict__ part) {
    const float *const a[1] = {da0};
    float *const p[1] = {part};
    train_wih0_grad_body<false, 1>(a, f, B, L, chunk, p, RecRows{});
}
__global__ void __launch_bounds__(128)
train_wih0_grad_record(const float *__restrict__ da0, const float *__restrict__ f, int64_t B, int L, int chunk, float *__restrict__ part, RecRows rr) {
    const float *const a[1] = {da0};
    float *const p[1] = {part};
    train_wih0_grad_body<true, 1>(a, f, B, L, chunk, p, rr);
}
// The K heads of a b2cnn_train_heads_* call, kWihHeads per CTA on gridDim.z (an odd K's last CTA repeats its head, as
// train_pre0_partial_heads does).  Head h reads its da0 at h B rows; with one batch chunk its sums go straight to its
// gradient blob, else to its slot of part [K][chunks][64][L].  The CTAs of the first position tile and chunk also zero
// their heads' conv entries of the gradient blob: the front end is frozen.
constexpr int kWihHeads = 2;
template <bool REC>
__global__ void __launch_bounds__(128)
train_wih0_grad_heads(const float *__restrict__ da0, const float *__restrict__ f, const __grid_constant__ ScanHeads hd, int n_heads, BlobOff o, int64_t B, int L,
                      int chunk, int n_chunks, float *__restrict__ part, RecRows rr) {
    const float *a[kWihHeads];
    float *p[kWihHeads];
#pragma unroll
    for (int i = 0; i < kWihHeads; ++i) {
        const int h = min((int)blockIdx.z * kWihHeads + i, n_heads - 1);
        a[i] = da0 + (int64_t)h * B * kGates;
        p[i] = n_chunks > 1 ? part + (int64_t)h * n_chunks * kGates * L : hd.grad[h] + o.wih0;
        if (blockIdx.x == 0 && blockIdx.y == 0)
            for (int e = threadIdx.x; e < o.wih0; e += 128) hd.grad[h][e] = 0.f;
    }
    train_wih0_grad_body<REC, kWihHeads>(a, f, B, L, chunk, p, rr);
}

// dW_ih_l0 of head blockIdx.y = the sum of its batch-chunk partials in chunk order (train_sum_chunks per head)
__global__ void __launch_bounds__(256)
train_wih0_sum_heads(const float *__restrict__ part, int n_chunks, int64_t n, const __grid_constant__ ScanHeads hd, BlobOff o) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    part += (int64_t)blockIdx.y * n_chunks * n;
    float a = part[e];
    for (int c = 1; c < n_chunks; ++c) a += part[(int64_t)c * n + e];
    hd.grad[blockIdx.y][o.wih0 + e] = a;
}

// d f[t][p] = sum_g da0[t][g] W_ih_l0[g][p], g ascending; thread = position p with its 64 weights in registers, grid
// (position tiles of 128, groups of kRowBatch windows)
__global__ void __launch_bounds__(128)
train_dfeat(const float *__restrict__ da0, const float *__restrict__ wih0, int64_t B, int L, float *__restrict__ dfeat) {
    __shared__ __align__(16) float sda[kRowBatch * kGates];
    const int p = blockIdx.x * 128 + threadIdx.x;
    const int64_t t0 = (int64_t)blockIdx.y * kRowBatch;
    const int rows = (int)min((int64_t)kRowBatch, B - t0);
    for (int e = threadIdx.x; e < rows * kGates; e += 128) sda[e] = da0[t0 * kGates + e];
    __syncthreads();
    if (p >= L) return;
    float w[kGates];
#pragma unroll
    for (int g = 0; g < kGates; ++g) w[g] = wih0[(int64_t)g * L + p];
    for (int r = 0; r < rows; ++r) {
        float a = 0.f;
#pragma unroll
        for (int g4 = 0; g4 < kGates / 4; ++g4) {
            const float4 v = *reinterpret_cast<const float4 *>(sda + r * kGates + 4 * g4);
            a = fmaf(v.x, w[4 * g4 + 0], a); a = fmaf(v.y, w[4 * g4 + 1], a); a = fmaf(v.z, w[4 * g4 + 2], a); a = fmaf(v.w, w[4 * g4 + 3], a);
        }
        dfeat[(t0 + r) * L + p] = a;
    }
}

// d f of recording b's feature p = the sum of the d f of the counted windows that hold it (dfw [rows][Lw]), in ascending
// window order, without atomics; 0 where no window holds it.  One thread per recording feature.
__global__ void __launch_bounds__(256)
train_dfeat_fold(const float *__restrict__ dfw, RecRows rr, float *__restrict__ dfeat) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= rr.nrec * rr.LN) return;
    const int64_t b = e / rr.LN;
    const int p = (int)(e - b * rr.LN);
    const int64_t r0 = rr.roff[b], lo = rec_first_window(rr, p), hi = rec_last_window(rr, rr.roff[b + 1] - r0, p);
    float a = 0.f;
    for (int64_t w = lo; w <= hi; ++w) {
        const float v = dfw[(r0 + w) * rr.Lw + p - w * rr.sf];
        a = w == lo ? v : a + v;
    }
    dfeat[e] = a;
}

// first maximum of a pooling window over every `stride`-th float (c1 is kept position-major in a tile), like ATen's
// max_pool1d ((v > m) || isnan(v) replaces).  This is the first maximum of the pre-activation; the reference pools after
// tanh and takes the first maximum there.  The two differ only where tanhf maps distinct pre-activations to one float:
// this choice is the one exact arithmetic makes.
__device__ __forceinline__ int pool_argmax(const float *v, int stride, int start, int pk) {
    int best = start;
    float m = v[start * stride];
    for (int j = 1; j < pk; ++j) {
        const float c = v[(start + j) * stride];
        if (c > m || c != c) { m = c; best = start + j; }
    }
    return best;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) v += __shfl_xor_sync(0xffffffffu, v, sft);
    return v;
}

// The conv backward of one tile for `win` consecutive windows; grid: groups x tiles CTAs, group-major.  Per window:
// conv_tile() again (same masks, so the pool arg-max is the forward's), then dropout 2 / pool 2 / tanh / conv2 / pool 1 /
// tanh / conv1 backward over the tile's own features in shared memory.  A warp owns each weight's partial sum (lanes
// stride the positions, one shuffle tree) and adds it to the CTA's running sum in window order; the CTA writes one row
// of part[groups x tiles][n_conv].
// dx != NULL: d x of the tile's span is added into the zeroed dx; adjacent spans overlap by less than a tile's stride
// (checked by the host), so a sample has at most two contributions and their sum does not depend on the order.
// REC: the rows are recordings (rr); a tile that no counted window reaches is skipped (its partial row stays 0), and the
// staged x span is 0 wherever no counted window reads it: a covered feature reads none of those samples, so every
// uncovered position sees a finite pre-activation times an exact 0 gradient, and no 0 * NaN reaches the partials or d x.
template <bool REC>
__device__ __forceinline__ void train_conv_bwd_body(const float *__restrict__ x, const float *__restrict__ prm, BlobOff o, Dims d, int tiles, int win, int64_t B,
               const float *__restrict__ mask1, const float *__restrict__ mask2, const float *__restrict__ dfeat,
               float *__restrict__ part, float *__restrict__ dx, const RecRows &rr) {
    extern __shared__ __align__(16) float sm[];
    const TileSmem s = tile_smem(d, true);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int kWarps = kThreads / 32;
    const Tile t = tile_of(d, blockIdx.x % tiles);
    const int64_t b0 = (int64_t)(blockIdx.x / tiles) * win, b1 = min(B, b0 + win);
    const int ck = d.C * d.K1, n_conv = kCMid * ck + kCMid + kCMid * d.K2 + 1;
    tile_stage_weights(prm, o, d, s, sm, tid);
    for (int e = tid; e < n_conv; e += kThreads) sm[s.g + e] = 0.f;
    for (int64_t b = b0; b < b1; ++b) {
        [[maybe_unused]] int64_t n = 0;
        if constexpr (REC) {
            n = rr.roff[b + 1] - rr.roff[b];
            if (!rec_covers(rr, n, t.i0, t.nf)) continue;       // the same for the whole CTA
        }
        const float *m1b = mask1 ? mask1 + b * kCMid * d.P1 : nullptr;
        __syncthreads();                                       // the previous window's readers are done
        for (int i = tid; i < t.nf; i += kThreads) sm[s.df + i] = dfeat[b * d.L + t.i0 + i] * (mask2 ? mask2[b * d.L + t.i0 + i] : 1.0f);
        conv_tile<REC>(x + b * d.C * d.W, m1b, d, t, s, sm, tid, &rr, n);
        // ---- dropout 2 + pool 2 + tanh, gather form over the tile's own features
        for (int j = tid; j < t.n2; j += kThreads) {
            float a = 0.f;
            int i_lo = (j - d.PK + d.PS) / d.PS;
            if (j - d.PK + 1 <= 0) i_lo = 0;
            for (int i = i_lo; i <= j / d.PS && i < t.nf; ++i)
                if (pool_argmax(sm + s.c2, 1, d.PS * i, d.PK) == j) a += sm[s.df + i];
            sm[s.dc2 + j] = a * dtanhf_(sm[s.c2 + j]);
        }
        __syncthreads();
        // ---- conv2: weight / bias partials, d d1
        for (int e = warp; e < kCMid * d.K2 + 1; e += kWarps) {
            float a = 0.f;
            if (e < kCMid * d.K2) {
                const float *dr = sm + s.d1 + (e / d.K2) * s.pp + e % d.K2;
                for (int j = lane; j < t.n2; j += 32) a = fmaf(sm[s.dc2 + j], dr[j], a);
            } else {
                for (int j = lane; j < t.n2; j += 32) a += sm[s.dc2 + j];
            }
            a = warp_sum(a);
            if (lane == 0) sm[s.g + (e < kCMid * d.K2 ? o.w2 + e : o.b2)] += a;
        }
        for (int e = tid; e < kCMid * t.np1; e += kThreads) {
            const int oc = e / t.np1, u = e % t.np1;
            float a = 0.f;
            for (int k = 0; k < d.K2; ++k) {
                const int j = u - k;
                if (j >= 0 && j < t.n2) a = fmaf(sm[s.w2 + oc * d.K2 + k], sm[s.dc2 + j], a);
            }
            sm[s.dd1 + oc * s.pp + u] = a * (m1b ? m1b[(int64_t)oc * d.P1 + t.s2 + u] : 1.0f);
        }
        __syncthreads();
        // ---- pool 1 + tanh
        for (int e = tid; e < kCMid * t.n1; e += kThreads) {
            const int j = e >> 2, oc = e & 3;
            const float *col = sm + s.c1 + oc;
            float a = 0.f;
            int i_lo = (j - d.PK + d.PS) / d.PS;
            if (j - d.PK + 1 <= 0) i_lo = 0;
            for (int i = i_lo; i <= j / d.PS && i < t.np1; ++i)
                if (pool_argmax(col, kCMid, d.PS * i, d.PK) == j) a += sm[s.dd1 + oc * s.pp + i];
            sm[s.dc1 + e] = a * dtanhf_(sm[s.c1 + e]);
        }
        __syncthreads();
        // ---- conv1: a warp per (channel, tap) with the four output channels' sums, then the biases
        for (int e = warp; e < ck + 1; e += kWarps) {
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
            if (e < ck) {
                const float *xr = sm + s.x + (e / d.K1) * s.xp + e % d.K1;
                for (int j = lane; j < t.n1; j += 32) {
                    const float4 g = *reinterpret_cast<const float4 *>(sm + s.dc1 + 4 * j);
                    const float xv = xr[j];
                    a.x = fmaf(g.x, xv, a.x); a.y = fmaf(g.y, xv, a.y); a.z = fmaf(g.z, xv, a.z); a.w = fmaf(g.w, xv, a.w);
                }
            } else {
                for (int j = lane; j < t.n1; j += 32) {
                    const float4 g = *reinterpret_cast<const float4 *>(sm + s.dc1 + 4 * j);
                    a.x += g.x; a.y += g.y; a.z += g.z; a.w += g.w;
                }
            }
            a.x = warp_sum(a.x); a.y = warp_sum(a.y); a.z = warp_sum(a.z); a.w = warp_sum(a.w);
            if (lane == 0) {
                const float av[4] = {a.x, a.y, a.z, a.w};
                for (int oc = 0; oc < kCMid; ++oc) sm[s.g + (e < ck ? o.w1 + oc * ck + e : o.b1 + oc)] += av[oc];
            }
        }
        if (dx) {
            for (int e = tid; e < d.C * t.nx; e += kThreads) {
                const int c = e / t.nx, u = e % t.nx;
                const int k_lo = max(0, u - (t.n1 - 1)), k_hi = min(d.K1 - 1, u);
                float a = 0.f;
                for (int oc = 0; oc < kCMid; ++oc)
                    for (int k = k_lo; k <= k_hi; ++k) a = fmaf(sm[s.w1 + (c * d.K1 + k) * kCMid + oc], sm[s.dc1 + 4 * (u - k) + oc], a);
                atomicAdd(dx + (b * d.C + c) * d.W + t.s1 + u, a);
            }
        }
    }
    __syncthreads();
    for (int e = tid; e < n_conv; e += kThreads) part[(int64_t)blockIdx.x * n_conv + e] = sm[s.g + e];
}
__global__ void __launch_bounds__(kThreads)
train_conv_bwd(const float *__restrict__ x, const float *__restrict__ prm, BlobOff o, Dims d, int tiles, int win, int64_t B,
               const float *__restrict__ mask1, const float *__restrict__ mask2, const float *__restrict__ dfeat,
               float *__restrict__ part, float *__restrict__ dx) {
    train_conv_bwd_body<false>(x, prm, o, d, tiles, win, B, mask1, mask2, dfeat, part, dx, RecRows{});
}
__global__ void __launch_bounds__(kThreads)
train_conv_bwd_record(const float *__restrict__ x, const float *__restrict__ prm, BlobOff o, Dims d, int tiles, int win, int64_t B,
               const float *__restrict__ mask1, const float *__restrict__ mask2, const float *__restrict__ dfeat,
               float *__restrict__ part, float *__restrict__ dx, RecRows rr) {
    train_conv_bwd_body<true>(x, prm, o, d, tiles, win, B, mask1, mask2, dfeat, part, dx, rr);
}

// grad[e] = the sum of part[.][e] over all rows in a fixed order: one CTA per conv parameter, thread i adds rows
// i, i + 256, ... in order, then the block's tree
__global__ void __launch_bounds__(256)
train_conv_grad_reduce(const float *__restrict__ part, int64_t rows, int n_conv, float *__restrict__ grad) {
    __shared__ float red[256];
    const int e = blockIdx.x, tid = threadIdx.x;
    float a = 0.f;
    for (int64_t r = tid; r < rows; r += 256) a += part[r * n_conv + e];
    red[tid] = a;
    __syncthreads();
    for (int sft = 128; sft > 0; sft >>= 1) {
        if (tid < sft) red[tid] += red[tid + sft];
        __syncthreads();
    }
    if (tid == 0) grad[e] = red[0];
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
// train_adam on the blob entries [o.wih0, o.total) of head blockIdx.y, with its own learning rate
__global__ void train_adam_heads(const __grid_constant__ AdamHeads ah, BlobOff o, float b1, float b2, float eps, float bc1, float bc2_sqrt) {
    const int64_t e = o.wih0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= o.total) return;
    const int h = blockIdx.y;
    float *__restrict__ prm = ah.prm[h], *__restrict__ m = ah.m[h], *__restrict__ v = ah.v[h];
    const float g = ah.grad[h][e], lr = ah.lr[h];
    const float mm = m[e] + (g - m[e]) * (1.f - b1);
    const float vv = b2 * v[e] + (1.f - b2) * g * g;
    m[e] = mm; v[e] = vv;
    const float denom = sqrtf(vv) / bc2_sqrt + eps;
    prm[e] = prm[e] - (lr / bc1) * (mm / denom);
}

// the geometry of a configuration, refusing what the training kernels do not cover; no CUDA call
static bool train_geometry(const b2cnn_config *cfg, Dims &d, const char **err) {
    if (!cfg) { *err = "training: null configuration"; return false; }
    const b2cnn_config &c = *cfg;
    if (c.c_mid != kCMid || c.hidden != kHidden || c.layers != 2) { *err = "training: c_mid / hidden / layers must be 4 / 16 / 2"; return false; }
    if (c.act != B2CNN_ACT_TANH || (c.flags & B2CNN_FLAG_AFFINE)) { *err = "training: tanh activations without affine only (bin/models.py:23,26)"; return false; }
    if (!derive_dims(c, d)) { *err = "training: bad geometry or window too short for the conv/pool stack"; return false; }
    if (d.L != c.lstm_input) { *err = "training: L_out(window) != lstm_input (x.view(-1, MAGICNUM) would straddle windows)"; return false; }
    return true;
}

// A _record call after its checks: the recording geometry rd, the window stride S, the row offsets of the recordings (the
// prefix sums of their window counts) and the rows (counted windows) of the scans.  Without one, rows is the batch.
struct Rec {
    bool on = false;
    Dims rd{};
    int64_t S = 0, rows = 0;
    std::vector<int64_t> roff;
};

// The windows of a _record call (include/b2cnn.h): stride S a positive multiple of the feature stride F, every count in
// [0, n_w] with n_w = (N - W) / S + 1 (0 when N < W), at least one window in all, and indices the kernels hold.  Fills
// rec and, in sequence mode, off with the offsets of one sequence per recording with windows.  No CUDA call.
static bool record_rows(const b2cnn_config &c, const Dims &d, int64_t B, int mode, const RecordArgs &ra, Rec &rec,
                        std::vector<int64_t> &off, const char **err) {
    if (!ra.counts) { *err = "training: NULL window_counts"; return false; }
    if (ra.S < 1 || ra.S % d.feature_stride() || ra.S > INT32_MAX) { *err = "training: stride must be a positive multiple of the feature stride pool_s^2"; return false; }
    if (ra.N < 1 || ra.N > INT32_MAX) { *err = "training: recording length N must be in [1, 2^31 - 1] (the kernels index samples with int)"; return false; }
    const int64_t n_w = ra.N >= d.W ? (ra.N - d.W) / ra.S + 1 : 0;
    rec.roff.assign((size_t)B + 1, 0);
    off.clear();
    if (mode == B2CNN_MODE_SEQUENCE) off.push_back(0);
    for (int64_t b = 0; b < B; ++b) {
        const int64_t v = ra.counts[b];
        if (v < 0 || v > n_w) { *err = "training: every window count must lie in [0, (N - W) / stride + 1]"; return false; }
        rec.roff[b + 1] = rec.roff[b] + v;
        if (v > 0 && mode == B2CNN_MODE_SEQUENCE) off.push_back(rec.roff[b + 1]);
    }
    if (rec.roff[B] < 1) { *err = "training: the window counts add up to 0"; return false; }
    if (rec.roff[B] > INT32_MAX) { *err = "training: more than 2^31 - 1 windows"; return false; }
    b2cnn_config rc = c;
    rc.window = (int)ra.N;
    derive_dims(rc, rec.rd);                     // N >= W: at least one window fits
    rec.on = true;
    rec.S = ra.S;
    rec.rows = rec.roff[B];
    return true;
}

// what the kernels need beyond a valid geometry (cd / B: the conv kernels' geometry and rows); no CUDA call
static bool plan_fits(const Dims &cd, const TrainPlan &pl, int64_t B, const char **err) {
    if (pl.smem_bwd > 227 * 1024) { *err = "training: too many input channels for a conv tile's shared memory"; return false; }
    // a tile's x span against the tiles' stride: d x relies on at most two tiles touching a sample
    const int np1 = cd.PS * (kT - 1) + cd.PK + cd.K2 - 1, span = cd.PS * (np1 - 1) + cd.PK + cd.K1 - 1, stride = cd.PS * cd.PS * kT;
    if (pl.tiles > 1 && span > 2 * stride) { *err = "training: receptive field longer than a conv tile"; return false; }
    if ((int64_t)pl.tiles * B > INT32_MAX) { *err = "training: batch too large"; return false; }
    return true;
}

int64_t train_workspace_bytes(const b2cnn_config *cfg, int64_t B, const SeqLengths &sl, const RecordArgs &ra, int mode, int heads) {
    Dims d;
    const char *err = "";
    std::vector<int64_t> off;
    Rec rec;
    if (heads < 0 || heads > kMaxHeads) return -1;
    if (B < 1 || !train_geometry(cfg, d, &err) || (sl.on && !seq_offsets(sl, B, off, &err))) return -1;
    if (ra.on && ((mode != B2CNN_MODE_INDEPENDENT && mode != B2CNN_MODE_SEQUENCE) || !record_rows(*cfg, d, B, mode, ra, rec, off, &err))) return -1;
    const TrainPlan pl = train_plan(d, ra.on ? rec.rows : B, off.empty() ? 0 : (int64_t)off.size() - 1, ra.on ? &rec.rd : nullptr, B, heads);
    if (ra.on && !plan_fits(rec.rd, pl, B, &err)) return -1;      // a shape the _record calls refuse has no workspace
    return pl.w.total * (int64_t)sizeof(float);
}

// A training call after the checks every entry point shares (check): the geometry, the plan, the sequence offsets of a
// _seq call and the windows of a _record call (rec.rows: the scans' rows, the batch without one).  open() then makes
// the call's device current for the life of this object and copies the offsets into the workspace, which every launch
// below addresses through it.
struct TrainCall {
    Dims d;
    TrainPlan pl;
    BlobOff o{};
    std::vector<int64_t> off;
    Rec rec;
    int64_t B = 0;
    int device = -1, sequence = 0;
    std::optional<DeviceGuard> dev;
    float *ws = nullptr;
    SeqSpan sq{nullptr, 0, 1, nullptr};
    RecRows rr{nullptr, 0, 0, 1, 0, 0, 0};

    // The checks of every training entry point, before any CUDA call: the configuration, the mode, the pointers the call
    // needs (ptrs_ok) and the batch, the sequence lengths of a _seq call (into off), the windows of a _record call (into
    // rec and off), what the kernels hold, and the workspace size.
    int check(const b2cnn_config *cfg, int64_t batch, int mode, const SeqLengths &sl, const RecordArgs &ra, bool ptrs_ok, int64_t ws_bytes,
              const char **err, int heads = 0) {
        if (!train_geometry(cfg, d, err)) return B2CNN_EINVAL;
        if (mode != B2CNN_MODE_INDEPENDENT && mode != B2CNN_MODE_SEQUENCE) { *err = "training: bad mode"; return B2CNN_EINVAL; }
        if (!ptrs_ok || batch < 1) { *err = "training: null argument / bad batch"; return B2CNN_EINVAL; }
        if (sl.on && !seq_offsets(sl, batch, off, err)) return B2CNN_EINVAL;
        if (ra.on && !record_rows(*cfg, d, batch, mode, ra, rec, off, err)) return B2CNN_EINVAL;
        if (ra.has_state() && (!ra.on || mode != B2CNN_MODE_SEQUENCE)) { *err = "training: an LSTM state needs sequence mode"; return B2CNN_EINVAL; }
        if (ra.states_overlap(batch)) { *err = "training: the LSTM state arrays overlap"; return B2CNN_EINVAL; }
        if (!ra.on) rec.rows = batch;
        pl = train_plan(d, rec.rows, off.empty() ? 0 : (int64_t)off.size() - 1, ra.on ? &rec.rd : nullptr, batch, heads);
        if (!plan_fits(cd(), pl, batch, err)) return B2CNN_EINVAL;
        if (ws_bytes < pl.w.total * (int64_t)sizeof(float)) {
            *err = heads ? (ra.on ? "training: workspace smaller than b2cnn_train_heads_workspace_bytes_record()"
                                  : "training: workspace smaller than b2cnn_train_heads_workspace_bytes()")
                 : ra.on ? "training: workspace smaller than b2cnn_train_workspace_bytes_record()"
                 : sl.on ? "training: workspace smaller than b2cnn_train_workspace_bytes_seq()" : "training: workspace smaller than b2cnn_train_workspace_bytes()";
            return B2CNN_ESTATE;
        }
        o = blob_offsets(d);
        B = batch;
        device = cfg->device;
        sequence = mode == B2CNN_MODE_SEQUENCE ? 1 : 0;
        return B2CNN_OK;
    }

    // After the entry point's own checks.  The offsets are copied from pageable memory: the copies have read them when
    // they return.
    int open(void *workspace, cudaStream_t st, const char **err) {
        dev.emplace(device);
        if (dev->err != cudaSuccess) { *err = "cudaSetDevice"; return B2CNN_ECUDA; }
        ws = reinterpret_cast<float *>(workspace);
        if (!off.empty()) {
            int64_t *doff = reinterpret_cast<int64_t *>(ws + pl.w.off);
            if (cudaMemcpyAsync(doff, off.data(), sizeof(int64_t) * off.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) {
                *err = "copy sequence offsets";
                return B2CNN_ECUDA;
            }
            sq = SeqSpan{doff, (int64_t)off.size() - 1, pl.seq_per, pl.seq_ctas > 1 ? ws + pl.w.part : nullptr};
        }
        if (rec.on) {
            int64_t *droff = reinterpret_cast<int64_t *>(ws + pl.w.roff);
            if (cudaMemcpyAsync(droff, rec.roff.data(), sizeof(int64_t) * rec.roff.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) {
                *err = "copy row offsets";
                return B2CNN_ECUDA;
            }
            rr = RecRows{droff, B, (int)rec.S, (int)(rec.S / d.feature_stride()), d.W, d.L, rec.rd.L};
        }
        return B2CNN_OK;
    }

    // the conv kernels' geometry: the recordings' with a _record call, else the windows'
    const Dims &cd() const { return rec.on ? rec.rd : d; }
    // the layer-0 pre-activation GEMM of n_heads heads: (row tiles of 64, split-K slices, head pairs), written to the
    // slices' partials, or with one slice (the whole sum: no reduction) to ws.pre0
    dim3 pre0_grid(int n_heads) const {
        return dim3((unsigned)((rec.rows + 63) / 64), (unsigned)pl.slices, (unsigned)((n_heads + kPre0Heads - 1) / kPre0Heads));
    }
    float *pre0_out() const { return ws + (pl.slices > 1 ? pl.w.part : pl.w.pre0); }
};

// the conv forward into ws.f over the windows, or with a _record call over the recordings, on the conv entries of params
static void launch_conv_forward(const TrainCall &c, const float *params, const float *x, const float *mask1, const float *mask2,
                                cudaStream_t st) {
    const TrainPlan &pl = c.pl;
    const dim3 conv((unsigned)(c.B * pl.tiles));
    if (c.rec.on) {
        if (pl.smem_fwd > 48 * 1024) cudaFuncSetAttribute(train_conv_fwd_record, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem_fwd);
        train_conv_fwd_record<<<conv, kThreads, pl.smem_fwd, st>>>(x, params, c.o, c.rec.rd, pl.tiles, mask1, mask2, c.ws + pl.w.f, c.rr);
    } else {
        if (pl.smem_fwd > 48 * 1024) cudaFuncSetAttribute(train_conv_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem_fwd);
        train_conv_fwd<<<conv, kThreads, pl.smem_fwd, st>>>(x, params, c.o, c.d, pl.tiles, mask1, mask2, c.ws + pl.w.f);
    }
}
// with several split-K slices: the layer-0 pre-activations [n_heads][R][64] summed from their partials into ws.pre0
static void sum_pre0(const TrainCall &c, int n_heads, cudaStream_t st) {
    if (c.pl.slices <= 1) return;
    const int64_t n = (int64_t)n_heads * c.rec.rows * kGates;
    train_sum_chunks<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c.ws + c.pl.w.part, c.pl.slices, n, c.ws + c.pl.w.pre0);
}
// the conv forward and the layer-0 pre-activations of the one model a call trains
static void conv_forward(const TrainCall &c, const float *params, const float *x, const float *mask1, const float *mask2, cudaStream_t st) {
    launch_conv_forward(c, params, x, mask1, mask2, st);
    const float *const f = c.ws + c.pl.w.f;
    if (c.rec.on) train_pre0_partial_record<<<c.pre0_grid(1), 256, 0, st>>>(f, params + c.o.wih0, c.rec.rows, c.d.L, c.pre0_out(), c.rr);
    else train_pre0_partial<<<c.pre0_grid(1), 256, 0, st>>>(f, params + c.o.wih0, c.rec.rows, c.d.L, c.pre0_out());
    sum_pre0(c, 1, st);
}

// everything after d(head): d W_ih_l0 and, unless the front end is frozen, d f (with REC folded onto the recordings), the
// convolutional backward into `grads` and, when dx != NULL, the input gradient (added into dx, zeroed here)
template <bool REC>
static bool launch_backward_tail(const TrainCall &c, const float *params, const float *x, const float *mask1, const float *mask2,
                                 float *grads, float *dx, bool frozen_conv, cudaStream_t st) {
    const Dims &d = c.d, &cd = c.cd();
    const TrainPlan &pl = c.pl;
    const TrainWs &w = pl.w;
    const BlobOff &o = c.o;
    const RecRows &rr = c.rr;
    float *const ws = c.ws;
    const int64_t B = c.B, R = c.rec.rows;
    const int64_t n1 = (int64_t)kGates * d.L;
    const unsigned ptiles = (unsigned)((d.L + 127) / 128);
    const dim3 wgrid(ptiles, (unsigned)pl.wih_chunks);
    float *const wout = pl.wih_chunks > 1 ? ws + w.part : grads + o.wih0;
    if constexpr (REC) train_wih0_grad_record<<<wgrid, 128, 0, st>>>(ws + w.da0, ws + w.f, R, d.L, pl.wih_chunk, wout, rr);
    else train_wih0_grad<<<wgrid, 128, 0, st>>>(ws + w.da0, ws + w.f, R, d.L, pl.wih_chunk, wout);
    if (pl.wih_chunks > 1)
        train_sum_chunks<<<(unsigned)((n1 + 255) / 256), 256, 0, st>>>(ws + w.part, pl.wih_chunks, n1, grads + o.wih0);
    if (frozen_conv) return true;
    train_dfeat<<<dim3(ptiles, (unsigned)((R + kRowBatch - 1) / kRowBatch)), 128, 0, st>>>(ws + w.da0, params + o.wih0, R, d.L,
                                                                                          ws + (REC ? w.dfw : w.dfeat));
    if (REC) {
        const int64_t n = B * cd.L;
        train_dfeat_fold<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws + w.dfw, rr, ws + w.dfeat);
    }
    if (dx && cudaMemsetAsync(dx, 0, sizeof(float) * B * cd.C * cd.W, st) != cudaSuccess) return false;
    if constexpr (REC) {
        if (pl.smem_bwd > 48 * 1024) cudaFuncSetAttribute(train_conv_bwd_record, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem_bwd);
        train_conv_bwd_record<<<(unsigned)pl.part_rows, kThreads, pl.smem_bwd, st>>>(x, params, o, cd, pl.tiles, pl.win, B, mask1, mask2,
                                                                                     ws + w.dfeat, ws + w.part, dx, rr);
    } else {
        if (pl.smem_bwd > 48 * 1024) cudaFuncSetAttribute(train_conv_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem_bwd);
        train_conv_bwd<<<(unsigned)pl.part_rows, kThreads, pl.smem_bwd, st>>>(x, params, o, cd, pl.tiles, pl.win, B, mask1, mask2,
                                                                              ws + w.dfeat, ws + w.part, dx);
    }
    train_conv_grad_reduce<<<(unsigned)pl.n_conv, 256, 0, st>>>(ws + w.part, pl.part_rows, pl.n_conv, grads);
    return true;
}
static bool backward_tail(const TrainCall &c, const float *params, const float *x, const float *mask1, const float *mask2, float *grads,
                          float *dx, bool frozen_conv, cudaStream_t st) {
    if (c.rec.on) return launch_backward_tail<true>(c, params, x, mask1, mask2, grads, dx, frozen_conv, st);
    return launch_backward_tail<false>(c, params, x, mask1, mask2, grads, dx, frozen_conv, st);
}

// the scans' view of the one model a call trains (gridDim.y = 1)
static ScanHeads one_head(const float *params, float *grads) {
    ScanHeads hd{};
    hd.prm[0] = params;
    hd.grad[0] = grads;
    return hd;
}

// with more than one scan CTA: each head's gradients (and, with loss_out, its mean loss) from its CTAs' rows
static void launch_head_reduce(const TrainCall &c, const ScanHeads &hd, int n_heads, float *loss_out, cudaStream_t st) {
    if (!c.sq.rows) return;
    const dim3 grid((unsigned)((head_row_len(c.o) + 255) / 256), (unsigned)n_heads);
    train_head_reduce<<<grid, 256, 0, st>>>(c.sq.rows, c.pl.seq_ctas, c.o, c.rec.rows, hd, loss_out);
}

// the scan kernels of one HEAD, the STATE instance for a call with states
template <int HEAD, typename... A>
static void lstm_fwd(dim3 grid, cudaStream_t st, bool state, A... a) {
    if (state) train_lstm_fwd<HEAD, true><<<grid, 64, 0, st>>>(a...);
    else train_lstm_fwd<HEAD, false><<<grid, 64, 0, st>>>(a...);
}
template <int HEAD, typename... A>
static void lstm_bwd(dim3 grid, cudaStream_t st, bool state, A... a) {
    if (state) train_lstm_bwd<HEAD, true><<<grid, 64, 0, st>>>(a...);
    else train_lstm_bwd<HEAD, false><<<grid, 64, 0, st>>>(a...);
}

// The scans' view of a _record_state call's states (all null otherwise).  Before the scan that writes `dst` (state_out in
// the forward, d_state_in in the backward), dst = src, or zeros for a null src: the rows of recordings without windows
// keep that value, the scan overwrites the others.
static ScanState scan_state(const RecordArgs &ra, const RecRows &rr) {
    return ScanState{ra.state_in, ra.state_out, ra.d_state_out, ra.d_state_in, rr.roff, rr.nrec};
}
static bool pass_state(float *dst, const float *src, int64_t B, cudaStream_t st) {
    if (!dst) return true;
    const size_t bytes = sizeof(float) * (size_t)B * kGates;
    return (src ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st) : cudaMemsetAsync(dst, 0, bytes, st)) == cudaSuccess;
}

// The fused step's forward and backward scans of the n_heads heads hd, one grid row per head, on the BCE loss of HEAD
// (the unweighted loss takes pos_weight 1); `state`: they start from and end in the states of ss
template <int HEAD>
static void fused_scans(const TrainCall &c, const ScanHeads &hd, int n_heads, const float *age, const float *target, float pos_weight,
                        float *loss_out, bool state, const ScanState &ss, cudaStream_t st) {
    const TrainWs &w = c.pl.w;
    float *const ws = c.ws;
    const dim3 grid((unsigned)c.pl.seq_ctas, (unsigned)n_heads);
    lstm_fwd<HEAD>(grid, st, state, ws + w.pre0, hd, c.o, c.d, c.rec.rows, c.sequence, c.sq, age, target, pos_weight, ws + w.acts, ws + w.cs,
                   ws + w.hs, ws + w.lin, ws + w.z, loss_out, ss);
    lstm_bwd<HEAD>(grid, st, state, hd, c.o, c.d, c.rec.rows, c.sequence, c.sq, age, target, pos_weight, (const float *)nullptr, ws + w.acts,
                   ws + w.cs, ws + w.hs, ws + w.lin, ws + w.z, ws + w.da0, (float *)nullptr, ss);
}
static void launch_scans(const TrainCall &c, const ScanHeads &hd, int n_heads, const float *age, const float *target, bool weighted,
                         float pos_weight, float *loss_out, bool state, const ScanState &ss, cudaStream_t st) {
    (weighted ? fused_scans<kHeadBcePw> : fused_scans<kHeadBce>)(c, hd, n_heads, age, target, weighted ? pos_weight : 1.f, loss_out, state, ss, st);
}

// B: the windows, or with a _record call (ra.on) the recordings x [B][C][N], whose R counted windows are the rows that age,
// target and the scans see
int train_step(const b2cnn_config *cfg, float *params, float *adam_m, float *adam_v, float *grads, int64_t step, float lr, float beta1,
               float beta2, float eps, int apply_update, const float *x, int64_t B, const float *age, const float *target,
               int weighted, float pos_weight, int mode, const SeqLengths &sl, const RecordArgs &ra, const float *mask1, const float *mask2,
               float *loss_out, void *workspace, int64_t ws_bytes, cudaStream_t st, const char **err) {
    TrainCall c;
    int rc = c.check(cfg, B, mode, sl, ra, params && grads && x && age && target && loss_out && workspace, ws_bytes, err);
    if (rc != B2CNN_OK) return rc;
    if (step < 1) { *err = "training: step must be >= 1"; return B2CNN_EINVAL; }
    if (apply_update && (!adam_m || !adam_v)) { *err = "training: Adam state missing"; return B2CNN_EINVAL; }
    if (weighted && !(pos_weight > 0.f && pos_weight <= FLT_MAX)) { *err = "training: pos_weight must be positive and finite"; return B2CNN_EINVAL; }
    if ((rc = c.open(workspace, st, err)) != B2CNN_OK) return rc;
    const BlobOff &o = c.o;
    if (cudaMemsetAsync(grads, 0, sizeof(float) * o.total, st) != cudaSuccess) { *err = "memset grads"; return B2CNN_ECUDA; }
    conv_forward(c, params, x, mask1, mask2, st);
    // the fused step is truncated back-propagation through time: no gradient enters through the final state
    const ScanState ss = scan_state(RecordArgs{ra.on, ra.N, ra.S, ra.counts, ra.state_in, ra.state_out}, c.rr);
    if (!pass_state(ra.state_out, ra.state_in, B, st)) { *err = "copy of the LSTM state"; return B2CNN_ECUDA; }
    const ScanHeads hd = one_head(params, grads);
    launch_scans(c, hd, 1, age, target, weighted, pos_weight, loss_out, ra.has_state(), ss, st);
    launch_head_reduce(c, hd, 1, loss_out, st);
    if (!backward_tail(c, params, x, mask1, mask2, grads, nullptr, false, st)) { *err = "memset dx"; return B2CNN_ECUDA; }
    if (apply_update) {
        const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
        train_adam<<<(unsigned)((o.total + 255) / 256), 256, 0, st>>>(params, adam_m, adam_v, grads, o.total, lr, beta1, beta2, eps, bc1, sqrtf(bc2));
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

int train_forward(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age, int mode, const SeqLengths &sl,
                  const RecordArgs &ra, const float *mask1, const float *mask2, float *z_out, void *workspace, int64_t ws_bytes,
                  cudaStream_t st, const char **err) {
    TrainCall c;
    int rc = c.check(cfg, B, mode, sl, ra, params && x && age && z_out && workspace, ws_bytes, err);
    if (rc != B2CNN_OK || (rc = c.open(workspace, st, err)) != B2CNN_OK) return rc;
    const TrainWs &w = c.pl.w;
    float *const ws = c.ws;
    conv_forward(c, params, x, mask1, mask2, st);
    if (!pass_state(ra.state_out, ra.state_in, B, st)) { *err = "copy of the LSTM state"; return B2CNN_ECUDA; }
    lstm_fwd<kHeadLogits>((unsigned)c.pl.seq_ctas, st, ra.has_state(), ws + w.pre0, one_head(params, nullptr), c.o, c.d, c.rec.rows, c.sequence,
                          c.sq, age, (const float *)nullptr, 1.f, ws + w.acts, ws + w.cs, ws + w.hs, ws + w.lin, z_out, (float *)nullptr,
                          scan_state(ra, c.rr));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

int train_backward(const b2cnn_config *cfg, const float *params, const float *x, int64_t B, const float *age, int mode, const SeqLengths &sl,
                   const RecordArgs &ra, const float *mask1, const float *mask2, const float *dz, float *grads, float *dx, float *dage,
                   int flags, void *workspace, int64_t ws_bytes, cudaStream_t st, const char **err) {
    TrainCall c;
    int rc = c.check(cfg, B, mode, sl, ra, params && x && age && dz && grads && workspace, ws_bytes, err);
    if (rc != B2CNN_OK) return rc;
    if (flags & ~B2CNN_TRAIN_FROZEN_CONV) { *err = "training: unknown flag"; return B2CNN_EINVAL; }
    const bool frozen_conv = (flags & B2CNN_TRAIN_FROZEN_CONV) != 0;
    if (frozen_conv && dx) { *err = "training: B2CNN_TRAIN_FROZEN_CONV computes no input gradient (dx must be NULL)"; return B2CNN_EINVAL; }
    if ((rc = c.open(workspace, st, err)) != B2CNN_OK) return rc;
    const TrainWs &w = c.pl.w;
    float *const ws = c.ws;
    // zeroed: a frozen front end leaves the conv entries as they are
    if (cudaMemsetAsync(grads, 0, sizeof(float) * c.o.total, st) != cudaSuccess) { *err = "memset grads"; return B2CNN_ECUDA; }
    if (!pass_state(ra.d_state_in, ra.d_state_out, B, st)) { *err = "copy of the LSTM state gradient"; return B2CNN_ECUDA; }
    const ScanHeads hd = one_head(params, grads);
    lstm_bwd<kHeadLogits>((unsigned)c.pl.seq_ctas, st, ra.has_state(), hd, c.o, c.d, c.rec.rows, c.sequence, c.sq, age,
                          (const float *)nullptr, 1.f, dz, ws + w.acts, ws + w.cs, ws + w.hs, ws + w.lin, (const float *)nullptr, ws + w.da0, dage,
                          scan_state(ra, c.rr));
    launch_head_reduce(c, hd, 1, nullptr, st);
    if (!backward_tail(c, params, x, mask1, mask2, grads, dx, frozen_conv, st)) { *err = "memset dx"; return B2CNN_ECUDA; }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

}  // namespace b2cnn

namespace b2cnn {

// K candidate heads on one frozen front end (b2cnn_train_heads_step / _record, include/b2cnn.h): the conv forward once
// on the front end's conv weights, then every later kernel of the fused step with a head axis -- the projection and
// dW_ih_l0 two heads per CTA on gridDim.z, the scans and their reductions one grid row per head, Adam over every head's
// entries from W_ih_l0 on -- and no conv backward.  Head h computes the bits b2cnn_train_step computes for its blob:
// every sum it makes is the fused step's, in the fused step's order.  The launch list does not depend on K.
int train_heads_step(const b2cnn_config *cfg, const float *frontend, int n_heads, float *const *params, float *const *adam_m,
                     float *const *adam_v, float *const *grads, const float *lr, int64_t step, float beta1, float beta2, float eps,
                     int apply_update, const float *x, int64_t B, const float *age, const float *target, int weighted, float pos_weight,
                     int mode, const SeqLengths &sl, const RecordArgs &ra, const float *mask1, const float *mask2, float *loss_out,
                     void *workspace, int64_t ws_bytes, cudaStream_t st, const char **err) {
    if (n_heads < 1 || n_heads > kMaxHeads) { *err = "training: n_heads must be in [1, B2CNN_SLIDE_MAX_HEADS = 8]"; return B2CNN_EINVAL; }
    if (!params || !grads || !lr || (apply_update && (!adam_m || !adam_v))) { *err = "training: null head array"; return B2CNN_EINVAL; }
    Dims d;
    if (!train_geometry(cfg, d, err)) return B2CNN_EINVAL;
    const size_t blob_bytes = sizeof(float) * blob_offsets(d).total;
    // every array a head writes: its blob, its gradients and (with an update) its Adam state, none shared with another's
    std::vector<const float *> arrays;
    for (int h = 0; h < n_heads; ++h) {
        if (!params[h] || !grads[h] || (apply_update && (!adam_m[h] || !adam_v[h]))) { *err = "training: null head pointer"; return B2CNN_EINVAL; }
        arrays.push_back(params[h]);
        arrays.push_back(grads[h]);
        if (apply_update) { arrays.push_back(adam_m[h]); arrays.push_back(adam_v[h]); }
    }
    for (size_t i = 0; i < arrays.size(); ++i)
        for (size_t j = i + 1; j < arrays.size(); ++j)
            if (overlap(arrays[i], arrays[j], blob_bytes)) {
                *err = "training: two heads share a blob (or a head's blob, gradients and Adam state overlap)";
                return B2CNN_EINVAL;
            }
    TrainCall c;
    int rc = c.check(cfg, B, mode, sl, ra, frontend && x && age && target && loss_out && workspace, ws_bytes, err, n_heads);
    if (rc != B2CNN_OK) return rc;
    if (ra.has_state()) { *err = "training: heads carry no LSTM state"; return B2CNN_EINVAL; }
    if (step < 1) { *err = "training: step must be >= 1"; return B2CNN_EINVAL; }
    if (weighted && !(pos_weight > 0.f && pos_weight <= FLT_MAX)) { *err = "training: pos_weight must be positive and finite"; return B2CNN_EINVAL; }
    if ((rc = c.open(workspace, st, err)) != B2CNN_OK) return rc;
    const TrainWs &w = c.pl.w;
    const BlobOff &o = c.o;
    float *const ws = c.ws;
    const int64_t R = c.rec.rows;
    ScanHeads hd{};
    AdamHeads ah{};
    for (int h = 0; h < n_heads; ++h) {
        hd.prm[h] = ah.prm[h] = params[h];
        hd.grad[h] = grads[h];
        ah.grad[h] = grads[h];
        ah.m[h] = apply_update ? adam_m[h] : nullptr;
        ah.v[h] = apply_update ? adam_v[h] : nullptr;
        ah.lr[h] = lr[h];
    }
    // the front end once, then every head's layer-0 pre-activations and the K heads' scans side by side
    launch_conv_forward(c, frontend, x, mask1, mask2, st);
    if (c.rec.on) train_pre0_partial_heads<true><<<c.pre0_grid(n_heads), 256, 0, st>>>(ws + w.f, hd, n_heads, o, R, c.d.L, c.pre0_out(), c.rr);
    else train_pre0_partial_heads<false><<<c.pre0_grid(n_heads), 256, 0, st>>>(ws + w.f, hd, n_heads, o, R, c.d.L, c.pre0_out(), c.rr);
    sum_pre0(c, n_heads, st);
    launch_scans(c, hd, n_heads, age, target, weighted, pos_weight, loss_out, false, ScanState{}, st);
    launch_head_reduce(c, hd, n_heads, loss_out, st);
    // dW_ih_l0 (and the zeroed conv entries), then Adam
    const int64_t n1 = (int64_t)kGates * c.d.L;
    const dim3 wgrid((unsigned)((c.d.L + 127) / 128), (unsigned)c.pl.wih_chunks, (unsigned)((n_heads + kWihHeads - 1) / kWihHeads));
    if (c.rec.on)
        train_wih0_grad_heads<true><<<wgrid, 128, 0, st>>>(ws + w.da0, ws + w.f, hd, n_heads, o, R, c.d.L, c.pl.wih_chunk, c.pl.wih_chunks, ws + w.part, c.rr);
    else
        train_wih0_grad_heads<false><<<wgrid, 128, 0, st>>>(ws + w.da0, ws + w.f, hd, n_heads, o, R, c.d.L, c.pl.wih_chunk, c.pl.wih_chunks, ws + w.part, c.rr);
    if (c.pl.wih_chunks > 1)
        train_wih0_sum_heads<<<dim3((unsigned)((n1 + 255) / 256), (unsigned)n_heads), 256, 0, st>>>(ws + w.part, c.pl.wih_chunks, n1, hd, o);
    if (apply_update) {
        const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
        train_adam_heads<<<dim3((unsigned)((o.total - o.wih0 + 255) / 256), (unsigned)n_heads), 256, 0, st>>>(ah, o, beta1, beta2, eps, bc1, sqrtf(bc2));
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

}  // namespace b2cnn
