// b2cnn_wire.cu -- the reference's wire formats, decoded on the device (SURVEY.md section 8, row f3).
//
//   bin/sendStream.py:59-64      one Kafka message per (sample, signal): value = json.dumps([i, val]), i = position of
//                                the signal in the record's selected list, val = physical value (NaN when missing)
//                                e.g.  [0, 81.0]   [3, NaN]   [2, 80.66666666666667]
//   bin/processStream.py:126-131 one message per (patient, channel) and trigger: key "<pid>_<chan>", value =
//                                to_json(collect_list(average3)) = a JSON array of doubles, e.g.  [81.0,80.4,1.0E-5]
//
// A trigger's messages arrive as one byte buffer + offsets (what a Kafka consumer poll() hands over); one thread
// parses one message and, for the sample format, scatters the value straight into the [rows][n_sig] fp64 frame
// that b2cnn_ring_push(B2CNN_SAMPLES_F64) consumes -- no per-message Python, no host-side json.loads.
//
// Decimal -> binary64 is CORRECTLY ROUNDED (the same double json.loads / float() / Java's Double.parseDouble give):
// up to 19 significant digits and a decimal exponent |e10| <= 27 after folding in the fraction digits, which covers
// every string Python's repr / Java's Double.toString emit for values between 1e-10 and 1e27 -- vital signs are
// O(1..1e3).  The digits are accumulated exactly in 64 bits and scaled by 5^k * 2^k with 128-bit integer arithmetic
// (one division or one multiplication, round-to-nearest-even on the exact remainder): no floating-point
// approximation is involved.  Anything outside that range, or malformed, is flagged (status != 0) and yields NaN.
#include <cmath>

#include "b2cnn_internal.cuh"

namespace b2cnn {

#if defined(__CUDA_ARCH__)
#define B2_CLZ64(v) __clzll((long long)(v))
#else
#define B2_CLZ64(v) __builtin_clzll((unsigned long long)(v))
#endif

__host__ __device__ inline unsigned long long pow5_u64(int k) {
    constexpr unsigned long long T[28] = {1ull, 5ull, 25ull, 125ull, 625ull, 3125ull, 15625ull, 78125ull, 390625ull, 1953125ull, 9765625ull, 48828125ull, 244140625ull, 1220703125ull, 6103515625ull, 30517578125ull, 152587890625ull, 762939453125ull, 3814697265625ull, 19073486328125ull, 95367431640625ull, 476837158203125ull, 2384185791015625ull, 11920928955078125ull, 59604644775390625ull, 298023223876953125ull, 1490116119384765625ull, 7450580596923828125ull};
    return T[k];
}

// exact: (-1)^neg * m * 10^e10, m < 2^64, |e10| <= 27  ->  nearest double (ties to even)
__host__ __device__ double scale_decimal(unsigned long long m, int e10, bool neg, int *status) {
    if (m == 0) return neg ? -0.0 : 0.0;
    if (e10 < -27 || e10 > 27) { *status = 2; return nan(""); }
    const unsigned long long p5 = pow5_u64(e10 < 0 ? -e10 : e10);
    unsigned __int128 q;          // value = q * 2^ex  (+ sticky below q's last bit)
    int ex;
    bool sticky = false;
    if (e10 >= 0) {
        q = (unsigned __int128)m * p5;                      // < 2^127, exact
        ex = e10;
    } else {
        const int lz = B2_CLZ64(m);
        const unsigned __int128 n = ((unsigned __int128)(m << lz)) << 63;      // top bit at 126
        q = n / p5;                                         // >= 2^63: at least 63 significant bits
        sticky = (n % p5) != 0;
        ex = e10 - 63 - lz;
    }
    // round q (with sticky) to 53 bits
    int bits = 0;
    {
        const unsigned long long hi = (unsigned long long)(q >> 64), lo = (unsigned long long)q;
        bits = hi ? 128 - B2_CLZ64(hi) : 64 - B2_CLZ64(lo);
    }
    unsigned long long mant;
    if (bits > 53) {
        const int sh = bits - 53;
        const unsigned __int128 rest = q & ((((unsigned __int128)1) << sh) - 1);
        const unsigned __int128 half = ((unsigned __int128)1) << (sh - 1);
        mant = (unsigned long long)(q >> sh);
        const bool up = rest > half || (rest == half && (sticky || (mant & 1ull)));
        if (up) ++mant;                                     // may carry to 2^53: still exact as a double
        ex += sh;
    } else {
        mant = (unsigned long long)q;                       // sticky can only be set with bits >= 63
    }
    const double v = ldexp((double)mant, ex);
    return neg ? -v : v;
}

// the whitespace json.loads skips between tokens
__host__ __device__ inline bool json_ws(uint8_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }

// parses a JSON number / NaN / Infinity / null starting at s[i]; advances i.  status: 0 ok, 1 malformed, 2 out of range
__host__ __device__ double parse_number(const uint8_t *s, int64_t &i, int64_t end, int *status) {
    while (i < end && json_ws(s[i])) ++i;
    bool neg = false;
    const bool quoted = i < end && s[i] == '"';              // Spark quotes non-finite doubles: "NaN", "Infinity", "-Infinity"
    if (quoted) ++i;
    if (i < end && (s[i] == '-' || s[i] == '+')) { neg = s[i] == '-'; ++i; }
    if (!quoted && i < end && s[i] == '"') ++i;
    if (i + 3 <= end && s[i] == 'N' && s[i + 1] == 'a' && s[i + 2] == 'N') { i += 3; if (i < end && s[i] == '"') ++i; return nan(""); }
    if (i + 4 <= end && s[i] == 'n' && s[i + 1] == 'u' && s[i + 2] == 'l' && s[i + 3] == 'l') { i += 4; return nan(""); }
    if (i + 8 <= end && s[i] == 'I' && s[i + 1] == 'n' && s[i + 2] == 'f' && s[i + 3] == 'i' && s[i + 4] == 'n' && s[i + 5] == 'i' &&
        s[i + 6] == 't' && s[i + 7] == 'y') {
        i += 8; if (i < end && s[i] == '"') ++i;
        return neg ? -INFINITY : INFINITY;
    }
    unsigned long long m = 0;
    int ndig = 0, e10 = 0;
    bool any = false, dropped_nonzero = false;
    for (; i < end && s[i] >= '0' && s[i] <= '9'; ++i) {
        any = true;
        if (ndig < 19) { m = m * 10 + (s[i] - '0'); if (m) ++ndig; }
        else { ++e10; dropped_nonzero |= s[i] != '0'; }
    }
    if (i < end && s[i] == '.') {
        ++i;
        for (; i < end && s[i] >= '0' && s[i] <= '9'; ++i) {
            any = true;
            if (ndig < 19) { m = m * 10 + (s[i] - '0'); if (m) ++ndig; --e10; }
            else dropped_nonzero |= s[i] != '0';
        }
    }
    if (!any) { *status = 1; return nan(""); }
    if (i < end && (s[i] == 'e' || s[i] == 'E')) {
        ++i;
        bool eneg = false;
        if (i < end && (s[i] == '-' || s[i] == '+')) { eneg = s[i] == '-'; ++i; }
        int ev = 0; bool eany = false;
        for (; i < end && s[i] >= '0' && s[i] <= '9'; ++i) { eany = true; if (ev < 10000) ev = ev * 10 + (s[i] - '0'); }
        if (!eany) { *status = 1; return nan(""); }
        e10 += eneg ? -ev : ev;
    }
    if (dropped_nonzero) { *status = 2; return nan(""); }        // more than 19 significant digits: not produced by repr / toString
    // trailing zeros of the mantissa keep |e10| small for strings like 1200000.0
    while (m && (m % 10) == 0 && e10 < 0) { m /= 10; ++e10; }
    return scale_decimal(m, e10, neg, status);
}

// value = "[<int>, <number>]"  (bin/sendStream.py:62)
__global__ void decode_pairs_kernel(const uint8_t *__restrict__ bytes, const int64_t *__restrict__ offsets, int64_t n_msgs,
                                    int *__restrict__ idx_out, double *__restrict__ val_out, const int64_t *__restrict__ row_of_msg,
                                    double *__restrict__ frame, int64_t frame_rows, int n_sig, int *__restrict__ n_bad) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_msgs) return;
    int64_t i = offsets[t];
    const int64_t end = offsets[t + 1];
    int status = 0, idx = -1;
    double v = nan("");
    while (i < end && json_ws(bytes[i])) ++i;
    if (i < end && bytes[i] == '[') {
        ++i;
        while (i < end && json_ws(bytes[i])) ++i;
        long long k = 0; bool any = false, big = false;      // an index idx_out cannot hold is malformed, not truncated
        for (; i < end && bytes[i] >= '0' && bytes[i] <= '9'; ++i) {
            any = true;
            k = k * 10 + (bytes[i] - '0');
            if (k > 0x7fffffffll) { big = true; k = 0x7fffffffll; }
        }
        while (i < end && json_ws(bytes[i])) ++i;
        if (big) status = 1;
        else if (any && i < end && bytes[i] == ',') {
            ++i;
            idx = (int)k;
            v = parse_number(bytes, i, end, &status);
            while (i < end && json_ws(bytes[i])) ++i;
            if (!(i < end && bytes[i] == ']')) status = status ? status : 1;
            else ++i;
        } else status = 1;
        while (i < end && json_ws(bytes[i])) ++i;
        if (i < end) status = status ? status : 1;            // nothing but whitespace after the closing bracket
    } else status = 1;
    if (status) { idx = -1; v = nan(""); atomicAdd(n_bad, 1); }
    if (idx_out) idx_out[t] = idx;
    if (val_out) val_out[t] = v;
    // the signal index comes from the message and the row from the caller: neither may leave the frame
    if (frame && row_of_msg && idx >= 0 && idx < n_sig) {
        const int64_t row = row_of_msg[t];
        if (row >= 0 && row < frame_rows) frame[row * n_sig + idx] = v;
    }
}

// value = "[v0,v1,...]"  (bin/processStream.py:128 to_json(collect_list(...)), read back by bin/predictStream.py:241)
__global__ void decode_arrays_kernel(const uint8_t *__restrict__ bytes, const int64_t *__restrict__ offsets, int64_t n_msgs,
                                     int max_vals, double *__restrict__ vals_out, int *__restrict__ counts_out, int *__restrict__ n_bad) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_msgs) return;
    int64_t i = offsets[t];
    const int64_t end = offsets[t + 1];
    int status = 0, n = 0;
    double *out = vals_out + t * max_vals;
    while (i < end && json_ws(bytes[i])) ++i;
    if (i < end && bytes[i] == '[') {
        ++i;
        while (i < end && json_ws(bytes[i])) ++i;
        if (i < end && bytes[i] == ']') { ++i; }
        else {
            while (true) {
                const double v = parse_number(bytes, i, end, &status);
                if (status) break;
                if (n < max_vals) out[n] = v;
                ++n;
                while (i < end && json_ws(bytes[i])) ++i;
                if (i < end && bytes[i] == ',') { ++i; continue; }
                if (i < end && bytes[i] == ']') { ++i; break; }
                status = 1; break;
            }
        }
        while (i < end && json_ws(bytes[i])) ++i;
        if (!status && i < end) status = 1;                    // nothing but whitespace after the closing bracket
    } else status = 1;
    if (status || n > max_vals) { atomicAdd(n_bad, 1); n = status ? -1 : n; }
    for (int k = n < 0 ? 0 : (n < max_vals ? n : max_vals); k < max_vals; ++k) out[k] = nan("");
    counts_out[t] = n;
}

__global__ void fill_nan_f64_kernel(double *p, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = nan("");
}

int wire_decode_pairs(const uint8_t *bytes, const int64_t *offsets, int64_t n_msgs, int *idx_out, double *val_out,
                      const int64_t *row_of_msg, double *frame, int64_t frame_rows, int n_sig, int *n_bad, cudaStream_t st,
                      const char **err) {
    if (!bytes || !offsets || n_msgs < 0 || !n_bad || (frame && (!row_of_msg || n_sig < 1 || frame_rows < 0))) { *err = "null pointer / bad shape"; return B2CNN_EINVAL; }
    cudaError_t e = cudaMemsetAsync(n_bad, 0, sizeof(int), st);
    if (e == cudaSuccess && frame && frame_rows > 0) {
        const int64_t n = frame_rows * n_sig;
        fill_nan_f64_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(frame, n);      // a signal without a message is missing
    }
    if (e == cudaSuccess && n_msgs > 0)
        decode_pairs_kernel<<<(unsigned)((n_msgs + 127) / 128), 128, 0, st>>>(bytes, offsets, n_msgs, idx_out, val_out, row_of_msg, frame, frame_rows, n_sig, n_bad);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

int wire_decode_arrays(const uint8_t *bytes, const int64_t *offsets, int64_t n_msgs, int max_vals, double *vals_out, int *counts_out,
                       int *n_bad, cudaStream_t st, const char **err) {
    // a trigger without messages has nothing to write: its (empty) output tensors may have null data pointers
    if (!bytes || !offsets || n_msgs < 0 || max_vals < 1 || (n_msgs > 0 && (!vals_out || !counts_out)) || !n_bad) {
        *err = "null pointer / bad shape"; return B2CNN_EINVAL;
    }
    cudaError_t e = cudaMemsetAsync(n_bad, 0, sizeof(int), st);
    if (e == cudaSuccess && n_msgs > 0)
        decode_arrays_kernel<<<(unsigned)((n_msgs + 127) / 128), 128, 0, st>>>(bytes, offsets, n_msgs, max_vals, vals_out, counts_out, n_bad);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return B2CNN_ECUDA; }
    return B2CNN_OK;
}

// the same parser compiled for the host: what tests/ check against Python's float() without a GPU
double wire_parse_decimal_host(const char *s, int64_t len, int *status) {
    int64_t i = 0;
    int st = 0;
    const double v = parse_number(reinterpret_cast<const uint8_t *>(s), i, len, &st);
    if (!st && i != len) st = 1;
    if (status) *status = st;
    return v;
}

}  // namespace b2cnn
