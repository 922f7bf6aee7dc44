// spectrum.cuh -- the power spectrum of a handle's input (include/ertgpu_spectrum.h): spectrum_kernel<F> reads each
// call's input once, as the caller passed it, and fuses fmt_wide_sample<F>, the Hann window, an in-place shared-memory
// FFT, |X|^2 and the row sums.  Spectrum holds a handle's tables, buffers and stream position, and launches the kernel.
//
// Determinism.  A row's sum is taken in an order fixed by frame index alone:
//   * groups: row r is cut into groups of G = max(4, 2^14 / N) consecutive frames (the last one of a row may be shorter),
//     small enough that a staging chunk gives the GPU several groups per SM at every N; a CTA
//     sums the frames of one group in frame order, starting from 0, or, for a group that an earlier call began, from
//     that call's partial sum (kept on the device);
//   * rows: the groups of a row are added in group order, starting from 0, or from the sum of the row's groups that
//     earlier calls completed; the CTA that completes the last of a row's groups in a call does it (a per-row counter).
// Peaks are maxima.  Every frame's FFT is the same sequence of float32 operations (-fmad=false), whatever CTA runs it.
// Raw bytes of the incomplete frame at the end of a call are kept for the next one.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>
#include <string>
#include <vector>

#include "../../include/ertgpu_spectrum.h"
#include "convert.cuh"
#include "cuda_owned.hpp"

namespace ert {

constexpr int kSpecPerThread = 16;     // points of a frame per thread (fewer below N = 1024)
constexpr int kSpecMaxThreads = (1 << ERTSPEC_LOG2_MAX) / kSpecPerThread;
constexpr int kSpecGroupLog2 = 14;     // N G = 2^14 samples per group, at least kSpecGroupMin frames
constexpr int kSpecGroupMin = 4;
constexpr int64_t kSpecLaunchSamples = 1 << 24;  // input samples one launch takes at most: a longer step is cut

__host__ __device__ inline int spec_threads(int log2n) {
    const int t = (1 << log2n) / kSpecPerThread;
    return t < 64 ? 64 : t;
}

// The frequency bin (0 .. N-1, ascending, 0 Hz at N/2) of FFT position p: the in-place decimation-in-frequency
// transform (one radix-2 stage first when log2n is odd, then radix-4 stages) leaves X[k'] at the mixed-radix reversal
// of k'.
__host__ __device__ inline int spec_bin(int p, int log2n) {
    int k = 0, mul = 1, sh = log2n;
    if (log2n & 1) {
        sh -= 1;
        k = p >> sh;
        p &= (1 << sh) - 1;
        mul = 2;
    }
    while (sh > 0) {
        sh -= 2;
        k += (p >> sh) * mul;
        p &= (1 << sh) - 1;
        mul *= 4;
    }
    const int N = 1 << log2n;
    return (k + N / 2) & (N - 1);
}

struct SpecArgs {
    const uint8_t* in;           // the call's input samples
    long long n;
    const uint8_t* carry_src;    // samples [f0 N, f0 N + carry_n) of the stream
    uint8_t* carry_dst;          // the samples after the call's last whole frame
    int carry_n;
    float g;                     // input gain
    int log2n, N;
    long long F;                 // frames per row
    int G;                       // frames per group
    long long f0, nf;            // first frame of the call and its whole frames
    const float* win;            // [N]
    const float2* tw;            // [N] e^(-2 pi i m / N)
    float scale;                 // ertspec_power_scale
    const float* gpart_src;      // [2][N] mean sum and peak of a group an earlier call began (by FFT position)
    float* gpart_dst;            // ... of the group the call ends inside
    const float* open_src;       // [2][N] the open row's sum over its completed groups (open_valid)
    float* open_dst;
    int open_valid;
    float* grp;                  // [items][2][N] the sums of the groups the call completes
    unsigned int* cnt;           // per row from f0 / F: groups completed so far in this launch
    float* rows_mean;            // [row_cap][N] by bin
    float* rows_peak;
    long long row_cap;
};

__device__ __forceinline__ float2 spec_mul(float2 a, float2 w) {
    return make_float2(__fsub_rn(__fmul_rn(a.x, w.x), __fmul_rn(a.y, w.y)), __fadd_rn(__fmul_rn(a.x, w.y), __fmul_rn(a.y, w.x)));
}
__device__ __forceinline__ float2 spec_add(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 spec_sub(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }

// In-place DIF FFT of the N points in x (natural order in, spec_bin order out).  Called by every thread of the CTA.
__device__ __forceinline__ void spec_fft(float2* x, const float2* __restrict__ tw, int log2n) {
    const int T = blockDim.x, t = threadIdx.x, N = 1 << log2n;
    int lg = log2n;  // log2 of the span L of the stage's sub-transforms
    if (log2n & 1) {
        __syncthreads();
        const int S = N >> 1;
        for (int b = t; b < S; b += T) {
            const float2 a0 = x[b], a1 = x[b + S];
            x[b] = spec_add(a0, a1);
            x[b + S] = spec_mul(spec_sub(a0, a1), __ldg(tw + b));
        }
        lg -= 1;
    }
    for (; lg >= 2; lg -= 2) {
        __syncthreads();
        const int ls = lg - 2, S = 1 << ls, tws = log2n - lg;
        for (int b = t; b < (N >> 2); b += T) {
            const int q = b & (S - 1), base = (b >> ls) << lg;
            float2* p = x + base + q;
            const float2 a0 = p[0], a1 = p[S], a2 = p[2 * S], a3 = p[3 * S];
            const float2 s02 = spec_add(a0, a2), d02 = spec_sub(a0, a2), s13 = spec_add(a1, a3), d13 = spec_sub(a1, a3);
            const float2 jd13 = make_float2(d13.y, -d13.x);  // -i * d13
            p[0] = spec_add(s02, s13);
            p[S] = spec_mul(spec_add(d02, jd13), __ldg(tw + (q << tws)));
            p[2 * S] = spec_mul(spec_sub(s02, s13), __ldg(tw + ((2 * q) << tws)));
            p[3 * S] = spec_mul(spec_sub(d02, jd13), __ldg(tw + ((3 * q) << tws)));
        }
    }
    __syncthreads();
}

// One launch per call of the handle, over the whole frames the call completes.  Grid-stride over the call's groups; any
// grid size gives the same rows.  Dynamic shared memory: N float2, then one int.  A group's sums and peaks are kept in place in its
// output (a group slot, or the partial group for the next call), each position by one thread.
template <int F>
__global__ void __launch_bounds__(kSpecMaxThreads) spectrum_kernel(SpecArgs a) {
    extern __shared__ float2 x[];
    int& s_last = *reinterpret_cast<int*>(x + a.N);  // (all of a CTA's shared memory is dynamic: allow_dynamic_smem)
    constexpr int S = ertfmt_bytes(F);
    const int T = blockDim.x, t = threadIdx.x, N = a.N;

    // the raw bytes after the last whole frame, for the next call
    {
        const long long v0 = a.nf * N, nb = (a.carry_n + a.n - v0) * S, cb = (long long)a.carry_n * S;
        for (long long b = (long long)blockIdx.x * T + t; b < nb; b += (long long)gridDim.x * T) {
            const long long vb = v0 * S + b;
            a.carry_dst[b] = vb < cb ? a.carry_src[vb] : a.in[vb - cb];
        }
    }
    if (a.nf == 0) return;

    const long long Fr = a.F, G = a.G, gpr = (Fr + G - 1) / G, fe = a.f0 + a.nf;
    const long long gg0 = (a.f0 / Fr) * gpr + (a.f0 % Fr) / G;
    const long long gg1 = ((fe - 1) / Fr) * gpr + ((fe - 1) % Fr) / G;
    const long long r_s = a.f0 / Fr;
    auto gstart = [&](long long gg) { return (gg / gpr) * Fr + (gg % gpr) * G; };
    auto gend = [&](long long gg) { return (gg / gpr) * Fr + min((gg % gpr + 1) * G, Fr); };
    const long long last_done = gend(gg1) <= fe ? gg1 : gg1 - 1;  // the last group the call completes

    for (long long item = blockIdx.x; item <= gg1 - gg0; item += gridDim.x) {
        const long long gg = gg0 + item, r = gg / gpr;
        const bool cont = gstart(gg) < a.f0, complete = gend(gg) <= fe;
        const long long fs = max(gstart(gg), a.f0), fend = min(gend(gg), fe);
        float* out = complete ? a.grp + item * 2 * N : a.gpart_dst;
        for (int p = t; p < N; p += T) {
            out[p] = cont ? a.gpart_src[p] : 0.0f;
            out[N + p] = cont ? a.gpart_src[N + p] : 0.0f;
        }
        for (long long f = fs; f < fend; f++) {
            __syncthreads();  // the previous frame's powers are read
            // frame f is stream samples [f N, (f+1) N): the carried ones first, then the call's
            const long long v0 = (f - a.f0) * N - a.carry_n;
            const uint8_t* src = a.in + v0 * S;
#pragma unroll 4
            for (int j = t; j < N; j += T) {
                const uint32_t w = v0 + j < 0 ? fmt_wide_sample<F>(a.carry_src, a.carry_n + v0 + j, a.g)
                                              : fmt_wide_sample<F>(src, j, a.g);
                const float wj = __ldg(a.win + j);
                x[j] = make_float2(__fmul_rn(wj, (float)(int16_t)(w & 0xffffu)), __fmul_rn(wj, (float)(int16_t)(w >> 16)));
            }
            spec_fft(x, a.tw, a.log2n);
            for (int p = t; p < N; p += T) {
                const float2 c = x[p];
                const float pw = __fmul_rn(__fadd_rn(__fmul_rn(c.x, c.x), __fmul_rn(c.y, c.y)), a.scale);
                out[p] = __fadd_rn(out[p], pw);
                out[N + p] = fmaxf(out[N + p], pw);
            }
        }
        if (!complete) continue;
        // the CTA that completes the last of the row's groups in this call adds them up in group order
        const long long ga = max(gg0, r * gpr), gb = min(last_done, r * gpr + gpr - 1);
        __threadfence();
        __syncthreads();
        if (t == 0) {
            unsigned int* c = a.cnt + (r - r_s);
            const bool last = atomicAdd(c, 1u) == (unsigned int)(gb - ga);
            if (last) *c = 0u;  // ready for the next launch
            s_last = last;
        }
        __syncthreads();
        if (!s_last) continue;
        __threadfence();
        const bool row_done = (r + 1) * Fr <= fe;
        const bool from_open = r == r_s && a.open_valid;
        for (int p = t; p < N; p += T) {
            float m = 0.0f, pk = 0.0f;
            if (from_open) {
                m = __ldcg(a.open_src + p);
                pk = __ldcg(a.open_src + N + p);
            }
            for (long long g = ga; g <= gb; g++) {
                const float* s = a.grp + (g - gg0) * 2 * N;
                m = __fadd_rn(m, __ldcg(s + p));
                pk = fmaxf(pk, __ldcg(s + N + p));
            }
            if (row_done) {
                const long long o = (r % a.row_cap) * N + spec_bin(p, a.log2n);
                a.rows_mean[o] = __fdiv_rn(m, (float)Fr);
                a.rows_peak[o] = pk;
            } else {
                a.open_dst[p] = m;
                a.open_dst[N + p] = pk;
            }
        }
    }
}

// A handle's spectrum: configuration, device tables and buffers, and the stream position.  Host code only.
struct Spectrum {
    bool on = false;
    int log2n = 0, N = 0, G = 0, threads = 0, grid = 0;
    int64_t F = 0;
    int S = 2;                                   // bytes per input sample
    int64_t row_cap = 0, item_cap = 0, cnt_cap = 0;  // rows held until fetched; groups and rows of one launch
    size_t smem = 0;
    std::string label;  // "spectrum_kernel<fmt>"
    decltype(&spectrum_kernel<ERTGPU_FORMAT_CU8>) kern = nullptr;

    // The device tables and buffers: the handle clears them (= {}) when it releases its own.
    struct Device {
        DeviceArray<float> win;
        DeviceArray<float2> tw;
        DeviceArray<uint8_t> carry[2];
        DeviceArray<float> gpart[2], open[2];
        DeviceArray<float> grp;
        DeviceArray<unsigned int> cnt;
        DeviceArray<float> mean, peak;
    } dev;

    // The stream position: all that a stream start resets.
    struct Pos {
        int64_t samples = 0;       // input samples since the stream start
        int64_t rows_fetched = 0;  // rows ertgpu_fetch_spectrum returned
        int cc = 0, gc = 0, oc = 0;  // which of dev.carry, dev.gpart, dev.open the next launch reads
        bool open_valid = false;     // dev.open[oc] holds the open row's completed groups
    } pos;

    int64_t frames() const { return pos.samples / N; }
    int64_t rows_done() const { return frames() / F; }

    // Rows a call over n more input samples completes.
    int64_t rows_after(int64_t n) const { return (pos.samples + n) / N / F - rows_done(); }

    // At allocate: the kernel of format fmt (sample_bytes per sample), row buffers for calls of up to in_max input
    // samples, and group buffers for one launch of up to kSpecLaunchSamples.
    int allocate(std::string& err, int fmt, int sample_bytes, const char* fmt_label, int64_t in_max, int sm_count) {
        S = sample_bytes;
        N = 1 << log2n;
        G = std::max(kSpecGroupMin, 1 << std::max(0, kSpecGroupLog2 - log2n));
        threads = spec_threads(log2n);
        smem = (size_t)N * sizeof(float2) + 16;
        label = std::string("spectrum_kernel<") + fmt_label + ">";
        fmt_visit(fmt, [&](auto f) { kern = spectrum_kernel<f()>; });
        if (const int rc = allow_dynamic_smem(err, (const void*)kern, smem, "spectrum_kernel")) return rc;
        int per_sm = 0;
        CUDA_TRY(err, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
        grid = std::max(1, per_sm) * sm_count;
        row_cap = (in_max / N + 1) / F + 2;
        const int64_t frames_max = kSpecLaunchSamples / N + 1;
        cnt_cap = frames_max / F + 2;
        item_cap = frames_max / G + cnt_cap + 2;
        std::vector<float> w((size_t)N);
        ertspec_window(log2n, w.data());
        std::vector<float2> tw((size_t)N);
        for (int m = 0; m < N; m++) {
            const double ph = -2.0 * ERTSPEC_PI * (double)m / (double)N;
            tw[(size_t)m] = make_float2((float)cos(ph), (float)sin(ph));
        }
        CUDA_TRY(err, dev.win.upload(w));
        CUDA_TRY(err, dev.tw.upload(tw));
        for (int k = 0; k < 2; k++) {
            CUDA_TRY(err, dev.carry[k].alloc((size_t)N * 16));
            CUDA_TRY(err, dev.gpart[k].alloc((size_t)2 * N));
            CUDA_TRY(err, dev.open[k].alloc((size_t)2 * N));
        }
        CUDA_TRY(err, dev.grp.alloc((size_t)item_cap * 2 * N));
        CUDA_TRY(err, dev.cnt.alloc((size_t)cnt_cap));
        CUDA_TRY(err, cudaMemset(dev.cnt, 0, (size_t)cnt_cap * sizeof(unsigned int)));
        CUDA_TRY(err, dev.mean.alloc((size_t)row_cap * N));
        CUDA_TRY(err, dev.peak.alloc((size_t)row_cap * N));
        pos = {};
        return ERTGPU_OK;
    }

    // Enqueue the kernel over n input samples at d_in (device) on st, with input gain g, and advance the position: one
    // launch per kSpecLaunchSamples (rows do not depend on the cut), each counted in *launches.
    int launch(std::string& err, const uint8_t* d_in, int64_t n, float g, cudaStream_t st, int64_t* launches) {
        for (int64_t done = 0; done < n; done += kSpecLaunchSamples) {
            if (const int rc = launch_one(err, d_in + done * S, std::min(n - done, kSpecLaunchSamples), g, st)) return rc;
            ++*launches;
        }
        return ERTGPU_OK;
    }

    int launch_one(std::string& err, const uint8_t* d_in, int64_t n, float g, cudaStream_t st) {
        const int64_t f0 = frames(), carry_n = pos.samples - f0 * N, nf = (carry_n + n) / N, fe = f0 + nf;
        const int64_t gpr = (F + G - 1) / G;
        const auto group = [&](int64_t f) { return (f / F) * gpr + (f % F) / G; };
        const auto gend = [&](int64_t gg) { return (gg / gpr) * F + std::min((gg % gpr + 1) * G, F); };
        const int64_t items = nf ? group(fe - 1) - group(f0) + 1 : 0;
        const int64_t rows = nf ? fe / F - f0 / F + 1 : 0;
        if (items > item_cap || rows > cnt_cap)   // n <= kSpecLaunchSamples: cannot happen
            return fail(err, ERTGPU_ESIZE, "spectrum: %lld input samples in one launch exceed its buffers", (long long)n);
        SpecArgs a{};
        a.in = d_in;
        a.n = n;
        a.carry_src = dev.carry[pos.cc];
        a.carry_dst = dev.carry[pos.cc ^ 1];
        a.carry_n = (int)carry_n;
        a.g = g;
        a.log2n = log2n;
        a.N = N;
        a.F = F;
        a.G = G;
        a.f0 = f0;
        a.nf = nf;
        a.win = dev.win;
        a.tw = dev.tw;
        a.scale = ertspec_power_scale(log2n);
        a.gpart_src = dev.gpart[pos.gc];
        a.gpart_dst = dev.gpart[pos.gc ^ 1];
        a.open_src = dev.open[pos.oc];
        a.open_dst = dev.open[pos.oc ^ 1];
        a.open_valid = pos.open_valid;
        a.grp = dev.grp;
        a.cnt = dev.cnt;
        a.rows_mean = dev.mean;
        a.rows_peak = dev.peak;
        a.row_cap = row_cap;
        const int64_t carry_bytes = (carry_n + n - nf * N) * 16;
        const int64_t want = std::max<int64_t>(items, (carry_bytes + threads - 1) / threads);
        const unsigned g_ = (unsigned)std::max<int64_t>(1, std::min<int64_t>(want, grid));
        kern<<<g_, threads, smem, st>>>(a);
        CUDA_TRY(err, cudaGetLastError());
        pos.samples += n;
        pos.cc ^= 1;
        if (nf == 0) return ERTGPU_OK;
        if (gend(group(fe - 1)) > fe) pos.gc ^= 1;  // the call ends inside a group: its partial sums were written
        const int64_t last_done = gend(group(fe - 1)) <= fe ? group(fe - 1) : group(fe - 1) - 1;
        const int64_t r_end = fe / F;
        if (last_done >= group(f0) && last_done >= r_end * gpr) {
            pos.oc ^= 1;
            pos.open_valid = true;
        } else if (r_end != f0 / F) {
            pos.open_valid = false;
        }
        return ERTGPU_OK;
    }

    // The open row (frames() % F frames, at least one): its mean and peak by bin, from the device state.
    int open_row(std::string& err, float* mean, float* peak, int64_t* frames_in_row) const {
        const int64_t fr = frames() % F;
        *frames_in_row = fr;
        if (fr == 0) return ERTGPU_OK;
        std::vector<float> m((size_t)2 * N, 0.0f), gp((size_t)2 * N, 0.0f);
        if (pos.open_valid) CUDA_TRY(err, cudaMemcpy(m.data(), dev.open[pos.oc], m.size() * sizeof(float), cudaMemcpyDeviceToHost));
        const bool mid_group = fr % G != 0;
        if (mid_group) CUDA_TRY(err, cudaMemcpy(gp.data(), dev.gpart[pos.gc], gp.size() * sizeof(float), cudaMemcpyDeviceToHost));
        for (int p = 0; p < N; p++) {
            volatile float s = m[(size_t)p];
            float pk = m[(size_t)N + p];
            if (mid_group) {
                s = s + gp[(size_t)p];
                pk = std::fmax(pk, gp[(size_t)N + p]);
            }
            const int k = spec_bin(p, log2n);
            mean[k] = (float)s / (float)fr;
            peak[k] = pk;
        }
        return ERTGPU_OK;
    }
};

}  // namespace ert
