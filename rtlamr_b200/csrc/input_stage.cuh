// input_stage.cuh -- the input stage of a libertgpu handle: everything between the caller's bytes and the uint8 IQ blocks
// the demod reads.  It owns the input's format, rate and tuning (ertgpu_set_input_*), the mode they resolve to, the
// resampler's plan, tables and stream position, and it launches the one kernel in front of the pipeline:
// convert_kernel<F> (convert.cuh) or resample_kernel<F, TUNED> (resample.cuh), or the two of a decimating handle:
// decimate_kernel<F> (decimate.cuh) into resample_kernel<cu8, false>.  The first stage of several decimating channels of
// one capture can run as one decimate_channels_kernel<F> (launch_channels).  A tuned handle on the wide channel path
// (ertgpu_set_channel_gain) runs resample_wide_kernel<F>, or decimate_wide_kernel<F> into resample_wide_kernel<kFmtMid>,
// instead.  allocate chooses a handle's first- and last-stage kernels once, from its format, mode and path, and launch
// runs whichever it chose.  It also measures the level of its input with level_kernel<F> (level.cuh) for
// ertgpu_measure_input, and that of its channel with the wide kernels (begin_measure) for ertgpu_measure_channel.  Host
// code only.
#pragma once

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "convert.cuh"
#include "cuda_owned.hpp"
#include "decimate.cuh"
#include "level.cuh"
#include "resample.cuh"

namespace ert {

// One step of the stage: input samples at rs.cur on the device, and the whole uint8 blocks they complete.
struct InputStep {
    const uint8_t* iq = nullptr;  // the blocks the pipeline reads: rs.cur itself in pass-through mode
    int64_t nblocks = 0;
    RsArgs rs{};                  // the kernel's arguments (convert_kernel reads rs.cur only)
    DcArgs dc{};                  // decimate_kernel's (kDecimate): rs.cur is then its output
    bool shared_first = false;    // decimate_channels_kernel ran the first stage for a group of channels (launch_channels)
};

struct InputStage {
    // kPass: uint8 IQ at the decoder's rate, read where the caller put it.  kConvert: another format at that rate,
    // convert_kernel<F> into dev.out[0].  kResample(Tuned): resample_kernel<F, false (true)> into dev.out[cur_out]; the tuned
    // instance runs for a tuned capture or a plan with P != ERTRS_P.  kDecimate: decimate_kernel<F> into dev.mid, then
    // resample_kernel<cu8, false> from dev.mid into dev.out[cur_out] (a tuned handle that allows decimation, above 10:1).
    enum Mode { kPass, kConvert, kResample, kResampleTuned, kDecimate };

    explicit InputStage(std::string& err) : err_(err) {}

    // configuration, resolved into `mode` by each setter
    int32_t fmt = ERTGPU_FORMAT_CU8;
    float scale = 0.0f;
    int sample_bytes = 2;
    int64_t rate_in = 0;        // set_rate's rate (0: none)
    bool tuned = false;         // set_tuning: the channel at center_hz of a capture centred at capture_hz
    int64_t capture_hz = 0, center_hz = 0;
    uint32_t nco_step = 0;      // W at the input rate in effect
    bool decimation = false;    // allow_decimation: a tuned handle may take up to 256:1
    bool wide = false;          // set_channel_gain before allocate: the wide channel path (include/ertgpu_resample.h)
    int32_t gain = 0;           // its channel gain k
    Mode mode = kPass;
    ertgpu_resampler_info rs{};  // the resampler (the second stage in kDecimate)
    std::vector<int16_t> table;
    ertgpu_decimator_info dec{};  // the first stage (decimation allowed and a plan made; D = 1: none)
    std::vector<int16_t> taps;

    // decoder geometry (allocate)
    int64_t block = 0, max_blocks = 0;

    // The stream position of both stages: all that a stream start resets.
    struct StreamPos {
        int64_t in_total = 0;   // input samples received since the stream start (the second stage's in kDecimate)
        int64_t out_next = 0;   // first output not yet computed
        int64_t hist_first = 0, hist_n = 0;  // the input samples held in dev.hist[cur_hist]
        int64_t pend = 0;       // outputs at the front of dev.out[cur_out] that wait for a whole block
        int cur_hist = 0, cur_out = 0;
        // the first stage of kDecimate (its next output is the second stage's in_total)
        int64_t in1_total = 0;  // input samples received since the stream start
        int64_t hist1_first = 0, hist1_n = 0;  // the input samples held in dev.hist1[cur_hist1]
        int cur_hist1 = 0;
    };
    StreamPos pos;

    // The kernels allocate chose: the first stage of kDecimate, and the last stage of every resampling mode.
    using FirstKernel = void (*)(const int16_t*, DcArgs);  // decimate_kernel<F>, decimate_wide_kernel<F>
    using LastKernel = void (*)(const int32_t*, const uint32_t*, RsArgs);  // resample_kernel<F, T>, resample_wide_kernel<F>
    FirstKernel first_kernel = nullptr;
    LastKernel last_kernel = nullptr;
    decltype(&decimate_channels_kernel<ERTGPU_FORMAT_CU8>) channels_kernel = nullptr;  // kDecimate's, for launch_channels

    // device state
    size_t smem = 0;
    int grid = 0;               // most CTAs of one launch
    int level_grid = 0;
    size_t smem1 = 0;           // the first stage of kDecimate
    int grid1 = 0, per1 = 0;
    size_t smem1c = 0;          // the same for decimate_channels_kernel
    int grid1c = 0, per1c = 0;
    StreamPos mpos;             // the wide path's channel measurement (begin_measure)
    // The stage's device tables and buffers: the handle clears them (= {}) when it releases its own.
    struct Device {
        DeviceArray<int32_t> A;     // the table as the kernel reads it (rs_pack_table)
        DeviceArray<uint32_t> D;
        DeviceArray<uint32_t> E;    // the mixer table (ertrs_nco_table)
        DeviceArray<uint8_t> hist[2];  // input samples the next outputs still read
        DeviceArray<uint8_t> out[2];   // [partial block | new outputs]; the demod reads whole blocks of it
        DeviceArray<unsigned long long> level;  // level_kernel's kLvCounters counters (converted input only)
        // the first stage of kDecimate: its taps, input history and output (the second stage's input)
        DeviceArray<int16_t> taps;
        DeviceArray<uint8_t> hist1[2];
        DeviceArray<uint8_t> mid;
        // the wide path's channel measurement: its own input histories (with mpos), which begin_measure and end_measure
        // swap with the stream's, and its counters
        DeviceArray<uint8_t> mhist[2];
        DeviceArray<uint8_t> mhist1[2];
        DeviceArray<unsigned long long> clevel;
    } dev;

    bool resamples() const { return mode >= kResample; }
    // Input samples received since the stream start.
    int64_t received() const { return mode == kDecimate ? pos.in1_total : pos.in_total; }

    // ---- configuration (the handle is not allocated; rate_out = DataRate * ChipLength) ----
    int set_rate(int64_t hz, int64_t rate_out) {
        if (const int rc = configure_rate(hz, rate_out)) return rc;
        rate_in = hz;
        return ERTGPU_OK;
    }

    // center_hz 0: default_center_hz, the decoder's CenterFreq
    int set_tuning(int64_t capture_center_hz, int64_t channel_hz, int64_t default_center_hz, int64_t rate_out) {
        if (rate_in) return fail(err_, ERTGPU_EINVAL, "set_input_tuning after set_input_rate");
        if (capture_center_hz <= 0 || channel_hz < 0)
            return fail(err_, ERTGPU_EINVAL, "capture centre %lld Hz must be > 0 and channel %lld Hz >= 0",
                        (long long)capture_center_hz, (long long)channel_hz);
        tuned = true;
        capture_hz = capture_center_hz;
        center_hz = channel_hz ? channel_hz : default_center_hz;  // decode.go:105: the last CenterFreq
        const int64_t off = center_hz - capture_hz, ad = off < 0 ? -off : off;
        nco_step = ad <= rate_out ? ertrs_nco_step(off, rate_out) : 0;  // at the decoder's rate until set_rate
        return ERTGPU_OK;
    }

    // A tuned handle may take up to 256:1 (ertrs_plan_decimated), between set_tuning and set_rate.
    int allow_decimation() {
        if (!tuned) return fail(err_, ERTGPU_EINVAL, "allow_input_decimation before set_input_tuning");
        if (rate_in) return fail(err_, ERTGPU_EINVAL, "allow_input_decimation after set_input_rate");
        decimation = true;
        return ERTGPU_OK;
    }

    int set_format(int32_t format, float g) {
        if (!fmt_name(format)) return fail(err_, ERTGPU_EINVAL, "unknown input format %d", format);
        if (!std::isfinite(g) || g < 0.0f) return fail(err_, ERTGPU_EINVAL, "input scale %g is not a finite value >= 0", (double)g);
        if (format == ERTGPU_FORMAT_CU8 && g != 0.0f) return fail(err_, ERTGPU_EINVAL, "cu8 input is not scaled (scale %g)", (double)g);
        if (g == 0.0f) g = fmt_default_scale(format);
        fmt = format;
        scale = g;
        sample_bytes = fmt_sample_bytes(format);
        if (!resamples()) mode = fmt == ERTGPU_FORMAT_CU8 ? kPass : kConvert;
        return ERTGPU_OK;
    }

    // The gain of a converted input, as set_format takes it; the caller allows it at a stream start only.
    int set_scale(float g) {
        if (fmt == ERTGPU_FORMAT_CU8) return fail(err_, ERTGPU_EINVAL, "cu8 input is not scaled");
        if (!std::isfinite(g) || g < 0.0f) return fail(err_, ERTGPU_EINVAL, "input scale %g is not a finite value >= 0", (double)g);
        scale = g == 0.0f ? fmt_default_scale(fmt) : g;
        return ERTGPU_OK;
    }

    // At allocate: a tuned handle at the decoder's own rate gets its plan here, and the channel must lie inside it.  A
    // wide handle's plan is made again here, whenever set_channel_gain came: it always filters.
    int plan_native(int64_t rate_out) {
        if (!tuned || (rate_in && !wide)) return ERTGPU_OK;
        return configure_rate(rate_in ? rate_in : rate_out, rate_out);
    }

    // The wide channel path with gain 2^k: before allocate (which plans it), or at a stream start of a wide handle (the
    // caller checks which).
    int set_channel_gain(int32_t k, bool allocated) {
        if (!tuned) return fail(err_, ERTGPU_EINVAL, "set_channel_gain on an untuned handle: it needs set_input_tuning");
        if (allocated && !wide) return fail(err_, ERTGPU_EINVAL, "set_channel_gain: the handle was allocated without the wide channel path");
        if (k < 0 || k > ERTRS_GAIN_K_MAX) return fail(err_, ERTGPU_EINVAL, "channel gain 2^%d: k must be within 0 ... %d", k, ERTRS_GAIN_K_MAX);
        wide = true;
        gain = k;
        return ERTGPU_OK;
    }

    int tuning(ertgpu_tuning_info* info) const {
        if (!tuned) return ERTGPU_EINVAL;
        if (info) {
            info->capture_center_hz = capture_hz;
            info->center_hz = center_hz;
            info->offset_hz = center_hz - capture_hz;
            info->nco_step = nco_step;
            info->nco_bits = ERTRS_NCO_BITS;
        }
        return ERTGPU_OK;
    }

    int resampler(ertgpu_resampler_info* info, int16_t* dst, size_t cap, size_t* n_out) const {
        if (!resamples()) return ERTGPU_EINVAL;
        if (info) *info = rs;
        if (n_out) *n_out = table.size();
        if (dst && cap >= table.size()) memcpy(dst, table.data(), table.size() * sizeof(int16_t));
        return ERTGPU_OK;
    }

    int decimator(ertgpu_decimator_info* info, int16_t* dst, size_t cap, size_t* n_out) const {
        if (!decimation || dec.rate_in == 0) return ERTGPU_EINVAL;
        if (info) *info = dec;
        if (n_out) *n_out = taps.size();
        if (dst && cap >= taps.size()) memcpy(dst, taps.data(), taps.size() * sizeof(int16_t));
        return ERTGPU_OK;
    }

    // ---- device buffers ----
    // Blocks of block_size samples, a step completes at most max_blocks_per_step of them; sm_count SMs.
    int allocate(int64_t block_size, int64_t max_blocks_per_step, int sm_count) {
        block = block_size;
        max_blocks = max_blocks_per_step;
        reset_stream();
        if (fmt != ERTGPU_FORMAT_CU8) {
            CUDA_TRY(err_, dev.level.alloc(kLvCounters));
            level_grid = sm_count * 4;
        }
        if (mode == kPass) return ERTGPU_OK;
        if (mode == kConvert) {
            grid = sm_count * 8;
            CUDA_TRY(err_, dev.out[0].alloc((size_t)max_blocks * block * 2));  // 256-byte aligned
            return ERTGPU_OK;
        }
        const bool mix = mode == kResampleTuned;
        std::vector<int32_t> A((size_t)rs.P * rs.T);
        std::vector<uint32_t> D((size_t)rs.P * (rs.T / 2));
        rs_pack_table(table.data(), rs.P, rs.T, A.data(), D.data());
        CUDA_TRY(err_, dev.A.upload(A));
        CUDA_TRY(err_, dev.D.upload(D));
        if (mix || mode == kDecimate) {
            std::vector<uint32_t> E(ERTRS_NCO_N);
            ertrs_nco_table(E.data());
            CUDA_TRY(err_, dev.E.upload(E));
        }
        const size_t hb = wide ? 4 : 2;  // bytes per carried sample: s_w words on the wide path
        for (int k = 0; k < 2; k++) {
            CUDA_TRY(err_, dev.hist[k].alloc((size_t)rs.T * hb + 16));
            // a step completes at most max_blocks blocks: less than (max_blocks + 1) * BS outputs are buffered
            CUDA_TRY(err_, dev.out[k].alloc((size_t)(max_blocks + 1) * block * 2 + 64));
        }
        fmt_visit(fmt, [&](auto f) {
            if (mode == kDecimate) {  // the second stage reads the first stage's bytes, or its s_w words on the wide path
                first_kernel = wide ? decimate_wide_kernel<f()> : decimate_kernel<f()>;
                last_kernel = wide ? resample_wide_kernel<kFmtMid> : resample_kernel<ERTGPU_FORMAT_CU8, false>;
                channels_kernel = decimate_channels_kernel<f()>;
            } else {
                last_kernel = wide ? resample_wide_kernel<f()> : mix ? resample_kernel<f(), true> : resample_kernel<f(), false>;
            }
        });
        smem = wide ? rs_wide_smem_bytes(rs.P, rs.T, rs.L, rs.M, mode == kDecimate) : rs_smem_bytes(rs.P, rs.T, rs.L, rs.M, mix);
        if (const int rc = fit((const void*)last_kernel, kRsThreads, smem, "resampler", sm_count, &grid)) return rc;
        if (wide) {
            CUDA_TRY(err_, dev.clevel.alloc(ERTRS_GAIN_BINS));
            for (int k = 0; k < 2; k++) CUDA_TRY(err_, dev.mhist[k].alloc((size_t)rs.T * 4 + 16));
        }
        return mode == kDecimate ? allocate_first(sm_count) : ERTGPU_OK;
    }

    void reset_stream() { pos = {}; }

    // ---- calls ----
    // Before anything else of a decode call: a resampling stage takes whole IQ samples of s bytes.
    int check_samples(size_t nbytes) const {
        if (resamples() && nbytes % sample_bytes)
            return fail(err_, ERTGPU_ESIZE, "nbytes %zu is not a whole number of %d-byte IQ samples", nbytes, sample_bytes);
        return ERTGPU_OK;
    }

    // The rest of a call's input rules: device input is s-byte aligned when resampling, 16-byte aligned otherwise; a
    // native stage takes whole blocks of BlockSize * s bytes; a device call completes at most max_blocks blocks.
    int check_call(const void* iq, size_t nbytes, bool device) const {
        const int align = resamples() ? sample_bytes : 16;
        if (device && (reinterpret_cast<uintptr_t>(iq) & (align - 1)) != 0)
            return fail(err_, ERTGPU_EINVAL, "device input must be %d-byte aligned", align);
        const size_t bs2 = (size_t)block * 2;
        if (mode == kPass && nbytes % bs2)
            return fail(err_, ERTGPU_ESIZE, "nbytes %zu is not a multiple of BlockSize2 %zu", nbytes, bs2);
        const size_t bsf = (size_t)block * sample_bytes;
        if (!resamples() && nbytes % bsf)
            return fail(err_, ERTGPU_ESIZE, "nbytes %zu is not a multiple of BlockSize * %d = %zu", nbytes, sample_bytes, bsf);
        if (device) {
            const int64_t nb = plan(nullptr, (int64_t)(nbytes / sample_bytes)).nblocks;
            if (nb > max_blocks)
                return fail(err_, ERTGPU_ESIZE, "%zu input bytes complete %lld blocks, more than max_blocks_per_call %lld", nbytes,
                            (long long)nb, (long long)max_blocks);
        }
        return ERTGPU_OK;
    }

    // Input samples per staging chunk of ertgpu_decode.  32 MiB of whole decoder blocks natively; a resampling chunk also
    // covers the filter's look-ahead.  Decimating by more than 4 (tuned handles, up to 10) the chunk grows with M / L,
    // so that it still reaches max_blocks blocks.
    int64_t chunk() const {
        if (!resamples()) return block * std::min<int64_t>(max_blocks, std::max<int64_t>(1, (32 << 20) / (block * 2)));
        if (mode == kDecimate) {  // and with the first stage's D
            const int64_t ratio = dec.D * std::max<int64_t>(4, (rs.M + rs.L - 1) / rs.L);
            return std::min<int64_t>(16 << 20, ratio * (max_blocks + 1) * block + dec.D * (rs.T + 8) + dec.T1 + 8);
        }
        const int64_t ratio = std::max<int64_t>(4, (rs.M + rs.L - 1) / rs.L);
        return std::min<int64_t>(16 << 20, ratio * (max_blocks + 1) * block + rs.T + 8);
    }

    // The next chunk when `left` input samples remain: when resampling, the step that takes it completes at most
    // max_blocks blocks.
    int64_t next_chunk(int64_t left) const {
        const int64_t c = std::min(chunk(), left);
        return resamples() ? std::min(c, max_input()) : c;
    }

    // At least the input samples of any step that completes at most max_blocks blocks (a device call, check_call), from
    // any stream position: max_input's bound with the history it carries at its largest.
    int64_t max_call_input() const {
        if (!resamples()) return max_blocks * block;
        const int64_t m2 = k_of((max_blocks + 1) * block) + rs.T + rs.M / rs.L + 16;
        return mode == kDecimate ? (m2 + 1) * dec.D + dec.T1 + 16 : m2;
    }

    // The step over n new input samples at d_in (device).  Nothing of the stage changes until commit.
    InputStep plan(const uint8_t* d_in, int64_t n) const {
        InputStep s;
        s.rs.cur = d_in;
        if (!resamples()) {
            s.iq = mode == kPass ? d_in : dev.out[0];
            s.nblocks = n / block;
            return s;
        }
        if (mode == kDecimate) {  // the second stage takes the first stage's outputs of this step
            n = plan_first(s.dc, d_in, n);
            s.rs.cur = dev.mid;
        }
        // every output whose window is complete
        const int64_t L = rs.L, M = rs.M, T = rs.T;
        const int64_t in_new = pos.in_total + n;
        const int64_t ne = ertrs_out_end(&rs, in_new);
        const int64_t cnt = ne - pos.out_next;
        s.nblocks = (pos.pend + cnt) / block;
        s.iq = dev.out[pos.cur_out];
        RsArgs* a = &s.rs;
        a->hist = dev.hist[pos.cur_hist];
        a->hist_first = pos.hist_first;
        a->hist_n = pos.hist_n;
        a->cur_n = n;
        a->n0 = pos.out_next;
        a->count = cnt;
        a->split = s.nblocks > 0 ? s.nblocks * block - pos.pend : LLONG_MAX;
        a->base_n = (pos.out_next / L) * L;
        a->base_k = (pos.out_next / L) * M;
        a->out = dev.out[pos.cur_out] + 2 * pos.pend;
        a->out2 = dev.out[pos.cur_out ^ 1];
        const int64_t first = std::min(in_new, std::max<int64_t>(0, k_of(ne) - T / 2 + 1));
        a->carry_dst = dev.hist[pos.cur_hist ^ 1];
        a->carry_first = first;
        a->carry_n = in_new - first;
        a->L = L;
        a->M = M;
        a->T = (int)T;
        a->scale = scale;
        a->E = dev.E;
        a->W = nco_step;
        a->P = rs.P;
        a->gain = gain;
        a->level = nullptr;
        const int64_t Q = (int64_t)rs.P << ERTRS_F, step = kRsThreads * M;
        a->step_k = step / L;
        a->step_phi = step % L;
        a->step_q = (int64_t)(((__int128)a->step_phi * Q) / L);
        a->step_r = (int64_t)(((__int128)a->step_phi * Q) % L);
        return s;
    }

    // Enqueue the step's kernels on st, if it has any, and count them in *launches.
    int launch(const InputStep& s, cudaStream_t st, int64_t* launches) const {
        if (mode == kConvert) {
            const long long groups = s.nblocks * block / 8;
            const unsigned g = grid_of(groups, kCvtThreads, grid);
            fmt_visit(fmt, [&](auto f) {
                if constexpr (f() != ERTGPU_FORMAT_CU8)
                    convert_kernel<f()><<<g, kCvtThreads, 0, st>>>(s.rs.cur, dev.out[0], groups, scale);
            });
            CUDA_TRY(err_, cudaGetLastError());
            ++*launches;
            return ERTGPU_OK;
        }
        if (first_kernel && !s.shared_first && (s.dc.count > 0 || s.dc.carry_n > 0)) {
            first_kernel<<<grid_of(s.dc.count, (long long)kDcThreads * per1, grid1), kDcThreads, smem1, st>>>(dev.taps, s.dc);
            CUDA_TRY(err_, cudaGetLastError());
            ++*launches;
        }
        if (last_kernel && (s.rs.count > 0 || s.rs.carry_n > 0)) {
            last_kernel<<<grid_of(s.rs.count, kRsTile, grid), kRsThreads, smem, st>>>(dev.A, dev.D, s.rs);
            CUDA_TRY(err_, cudaGetLastError());
            ++*launches;
        }
        return ERTGPU_OK;
    }

    // Enqueue decimate_channels_kernel on st for the first stage of the n steps s[0..n) of a group of decimating
    // channels of one capture (this stage is s[0]'s; the others share its format, gain, plan, tables and stream position),
    // and mark each step's first stage as done.  Counted in *launches.
    int launch_channels(InputStep* s, int n, cudaStream_t st, int64_t* launches) const {
        const DcArgs& a = s[0].dc;
        DcChannels ch{};
        ch.n = n;
        for (int k = 0; k < n; k++) {
            ch.W[k] = s[k].dc.W;
            ch.out[k] = s[k].dc.out;
            ch.carry_dst[k] = s[k].dc.carry_dst;
            s[k].shared_first = true;
        }
        if (a.count <= 0 && a.carry_n <= 0) return ERTGPU_OK;
        DcArgs ac = a;
        ac.per = per1c;
        channels_kernel<<<grid_of(a.count, (long long)kDcThreads * per1c, grid1c), kDcThreads, smem1c, st>>>(dev.taps, ac, ch);
        CUDA_TRY(err_, cudaGetLastError());
        ++*launches;
        return ERTGPU_OK;
    }

    // Enqueue level_kernel over n input samples at d_in (device, 16-byte aligned) on st: their counts are added to dev.level.
    int launch_level(const uint8_t* d_in, int64_t n, cudaStream_t st) const {
        const long long nbytes = n * sample_bytes, groups = (nbytes + 15) / 16;
        const unsigned g = grid_of(groups, kLvThreads, level_grid);
        fmt_visit(fmt, [&](auto f) {
            if constexpr (f() != ERTGPU_FORMAT_CU8) level_kernel<f()><<<g, kLvThreads, 0, st>>>(d_in, nbytes, dev.level);
        });
        CUDA_TRY(err_, cudaGetLastError());
        return ERTGPU_OK;
    }

    // The step's kernel is enqueued: advance the stream position.
    void commit(const InputStep& s) {
        if (!resamples()) {  // whole blocks only (check_call)
            pos.in_total += s.nblocks * block;
            return;
        }
        if (mode == kDecimate) {
            pos.in1_total += s.dc.cur_n;
            pos.hist1_first = s.dc.carry_first;
            pos.hist1_n = s.dc.carry_n;
            pos.cur_hist1 ^= 1;
        }
        const RsArgs& a = s.rs;
        pos.in_total += a.cur_n;
        pos.out_next += a.count;
        pos.hist_first = a.carry_first;
        pos.hist_n = a.carry_n;
        pos.cur_hist ^= 1;
        pos.pend += a.count - s.nblocks * block;
        if (s.nblocks > 0) pos.cur_out ^= 1;  // the outputs past the last whole block are already at the front of the other buffer
    }

    // The stage's kernels as ertgpu_last_kernels names them ("" in pass-through mode); `shared`: the first stage ran as
    // decimate_channels_kernel.
    std::string label(bool shared = false) const {
        const char* f = fmt_name(fmt);
        if (wide)
            return mode == kDecimate ? std::string("decimate_kernel<") + f + ",wide>;resample_kernel<mid16,tuned,wide>"
                                     : std::string("resample_kernel<") + f + ",tuned,wide>";
        switch (mode) {
            case kPass: return "";
            case kConvert: return std::string("convert_kernel<") + f + ">";
            case kResample: return fmt == ERTGPU_FORMAT_CU8 ? "resample_kernel" : std::string("resample_kernel<") + f + ">";
            case kDecimate: return std::string(shared ? "decimate_channels_kernel<" : "decimate_kernel<") + f + ">;resample_kernel<cu8>";
            default: return std::string("resample_kernel<") + f + ",tuned>";
        }
    }

    // A channel measurement (wide path) runs the stage's own steps from a stream start, with rs.level = dev.clevel in every
    // step.  begin_measure swaps the measurement's input histories and stream position in for the stream's, and
    // end_measure swaps them back.
    void begin_measure() {
        swap_measure();
        reset_stream();
    }

    void end_measure() { swap_measure(); }

private:
    std::string& err_;  // the handle's last error

    void swap_measure() {
        std::swap(pos, mpos);
        std::swap(dev.hist, dev.mhist);
        std::swap(dev.hist1, dev.mhist1);
    }

    // CTAs of a launch over n items, per to a tile: one per tile, at least one and at most cap.
    static unsigned grid_of(long long n, long long per, int cap) {
        return (unsigned)std::max<long long>(1, std::min<long long>((n + per - 1) / per, cap));
    }

    // A kernel of `threads` threads with `bytes` of dynamic shared memory (allow_dynamic_smem): *cap becomes the most CTAs
    // of it the device runs at once.
    int fit(const void* kernel, int threads, size_t bytes, const char* what, int sm_count, int* cap) {
        if (const int rc = allow_dynamic_smem(err_, kernel, bytes, what)) return rc;
        int per_sm = 0;
        CUDA_TRY(err_, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, bytes));
        *cap = std::max(1, per_sm) * sm_count;
        return ERTGPU_OK;
    }

    // The resampler for input at hz: ertrs_plan, or ertrs_plan_tuned and the NCO step on a tuned handle.  It runs when
    // the rates differ or a tuned handle mixes; the tuned instance when it mixes or its plan has P != ERTRS_P.
    int configure_rate(int64_t hz, int64_t rate_out) {
        ertgpu_resampler_info info{};
        ertgpu_decimator_info d{};
        std::vector<int16_t> t1;
        uint32_t w = 0;
        if (tuned && decimation) {
            const int64_t off = center_hz - capture_hz;
            if (ertrs_plan_decimated(hz, rate_out, off, &d, &info) != 0)  // up to 10:1 the message of a tuned handle
                return fail(err_, ERTGPU_EINVAL,
                            "input rate %lld Hz, channel offset %lld Hz: the decoder rate %lld Hz must be within %s ... 4 "
                            "times the input rate, and |offset| + 0.4 * min(rates) at most half the input rate",
                            (long long)hz, (long long)off, (long long)rate_out, hz <= 10 * rate_out ? "1/10" : "1/256");
            if (d.D > 1) {
                t1.resize((size_t)d.T1);
                if (ertrs_build_decimator(&d, t1.data()) != 0) return fail(err_, ERTGPU_EINVAL, "decimator taps do not fit int16");
            }
            w = ertrs_nco_step(off, hz);
        } else if (tuned) {
            const int64_t off = center_hz - capture_hz;
            if (ertrs_plan_tuned(hz, rate_out, off, &info) != 0)
                return fail(err_, ERTGPU_EINVAL,
                            "input rate %lld Hz, channel offset %lld Hz: the decoder rate %lld Hz must be within 1/10 ... 4 "
                            "times the input rate, and |offset| + 0.4 * min(rates) at most half the input rate",
                            (long long)hz, (long long)off, (long long)rate_out);
            w = ertrs_nco_step(off, hz);
        } else if (ertrs_plan(hz, rate_out, &info) != 0) {
            return fail(err_, ERTGPU_EINVAL, "input rate %lld Hz: the decoder rate %lld Hz must be within 1/4 ... 4 times it",
                        (long long)hz, (long long)rate_out);
        }
        const bool on = hz != rate_out || w != 0 || wide;
        std::vector<int16_t> t;
        if (on) {
            t.resize((size_t)(info.P + 1) * info.T);
            if (ertrs_build_table(&info, t.data()) != 0) return fail(err_, ERTGPU_EINVAL, "resampler table does not fit int16");
        }
        mode = !on ? (fmt == ERTGPU_FORMAT_CU8 ? kPass : kConvert) : w != 0 || info.P != ERTRS_P || wide ? kResampleTuned : kResample;
        if (d.D > 1) mode = kDecimate;
        nco_step = w;
        rs = info;
        table.swap(t);
        dec = d;
        taps.swap(t1);
        return ERTGPU_OK;
    }

    // The first stage's plan of the step over n new input samples at d_in; returns its number of outputs.
    int64_t plan_first(DcArgs& a, const uint8_t* d_in, int64_t n) const {
        const int64_t D = dec.D, T1 = dec.T1;
        const int64_t in_new = pos.in1_total + n;
        const int64_t ne = in_new - T1 / 2 > 0 ? (in_new - T1 / 2 + D - 1) / D : 0;  // ertrs_out_end at L = 1, M = D
        a.hist = dev.hist1[pos.cur_hist1];
        a.cur = d_in;
        a.hist_first = pos.hist1_first;
        a.hist_n = pos.hist1_n;
        a.cur_n = n;
        a.n0 = pos.in_total;  // the first stage's next output is the second stage's next input
        a.count = ne - pos.in_total;
        a.out = dev.mid;
        const int64_t first = std::min(in_new, std::max<int64_t>(0, ne * D - T1 / 2 + 1));
        a.carry_dst = dev.hist1[pos.cur_hist1 ^ 1];
        a.carry_first = first;
        a.carry_n = in_new - first;
        a.D = (int)D;
        a.T1 = (int)T1;
        a.per = per1;
        a.scale = scale;
        a.E = dev.E;
        a.W = nco_step;
        return a.count;
    }

    // The first stage's device buffers, after the second stage's.
    int allocate_first(int sm_count) {
        CUDA_TRY(err_, dev.taps.upload(taps));
        const size_t hb = wide ? 4 : 2;  // bytes per carried sample, and per stage-1 output
        for (int k = 0; k < 2; k++) CUDA_TRY(err_, dev.hist1[k].alloc((size_t)(dec.T1 + dec.D + 16) * hb));
        // A step hands the second stage fewer than (max_blocks + 1) * block * M / L + M / L + T samples (the blocks a
        // step may complete, plus the look-ahead).
        const int64_t mid = (int64_t)(((__int128)(max_blocks + 1) * block * rs.M + rs.L - 1) / rs.L) + rs.M / rs.L + rs.T + 64;
        CUDA_TRY(err_, dev.mid.alloc((size_t)mid * hb));
        per1 = dc_per_thread(dec.D, dec.T1);
        smem1 = dc_smem_bytes(dec.D, dec.T1, per1);
        if (const int rc = fit((const void*)first_kernel, kDcThreads, smem1, "decimator", sm_count, &grid1)) return rc;
        if (wide) {  // decimate_wide_kernel: decimate_kernel's tiles; groups run it per channel (DESIGN §3.12)
            for (int k = 0; k < 2; k++) CUDA_TRY(err_, dev.mhist1[k].alloc((size_t)(dec.T1 + dec.D + 16) * 4));
            return ERTGPU_OK;
        }
        per1c = dc_per_thread(dec.D, dec.T1, kDcChannelsSpanWords);
        smem1c = dc_channels_smem_bytes(dec.D, dec.T1, per1c);
        return fit((const void*)channels_kernel, kDcThreads, smem1c, "decimator", sm_count, &grid1c);
    }

    int64_t k_of(int64_t n) const { return (int64_t)((__int128)n * rs.M / rs.L); }

    // Most input samples the next step may take so that it completes at most max_blocks decoder blocks.
    int64_t max_input() const {
        const int64_t cap_out = (max_blocks + 1) * block - 1 - pos.pend;
        const int64_t m2 = rs.T / 2 + k_of(pos.out_next + cap_out) - pos.in_total;
        // decimating: the first stage completes at most m2 outputs, ceil((in1_total + x - T1/2) / D) <= in_total + m2
        return mode == kDecimate ? (pos.in_total + m2) * dec.D + dec.T1 / 2 - pos.in1_total : m2;
    }
};

}  // namespace ert
