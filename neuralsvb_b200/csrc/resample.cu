// Band-limited resampling with resampy's kaiser_best filter over a ragged batch of clips: what the reference's
// librosa.core.load(path, sr=...) does to every waveform it reads (data_gen/tts/data_gen_utils.py:111, librosa 0.8.0 /
// resampy 0.2.2).  oracle/resample.py states the algorithm; this file implements the same text in two launches:
//
//   1. resample_time_kernel   one thread per distinct source rate: the sequential float64 time register
//                             (time_register += 1 / ratio once per output), written once up to the longest clip of that rate.
//                             A sum in order is the text; t * increment is not the same number once the increment is inexact.
//   2. resample_kernel        one CTA per kOut consecutive output samples of one clip, one thread per output.  The input span
//                             the CTA's outputs read is staged in shared memory as double; each thread walks the left wing, then
//                             the right wing, one 16-byte {win, delta} load per tap from the rate's table (512 KB: served by
//                             L1 / L2), and rounds its float32 output after every tap (__dmul_rn / __dadd_rn, so that nothing
//                             is contracted to an FMA, then __double2float_rn).  Outputs past int(n_in ratio) are the
//                             fix_length zeros; a clip already at the target rate is copied.
//
// Each output reads only its own clip and accumulates in a fixed order without atomics, so a clip's output is bit-identical alone
// and in any batch.  The tables are built on the host from the caller's float64 window (scaled by the ratio and differenced with
// the same float64 operations as the oracle); every size and the workspace are worked out on the host before any launch.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"

namespace svb {
namespace {

constexpr int kOut = 128;                  // outputs per CTA (one per thread)
constexpr size_t kMaxSmem = 200 * 1024;    // the staged input span of one CTA

struct ResClip {
    long long in_off;    // first input sample in the concatenated waveforms
    long long out_off;   // first output sample in the concatenated outputs
    int n_in;            // input samples
    int n_res;           // int(n_in ratio): computed outputs
    int n_out;           // ceil(n_in ratio): outputs after the fix_length zeros (n_in when the rate is the target)
    int rate;            // index of the clip's source rate in the rate table, -1 when it is the target rate
    int blk_off;         // first CTA of the clip
};

struct ResRate {
    double inc;          // 1 / ratio
    double scale;        // min(1, ratio)
    long long tr_off;    // first entry of the rate's time register
    long long tab_off;   // first {win, delta} entry of the rate's table
    int step;            // index_step = int(scale num_table)
    int wmax;            // nwin / step: the longest wing
    int n_max;           // the longest clip's n_res
    int src_sr;
};

struct Layout {
    std::vector<ResClip> clips;
    std::vector<ResRate> rates;
    size_t off_clip, off_rate, off_tab, off_tr, total, smem;
    long long out_total;
    int blocks;
};

size_t align_up(size_t x) { return (x + 255) / 256 * 256; }

int plan(int32_t target_sr, const int32_t *src_sr, const int64_t *lengths, int32_t n_clips, int32_t nwin, int32_t num_table, Layout *lay) {
    SVB_CHECK(src_sr && lengths && n_clips > 0, SVB_ERR_INVALID, "resample: null rates or lengths, or no clips");
    SVB_CHECK(target_sr > 0, SVB_ERR_INVALID, "resample: target rate %d", target_sr);
    SVB_CHECK(nwin >= 2 && num_table >= 1, SVB_ERR_INVALID, "resample: filter of %d taps at %d per zero crossing", nwin, num_table);
    lay->clips.resize(n_clips);
    lay->rates.clear();
    long long in = 0, out = 0, blk = 0, tr = 0;
    size_t smem = 0;
    for (int c = 0; c < n_clips; ++c) {
        const long long N = lengths[c];
        SVB_CHECK(src_sr[c] > 0, SVB_ERR_INVALID, "resample: clip %d has sample rate %d", c, src_sr[c]);
        SVB_CHECK(N >= 0 && N < (1LL << 31), SVB_ERR_INVALID, "resample: clip %d has %lld samples", c, N);
        ResClip cl{in, out, (int)N, (int)N, (int)N, -1, (int)blk};
        if (src_sr[c] != target_sr) {
            const double ratio = (double)target_sr / (double)src_sr[c];
            const double n_res = std::floor((double)N * ratio), n_out = std::ceil((double)N * ratio);
            SVB_CHECK(n_res >= 1.0, SVB_ERR_INVALID, "resample: clip %d: %lld samples are too few to resample from %d to %d Hz", c, N,
                      src_sr[c], target_sr);
            SVB_CHECK(n_out < (double)(1LL << 31), SVB_ERR_INVALID, "resample: clip %d: %.0f output samples", c, n_out);
            cl.n_res = (int)n_res, cl.n_out = (int)n_out;
            int r = 0;
            while (r < (int)lay->rates.size() && lay->rates[r].src_sr != src_sr[c]) ++r;
            if (r == (int)lay->rates.size()) {
                const double scale = std::min(1.0, ratio);
                const int step = (int)(scale * num_table);
                SVB_CHECK(step >= 1, SVB_ERR_INVALID, "resample: ratio %d / %d is below 1 / %d", target_sr, src_sr[c], num_table);
                ResRate R{1.0 / ratio, scale, 0, (long long)r * nwin, step, nwin / step, 0, src_sr[c]};
                // the span of kOut outputs: (kOut - 1) increments (plus the time register's rounding), then a wing on each side
                const double span = std::ceil((kOut - 1) * R.inc * (1.0 + 1e-9)) + 2.0 + 2.0 * R.wmax + 2.0;
                SVB_CHECK(span * sizeof(double) <= kMaxSmem, SVB_ERR_INVALID, "resample: ratio %d / %d needs %.0f staged samples per CTA",
                          target_sr, src_sr[c], span);
                smem = std::max(smem, (size_t)span * sizeof(double));
                lay->rates.push_back(R);
            }
            cl.rate = r;
            lay->rates[r].n_max = std::max(lay->rates[r].n_max, cl.n_res);
        }
        lay->clips[c] = cl;
        in += N, out += cl.n_out;
        blk += (cl.n_out + kOut - 1) / kOut;
    }
    SVB_CHECK(blk < (1LL << 31), SVB_ERR_INVALID, "resample: %lld output samples are too many for one call", out);
    for (auto &R : lay->rates) R.tr_off = tr, tr += R.n_max;
    lay->out_total = out, lay->blocks = (int)blk, lay->smem = smem;
    lay->off_clip = 0;
    lay->off_rate = align_up((size_t)n_clips * sizeof(ResClip));
    lay->off_tab = lay->off_rate + align_up(std::max<size_t>(1, lay->rates.size()) * sizeof(ResRate));
    lay->off_tr = lay->off_tab + align_up(lay->rates.size() * (size_t)nwin * sizeof(double2));
    lay->total = lay->off_tr + align_up((size_t)tr * sizeof(double));
    return SVB_OK;
}

// ---- kernel 1: the time register ------------------------------------------------------------------------------------------
__global__ void resample_time_kernel(const ResRate *__restrict__ rates, double *__restrict__ trs) {
    const ResRate R = rates[blockIdx.x];
    double *tr = trs + R.tr_off;
    double v = 0.0;
    for (int t = 0; t < R.n_max; ++t) {
        tr[t] = v;
        v = __dadd_rn(v, R.inc);
    }
}

// ---- kernel 2: the filter -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void phase(double frac, int num_table, int *off, double *eta) {
    const double idx = __dmul_rn(frac, (double)num_table);
    *off = (int)idx;                                               // int() of a non-negative value: truncation
    *eta = __dsub_rn(idx, (double)*off);
}

// y = float32(float64(y) + (win + eta delta) float64(x)), each operation rounded on its own
__device__ __forceinline__ float tap(float y, double2 w, double eta, double x) {
    const double weight = __dadd_rn(w.x, __dmul_rn(eta, w.y));
    return __double2float_rn(__dadd_rn((double)y, __dmul_rn(weight, x)));
}

__global__ void __launch_bounds__(kOut) resample_kernel(const float *__restrict__ wav, const ResClip *__restrict__ clips, int n_clips,
                                                        const ResRate *__restrict__ rates, const double2 *__restrict__ tabs,
                                                        const double *__restrict__ trs, int nwin, int num_table, float *__restrict__ out) {
    extern __shared__ double xs[];
    int lo_c = 0, hi_c = n_clips - 1;                               // the last clip with blk_off <= blockIdx.x
    while (lo_c < hi_c) {
        const int mid = (lo_c + hi_c + 1) >> 1;
        if (clips[mid].blk_off <= (int)blockIdx.x) lo_c = mid;
        else hi_c = mid - 1;
    }
    const ResClip cl = clips[lo_c];
    const int t0 = ((int)blockIdx.x - cl.blk_off) * kOut, t = t0 + (int)threadIdx.x;
    const float *x = wav + cl.in_off;
    float *o = out + cl.out_off;
    if (cl.rate < 0) {                                              // already at the target rate
        if (t < cl.n_out) o[t] = x[t];
        return;
    }
    if (t0 >= cl.n_res) {                                           // the whole CTA is in the fix_length tail
        if (t < cl.n_out) o[t] = 0.f;
        return;
    }
    const ResRate R = rates[cl.rate];
    const double *tr = trs + R.tr_off;
    const long long n_first = (long long)tr[t0], n_last = (long long)tr[min(t0 + kOut, cl.n_res) - 1];
    const long long lo = max(0LL, n_first - R.wmax), hi = min((long long)cl.n_in, n_last + R.wmax + 1);
    for (long long i = threadIdx.x; i < hi - lo; i += kOut) xs[i] = (double)x[lo + i];
    __syncthreads();                                                // no block-wide barrier below this point
    if (t >= cl.n_out) return;
    if (t >= cl.n_res) {
        o[t] = 0.f;
        return;
    }
    const double trv = tr[t];
    const long long n = (long long)trv;
    const double2 *tab = tabs + R.tab_off;
    const double *xc = xs + (n - lo);
    float y = 0.f;
    double frac = __dmul_rn(R.scale, __dsub_rn(trv, (double)n)), eta;
    int off;
    phase(frac, num_table, &off, &eta);
    const int left = (int)min(n + 1, (long long)((nwin - off) / R.step));
    for (int i = 0; i < left; ++i) y = tap(y, __ldg(tab + off + i * R.step), eta, xc[-i]);
    frac = __dsub_rn(R.scale, frac);
    phase(frac, num_table, &off, &eta);
    const int right = (int)min((long long)cl.n_in - n - 1, (long long)((nwin - off) / R.step));
    for (int k = 0; k < right; ++k) y = tap(y, __ldg(tab + off + k * R.step), eta, xc[k + 1]);
    o[t] = y;
}

int run(int32_t target_sr, const int32_t *src_sr, const int64_t *lengths, int32_t n_clips, const double *win, int32_t nwin, int32_t num_table,
        const float *wav_dev, float *out_dev, void *ws, int64_t ws_bytes, float *stage_ms, cudaStream_t st) {
    Layout lay;
    SVB_TRY(plan(target_sr, src_sr, lengths, n_clips, nwin, num_table, &lay));
    SVB_CHECK(win && wav_dev && out_dev && ws, SVB_ERR_INVALID, "resample: null buffer");
    SVB_CHECK(ws_bytes >= (int64_t)lay.total, SVB_ERR_INVALID, "resample: workspace of %lld bytes, %zu needed", (long long)ws_bytes, lay.total);
    if (lay.out_total == 0) return SVB_OK;
    // one table per source rate: the window scaled by the ratio below 1, then differenced (oracle/resample.tables)
    std::vector<double2> tabs(lay.rates.size() * (size_t)nwin);
    std::vector<double> s(nwin);
    for (size_t r = 0; r < lay.rates.size(); ++r) {
        const double ratio = (double)target_sr / (double)lay.rates[r].src_sr;
        for (int j = 0; j < nwin; ++j) s[j] = ratio < 1.0 ? win[j] * ratio : win[j];
        double2 *tb = tabs.data() + r * nwin;
        for (int j = 0; j < nwin; ++j) tb[j] = make_double2(s[j], j + 1 < nwin ? s[j + 1] - s[j] : 0.0);
    }
    char *base = static_cast<char *>(ws);
    ResClip *d_clips = reinterpret_cast<ResClip *>(base + lay.off_clip);
    ResRate *d_rates = reinterpret_cast<ResRate *>(base + lay.off_rate);
    double2 *d_tabs = reinterpret_cast<double2 *>(base + lay.off_tab);
    double *d_tr = reinterpret_cast<double *>(base + lay.off_tr);
    SVB_CUDA(cudaMemcpyAsync(d_clips, lay.clips.data(), lay.clips.size() * sizeof(ResClip), cudaMemcpyHostToDevice, st));
    if (!lay.rates.empty()) {
        SVB_CUDA(cudaMemcpyAsync(d_rates, lay.rates.data(), lay.rates.size() * sizeof(ResRate), cudaMemcpyHostToDevice, st));
        SVB_CUDA(cudaMemcpyAsync(d_tabs, tabs.data(), tabs.size() * sizeof(double2), cudaMemcpyHostToDevice, st));
    }
    // the copies read pageable host vectors: finish them before the vectors go out of scope
    SVB_CUDA(cudaStreamSynchronize(st));

    cudaEvent_t ev[3] = {};
    if (stage_ms)
        for (auto &e : ev) SVB_CUDA(cudaEventCreate(&e));
    int rc = SVB_OK;
    auto mark = [&](int k) {
        if (stage_ms && rc == SVB_OK && cudaEventRecord(ev[k], st) != cudaSuccess) rc = SVB_ERR_CUDA;
    };
    mark(0);
    if (!lay.rates.empty()) resample_time_kernel<<<(int)lay.rates.size(), 1, 0, st>>>(d_rates, d_tr);
    mark(1);
    static size_t configured[kSmemCacheDevices] = {};
    if (rc == SVB_OK && cudaGetLastError() != cudaSuccess) rc = SVB_ERR_CUDA;
    if (rc == SVB_OK) rc = raise_smem_limit(resample_kernel, lay.smem, configured);
    if (rc == SVB_OK) {
        resample_kernel<<<lay.blocks, kOut, lay.smem, st>>>(wav_dev, d_clips, n_clips, d_rates, d_tabs, d_tr, nwin, num_table, out_dev);
        if (cudaGetLastError() != cudaSuccess) rc = SVB_ERR_CUDA;
    }
    mark(2);
    if (stage_ms && rc == SVB_OK) {
        if (cudaEventSynchronize(ev[2]) != cudaSuccess || cudaEventElapsedTime(stage_ms, ev[0], ev[1]) != cudaSuccess ||
            cudaEventElapsedTime(stage_ms + 1, ev[1], ev[2]) != cudaSuccess)
            rc = SVB_ERR_CUDA;
    }
    for (auto e : ev)
        if (e) cudaEventDestroy(e);
    if (rc != SVB_OK) set_error("resample: launch or timing failed: %s", cudaGetErrorString(cudaGetLastError()));
    return rc;
}

}  // namespace
}  // namespace svb

using namespace svb;

extern "C" int64_t svb_resample_plan(int32_t target_sr, const int32_t *src_sr, const int64_t *lengths, int32_t n_clips, int32_t nwin,
                                     int32_t num_table, int64_t *res_lengths_out, int64_t *out_lengths_out) {
    Layout lay;
    if (plan(target_sr, src_sr, lengths, n_clips, nwin, num_table, &lay) != SVB_OK) return -1;
    for (int c = 0; c < n_clips; ++c) {
        if (res_lengths_out) res_lengths_out[c] = lay.clips[c].n_res;
        if (out_lengths_out) out_lengths_out[c] = lay.clips[c].n_out;
    }
    return (int64_t)lay.total;
}

extern "C" int svb_resample_batch(int32_t target_sr, const int32_t *src_sr, const int64_t *lengths, int32_t n_clips, const double *win_host,
                                  int32_t nwin, int32_t num_table, const float *wav_concat_dev, float *out_dev, void *workspace_dev,
                                  int64_t workspace_bytes, float *stage_ms_host, void *stream) {
    return run(target_sr, src_sr, lengths, n_clips, win_host, nwin, num_table, wav_concat_dev, out_dev, workspace_dev, workspace_bytes,
               stage_ms_host, as_stream(stream));
}
