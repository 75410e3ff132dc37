// Autocorrelation pitch tracker (Boersma 1993, the method of Praat's "To Pitch (ac)") over a ragged batch of clips: the f0
// extractor of the binarizer (reference data_gen/tts/data_gen_utils.py:150-184, `get_pitch`).  oracle/pitch_ac.py states the
// algorithm in full; this file implements the same text in three launches:
//
//   1. pitch_clip_stats_kernel   one CTA per clip: the clip's mean (double, fixed strided order + fixed tree) and
//                                globalPeak = max |x - mean|.
//   2. pitch_cand_kernel         one CTA per run of kFPC consecutive frames of one clip, one warp per frame.  The samples the
//                                kFPC windows share are staged in shared memory once (827 + 7 * 128 at 22050 Hz / hop 128);
//                                each warp removes its window's mean, takes the local peak, applies the Hann window and
//                                computes r_a(tau) for tau = 0 .. tau_max + 1 with fp32 FMAs from shared memory: lane l owns
//                                the R consecutive lags l R .. l R + R - 1 and slides a register window over the frame, so a
//                                step is two shared loads (one a broadcast) for R FMAs.  Then it normalises by the window's
//                                own autocorrelation (a host-computed table), finds and refines the peaks, compacts them in
//                                lag order with ballots and selects the 14 strongest (ties to the smaller lag) by repeated
//                                warp arg-max.  Output: [frames, 15] (frequency, strength) pairs and a count per frame.
//   3. pitch_path_kernel         one warp per clip, lane j = candidate j: the Viterbi recursion in double, each step a max over
//                                the 16 predecessors by shuffles (ties to the lower index), uint8 back-pointers [frames, 16] in
//                                global memory, then the backtrack writes f0 straight into the placed [len(mel)] output.
//
// Every launch reads only its own clip's samples and reduces in a fixed order without atomics, so a clip's output is
// bit-identical alone and in any batch.  Sizes (frames, window, workspace) are worked out on the host before any launch.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace svb {
namespace {

constexpr int kFPC = 8;             // frames per CTA of the candidate kernel (one warp each)
constexpr int kMaxCand = 15;        // unvoiced + 14 voiced
constexpr int kMaxR = 18;           // lags per lane: tau_max + 2 <= 32 * 18

struct PitchClip {
    long long wav_off;   // first sample in the concatenated waveforms
    long long out_off;   // first placed output frame
    int N;               // samples
    int n;               // analysis frames
    int c0;              // centre sample of frame 0
    int frame_off;       // first analysis frame in the batch's frame arrays
    int blk_off;         // first CTA of the candidate kernel
    int T;               // placed output frames (len(mel))
};

struct PitchParams {
    int sr, hop, L, h, tau_max, nlag, lpad, n_clips;
    float sr_f, lag_min, lag_max, half_vt, vt, st, oc, floor_hz;
    double c_vu, c_oj;   // voiced_unvoiced_cost * c, octave_jump_cost * c (c = 0.01 / dt)
};

struct Grid {
    int n, L, c0, tau_max;
};

// oracle/pitch_ac.grid, the same float64 operations in the same order
int pitch_grid(const svb_pitch_config *cfg, long long N, int clip, Grid *g) {
    const double D = (double)N / cfg->sr, W = 3.0 / cfg->floor;
    g->L = 2 * (int)std::floor(W * cfg->sr / 2.0) + 1;
    const double nf = std::floor((D - W) / cfg->time_step) + 1.0;
    SVB_CHECK(nf >= 1.0, SVB_ERR_INVALID, "pitch_ac: clip %d has %lld samples (%.4f s), shorter than one pitch window (%.4f s at floor %g Hz)",
              clip, N, D, W, cfg->floor);
    g->n = (int)nf;
    g->c0 = (int)((N - (long long)(g->n - 1) * cfg->hop) / 2);
    g->tau_max = (int)std::ceil(cfg->sr / cfg->floor);
    return SVB_OK;
}

int validate(const svb_pitch_config *cfg) {
    SVB_CHECK(cfg, SVB_ERR_INVALID, "pitch_ac: null config");
    SVB_CHECK(cfg->sr > 0 && cfg->hop > 0 && cfg->floor > 0 && cfg->ceiling > cfg->floor && cfg->time_step > 0, SVB_ERR_INVALID,
              "pitch_ac: bad sr %d / hop %d / floor %g / ceiling %g / time_step %g", cfg->sr, cfg->hop, cfg->floor, cfg->ceiling,
              cfg->time_step);
    SVB_CHECK(std::fabs(cfg->time_step * cfg->sr - cfg->hop) < 1e-6, SVB_ERR_INVALID,
              "pitch_ac: time_step %g s is not hop / sr = %d / %d", cfg->time_step, cfg->hop, cfg->sr);
    SVB_CHECK(cfg->lpad >= 0, SVB_ERR_INVALID, "pitch_ac: negative lpad %d", cfg->lpad);
    SVB_CHECK(cfg->voicing_threshold >= 0 && cfg->silence_threshold > 0 && cfg->octave_cost >= 0 && cfg->octave_jump_cost >= 0 &&
                  cfg->voiced_unvoiced_cost >= 0, SVB_ERR_INVALID, "pitch_ac: negative threshold or cost");
    const int tau_max = (int)std::ceil(cfg->sr / cfg->floor);
    SVB_CHECK(tau_max + 2 <= 32 * kMaxR, SVB_ERR_INVALID, "pitch_ac: sr / floor = %g needs %d lags, more than %d", cfg->sr / cfg->floor,
              tau_max + 2, 32 * kMaxR);
    SVB_CHECK(cfg->sr / cfg->ceiling >= 2.0, SVB_ERR_INVALID, "pitch_ac: ceiling %g is above sr / 2", cfg->ceiling);
    return SVB_OK;
}

// ---- workspace ----------------------------------------------------------------------------------------------------------------
struct Layout {
    size_t off_clip, off_stats, off_win, off_rwn, off_cand, off_count, off_bp, total;
    long long frames;
    int blocks, L, tau_max;
};

size_t align_up(size_t x) { return (x + 255) / 256 * 256; }

int plan(const svb_pitch_config *cfg, const int64_t *lengths, const int64_t *mel_frames, int32_t n_clips,
         std::vector<PitchClip> *clips, Layout *lay) {
    SVB_TRY(validate(cfg));
    SVB_CHECK(lengths && n_clips > 0, SVB_ERR_INVALID, "pitch_ac: null lengths or no clips");
    if (clips) clips->resize(n_clips);
    long long wav = 0, fr = 0, out = 0;
    int blk = 0, L = 0, tau_max = 0;
    for (int c = 0; c < n_clips; ++c) {
        SVB_CHECK(lengths[c] > 0 && lengths[c] < (1LL << 31), SVB_ERR_INVALID, "pitch_ac: clip %d has %lld samples", c, (long long)lengths[c]);
        Grid g;
        SVB_TRY(pitch_grid(cfg, lengths[c], c, &g));
        const long long T = mel_frames ? mel_frames[c] : 0;
        SVB_CHECK(T >= 0 && T < (1LL << 31), SVB_ERR_INVALID, "pitch_ac: clip %d has %lld mel frames", c, T);
        if (clips) (*clips)[c] = PitchClip{wav, out, (int)lengths[c], g.n, g.c0, (int)fr, blk, (int)T};
        wav += lengths[c], fr += g.n, out += T;
        blk += (g.n + kFPC - 1) / kFPC;
        L = g.L, tau_max = g.tau_max;
    }
    SVB_CHECK(blk < (1 << 30), SVB_ERR_INVALID, "pitch_ac: %lld frames are too many for one call", fr);
    lay->frames = fr, lay->blocks = blk, lay->L = L, lay->tau_max = tau_max;
    lay->off_clip = 0;
    lay->off_stats = align_up((size_t)n_clips * sizeof(PitchClip));
    lay->off_win = lay->off_stats + align_up((size_t)n_clips * 2 * sizeof(float));
    lay->off_rwn = lay->off_win + align_up((size_t)L * sizeof(float));
    lay->off_cand = lay->off_rwn + align_up((size_t)(tau_max + 2) * sizeof(float));
    lay->off_count = lay->off_cand + align_up((size_t)fr * kMaxCand * sizeof(float2));
    lay->off_bp = lay->off_count + align_up((size_t)fr * sizeof(int));
    lay->total = lay->off_bp + align_up((size_t)fr * 16);
    return SVB_OK;
}

// ---- kernel 1: clip statistics ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pitch_clip_stats_kernel(const float *__restrict__ wav, const PitchClip *__restrict__ clips,
                                                               float2 *__restrict__ stats) {
    const PitchClip cl = clips[blockIdx.x];
    const float *x = wav + cl.wav_off;
    __shared__ double ssum[256];
    __shared__ float smax[256];
    double s = 0.0;
    for (int i = threadIdx.x; i < cl.N; i += 256) s += (double)x[i];
    ssum[threadIdx.x] = s;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) ssum[threadIdx.x] += ssum[threadIdx.x + w];
        __syncthreads();
    }
    const float mean = (float)(ssum[0] / cl.N);
    float m = 0.f;
    for (int i = threadIdx.x; i < cl.N; i += 256) m = fmaxf(m, fabsf(x[i] - mean));
    smax[threadIdx.x] = m;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) smax[threadIdx.x] = fmaxf(smax[threadIdx.x], smax[threadIdx.x + w]);
        __syncthreads();
    }
    if (threadIdx.x == 0) stats[blockIdx.x] = make_float2(mean, smax[0]);
}

// ---- kernel 2: frame analysis and candidates ----------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// (strength, lag) a beats b: stronger, or as strong with the smaller lag
__device__ __forceinline__ bool beats(float sa, float la, float sb, float lb) { return sa > sb || (sa == sb && la < lb); }

template <int R>
__global__ void __launch_bounds__(32 * kFPC) pitch_cand_kernel(const float *__restrict__ wav, const PitchClip *__restrict__ clips,
                                                               const float2 *__restrict__ stats, const float *__restrict__ win,
                                                               const float *__restrict__ rwn, PitchParams p, float2 *__restrict__ cand,
                                                               int *__restrict__ count, float *__restrict__ r_out) {
    extern __shared__ float smem[];
    // every section starts on a 16-byte boundary: the peak list below is read as float2
    const int FB = round_up(p.L + 32 * R, 4);                      // frame buffer: the windowed frame + zero tail for the lags
    float *stage = smem;                                           // [L + (kFPC - 1) hop], rounded up to 4 floats
    float *fbuf = stage + round_up(p.L + (kFPC - 1) * p.hop, 4);   // [kFPC][FB]
    float *rbuf = fbuf + kFPC * FB;                                // [kFPC][32 R]
    float2 *pk = reinterpret_cast<float2 *>(rbuf + kFPC * 32 * R); // [kFPC][16 R] (strength, lag)

    int lo = 0, hi = p.n_clips - 1;                                // the last clip with blk_off <= blockIdx.x
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (clips[mid].blk_off <= (int)blockIdx.x) lo = mid;
        else hi = mid - 1;
    }
    const PitchClip cl = clips[lo];
    const int j0 = ((int)blockIdx.x - cl.blk_off) * kFPC;
    const float *x = wav + cl.wav_off;
    const long long first = (long long)cl.c0 + (long long)j0 * p.hop - p.h;
    const int S = p.L + (kFPC - 1) * p.hop;
    for (int i = threadIdx.x; i < S; i += blockDim.x) {
        const long long k = first + i;
        stage[i] = (k >= 0 && k < cl.N) ? x[k] : 0.f;
    }
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = j0 + warp;
    if (j >= cl.n) return;                                         // no block-wide barrier below this point
    const float *xs = stage + warp * p.hop;
    float *fb = fbuf + warp * FB;
    float s = 0.f;
    for (int k = lane; k < p.L; k += 32) s += xs[k];
    const float mean = warp_sum(s) / (float)p.L;
    float lp = 0.f;
    for (int k = lane; k < p.L; k += 32) {
        const float v = xs[k] - mean;
        lp = fmaxf(lp, fabsf(v));
        fb[k] = v * win[k];
    }
    for (int k = p.L + lane; k < FB; k += 32) fb[k] = 0.f;
    lp = warp_max(lp);
    __syncwarp();

    // r_a(tau) for tau = lane R .. lane R + R - 1, summed over k = 0 .. L - 1 in order
    const int tau0 = lane * R;
    float acc[R], wv[R];
#pragma unroll
    for (int i = 0; i < R; ++i) acc[i] = 0.f, wv[i] = fb[tau0 + i];
    for (int k = 0; k < p.L; ++k) {
        const float a = fb[k];
#pragma unroll
        for (int i = 0; i < R; ++i) acc[i] = fmaf(a, wv[i], acc[i]);
#pragma unroll
        for (int i = 0; i < R - 1; ++i) wv[i] = wv[i + 1];
        wv[R - 1] = fb[k + tau0 + R];
    }
    // An exactly constant window has r_a(0) = 0 and localPeak = 0: the text's float64 mean of equal floats is exact.  The fp32 mean
    // above need not be, and the +-1-ulp residue it leaves would normalise to r(tau) ~ 1.  Such a window leaves |x - mean| within
    // a few ulps of |mean| (the fp32 sum of L <= 1723 equal terms is within 60 ulps), so only a window that small pays for the
    // exact test.
    bool flat = false;
    if (lp <= 1e-4f * fabsf(mean)) {
        bool same = true;
        for (int k = lane; k < p.L; k += 32) same = same && xs[k] == xs[0];
        flat = __all_sync(0xffffffffu, same);
    }
    if (flat) lp = 0.f;
    const float ra0 = flat ? 0.f : __shfl_sync(0xffffffffu, acc[0], 0);
    float *rr = rbuf + warp * 32 * R;
    const long long fg = (long long)cl.frame_off + j;
#pragma unroll
    for (int i = 0; i < R; ++i) {
        const int tau = tau0 + i;
        if (tau < p.nlag) {
            const float v = ra0 != 0.f ? (acc[i] / ra0) / rwn[tau] : 0.f;
            rr[tau] = v;
            if (r_out) r_out[fg * p.nlag + tau] = v;
        }
    }
    __syncwarp();

    const float2 st = stats[lo];
    float2 *out = cand + fg * kMaxCand;
    float s_unv;
    if (st.y == 0.f) s_unv = p.vt + 2.f;
    else s_unv = p.vt + fmaxf(0.f, 2.f - (lp / st.y) / (p.st / (1.f + p.vt)));
    int nc = 1;
    if (st.y != 0.f && ra0 != 0.f) {
        // peaks in lag order, compacted with ballots
        float2 *mine = pk + warp * 16 * R;
        int np = 0;
        for (int t0 = 1; t0 <= p.tau_max; t0 += 32) {
            const int t = t0 + lane;
            bool ok = false;
            float str = 0.f, lag = 0.f;
            if (t <= p.tau_max) {
                const float a = rr[t - 1], b = rr[t], c = rr[t + 1];
                if (a < b && b >= c) {
                    const float d = 0.5f * (a - c) / (a - 2.f * b + c);
                    lag = (float)t + d;
                    const float height = b - 0.25f * (a - c) * d;
                    if (lag >= p.lag_min && lag <= p.lag_max && height > p.half_vt) {
                        ok = true;
                        str = height - p.oc * log2f(p.floor_hz * lag / p.sr_f);
                    }
                }
            }
            const unsigned bal = __ballot_sync(0xffffffffu, ok);
            if (ok) mine[np + __popc(bal & ((1u << lane) - 1u))] = make_float2(str, lag);
            np += __popc(bal);
        }
        __syncwarp();
        // the 14 strongest, ties to the smaller lag
        for (int r = 0; r < kMaxCand - 1 && r < np; ++r) {
            float bs = -INFINITY, bl = INFINITY;
            int bi = -1;
            for (int i = lane; i < np; i += 32) {
                const float2 q = mine[i];
                if (q.x != -INFINITY && (bi < 0 || beats(q.x, q.y, bs, bl))) bs = q.x, bl = q.y, bi = i;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float os = __shfl_xor_sync(0xffffffffu, bs, o), ol = __shfl_xor_sync(0xffffffffu, bl, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (oi >= 0 && (bi < 0 || beats(os, ol, bs, bl))) bs = os, bl = ol, bi = oi;
            }
            if (bi < 0) break;
            if (lane == 0) {
                out[nc] = make_float2(p.sr_f / bl, bs);
                mine[bi].x = -INFINITY;
            }
            ++nc;
            __syncwarp();
        }
    }
    if (lane == 0) {
        out[0] = make_float2(0.f, s_unv);
        count[fg] = nc;
    }
    for (int i = nc + lane; i < kMaxCand; i += 32)
        if (i >= 1) out[i] = make_float2(0.f, -INFINITY);
}

// ---- kernel 3: path search and placement --------------------------------------------------------------------------------------
__device__ __forceinline__ double trans_cost(float fp, float fc, const PitchParams &p) {
    const bool vp = fp > 0.f, vc = fc > 0.f;
    if (vp && vc) return p.c_oj * fabs(log2((double)fp / (double)fc));
    return vp != vc ? p.c_vu : 0.0;
}

__global__ void __launch_bounds__(128) pitch_path_kernel(const PitchClip *__restrict__ clips, const float2 *__restrict__ cand,
                                                         const int *__restrict__ count, unsigned char *__restrict__ bp, PitchParams p,
                                                         float *__restrict__ f0_out) {
    const int clip = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (clip >= p.n_clips) return;
    const PitchClip cl = clips[clip];
    const float2 *cd = cand + (long long)cl.frame_off * kMaxCand;
    const int *cnt = count + cl.frame_off;
    unsigned char *b = bp + (long long)cl.frame_off * 16;
    const int li = lane < 16 ? lane : 15;                          // lanes 16..31 mirror lane 15 (never valid)
    int kc = cnt[0];
    float f = li < kMaxCand ? cd[li].x : 0.f;
    double delta = (li < kc && lane < kMaxCand) ? (double)cd[li].y : -INFINITY;
    for (int j = 1; j < cl.n; ++j) {
        const int kp = kc;
        kc = cnt[j];
        const float2 me = cd[(long long)j * kMaxCand + (li < kMaxCand ? li : 0)];
        double best = -INFINITY;
        int arg = 0;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const double dk = __shfl_sync(0xffffffffu, delta, k);
            const float fk = __shfl_sync(0xffffffffu, f, k);
            if (k < kp) {
                const double sc = dk - trans_cost(fk, me.x, p);
                if (sc > best) best = sc, arg = k;
            }
        }
        const bool valid = lane < kMaxCand && li < kc;
        if (lane < 16) b[(long long)j * 16 + lane] = (unsigned char)arg;
        delta = valid ? best + (double)me.y : -INFINITY;
        f = me.x;
    }
    // the last frame's best candidate, ties to the lower index
    double bv = delta;
    int bi = lane < kMaxCand ? lane : 31;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) bv = ov, bi = oi;
    }
    float *out = f0_out + cl.out_off;
    const long long T = cl.T, lpad = p.lpad;
    const float last = cd[(long long)(cl.n - 1) * kMaxCand + bi].x;
    for (long long i = lane; i < T; i += 32) {
        if (i < lpad) out[i] = 0.f;
        else if (i >= lpad + cl.n) out[i] = last;                  // extended with the last value
    }
    if (lane == 0) {
        int k = bi;
        for (int j = cl.n - 1; j >= 0; --j) {
            if (lpad + j < T) out[lpad + j] = cd[(long long)j * kMaxCand + k].x;
            if (j > 0) k = b[(long long)j * 16 + k];
        }
    }
}

template <int R>
size_t cand_smem(int L, int hop) {
    return ((size_t)round_up(L + (kFPC - 1) * hop, 4) + (size_t)kFPC * round_up(L + 32 * R, 4) + (size_t)kFPC * 32 * R) * sizeof(float) +
           (size_t)kFPC * 16 * R * sizeof(float2);
}

template <int R>
int launch_cand(const float *wav, const PitchClip *clips, const float2 *stats, const float *win, const float *rwn, const PitchParams &p,
                int blocks, float2 *cand, int *count, float *r_out, cudaStream_t st) {
    const size_t smem = cand_smem<R>(p.L, p.hop);
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(pitch_cand_kernel<R>, smem, configured));
    pitch_cand_kernel<R><<<blocks, 32 * kFPC, smem, st>>>(wav, clips, stats, win, rwn, p, cand, count, r_out);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

struct StageTimer {
    cudaEvent_t ev[4] = {};
    bool on;
    explicit StageTimer(bool on_) : on(on_) {}
    ~StageTimer() {
        for (auto e : ev)
            if (e) cudaEventDestroy(e);
    }
    int create() {
        if (on)
            for (auto &e : ev) SVB_CUDA(cudaEventCreate(&e));
        return SVB_OK;
    }
    int mark(int k, cudaStream_t st) {
        if (on) SVB_CUDA(cudaEventRecord(ev[k], st));
        return SVB_OK;
    }
    int read(float *ms) {
        if (!on) return SVB_OK;
        SVB_CUDA(cudaEventSynchronize(ev[3]));
        for (int k = 0; k < 3; ++k) SVB_CUDA(cudaEventElapsedTime(ms + k, ev[k], ev[k + 1]));
        return SVB_OK;
    }
};

int run(const svb_pitch_config *cfg, const float *wav_dev, const int64_t *lengths, int32_t n_clips, const int64_t *mel_frames,
        float *f0_dev, void *ws, int64_t ws_bytes, float *cand_dev, int32_t *count_dev, float *r_dev, float *stage_ms, cudaStream_t st) {
    std::vector<PitchClip> clips;
    Layout lay;
    SVB_TRY(plan(cfg, lengths, mel_frames, n_clips, &clips, &lay));
    SVB_CHECK(wav_dev && mel_frames && f0_dev && ws, SVB_ERR_INVALID, "pitch_ac: null buffer");
    SVB_CHECK(ws_bytes >= (int64_t)lay.total, SVB_ERR_INVALID, "pitch_ac: workspace of %lld bytes, %zu needed", (long long)ws_bytes, lay.total);
    // host tables: the Hann window and the window's normalised autocorrelation, in double then rounded once
    const int L = lay.L, nlag = lay.tau_max + 2;
    std::vector<double> w(L);
    for (int k = 0; k < L; ++k) w[k] = 0.5 - 0.5 * std::cos(2.0 * M_PI * (k + 1) / (L + 1));
    std::vector<float> winf(L), rwn(nlag);
    for (int k = 0; k < L; ++k) winf[k] = (float)w[k];
    double rw0 = 0.0;
    for (int k = 0; k < L; ++k) rw0 += w[k] * w[k];
    for (int t = 0; t < nlag; ++t) {
        double s = 0.0;
        for (int k = 0; k + t < L; ++k) s += w[k] * w[k + t];
        rwn[t] = (float)(s / rw0);
    }
    char *base = static_cast<char *>(ws);
    PitchClip *d_clips = reinterpret_cast<PitchClip *>(base + lay.off_clip);
    float2 *d_stats = reinterpret_cast<float2 *>(base + lay.off_stats);
    float *d_win = reinterpret_cast<float *>(base + lay.off_win);
    float *d_rwn = reinterpret_cast<float *>(base + lay.off_rwn);
    float2 *d_cand = cand_dev ? reinterpret_cast<float2 *>(cand_dev) : reinterpret_cast<float2 *>(base + lay.off_cand);
    int *d_count = count_dev ? count_dev : reinterpret_cast<int *>(base + lay.off_count);
    unsigned char *d_bp = reinterpret_cast<unsigned char *>(base + lay.off_bp);
    SVB_CUDA(cudaMemcpyAsync(d_clips, clips.data(), clips.size() * sizeof(PitchClip), cudaMemcpyHostToDevice, st));
    SVB_CUDA(cudaMemcpyAsync(d_win, winf.data(), L * sizeof(float), cudaMemcpyHostToDevice, st));
    SVB_CUDA(cudaMemcpyAsync(d_rwn, rwn.data(), nlag * sizeof(float), cudaMemcpyHostToDevice, st));
    // the copies read pageable host vectors: finish them before the vectors go out of scope
    SVB_CUDA(cudaStreamSynchronize(st));

    PitchParams p;
    p.sr = cfg->sr, p.hop = cfg->hop, p.L = L, p.h = (L - 1) / 2, p.tau_max = lay.tau_max, p.nlag = nlag, p.lpad = cfg->lpad;
    p.n_clips = n_clips;
    p.sr_f = (float)cfg->sr, p.lag_min = (float)(cfg->sr / cfg->ceiling), p.lag_max = (float)(cfg->sr / cfg->floor);
    p.half_vt = (float)(0.5 * cfg->voicing_threshold), p.vt = (float)cfg->voicing_threshold, p.st = (float)cfg->silence_threshold;
    p.oc = (float)cfg->octave_cost, p.floor_hz = (float)cfg->floor;
    const double c = 0.01 / cfg->time_step;
    p.c_vu = cfg->voiced_unvoiced_cost * c, p.c_oj = cfg->octave_jump_cost * c;

    StageTimer tm(stage_ms != nullptr);
    SVB_TRY(tm.create());
    SVB_TRY(tm.mark(0, st));
    pitch_clip_stats_kernel<<<n_clips, 256, 0, st>>>(wav_dev, d_clips, d_stats);
    SVB_CUDA(cudaGetLastError());
    SVB_TRY(tm.mark(1, st));
    if (nlag <= 32 * 9)
        SVB_TRY(launch_cand<9>(wav_dev, d_clips, d_stats, d_win, d_rwn, p, lay.blocks, d_cand, d_count, r_dev, st));
    else
        SVB_TRY(launch_cand<kMaxR>(wav_dev, d_clips, d_stats, d_win, d_rwn, p, lay.blocks, d_cand, d_count, r_dev, st));
    SVB_TRY(tm.mark(2, st));
    pitch_path_kernel<<<(n_clips + 3) / 4, 128, 0, st>>>(d_clips, d_cand, d_count, d_bp, p, f0_dev);
    SVB_CUDA(cudaGetLastError());
    SVB_TRY(tm.mark(3, st));
    SVB_TRY(tm.read(stage_ms));
    return SVB_OK;
}

}  // namespace
}  // namespace svb

using namespace svb;

extern "C" int64_t svb_pitch_ac_workspace_bytes(const svb_pitch_config *cfg, const int64_t *lengths, int32_t n_clips, int32_t *frames_out) {
    std::vector<PitchClip> clips;
    Layout lay;
    if (plan(cfg, lengths, nullptr, n_clips, &clips, &lay) != SVB_OK) return -1;
    if (frames_out)
        for (int c = 0; c < n_clips; ++c) frames_out[c] = clips[c].n;
    return (int64_t)lay.total;
}

extern "C" int svb_pitch_ac_batch(const svb_pitch_config *cfg, const float *wav_concat_dev, const int64_t *lengths, int32_t n_clips,
                                  const int64_t *mel_frames, float *f0_out_dev, void *workspace_dev, int64_t workspace_bytes,
                                  float *cand_dev, int32_t *count_dev, float *r_dev, float *stage_ms_host, void *stream) {
    return run(cfg, wav_concat_dev, lengths, n_clips, mel_frames, f0_out_dev, workspace_dev, workspace_bytes, cand_dev, count_dev, r_dev,
               stage_ms_host, as_stream(stream));
}
