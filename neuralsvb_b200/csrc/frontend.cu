// Fused STFT front end: framing + padding + hann window + real FFT + magnitude + mel matmul + log,
// no cuFFT, no intermediate spectrogram in HBM.
//
// Forward (stft_mel_v2_kernel): kFPB = 4 consecutive frames of one clip per CTA.  A real frame of N samples is
// transformed as ONE N/2-point complex FFT of z[n] = x[2n] + i x[2n+1] plus a post-twiddle pass (half the
// butterflies of a complex N-point FFT on a zero imaginary part); twiddles, the hann window and the mel filters are
// staged once per CTA in shared memory; the mel filters come in a span-compressed form (mel_pack_kernel: first / last
// non-zero bin of every row + the values in between, ~2 values per frequency bin for triangular filters), so the
// projection walks only the non-zero span of each filter.  Clips of different lengths are served by one launch
// through a per-clip table (ragged batches of the binarizer, svb_wav2spec_batch).
// Backward / denoise keep the one-CTA-per-frame complex FFT below (they need the full inverse transform).
//
// Replaces (see include/svb_vocoder.h for the per-mode citations):
//   process_utterance            data_gen/tts/data_gen_utils.py:123-134   (librosa.stft, |.|, mel @, log10)
//   mel_spectrogram              modules/hifigan/mel_utils.py:59-76       (reflect pad, torch.stft, sqrt(.+1e-9), ln)
//   stft() of the STFT losses    modules/parallel_wavegan/losses/stft_loss.py:26-31
//
// The frame is loaded bit-reversed into shared memory, transformed by an in-place radix-2 DIT FFT
// with twiddles from sincospif (accurate to 1 ulp), and the n_fft/2+1 magnitudes stay in shared
// memory for the mel projection: each warp owns mel bins and walks only the non-zero span of the
// triangular filter.  HBM traffic = the waveform once (L2 absorbs the n_fft/hop overlap) + the
// output; the kernel is bandwidth/latency bound (about 18.6 MFLOP per 2 s clip).
#include <algorithm>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace svb {

struct StftArgs {
    const float *wav;        // [B, n]
    const float *mel_basis;  // [n_mels, n_bins] or nullptr
    float *out;
    long long n;
    int n_fft, log2n, hop, win, n_bins, n_mels;
    int frames;
    int pad_mode, out_kind, clamp_input, frames_major;
    float eps;
};

__device__ __forceinline__ long long reflect_index(long long i, long long n) {
    // numpy / torch 'reflect' (no edge repeat); valid for |overshoot| < n
    if (i < 0) i = -i;
    if (i >= n) i = 2 * (n - 1) - i;
    return i;
}

// radix-2 decimation-in-time on bit-reversed input, natural-order output; sign = +1: forward (e^{-i..}), -1: inverse
__device__ __forceinline__ void fft_radix2(float *re, float *im, const float *twc, const float *tws, int N, int log2n,
                                           float sign) {
    const int tid = threadIdx.x;
    for (int s = 1; s <= log2n; ++s) {
        const int half = 1 << (s - 1);
        const int tw_stride = N >> s;
        for (int i = tid; i < N / 2; i += 256) {
            const int grp = i / half, k = i - grp * half;
            const int i0 = grp * 2 * half + k, i1 = i0 + half;
            const float c = twc[k * tw_stride], sn = sign * tws[k * tw_stride];
            const float xr = re[i1], xi = im[i1];
            const float tr = xr * c - xi * sn, ti = xr * sn + xi * c;
            const float ur = re[i0], ui = im[i0];
            re[i0] = ur + tr, im[i0] = ui + ti;
            re[i1] = ur - tr, im[i1] = ui - ti;
        }
        __syncthreads();
    }
}

__device__ __forceinline__ long long frame_start(const StftArgs &a, int frame) {
    if (a.pad_mode == SVB_PAD_HALF_REFLECT) return (long long)frame * a.hop - (a.n_fft - a.hop) / 2;
    return (long long)frame * a.hop - a.n_fft / 2;
}

// windowed frame (bit-reversed) + twiddles into shared memory, then the forward FFT
__device__ __forceinline__ void load_frame_fft(const StftArgs &a, float *re, float *im, float *twc, float *tws, int frame, int b) {
    const int tid = threadIdx.x, N = a.n_fft;
    const float *w = a.wav + (size_t)b * a.n;
    const long long start = frame_start(a, frame);
    const int wl = (N - a.win) / 2;   // window is centred in the n_fft frame (librosa pad_center / torch.stft)

    for (int i = tid; i < N; i += 256) {
        float v = 0.f;
        const int wi = i - wl;
        if (wi >= 0 && wi < a.win) {
            long long s = start + i;
            bool ok = true;
            if (s < 0 || s >= a.n) {
                if (a.pad_mode == SVB_PAD_CENTER_ZERO) ok = false;
                else s = reflect_index(s, a.n);
            }
            if (ok) {
                float x = __ldg(w + s);
                if (a.clamp_input) x = fminf(fmaxf(x, -1.f), 1.f);
                const float hann = 0.5f - 0.5f * cospif(2.0f * (float)wi / (float)a.win);   // periodic hann
                v = x * hann;
            }
        }
        const int j = __brev((unsigned)i) >> (32 - a.log2n);
        re[j] = v;
        im[j] = 0.f;
    }
    for (int i = tid; i < N / 2; i += 256) {
        float s, c;
        sincospif(2.0f * (float)i / (float)N, &s, &c);
        twc[i] = c;
        tws[i] = -s;
    }
    __syncthreads();
    fft_radix2(re, im, twc, tws, N, a.log2n, 1.f);
}

// ---------------------------------------------------------------------------------------------------------------
// v2 forward: real FFT via a half-size complex FFT, kFPB frames per CTA, span-compressed mel filters, ragged batches
constexpr int kFPB = 4;

struct ClipTable {              // per clip c: first CTA, waveform offset / length, output frame offset / count
    const int *blk_off;         // [n_clips + 1]
    const long long *wav_off;   // [n_clips + 1] (element offsets into the concatenated waveforms)
    const long long *frm_off;   // [n_clips + 1] (frame offsets into the concatenated output)
};

struct MelPack {                // produced by mel_pack_kernel in the same stream
    const int *lo, *hi, *off;   // [n_mels]: span [lo, hi) of row m, its values at val[off[m] .. off[m] + hi - lo)
    const float *val;
    const int *total;           // [1]: number of packed values
};

// one block: row m -> [lo, hi), exclusive scan of the span lengths, packed values
__global__ void __launch_bounds__(256) mel_pack_kernel(const float *__restrict__ basis, int n_mels, int n_bins, int *lo, int *hi,
                                                       int *off, float *val, int *total) {
    __shared__ int s_len[1024];
    for (int m = threadIdx.x; m < n_mels; m += 256) {
        const float *row = basis + (size_t)m * n_bins;
        int a = n_bins, b = 0;
        for (int i = 0; i < n_bins; ++i)
            if (row[i] != 0.f) {
                a = min(a, i);
                b = i + 1;
            }
        if (b == 0) a = 0;
        lo[m] = a, hi[m] = b, s_len[m] = b - a;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int m = 0; m < n_mels; ++m) {
            off[m] = acc;
            acc += s_len[m];
        }
        *total = acc;
    }
    __syncthreads();
    for (int m = 0; m < n_mels; ++m) {
        const int a = lo[m], len = s_len[m], o = off[m];
        for (int i = threadIdx.x; i < len; i += 256) val[o + i] = basis[(size_t)m * n_bins + a + i];
    }
}

__global__ void __launch_bounds__(256) stft_mel_v2_kernel(StftArgs a, ClipTable ct, int n_clips, MelPack mp, int pack_cap) {
    extern __shared__ float smem[];
    const int N = a.n_fft, H = N / 2, tid = threadIdx.x;
    float *zr = smem;                       // [kFPB][H]
    float *zi = zr + kFPB * H;              // [kFPB][H]
    float *twc = zi + kFPB * H;             // [H]  cos(2 pi k / N)
    float *tws = twc + H;                   // [H]  sin(2 pi k / N)
    float *wnd = tws + H;                   // [win]
    float *mag = wnd + a.win;               // [kFPB][n_bins]
    float *pval = mag + kFPB * a.n_bins;    // [pack_cap] (mel outputs only)
    // ---- which clip / frames
    int clip = 0, blk_in_clip = blockIdx.x;
    long long n = a.n, wav_base = 0, out_frame0 = 0;
    int frames = a.frames;
    if (ct.blk_off) {
        int lo = 0, hi = n_clips - 1;                               // last clip with blk_off[c] <= blockIdx.x
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (ct.blk_off[mid] <= (int)blockIdx.x) lo = mid;
            else hi = mid - 1;
        }
        clip = lo, blk_in_clip = blockIdx.x - ct.blk_off[clip];
        wav_base = ct.wav_off[clip], n = ct.wav_off[clip + 1] - wav_base;
        out_frame0 = ct.frm_off[clip], frames = (int)(ct.frm_off[clip + 1] - out_frame0);
    } else {
        const int bpc = (a.frames + kFPB - 1) / kFPB;
        clip = blockIdx.x / bpc, blk_in_clip = blockIdx.x - clip * bpc;
        wav_base = (long long)clip * a.n, out_frame0 = (long long)clip * a.frames;
    }
    const int f0 = blk_in_clip * kFPB, nf = min(kFPB, frames - f0);
    const float *w = a.wav + wav_base;
    const bool want_mel = a.out_kind == SVB_OUT_LOG10_MEL || a.out_kind == SVB_OUT_LN_MEL || a.out_kind == SVB_OUT_MEL_MAG;

    // ---- tables: twiddles, window, packed mel filters
    for (int k = tid; k < H; k += 256) {
        float sn, cs;
        sincospif(2.0f * (float)k / (float)N, &sn, &cs);
        twc[k] = cs, tws[k] = sn;
    }
    for (int i = tid; i < a.win; i += 256) wnd[i] = 0.5f - 0.5f * cospif(2.0f * (float)i / (float)a.win);   // periodic hann
    int n_pack = 0;
    if (want_mel) {
        n_pack = *mp.total;
        if (n_pack <= pack_cap)
            for (int i = tid; i < n_pack; i += 256) pval[i] = mp.val[i];
    }
    __syncthreads();

    // ---- windowed frames -> z (bit-reversed over log2(H) bits)
    const int wl = (N - a.win) / 2, lh = a.log2n - 1;
    for (int i = tid; i < nf * H; i += 256) {
        const int f = i / H, j = i - f * H;
        long long start = (long long)(f0 + f) * a.hop - (a.pad_mode == SVB_PAD_HALF_REFLECT ? (N - a.hop) / 2 : N / 2);
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int idx = 2 * j + e, wi = idx - wl;
            float x = 0.f;
            if (wi >= 0 && wi < a.win) {
                long long s = start + idx;
                bool ok = true;
                if (s < 0 || s >= n) {
                    if (a.pad_mode == SVB_PAD_CENTER_ZERO) ok = false;
                    else s = reflect_index(s, n);
                }
                if (ok) {
                    x = __ldg(w + s);
                    if (a.clamp_input) x = fminf(fmaxf(x, -1.f), 1.f);
                    x *= wnd[wi];
                }
            }
            v[e] = x;
        }
        const int br = lh > 0 ? (int)(__brev((unsigned)j) >> (32 - lh)) : 0;
        zr[f * H + br] = v[0], zi[f * H + br] = v[1];
    }
    __syncthreads();
    // ---- N/2-point radix-2 DIT on all frames of the CTA
    for (int st = 1; st <= lh; ++st) {
        const int half = 1 << (st - 1), tw_stride = N >> st;          // e^{-2 pi i k / (2 half)} = table[k * N / (2 half)]
        for (int i = tid; i < nf * (H / 2); i += 256) {
            const int f = i / (H / 2), q = i - f * (H / 2);
            const int grp = q / half, k = q - grp * half;
            const int i0 = f * H + grp * 2 * half + k, i1 = i0 + half;
            const float c = twc[k * tw_stride], sn = -tws[k * tw_stride];
            const float xr = zr[i1], xi = zi[i1];
            const float tr = xr * c - xi * sn, ti = xr * sn + xi * c;
            const float ur = zr[i0], ui = zi[i0];
            zr[i0] = ur + tr, zi[i0] = ui + ti;
            zr[i1] = ur - tr, zi[i1] = ui - ti;
        }
        __syncthreads();
    }
    // ---- post-twiddle: X[k] = (A + B)/2 + w_k (A - B)/(2i),  A = Z[k], B = conj(Z[H - k]),  w_k = e^{-2 pi i k / N}
    for (int i = tid; i < nf * a.n_bins; i += 256) {
        const int f = i / a.n_bins, k = i - f * a.n_bins;
        const int ka = k == H ? 0 : k, kb = k == 0 ? 0 : H - k;
        const float ar = zr[f * H + ka], ai = zi[f * H + ka];
        const float br = zr[f * H + kb], bi = -zi[f * H + kb];
        const float er = 0.5f * (ar + br), ei = 0.5f * (ai + bi);     // even part
        const float dr = 0.5f * (ar - br), di = 0.5f * (ai - bi);
        const float orr = di, oi = -dr;                                // (A - B) / (2i) = -i (A - B) / 2
        const float c = k == H ? -1.f : twc[k], sn = k == H ? 0.f : -tws[k];
        const float re = er + orr * c - oi * sn, im = ei + orr * sn + oi * c;
        const float p = re * re + im * im;
        float m;
        if (a.out_kind == SVB_OUT_LN_MEL) m = sqrtf(p + 1e-9f);           // mel_utils.py:74
        else if (a.out_kind == SVB_OUT_MAG || a.out_kind == SVB_OUT_MEL_MAG) m = sqrtf(fmaxf(p, a.eps));   // stft_loss.py:31
        else m = sqrtf(p);                                                // np.abs, data_gen_utils.py:125
        if (want_mel) mag[i] = m;
        else {
            const long long fr = f0 + f;
            const size_t o = a.frames_major ? ((size_t)(out_frame0 + fr)) * a.n_bins + k
                                            : ((size_t)clip * a.n_bins + k) * a.frames + fr;
            a.out[o] = m;
        }
    }
    if (!want_mel) return;
    __syncthreads();
    // ---- mel projection over the non-zero span of each filter: one thread per (frame, mel)
    const float *pv = n_pack <= pack_cap ? pval : mp.val;
    for (int i = tid; i < nf * a.n_mels; i += 256) {
        const int f = i / a.n_mels, m = i - f * a.n_mels;
        const int lo = mp.lo[m], len = mp.hi[m] - lo, o0 = mp.off[m];
        const float *mg = mag + f * a.n_bins + lo;
        float acc = 0.f;
        for (int j = 0; j < len; ++j) acc = fmaf(pv[o0 + j], mg[j], acc);
        float v;
        if (a.out_kind == SVB_OUT_LOG10_MEL) v = log10f(fmaxf(a.eps, acc));   // data_gen_utils.py:134
        else if (a.out_kind == SVB_OUT_MEL_MAG) v = acc;                      // parallel_wavegan/stft_loss.py:46 (no log)
        else v = logf(fmaxf(acc, a.eps));                                     // mel_utils.py:23-24
        const long long fr = f0 + f;
        const size_t o = a.frames_major ? ((size_t)(out_frame0 + fr)) * a.n_mels + m
                                        : ((size_t)clip * a.n_mels + m) * a.frames + fr;
        a.out[o] = v;
    }
}

// Backward of stft_mel_kernel: one CTA per frame recomputes the frame's spectrum, pulls the output gradient back to
// (d re, d im) of the one-sided bins, runs the inverse (adjoint) FFT  g_n = Re sum_k (d re_k + i d im_k) e^{+2 pi i k n / N}
// and scatters window * g through the padding's adjoint into d wav (atomics: frames overlap).
struct StftBwdArgs {
    const float *dout;
    float *dwav;
};

__global__ void __launch_bounds__(256) stft_mel_bwd_kernel(StftArgs a, StftBwdArgs g) {
    extern __shared__ float smem[];
    float *re = smem;
    float *im = re + a.n_fft;
    float *twc = im + a.n_fft;
    float *tws = twc + a.n_fft / 2;
    float *mag = tws + a.n_fft / 2;   // [n_bins]: magnitudes, then d magnitude
    float *dmel = mag + a.n_bins;     // [n_mels]
    const int tid = threadIdx.x, N = a.n_fft;
    const int frame = blockIdx.x, b = blockIdx.y;
    load_frame_fft(a, re, im, twc, tws, frame, b);

    const bool want_mel = a.out_kind == SVB_OUT_LOG10_MEL || a.out_kind == SVB_OUT_LN_MEL || a.out_kind == SVB_OUT_MEL_MAG;
    constexpr int kMaxPer = 9;        // bins per thread for n_fft <= 4096
    float zr[kMaxPer], zi[kMaxPer];
    if (want_mel) {
        for (int i = tid; i < a.n_bins; i += 256) {
            const float p = re[i] * re[i] + im[i] * im[i];
            mag[i] = a.out_kind == SVB_OUT_LN_MEL ? sqrtf(p + 1e-9f) : (a.out_kind == SVB_OUT_MEL_MAG ? sqrtf(fmaxf(p, a.eps)) : sqrtf(p));
        }
        __syncthreads();
        const int lane = tid & 31, warp = tid >> 5;
        for (int m = warp; m < a.n_mels; m += 8) {
            const float *row = a.mel_basis + (size_t)m * a.n_bins;
            float acc = 0.f;
            for (int i = lane; i < a.n_bins; i += 32) acc = fmaf(__ldg(row + i), mag[i], acc);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0) {
                const size_t o = a.frames_major ? ((size_t)b * a.frames + frame) * a.n_mels + m
                                                : ((size_t)b * a.n_mels + m) * a.frames + frame;
                float d;
                if (a.out_kind == SVB_OUT_MEL_MAG) d = __ldg(g.dout + o);
                else d = acc >= a.eps ? __ldg(g.dout + o) / acc : 0.f;           // d log(max(mel, eps))
                if (a.out_kind == SVB_OUT_LOG10_MEL) d *= 0.4342944819032518f;
                dmel[m] = d;
            }
        }
        __syncthreads();
    }
    {
        int j = 0;
        for (int i = tid; i < a.n_bins; i += 256, ++j) {
            const float r = re[i], q = im[i];
            const float p = r * r + q * q;
            float dm, m;
            if (want_mel) {
                dm = 0.f;
                for (int k = 0; k < a.n_mels; ++k) dm = fmaf(__ldg(a.mel_basis + (size_t)k * a.n_bins + i), dmel[k], dm);
                m = mag[i];
                if (a.out_kind == SVB_OUT_MEL_MAG && p < a.eps) dm = 0.f;        // clamp(min) floor of the magnitude
            } else {
                const size_t o = a.frames_major ? ((size_t)b * a.frames + frame) * a.n_bins + i
                                                : ((size_t)b * a.n_bins + i) * a.frames + frame;
                dm = __ldg(g.dout + o);
                if (a.out_kind == SVB_OUT_MAG) {
                    m = sqrtf(fmaxf(p, a.eps));
                    if (p < a.eps) dm = 0.f;                                     // clamp(min): no gradient below the floor
                } else {
                    m = sqrtf(p);
                }
            }
            const float s = m > 0.f ? dm / m : 0.f;
            zr[j] = s * r, zi[j] = s * q;
        }
    }
    __syncthreads();
    for (int i = tid; i < N; i += 256) re[i] = 0.f, im[i] = 0.f;
    __syncthreads();
    {
        int j = 0;
        for (int i = tid; i < a.n_bins; i += 256, ++j) {
            const int br = __brev((unsigned)i) >> (32 - a.log2n);
            re[br] = zr[j], im[br] = zi[j];
        }
    }
    __syncthreads();
    fft_radix2(re, im, twc, tws, N, a.log2n, -1.f);

    const long long start = frame_start(a, frame);
    const int wl = (N - a.win) / 2;
    const float *w = a.wav + (size_t)b * a.n;
    float *dw = g.dwav + (size_t)b * a.n;
    for (int i = tid; i < N; i += 256) {
        const int wi = i - wl;
        if (wi < 0 || wi >= a.win) continue;
        long long s = start + i;
        if (s < 0 || s >= a.n) {
            if (a.pad_mode == SVB_PAD_CENTER_ZERO) continue;
            s = reflect_index(s, a.n);
        }
        if (a.clamp_input) {
            const float x = __ldg(w + s);
            if (x < -1.f || x > 1.f) continue;
        }
        const float hann = 0.5f - 0.5f * cospif(2.0f * (float)wi / (float)a.win);
        atomicAdd(dw + s, hann * re[i]);
    }
}

// Spectral-subtraction post-filter (vocoders/vocoder_utils.py:7-15): per frame STFT -> |X| - v clipped at 0, phase kept
// -> inverse real FFT -> window -> overlap-add; a second kernel divides by the window sum-square (librosa.istft) and
// trims the centre padding.
__global__ void __launch_bounds__(256) denoise_frames_kernel(StftArgs a, float v, float *__restrict__ acc, long long out_len) {
    extern __shared__ float smem[];
    float *re = smem;
    float *im = re + a.n_fft;
    float *twc = im + a.n_fft;
    float *tws = twc + a.n_fft / 2;
    __shared__ float edge[2];         // Re Z_0, Re Z_{N/2}
    const int tid = threadIdx.x, N = a.n_fft;
    const int frame = blockIdx.x, b = blockIdx.y;
    load_frame_fft(a, re, im, twc, tws, frame, b);
    constexpr int kMaxPer = 9;
    float zr[kMaxPer], zi[kMaxPer];
    {
        int j = 0;
        for (int i = tid; i < a.n_bins; i += 256, ++j) {
            const float r = re[i], q = im[i];
            const float m = sqrtf(r * r + q * q);
            const float sc = m > 0.f ? fmaxf(m - v, 0.f) / m : 0.f;
            zr[j] = sc * r, zi[j] = sc * q;
            if (i == 0) edge[0] = zr[j];
            if (i == N / 2) edge[1] = zr[j];
        }
    }
    __syncthreads();
    for (int i = tid; i < N; i += 256) re[i] = 0.f, im[i] = 0.f;
    __syncthreads();
    {
        int j = 0;
        for (int i = tid; i < a.n_bins; i += 256, ++j) {
            const int br = __brev((unsigned)i) >> (32 - a.log2n);
            re[br] = zr[j], im[br] = zi[j];
        }
    }
    __syncthreads();
    fft_radix2(re, im, twc, tws, N, a.log2n, -1.f);
    // irfft_n = (2 Re sum_{k<=N/2} Z_k e^{+i..} - Re Z_0 - (-1)^n Re Z_{N/2}) / N
    const int wl = (N - a.win) / 2;
    const long long start = (long long)frame * a.hop - N / 2;
    float *out = acc + (size_t)b * out_len;
    for (int i = tid; i < N; i += 256) {
        const int wi = i - wl;
        if (wi < 0 || wi >= a.win) continue;
        const long long s = start + i;
        if (s < 0 || s >= out_len) continue;
        const float x = (2.f * re[i] - edge[0] - ((i & 1) ? -edge[1] : edge[1])) / (float)N;
        const float hann = 0.5f - 0.5f * cospif(2.0f * (float)wi / (float)a.win);
        atomicAdd(out + s, hann * x);
    }
}

__global__ void denoise_norm_kernel(float *__restrict__ y, long long out_len, int B, int N, int hop, int win, int frames) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * out_len) return;
    const long long s = i % out_len;
    const int wl = (N - win) / 2;
    // frames f with 0 <= s + N/2 - f*hop < N
    const long long p = s + N / 2;
    long long f_hi = p / hop, f_lo = (p - N + hop) / hop;       // ceil((p - N + 1) / hop)
    if (p - N + 1 <= 0) f_lo = 0;
    if (f_hi > frames - 1) f_hi = frames - 1;
    float wss = 0.f;
    for (long long f = f_lo; f <= f_hi; ++f) {
        const int wi = (int)(p - f * hop) - wl;
        if (wi < 0 || wi >= win) continue;
        const float h = 0.5f - 0.5f * cospif(2.0f * (float)wi / (float)win);
        wss += h * h;
    }
    if (wss > 1.1754944e-38f) y[i] /= wss;
}

static int ilog2(int n) {
    int l = 0;
    while ((1 << l) < n) ++l;
    return l;
}

}  // namespace svb

using namespace svb;

extern "C" int64_t svb_stft_num_frames(const svb_stft_config *cfg, int64_t n) {
    if (!cfg || cfg->hop <= 0) return SVB_ERR_INVALID;
    if (cfg->pad_mode == SVB_PAD_HALF_REFLECT) {
        const int64_t padded = n + 2 * (int64_t)((cfg->n_fft - cfg->hop) / 2);
        return padded < cfg->n_fft ? 0 : 1 + (padded - cfg->n_fft) / cfg->hop;
    }
    return 1 + n / cfg->hop;
}

static int validate_stft(const svb_stft_config *cfg, int64_t n, bool need_mel) {
    SVB_CHECK(cfg != nullptr, SVB_ERR_INVALID, "stft: null config");
    SVB_CHECK(cfg->n_fft >= 64 && cfg->n_fft <= 4096 && (cfg->n_fft & (cfg->n_fft - 1)) == 0, SVB_ERR_INVALID,
              "stft: n_fft %d must be a power of two in [64, 4096]", cfg->n_fft);
    SVB_CHECK(cfg->hop > 0 && cfg->win > 0 && cfg->win <= cfg->n_fft, SVB_ERR_INVALID,
              "stft: bad hop %d / win %d", cfg->hop, cfg->win);
    SVB_CHECK(cfg->pad_mode >= 0 && cfg->pad_mode <= 2 && cfg->out_kind >= 0 && cfg->out_kind <= 4, SVB_ERR_INVALID,
              "stft: bad pad_mode / out_kind");
    SVB_CHECK(n >= 1, SVB_ERR_INVALID, "stft: empty waveform");
    if (cfg->pad_mode != SVB_PAD_CENTER_ZERO) {
        const int64_t reach = cfg->pad_mode == SVB_PAD_HALF_REFLECT ? (cfg->n_fft - cfg->hop) / 2 : cfg->n_fft / 2;
        SVB_CHECK(reach < n, SVB_ERR_INVALID, "stft: reflect padding %lld needs a longer signal than %lld",
                  (long long)reach, (long long)n);   // same condition torch's reflect pad enforces
    }
    if (need_mel) SVB_CHECK(cfg->n_mels > 0, SVB_ERR_INVALID, "stft: n_mels must be positive for mel outputs");
    return SVB_OK;
}

namespace {

int fill_args(const svb_stft_config *cfg, const float *wav_dev, const float *mel_basis_dev, float *out_dev, int64_t n, StftArgs *a) {
    a->wav = wav_dev, a->mel_basis = mel_basis_dev, a->out = out_dev, a->n = n;
    a->n_fft = cfg->n_fft, a->log2n = ilog2(cfg->n_fft), a->hop = cfg->hop, a->win = cfg->win;
    a->n_bins = cfg->n_fft / 2 + 1, a->n_mels = cfg->n_mels;
    a->frames = (int)svb_stft_num_frames(cfg, n);
    a->pad_mode = cfg->pad_mode, a->out_kind = cfg->out_kind, a->clamp_input = cfg->clamp_input;
    a->frames_major = cfg->frames_major, a->eps = cfg->eps;
    return SVB_OK;
}

// launch of the v2 forward: `ct` = per-clip table on the device (nullptr members: B equal-length clips); `pack_ws` = caller-owned
// room for the packed mel filters (mel_pack_bytes), nullptr: allocated on the stream
size_t mel_pack_bytes(int n_mels, int n_bins) { return ((size_t)3 * n_mels + 4) * sizeof(int) + (size_t)n_mels * n_bins * sizeof(float); }

int launch_stft_v2(const StftArgs &a, bool want_mel, const ClipTable &ct, int n_clips, int total_blocks, cudaStream_t st,
                   char *pack_ws = nullptr) {
    MelPack mp = {};
    char *ws = nullptr;
    int pack_cap = 0;
    if (want_mel) {
        SVB_CHECK(a.n_mels <= 1024, SVB_ERR_INVALID, "stft: n_mels %d > 1024", a.n_mels);
        const size_t n_val = (size_t)a.n_mels * a.n_bins;
        const size_t ints = (size_t)3 * a.n_mels + 4;
        if (!pack_ws) SVB_CUDA(cudaMallocAsync((void **)&ws, mel_pack_bytes(a.n_mels, a.n_bins), st));
        char *p = pack_ws ? pack_ws : ws;
        int *ip = reinterpret_cast<int *>(p);
        mp.lo = ip, mp.hi = ip + a.n_mels, mp.off = ip + 2 * a.n_mels, mp.total = ip + 3 * a.n_mels;
        float *val = reinterpret_cast<float *>(p + ints * sizeof(int));
        mp.val = val;
        mel_pack_kernel<<<1, 256, 0, st>>>(a.mel_basis, a.n_mels, a.n_bins, ip, ip + a.n_mels, ip + 2 * a.n_mels, val, ip + 3 * a.n_mels);
        pack_cap = (int)std::min<size_t>(n_val, 4096);
    }
    const size_t smem = ((size_t)2 * kFPB * (a.n_fft / 2) + a.n_fft + a.win + (size_t)kFPB * a.n_bins + pack_cap) * sizeof(float);
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(stft_mel_v2_kernel, smem, configured));
    stft_mel_v2_kernel<<<total_blocks, 256, smem, st>>>(a, ct, n_clips, mp, pack_cap);
    SVB_CUDA(cudaGetLastError());
    if (ws) SVB_CUDA(cudaFreeAsync(ws, st));
    return SVB_OK;
}

}  // namespace

extern "C" int svb_stft_forward(const svb_stft_config *cfg, const float *wav_dev, int32_t B, int64_t n,
                                const float *mel_basis_dev, float *out_dev, void *stream) {
    const bool want_mel = cfg && (cfg->out_kind == SVB_OUT_LOG10_MEL || cfg->out_kind == SVB_OUT_LN_MEL || cfg->out_kind == SVB_OUT_MEL_MAG);
    SVB_TRY(validate_stft(cfg, n, want_mel));
    SVB_CHECK(wav_dev && out_dev && B > 0, SVB_ERR_INVALID, "stft: null buffer or empty batch");
    SVB_CHECK(!want_mel || mel_basis_dev, SVB_ERR_INVALID, "stft: mel output needs mel_basis_dev");
    StftArgs a;
    SVB_TRY(fill_args(cfg, wav_dev, mel_basis_dev, out_dev, n, &a));
    if (a.frames <= 0) return SVB_OK;
    const int bpc = (a.frames + kFPB - 1) / kFPB;
    return launch_stft_v2(a, want_mel, ClipTable{nullptr, nullptr, nullptr}, B, B * bpc, as_stream(stream));
}

// The ragged batch of wav2spec: per clip c, the first CTA, the waveform offset and the output frame offset (1 + lengths[c] / hop
// frames each, the centre-zero-padded STFT of data_gen_utils.process_utterance).  Checks every clip; frames_out (nullable) receives
// the frame counts.
struct Wav2SpecPlan {
    std::vector<long long> wav_off, frm_off;
    std::vector<int> blk_off;
    size_t tab_bytes, pack_off, total;
};

static int plan_wav2spec(const svb_stft_config *cfg, const int64_t *lengths, int32_t n_clips, int64_t *frames_out, Wav2SpecPlan *p) {
    SVB_CHECK(cfg && lengths && n_clips > 0, SVB_ERR_INVALID, "wav2spec: null config / lengths or no clips");
    p->wav_off.assign(n_clips + 1, 0), p->frm_off.assign(n_clips + 1, 0), p->blk_off.assign(n_clips + 1, 0);
    for (int c = 0; c < n_clips; ++c) {
        SVB_TRY(validate_stft(cfg, lengths[c], true));
        const int64_t fr = svb_stft_num_frames(cfg, lengths[c]);
        p->wav_off[c + 1] = p->wav_off[c] + lengths[c];
        p->frm_off[c + 1] = p->frm_off[c] + fr;
        p->blk_off[c + 1] = p->blk_off[c] + (int)((fr + kFPB - 1) / kFPB);
        if (frames_out) frames_out[c] = fr;
    }
    SVB_CHECK(cfg->n_mels <= 1024, SVB_ERR_INVALID, "stft: n_mels %d > 1024", cfg->n_mels);
    p->tab_bytes = (size_t)(n_clips + 1) * (2 * sizeof(long long) + sizeof(int));
    p->pack_off = (p->tab_bytes + 255) / 256 * 256;
    p->total = p->pack_off + mel_pack_bytes(cfg->n_mels, cfg->n_fft / 2 + 1);
    return SVB_OK;
}

// every clip's waveform zero-padded (or cut) to frames * hop samples, back to back (audio.librosa_pad_lr + wav[:T * hop])
__global__ void pad_to_frames_kernel(const float *__restrict__ wav, const long long *__restrict__ wav_off,
                                     const long long *__restrict__ frm_off, int hop, float *__restrict__ out) {
    const int c = blockIdx.y;
    const long long w0 = wav_off[c], n = wav_off[c + 1] - w0;
    const long long o0 = frm_off[c] * hop, m = (frm_off[c + 1] - frm_off[c]) * hop;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x)
        out[o0 + i] = i < n ? wav[w0 + i] : 0.f;
}

extern "C" int64_t svb_wav2spec_workspace_bytes(const svb_stft_config *cfg, const int64_t *lengths, int32_t n_clips, int64_t *frames_out) {
    Wav2SpecPlan p;
    SVB_TRY(plan_wav2spec(cfg, lengths, n_clips, frames_out, &p));
    return (int64_t)p.total;
}

extern "C" int64_t svb_wav2spec_batch(const svb_stft_config *cfg, const float *wav_concat_dev, const int64_t *lengths, int32_t n_clips,
                                      const float *mel_basis_dev, float *mel_concat_dev, float *wav_out_dev, int64_t *frames_out,
                                      void *workspace_dev, int64_t workspace_bytes, void *stream) {
    Wav2SpecPlan p;
    SVB_TRY(plan_wav2spec(cfg, lengths, n_clips, frames_out, &p));
    SVB_CHECK(wav_concat_dev && mel_basis_dev && mel_concat_dev && workspace_dev, SVB_ERR_INVALID, "wav2spec: null buffer");
    SVB_CHECK(workspace_bytes >= (int64_t)p.total, SVB_ERR_INVALID, "wav2spec: workspace of %lld bytes, %lld needed",
              (long long)workspace_bytes, (long long)p.total);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace_dev);
    std::vector<char> tab(p.tab_bytes);
    memcpy(tab.data(), p.wav_off.data(), (n_clips + 1) * sizeof(long long));
    memcpy(tab.data() + (n_clips + 1) * sizeof(long long), p.frm_off.data(), (n_clips + 1) * sizeof(long long));
    memcpy(tab.data() + 2 * (n_clips + 1) * sizeof(long long), p.blk_off.data(), (n_clips + 1) * sizeof(int));
    SVB_CUDA(cudaMemcpyAsync(ws, tab.data(), p.tab_bytes, cudaMemcpyHostToDevice, st));
    svb_stft_config c = *cfg;
    c.frames_major = 1;
    StftArgs a;
    SVB_TRY(fill_args(&c, wav_concat_dev, mel_basis_dev, mel_concat_dev, lengths[0], &a));
    ClipTable ct;
    ct.wav_off = reinterpret_cast<const long long *>(ws);
    ct.frm_off = ct.wav_off + (n_clips + 1);
    ct.blk_off = reinterpret_cast<const int *>(ws + 2 * (n_clips + 1) * sizeof(long long));
    SVB_TRY(launch_stft_v2(a, true, ct, n_clips, p.blk_off[n_clips], st, ws + p.pack_off));
    if (wav_out_dev) {
        long long longest = 0;
        for (int k = 0; k < n_clips; ++k) longest = std::max(longest, (p.frm_off[k + 1] - p.frm_off[k]) * cfg->hop);
        const dim3 grid((unsigned)std::min<long long>((longest + 255) / 256, 132 * 4), (unsigned)n_clips);
        pad_to_frames_kernel<<<grid, 256, 0, st>>>(wav_concat_dev, ct.wav_off, ct.frm_off, cfg->hop, wav_out_dev);
        SVB_CUDA(cudaGetLastError());
    }
    return (int64_t)p.frm_off[n_clips];
}

extern "C" int svb_stft_backward(const svb_stft_config *cfg, const float *wav_dev, int32_t B, int64_t n,
                                 const float *mel_basis_dev, const float *dout_dev, float *dwav_dev, void *stream) {
    const bool want_mel = cfg && (cfg->out_kind == SVB_OUT_LOG10_MEL || cfg->out_kind == SVB_OUT_LN_MEL || cfg->out_kind == SVB_OUT_MEL_MAG);
    SVB_TRY(validate_stft(cfg, n, want_mel));
    SVB_CHECK(wav_dev && dout_dev && dwav_dev && B > 0, SVB_ERR_INVALID, "stft_backward: null buffer or empty batch");
    SVB_CHECK(!want_mel || mel_basis_dev, SVB_ERR_INVALID, "stft_backward: mel output needs mel_basis_dev");
    StftArgs a;
    a.wav = wav_dev, a.mel_basis = mel_basis_dev, a.out = nullptr, a.n = n;
    a.n_fft = cfg->n_fft, a.log2n = ilog2(cfg->n_fft), a.hop = cfg->hop, a.win = cfg->win;
    a.n_bins = cfg->n_fft / 2 + 1, a.n_mels = cfg->n_mels;
    a.frames = (int)svb_stft_num_frames(cfg, n);
    a.pad_mode = cfg->pad_mode, a.out_kind = cfg->out_kind, a.clamp_input = cfg->clamp_input;
    a.frames_major = cfg->frames_major, a.eps = cfg->eps;
    if (a.frames <= 0) return SVB_OK;
    StftBwdArgs g;
    g.dout = dout_dev, g.dwav = dwav_dev;
    const size_t smem = (size_t)(3 * a.n_fft + a.n_bins + (want_mel ? a.n_mels : 0)) * sizeof(float);
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(stft_mel_bwd_kernel, smem, configured));
    stft_mel_bwd_kernel<<<dim3(a.frames, B), 256, smem, as_stream(stream)>>>(a, g);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_denoise(const svb_stft_config *cfg, const float *wav_dev, int32_t B, int64_t n, float v, float *out_dev,
                           void *stream) {
    svb_stft_config c;
    SVB_CHECK(cfg && wav_dev && out_dev && B > 0 && v >= 0.f, SVB_ERR_INVALID, "denoise: bad argument");
    c = *cfg;
    c.pad_mode = SVB_PAD_CENTER_ZERO, c.out_kind = SVB_OUT_MAG_RAW, c.clamp_input = 0;
    SVB_TRY(validate_stft(&c, n, false));
    StftArgs a;
    a.wav = wav_dev, a.mel_basis = nullptr, a.out = nullptr, a.n = n;
    a.n_fft = c.n_fft, a.log2n = ilog2(c.n_fft), a.hop = c.hop, a.win = c.win;
    a.n_bins = c.n_fft / 2 + 1, a.n_mels = 0;
    a.frames = (int)svb_stft_num_frames(&c, n);
    a.pad_mode = c.pad_mode, a.out_kind = c.out_kind, a.clamp_input = 0, a.frames_major = 1, a.eps = 0.f;
    const long long out_len = (long long)c.hop * (a.frames - 1);      // librosa.istft length (centre padding trimmed)
    SVB_CHECK(out_len > 0, SVB_ERR_INVALID, "denoise: signal shorter than one hop");
    cudaStream_t st = as_stream(stream);
    SVB_CUDA(cudaMemsetAsync(out_dev, 0, (size_t)B * out_len * sizeof(float), st));
    const size_t smem = (size_t)(3 * a.n_fft) * sizeof(float);
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(denoise_frames_kernel, smem, configured));
    denoise_frames_kernel<<<dim3(a.frames, B), 256, smem, st>>>(a, v, out_dev, out_len);
    const long long tot = (long long)B * out_len;
    denoise_norm_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(out_dev, out_len, B, c.n_fft, c.hop, c.win, a.frames);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}
