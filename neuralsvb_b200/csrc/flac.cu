// FLAC decoding (RFC 9639) over a ragged batch of streams: what librosa.core.load does to a .flac take through libsndfile, with
// oracle/flac.py as the reference.  The host parses the metadata (utils/audio.flac_info) and hands over, per stream, its bytes (the
// whole file), the offset of its first frame and the STREAMINFO fields.  Seven launches:
//
//   1. flac_scan_kernel      one thread per 16 bytes: flag every offset holding a frame header (sync code, codes, UTF-8 number,
//                            CRC-8) inside a stream's frame region; per-4096-byte chunk counts.
//   2. flac_chunk_scan       one CTA: exclusive prefix of the chunk counts.
//   3. flac_compact_kernel   the flagged offsets in order: the candidate list, grouped by stream.
//   4. flac_span_crc_kernel  one warp per candidate: CRC-16 of the bytes up to the next candidate (lanes combine their slices
//                            through x^(8n) mod P; the CRC is linear with zero init and no final xor).
//   5. flac_walk_kernel      one thread per stream: the frame chain.  A candidate becomes a frame only when the CRC-16 of the span to
//                            the next accepted frame checks out and its number continues the chain; spans of rejected candidates
//                            (sync patterns inside coded data) are merged.  The chain must match STREAMINFO and its total.
//   6. flac_bounds_kernel    one thread per frame: skims the subframes (Rice runs by count of leading zeros) to find where each
//                            channel starts, and checks that the frame's bits end where its CRC-16 starts.
//   7. flac_subframe_kernel  one thread per (frame, channel): decodes the subframe to int32 (LPC / FIXED restoration is the serial
//                            recurrence of the subframe); flac_output_kernel then undoes the stereo decorrelation and writes float32
//                            mono as utils.audio.read_wav converts a WAV of the same PCM.
//
// Every read is bounded by the frame's extent, so a damaged stream ends in an error naming the stream and byte offset, never in a
// read past the buffer.  Errors are collected per stream on the device (the earliest offset wins) and read back once at the end.
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace svb {
namespace {

constexpr int kChunk = 4096;      // bytes per scan CTA (256 threads x 16)
constexpr int kMaxLpc = 32;
constexpr int kSubThreads = 64;

enum FlacErr : unsigned { E_NONE = 0, E_START, E_CHAIN, E_CRC, E_SHORT, E_FRAMES, E_SUBFRAME, E_LENGTH, E_TRAIL };

struct FStream {
    long long base, first, end;   // global byte offsets: the stream's first byte, its first frame, one past its last byte
    long long out_off, pcm_off;   // first output sample, first int32 of its channel-planar PCM
    long long total;              // samples per channel
    long long frame_base, frame_cap;
    int sr, ch, bits, pad;
};

struct FFrame {
    long long start;              // global byte offset of the header
    long long first;              // first sample within the stream
    int bytes;                    // header .. CRC-16 inclusive
    int bs, stream, assign;       // assign: 0-7 independent, 8 left/side, 9 side/right, 10 mid/side
    int hdr;                      // header bytes
    unsigned sub[8];              // bit offset of each subframe from the frame's start
};

struct FHeader {
    int ok, variable, bs, sr, ch_code, bits, hdr;
    unsigned long long number;
};

struct Layout {
    std::vector<FStream> st;
    long long bytes, samples, pcm, frames;
    int chunks;
    size_t off_st, off_flag, off_cnt, off_cand, off_crc, off_frame, off_nf, off_err, off_pcm, total;
};

size_t align_up(size_t x) { return (x + 255) / 256 * 256; }

int plan(int32_t n, const int64_t *nbytes, const int64_t *first, const int32_t *sr, const int32_t *ch, const int32_t *bits,
         const int64_t *total, Layout *lay) {
    SVB_CHECK(n > 0 && nbytes && first && sr && ch && bits && total, SVB_ERR_INVALID, "flac: null stream arrays, or no streams");
    lay->st.resize(n);
    long long b = 0, o = 0, p = 0, f = 0;
    for (int s = 0; s < n; ++s) {
        SVB_CHECK(bits[s] >= 4 && bits[s] <= 24, SVB_ERR_INVALID, "flac: stream %d: %d bits per sample (4 to 24 are decoded)", s, bits[s]);
        SVB_CHECK(total[s] > 0, SVB_ERR_INVALID, "flac: stream %d: STREAMINFO gives no total sample count (0 = unknown)", s);
        SVB_CHECK(ch[s] >= 1 && ch[s] <= 8, SVB_ERR_INVALID, "flac: stream %d: %d channels (at most 8)", s, ch[s]);
        SVB_CHECK(sr[s] > 0, SVB_ERR_INVALID, "flac: stream %d: sample rate %d", s, sr[s]);
        SVB_CHECK(nbytes[s] > 0 && first[s] >= 0 && first[s] <= nbytes[s], SVB_ERR_INVALID,
                  "flac: stream %d: first frame at byte %lld of %lld", s, (long long)first[s], (long long)nbytes[s]);
        SVB_CHECK(total[s] < (1LL << 31), SVB_ERR_INVALID, "flac: stream %d: %lld samples (under 2^31 are decoded)", s, (long long)total[s]);
        FStream S{};
        S.base = b, S.first = b + first[s], S.end = b + nbytes[s];
        S.out_off = o, S.pcm_off = p, S.total = total[s];
        S.frame_base = f, S.frame_cap = std::min<long long>(total[s], (nbytes[s] - first[s]) / 9 + 1);
        S.sr = sr[s], S.ch = ch[s], S.bits = bits[s];
        lay->st[s] = S;
        b += nbytes[s], o += total[s], p += total[s] * ch[s], f += S.frame_cap;
    }
    SVB_CHECK(b < (1LL << 31), SVB_ERR_INVALID, "flac: %lld bytes are too many for one call (under 2 GiB)", b);
    lay->bytes = b, lay->samples = o, lay->pcm = p, lay->frames = f;
    lay->chunks = (int)((b + kChunk - 1) / kChunk);
    const long long cap = b / 2 + 1;    // two candidates are never adjacent: byte 1 of a sync code is not 0xFF
    lay->off_st = 0;
    lay->off_flag = align_up(n * sizeof(FStream));
    lay->off_cnt = lay->off_flag + align_up(b);
    lay->off_cand = lay->off_cnt + align_up((lay->chunks + 1) * sizeof(int));
    lay->off_crc = lay->off_cand + align_up(cap * sizeof(unsigned));
    lay->off_frame = lay->off_crc + align_up(cap * sizeof(unsigned short));
    lay->off_nf = lay->off_frame + align_up(f * sizeof(FFrame));
    lay->off_err = lay->off_nf + align_up(n * sizeof(long long));
    lay->off_pcm = lay->off_err + align_up(n * sizeof(unsigned long long));
    lay->total = lay->off_pcm + align_up(p * sizeof(int));
    return SVB_OK;
}

// ---- CRCs ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned crc8_byte(unsigned c, unsigned b) {
    c ^= b;
#pragma unroll
    for (int i = 0; i < 8; ++i) c = (c & 0x80) ? ((c << 1) ^ 0x07) & 0xFF : (c << 1) & 0xFF;
    return c;
}

// a(x) b(x) mod P(x), P = x^16 + x^15 + x^2 + 1 (0x8005)
__device__ unsigned gf_mul(unsigned a, unsigned b) {
    unsigned r = 0;
    for (int i = 15; i >= 0; --i) {
        r = (r & 0x8000) ? ((r << 1) ^ 0x8005) & 0xFFFF : (r << 1) & 0xFFFF;
        if ((b >> i) & 1) r ^= a;
    }
    return r;
}

// x^(8 n) mod P: what appending n bytes does to a CRC register
__device__ unsigned gf_xpow8(unsigned long long n) {
    unsigned r = 1, base = 0x100;       // x^8
    while (n) {
        if (n & 1) r = gf_mul(r, base);
        base = gf_mul(base, base);
        n >>= 1;
    }
    return r;
}

__constant__ int kRates[12] = {0, 88200, 176400, 192000, 8000, 16000, 22050, 24000, 32000, 44100, 48000, 96000};
__constant__ int kSizes[8] = {0, 8, 12, 0, 16, 20, 24, 32};

// ---- frame header ----------------------------------------------------------------------------------------------------------
__device__ FHeader parse_header(const unsigned char *d, long long off, long long end) {
    FHeader h{};
    if (off + 6 > end || d[off] != 0xFF || (d[off + 1] & 0xFE) != 0xF8) return h;
    const unsigned b2 = d[off + 2], b3 = d[off + 3];
    const int bs_code = b2 >> 4, sr_code = b2 & 15, ch_code = b3 >> 4, ss = (b3 >> 1) & 7;
    if (bs_code == 0 || sr_code == 15 || ch_code > 10 || ss == 3 || (b3 & 1)) return h;
    h.variable = d[off + 1] & 1;
    long long p = off + 4;
    unsigned b = d[p];
    int extra;
    unsigned long long num;
    if (b < 0x80) extra = 0, num = b;
    else if (b >= 0xC0 && b < 0xFE) {
        extra = 1;
        while (b & (0x40u >> extra)) ++extra;
        num = b & (0x3Fu >> extra);
    } else return h;
    if (extra > (h.variable ? 6 : 5) || p + 1 + extra > end) return h;
    for (int i = 0; i < extra; ++i) {
        const unsigned c = d[p + 1 + i];
        if ((c & 0xC0) != 0x80) return h;
        num = (num << 6) | (c & 0x3F);
    }
    p += 1 + extra;
    int bs;
    if (bs_code == 6 || bs_code == 7) {
        const int nb = bs_code - 5;
        if (p + nb > end) return h;
        bs = (nb == 1 ? d[p] : (d[p] << 8) | d[p + 1]) + 1, p += nb;
    } else bs = bs_code == 1 ? 192 : bs_code <= 5 ? 576 << (bs_code - 2) : 256 << (bs_code - 8);
    int rate;
    if (sr_code >= 12) {
        const int nb = sr_code == 12 ? 1 : 2;
        if (p + nb > end) return h;
        const int v = nb == 1 ? d[p] : (d[p] << 8) | d[p + 1];
        p += nb;
        rate = sr_code == 12 ? v * 1000 : sr_code == 13 ? v : v * 10;
    } else rate = kRates[sr_code];
    if (p + 1 > end) return h;
    unsigned c = 0;
    for (long long q = off; q < p; ++q) c = crc8_byte(c, d[q]);
    if (c != d[p]) return h;
    h.ok = 1, h.bs = bs, h.sr = rate, h.ch_code = ch_code, h.bits = kSizes[ss], h.hdr = (int)(p + 1 - off), h.number = num;
    return h;
}

__device__ __forceinline__ int find_stream(const FStream *st, int n, long long byte) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (st[mid].base <= byte) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ void report(unsigned long long *err, int s, const FStream &S, long long at, unsigned code) {
    atomicMin(err + s, ((unsigned long long)(at - S.base) << 8) | code);
}

// ---- 1-3: candidates -------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) flac_scan_kernel(const unsigned char *__restrict__ d, const FStream *__restrict__ st, int n,
                                                       long long bytes, unsigned char *__restrict__ flag, int *__restrict__ counts) {
    const long long b0 = (long long)blockIdx.x * kChunk + threadIdx.x * 16;
    int cnt = 0;
    for (int i = 0; i < 16; ++i) {
        const long long b = b0 + i;
        if (b >= bytes) break;
        unsigned char f = 0;
        if (d[b] == 0xFF) {
            const FStream &S = st[find_stream(st, n, b)];
            f = b >= S.first && parse_header(d, b, S.end).ok;
        }
        flag[b] = f, cnt += f;
    }
    __shared__ int red[256];
    red[threadIdx.x] = cnt;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) counts[blockIdx.x] = red[0];
}

__global__ void __launch_bounds__(1024) flac_chunk_scan(int *__restrict__ counts, int chunks) {
    __shared__ int part[1024];
    const int per = (chunks + 1023) / 1024, lo = min(chunks, (int)threadIdx.x * per), hi = min(chunks, lo + per);
    int s = 0;
    for (int i = lo; i < hi; ++i) s += counts[i];
    part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int i = 0; i < 1024; ++i) {
            const int v = part[i];
            part[i] = run, run += v;
        }
        counts[chunks] = run;
    }
    __syncthreads();
    int run = part[threadIdx.x];
    for (int i = lo; i < hi; ++i) {
        const int v = counts[i];
        counts[i] = run, run += v;
    }
}

__global__ void __launch_bounds__(256) flac_compact_kernel(const unsigned char *__restrict__ flag, long long bytes,
                                                          const int *__restrict__ counts, unsigned *__restrict__ cand) {
    const long long b0 = (long long)blockIdx.x * kChunk + threadIdx.x * 16;
    int cnt = 0;
    for (int i = 0; i < 16 && b0 + i < bytes; ++i) cnt += flag[b0 + i];
    __shared__ int pre[256];
    pre[threadIdx.x] = cnt;
    __syncthreads();
    for (int w = 1; w < 256; w <<= 1) {               // inclusive Hillis-Steele scan
        const int v = (int)threadIdx.x >= w ? pre[threadIdx.x - w] : 0;
        __syncthreads();
        pre[threadIdx.x] += v;
        __syncthreads();
    }
    int at = counts[blockIdx.x] + pre[threadIdx.x] - cnt;
    for (int i = 0; i < 16 && b0 + i < bytes; ++i)
        if (flag[b0 + i]) cand[at++] = (unsigned)(b0 + i);
}

// ---- 4: CRC-16 of every span between consecutive candidates ----------------------------------------------------------------
__global__ void __launch_bounds__(256) flac_span_crc_kernel(const unsigned char *__restrict__ d, const FStream *__restrict__ st, int n,
                                                           const int *__restrict__ count, const unsigned *__restrict__ cand,
                                                           unsigned short *__restrict__ crc) {
    __shared__ unsigned short tab[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        unsigned c = (unsigned)i << 8;
        for (int k = 0; k < 8; ++k) c = (c & 0x8000) ? ((c << 1) ^ 0x8005) & 0xFFFF : (c << 1) & 0xFFFF;
        tab[i] = (unsigned short)c;
    }
    __syncthreads();
    const int ncand = *count, lane = threadIdx.x & 31;
    for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < ncand; i += ((long long)gridDim.x * blockDim.x) >> 5) {
        const long long a = cand[i];
        const FStream &S = st[find_stream(st, n, a)];
        const long long e = (i + 1 < ncand && (long long)cand[i + 1] < S.end) ? (long long)cand[i + 1] : S.end;
        const long long len = e - a, per = (len + 31) / 32;
        const long long lo = min(e, a + lane * per), hi = min(e, lo + per);
        unsigned c = 0;
        for (long long q = lo; q < hi; ++q) c = ((c << 8) & 0xFFFF) ^ tab[(c >> 8) ^ d[q]];
        unsigned long long l = hi - lo;
        for (int w = 1; w < 32; w <<= 1) {            // lane L absorbs lane L + w: crc(A B) = crc(A) x^(8|B|) + crc(B)
            const unsigned cr = __shfl_down_sync(0xFFFFFFFFu, c, w);
            const unsigned long long lr = __shfl_down_sync(0xFFFFFFFFu, l, w);
            if ((lane & (2 * w - 1)) == 0 && lane + w < 32) c = gf_mul(c, gf_xpow8(lr)) ^ cr, l += lr;
        }
        if (lane == 0) crc[i] = (unsigned short)c;
    }
}

// ---- 5: the frame chain of each stream -------------------------------------------------------------------------------------
__device__ int lower_bound(const unsigned *cand, int n, long long v) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((long long)cand[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void flac_walk_kernel(const unsigned char *__restrict__ d, const FStream *__restrict__ st, int n, const int *__restrict__ count,
                                 const unsigned *__restrict__ cand, const unsigned short *__restrict__ crc, FFrame *__restrict__ frames,
                                 long long *__restrict__ nframes, unsigned long long *__restrict__ err) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const FStream S = st[s];
    const int ncand = *count;
    int i = lower_bound(cand, ncand, S.first);
    const int hi = lower_bound(cand, ncand, S.end);
    long long done = 0, k = 0, nf = 0;
    nframes[s] = 0;
    if (i >= hi || (long long)cand[i] != S.first) {
        report(err, s, S, S.first, E_START);
        return;
    }
    while (done < S.total) {
        const long long at = cand[i];
        const FHeader h = parse_header(d, at, S.end);
        const int ch = h.ch_code < 8 ? h.ch_code + 1 : 2;
        if (h.number != (unsigned long long)(h.variable ? done : k) || ch != S.ch || (h.bits && h.bits != S.bits) ||
            (h.sr && h.sr != S.sr) || done + h.bs > S.total) {
            report(err, s, S, at, E_CHAIN);
            break;
        }
        const unsigned long long want = h.variable ? done + h.bs : k + 1;
        unsigned c = 0;
        int j = i;
        bool found = false;
        long long trail = -1;                         // the last frame checks out here, but bytes follow it
        while (j < hi) {
            const long long a = cand[j], e = j + 1 < hi ? (long long)cand[j + 1] : S.end;
            c = gf_mul(c, gf_xpow8(e - a)) ^ crc[j];
            ++j;
            if (c != 0) continue;
            if (j == hi) {
                found = true;
                break;
            }
            if (done + h.bs == S.total) {             // the last frame must end where the stream does
                if (trail < 0) trail = cand[j];
                continue;
            }
            const FHeader nx = parse_header(d, cand[j], S.end);
            if (nx.variable == h.variable && nx.number == want) {
                found = true;
                break;
            }
        }
        if (!found) {
            if (trail >= 0) report(err, s, S, trail, E_TRAIL);
            else report(err, s, S, at, E_CRC);
            break;
        }
        if (nf >= S.frame_cap) {
            report(err, s, S, at, E_FRAMES);
            break;
        }
        const long long e = j < hi ? (long long)cand[j] : S.end;
        FFrame F{};
        F.start = at, F.first = done, F.bytes = (int)(e - at), F.bs = h.bs, F.stream = s, F.assign = h.ch_code, F.hdr = h.hdr;
        frames[S.frame_base + nf++] = F;
        done += h.bs, ++k, i = j;
        if (done < S.total && i >= hi) {
            report(err, s, S, e, E_SHORT);
            break;
        }
    }
    nframes[s] = nf;
}

// ---- 6-7: subframes --------------------------------------------------------------------------------------------------------
// MSB-first bit reader over one frame's bytes, the CRC-16 excluded; a read past them sets `bad` and returns zeros
struct Bits {
    const unsigned char *p;
    unsigned nbytes, next;
    unsigned long long cache;
    int avail;
    bool bad;

    __device__ void init(const unsigned char *frame, unsigned n, unsigned bitpos) {
        p = frame, nbytes = n, next = bitpos >> 3, cache = 0, avail = 0, bad = false;
        refill();
        skip(bitpos & 7);
    }
    __device__ __forceinline__ void refill() {
        while (avail <= 56 && next < nbytes) cache |= (unsigned long long)p[next++] << (56 - avail), avail += 8;
    }
    __device__ __forceinline__ unsigned pos() const { return next * 8 - avail; }
    __device__ __forceinline__ void skip(int k) { cache <<= k, avail -= k; }
    __device__ __forceinline__ unsigned read(int k) {          // 0 <= k <= 32
        if (k == 0) return 0;
        if (avail < k) refill();
        if (avail < k) {
            bad = true, avail = 0, cache = 0;
            return 0;
        }
        const unsigned v = (unsigned)(cache >> (64 - k));
        cache <<= k, avail -= k;
        return v;
    }
    __device__ __forceinline__ int sread(int k) {
        const unsigned v = read(k);
        return k == 0 ? 0 : k == 32 ? (int)v : (int)(v << (32 - k)) >> (32 - k);
    }
    __device__ __forceinline__ unsigned long long unary() {    // zeros before the next one, by count of leading zeros
        unsigned long long q = 0;
        for (;;) {
            if (avail == 0) refill();
            if (avail == 0) {
                bad = true;
                return 0;
            }
            const int z = min(__clzll(cache), avail);
            if (z < avail) {
                cache = z + 1 >= 64 ? 0ULL : cache << (z + 1);
                avail -= z + 1;
                return q + z;
            }
            q += avail, cache = 0, avail = 0;
        }
    }
};

// Decode (kStore) or skim one subframe.  bits: the channel's sample width (the side channel's is one more).  Returns false on a
// malformed subframe; x receives bs int32 samples when storing.
template <bool kStore>
__device__ bool subframe(Bits &r, int bs, int bits, int *__restrict__ x, int *__restrict__ coef) {
    if (r.read(1)) return false;
    const int t = (int)r.read(6);
    int wasted = 0;
    if (r.read(1)) wasted = (int)min(r.unary() + 1, 64ULL);
    if (wasted >= bits || r.bad) return false;
    bits -= wasted;
    if (t == 0) {
        const int v = r.sread(bits);
        if (kStore)
            for (int i = 0; i < bs; ++i) x[i] = (int)((unsigned)v << wasted);
        return !r.bad;
    }
    if (t == 1) {
        for (int i = 0; i < bs; ++i) {
            const int v = r.sread(bits);
            if (kStore) x[i] = (int)((unsigned)v << wasted);
        }
        return !r.bad;
    }
    int order, shift = 0, prec = 0;
    if (t >= 8 && t <= 12) order = t - 8;
    else if (t >= 32) order = t - 31;
    else return false;
    if (order > bs) return false;
    for (int i = 0; i < order; ++i) {
        const int v = r.sread(bits);
        if (kStore) x[i] = v;
    }
    if (t >= 32) {
        prec = (int)r.read(4) + 1;
        shift = r.sread(5);
        if (prec == 16 || shift < 0) return false;
        for (int j = 0; j < order; ++j) {
            const int c = r.sread(prec);
            if (kStore) coef[j * kSubThreads] = c;
        }
    }
    const int method = (int)r.read(2);
    if (method > 1) return false;
    const int pbits = method ? 5 : 4, esc = method ? 31 : 15, porder = (int)r.read(4);
    if ((bs & ((1 << porder) - 1)) || (bs >> porder) < order || r.bad) return false;
    int i = order;
    for (int part = 0; part < (1 << porder); ++part) {
        const int cnt = (bs >> porder) - (part == 0 ? order : 0);
        const int k = (int)r.read(pbits);
        if (k == esc) {
            const int nb = (int)r.read(5);
            for (int q = 0; q < cnt; ++q, ++i) {
                const int v = r.sread(nb);
                if (kStore) x[i] = v;
            }
        } else {
            for (int q = 0; q < cnt; ++q, ++i) {
                const unsigned long long hiq = r.unary();
                if (hiq >> 32) return false;
                const unsigned long long u = (hiq << k) | r.read(k);
                if (u >> 32) return false;
                if (kStore) x[i] = (int)((unsigned)(u >> 1) ^ (0u - (unsigned)(u & 1)));
            }
        }
        if (r.bad) return false;
    }
    if (!kStore) return !r.bad;
    // restoration: the serial recurrence of the subframe, in int64 like the oracle's unbounded integers
    if (t <= 12) {
        for (int q = order; q < bs; ++q) {
            long long pr = 0;
            if (order == 1) pr = x[q - 1];
            else if (order == 2) pr = 2LL * x[q - 1] - x[q - 2];
            else if (order == 3) pr = 3LL * x[q - 1] - 3LL * x[q - 2] + x[q - 3];
            else if (order == 4) pr = 4LL * x[q - 1] - 6LL * x[q - 2] + 4LL * x[q - 3] - x[q - 4];
            x[q] = (int)(x[q] + pr);
        }
    } else {
        for (int q = order; q < bs; ++q) {
            long long pr = 0;
            for (int j = 0; j < order; ++j) pr += (long long)coef[j * kSubThreads] * x[q - 1 - j];
            x[q] = (int)(x[q] + (pr >> shift));
        }
    }
    if (wasted)
        for (int q = 0; q < bs; ++q) x[q] = (int)((unsigned)x[q] << wasted);
    return true;
}

__device__ __forceinline__ int channel_bits(int assign, int c, int bits) {
    return bits + ((assign == 8 && c == 1) || (assign == 9 && c == 0) || (assign == 10 && c == 1));
}

__device__ __forceinline__ int frame_stream(const FStream *st, int n, long long slot) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (st[mid].frame_base <= slot) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(128) flac_bounds_kernel(const unsigned char *__restrict__ d, const FStream *__restrict__ st, int n,
                                                         long long slots, FFrame *__restrict__ frames, const long long *__restrict__ nframes,
                                                         unsigned long long *__restrict__ err) {
    for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < slots; f += (long long)gridDim.x * blockDim.x) {
        const int s = frame_stream(st, n, f);
        const FStream &S = st[s];
        if (f - S.frame_base >= nframes[s]) continue;
        FFrame &F = frames[f];
        Bits r;
        r.init(d + F.start, (unsigned)(F.bytes - 2), (unsigned)F.hdr * 8);
        bool ok = true;
        for (int c = 0; c < S.ch && ok; ++c) {
            F.sub[c] = r.pos();
            ok = subframe<false>(r, F.bs, channel_bits(F.assign, c, S.bits), nullptr, nullptr);
        }
        if (!ok) report(err, s, S, F.start, E_SUBFRAME);
        else if ((r.pos() + 7) / 8 != (unsigned)(F.bytes - 2)) report(err, s, S, F.start, E_LENGTH);
    }
}

__global__ void __launch_bounds__(kSubThreads) flac_subframe_kernel(const unsigned char *__restrict__ d, const FStream *__restrict__ st, int n,
                                                                   long long slots, const FFrame *__restrict__ frames,
                                                                   const long long *__restrict__ nframes, int *__restrict__ pcm,
                                                                   unsigned long long *__restrict__ err) {
    __shared__ int coef[kMaxLpc * kSubThreads];
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < slots * 8; g += (long long)gridDim.x * blockDim.x) {
        const long long f = g >> 3;
        const int c = (int)(g & 7);
        const int s = frame_stream(st, n, f);
        const FStream &S = st[s];
        if (c >= S.ch || f - S.frame_base >= nframes[s]) continue;
        const FFrame &F = frames[f];
        Bits r;
        r.init(d + F.start, (unsigned)(F.bytes - 2), F.sub[c]);
        int *x = pcm + S.pcm_off + (long long)c * S.total + F.first;
        if (!subframe<true>(r, F.bs, channel_bits(F.assign, c, S.bits), x, coef + threadIdx.x)) report(err, s, S, F.start, E_SUBFRAME);
    }
}

// one CTA per frame: undo the stereo decorrelation, scale by 2^-(bits - 1), average the channels as read_wav does
__global__ void __launch_bounds__(256) flac_output_kernel(const FStream *__restrict__ st, int n, long long slots,
                                                         const FFrame *__restrict__ frames, const long long *__restrict__ nframes,
                                                         const int *__restrict__ pcm, float *__restrict__ out) {
    for (long long f = blockIdx.x; f < slots; f += gridDim.x) {
        const int s = frame_stream(st, n, f);
        const FStream &S = st[s];
        if (f - S.frame_base >= nframes[s]) continue;
        const FFrame &F = frames[f];
        const float scale = 1.0f / (float)(1 << (S.bits - 1));
        const int *x = pcm + S.pcm_off + F.first;
        for (int i = threadIdx.x; i < F.bs; i += blockDim.x) {
            float v[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) v[c] = c < S.ch ? (float)x[(long long)c * S.total + i] * scale : 0.f;
            if (F.assign >= 8) {
                const int a = x[i], b = x[S.total + i];
                int L, R;
                if (F.assign == 8) L = a, R = a - b;
                else if (F.assign == 9) L = a + b, R = b;
                else {
                    const int m = (int)(((unsigned)a << 1) | (unsigned)(b & 1));
                    L = (m + b) >> 1, R = (m - b) >> 1;
                }
                v[0] = (float)L * scale, v[1] = (float)R * scale;
            }
            // numpy's float32 mean(axis=1) over scipy's C-ordered [n, ch] samples: channels in order, except that its pairwise sum
            // takes exactly 8 elements as ((c0 + c1) + (c2 + c3)) + ((c4 + c5) + (c6 + c7))
            float y;
            if (S.ch == 8) y = ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
            else {
                y = v[0];
#pragma unroll
                for (int c = 1; c < 8; ++c)
                    if (c < S.ch) y += v[c];
            }
            out[S.out_off + F.first + i] = S.ch == 1 ? y : y / (float)S.ch;
        }
    }
}

const char *what(unsigned code) {
    switch (code) {
    case E_START: return "no frame header where the metadata ends";
    case E_CHAIN: return "frame does not continue the stream or disagrees with STREAMINFO (number, rate, bits, channels or total)";
    case E_CRC: return "frame fails its CRC-16";
    case E_SHORT: return "the frames stop short of STREAMINFO's total sample count";
    case E_FRAMES: return "more frames than the stream's bytes can hold";
    case E_SUBFRAME: return "malformed or truncated subframe";
    case E_LENGTH: return "subframes end away from the frame's CRC-16";
    case E_TRAIL: return "data after the last frame";
    default: return "unknown error";
    }
}

int run(const Layout &lay, const unsigned char *data, float *out, void *ws, int64_t ws_bytes, float *stage_ms, cudaStream_t stream) {
    const int n = (int)lay.st.size();
    SVB_CHECK(data && out && ws, SVB_ERR_INVALID, "flac: null buffer");
    SVB_CHECK(ws_bytes >= (int64_t)lay.total, SVB_ERR_INVALID, "flac: workspace of %lld bytes, %zu needed", (long long)ws_bytes, lay.total);
    char *base = static_cast<char *>(ws);
    FStream *d_st = reinterpret_cast<FStream *>(base + lay.off_st);
    unsigned char *d_flag = reinterpret_cast<unsigned char *>(base + lay.off_flag);
    int *d_cnt = reinterpret_cast<int *>(base + lay.off_cnt);
    unsigned *d_cand = reinterpret_cast<unsigned *>(base + lay.off_cand);
    unsigned short *d_crc = reinterpret_cast<unsigned short *>(base + lay.off_crc);
    FFrame *d_frames = reinterpret_cast<FFrame *>(base + lay.off_frame);
    long long *d_nf = reinterpret_cast<long long *>(base + lay.off_nf);
    unsigned long long *d_err = reinterpret_cast<unsigned long long *>(base + lay.off_err);
    int *d_pcm = reinterpret_cast<int *>(base + lay.off_pcm);
    SVB_CUDA(cudaMemcpyAsync(d_st, lay.st.data(), n * sizeof(FStream), cudaMemcpyHostToDevice, stream));
    SVB_CUDA(cudaMemsetAsync(d_err, 0xFF, n * sizeof(unsigned long long), stream));
    cudaEvent_t ev[2] = {};
    if (stage_ms) {
        for (auto &e : ev) SVB_CUDA(cudaEventCreate(&e));
        SVB_CUDA(cudaEventRecord(ev[0], stream));
    }
    const int sms = 132 * 4;
    flac_scan_kernel<<<lay.chunks, 256, 0, stream>>>(data, d_st, n, lay.bytes, d_flag, d_cnt);
    flac_chunk_scan<<<1, 1024, 0, stream>>>(d_cnt, lay.chunks);
    flac_compact_kernel<<<lay.chunks, 256, 0, stream>>>(d_flag, lay.bytes, d_cnt, d_cand);
    flac_span_crc_kernel<<<sms, 256, 0, stream>>>(data, d_st, n, d_cnt + lay.chunks, d_cand, d_crc);
    flac_walk_kernel<<<(n + 31) / 32, 32, 0, stream>>>(data, d_st, n, d_cnt + lay.chunks, d_cand, d_crc, d_frames, d_nf, d_err);
    flac_bounds_kernel<<<sms, 128, 0, stream>>>(data, d_st, n, lay.frames, d_frames, d_nf, d_err);
    flac_subframe_kernel<<<sms, kSubThreads, 0, stream>>>(data, d_st, n, lay.frames, d_frames, d_nf, d_pcm, d_err);
    flac_output_kernel<<<sms, 256, 0, stream>>>(d_st, n, lay.frames, d_frames, d_nf, d_pcm, out);
    SVB_CUDA(cudaGetLastError());
    std::vector<unsigned long long> err(n);
    if (stage_ms) SVB_CUDA(cudaEventRecord(ev[1], stream));
    SVB_CUDA(cudaMemcpyAsync(err.data(), d_err, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
    SVB_CUDA(cudaStreamSynchronize(stream));
    if (stage_ms) {
        SVB_CUDA(cudaEventElapsedTime(stage_ms, ev[0], ev[1]));
        for (auto e : ev) cudaEventDestroy(e);
    }
    for (int s = 0; s < n; ++s)
        SVB_CHECK(err[s] == ~0ULL, SVB_ERR_INVALID, "flac: stream %d: %s at byte %llu", s, what((unsigned)(err[s] & 0xFF)), err[s] >> 8);
    return SVB_OK;
}

}  // namespace
}  // namespace svb

using namespace svb;

extern "C" int64_t svb_flac_plan(int32_t n_streams, const int64_t *nbytes, const int64_t *first_frame, const int32_t *sample_rate,
                                 const int32_t *channels, const int32_t *bits, const int64_t *total_samples, int64_t *out_samples) {
    Layout lay;
    if (plan(n_streams, nbytes, first_frame, sample_rate, channels, bits, total_samples, &lay) != SVB_OK) return -1;
    if (out_samples)
        for (int s = 0; s < n_streams; ++s) out_samples[s] = total_samples[s];
    return (int64_t)lay.total;
}

extern "C" int svb_flac_decode_batch(int32_t n_streams, const int64_t *nbytes, const int64_t *first_frame, const int32_t *sample_rate,
                                     const int32_t *channels, const int32_t *bits, const int64_t *total_samples, const void *data_dev,
                                     float *out_dev, void *workspace_dev, int64_t workspace_bytes, float *stage_ms_host, void *stream) {
    Layout lay;
    SVB_TRY(plan(n_streams, nbytes, first_frame, sample_rate, channels, bits, total_samples, &lay));
    return run(lay, static_cast<const unsigned char *>(data_dev), out_dev, workspace_dev, workspace_bytes, stage_ms_host, as_stream(stream));
}
