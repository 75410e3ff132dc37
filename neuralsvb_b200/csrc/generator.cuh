// Shared definitions of the generator handle (generator.cu: forward; generator_bwd.cu: training backward).
#pragma once
#include <map>
#include <string>
#include <vector>

#include "conv_ffma.cuh"
#include "conv_tc.cuh"
#include "nsf_source.cuh"

namespace svb {

struct HostTensor {
    std::vector<int64_t> shape;
    std::vector<float> data;
};

struct ConvLayer {          // one GEMM-shaped layer on the C4T layout
    float *w = nullptr;     // FFMA packing [KS][Cin][CoutP]
    float *b = nullptr;     // [Cout]
    TcWeights tc;           // tensor-core packing (optional)
    int Cin = 0, Cout = 0, CoutP = 0, KS = 1, dil = 1, ups_u = 0;
    double macs_per_row = 0;   // algorithmic MACs per GEMM row (true taps only)
};

struct NoiseConv {
    float *w = nullptr, *b = nullptr;
    int C = 0, K = 1, stride = 1, pad = 0;
};

struct Stage {
    int C = 0;              // channels after the upsampler
    int u = 1;
    ConvLayer up;
    NoiseConv noise;
    // resblocks[j].c1[m], c2[m]  (ResBlock2: only c1 used)
    std::vector<std::vector<ConvLayer>> c1, c2;
};

struct Tap {
    const float *p = nullptr;
    int C = 0, T = 0, Tp = 0;
    bool plain = false;     // [B][T] instead of C4T
};

// How a stage runs its ResBlock steps (decided per forward by plan_workspace): one launch per conv, chain by chain; or step
// by step, one launch over all chains' c1 and one over their c2 (merged), or one over both (fused: no A buffers)
enum class Schedule : char { PerConv, Merged, Fused };

// byte offsets into the workspace of one forward (in training mode this is also the tape of the backward)
struct Buffers {
    size_t mel = 0, pre = 0, har = 0, nsf = 0, sines = 0, wav = 0;
    size_t f0 = 0;                                           // [B][T] f0 of a ragged host call (clips unpacked)
    std::vector<Schedule> sched;                             // per stage
    std::vector<size_t> X, S;
    std::vector<std::vector<std::vector<size_t>>> A, R;      // [stage][ResBlock chain][dilation]
};

// Step m of ResBlock chain j of a stage: it reads x (also its residual) and leaves its result in dst, the stage sum S on
// the last step (scaled by 1 / nk and, after the first chain, accumulated), else the next step's x.  t: c1's output of a
// ResBlock1 step; nullptr for ResBlock2 and in fused stages.
struct StepBufs {
    float *x, *t, *dst;
    float scale;
    int accumulate;
};

// dgrad twins of the ResBlock convs of one stage (flipped taps, transposed channels) + upsampler weights
// in the [K][Cout][Cin] order the strided data-gradient kernel reads
struct BwdStage {
    std::vector<std::vector<ConvLayer>> d1, d2;
    float *up_wt = nullptr;
};

// one device-side re-packing step: dst[i] = idx[i] ? nat[src][idx[i] - 1] : 0, then (optionally) the wgmma tiles
struct PackJob {
    std::string src;            // name of the folded tensor in the reference's layout
    float *dst = nullptr;
    int *idx = nullptr;         // nullptr: plain copy
    size_t n = 0;
    const TcWeights *tc = nullptr;
};

struct GradBuf {
    float *p = nullptr;
    size_t n = 0;
};
}  // namespace svb

struct svb_gen {
    svb_gen_config cfg{};
    int device = 0;
    bool finalized = false;
    std::map<std::string, svb::HostTensor> host_w;
    std::vector<void *> dev_allocs;

    svb::ConvLayer conv_pre;
    std::vector<svb::Stage> stages;
    float *post_wq = nullptr;
    int post_K = 7, post_C = 0;
    float *lin_w = nullptr;
    float *lin_b_dev = nullptr;     // m_source.l_linear.bias [1]
    int hop = 1;

    // workspace
    char *ws = nullptr;
    size_t ws_cap = 0;
    int ws_B = 0, ws_T = 0;
    std::map<std::string, svb::Tap> taps;
    int last_B = 0, last_T = 0;
    bool last_nsf = false;
    svb::Buffers bf;            // layout of the last forward

    // training (generator_bwd.cu): tape kept by forward, dgrad packings, gradient buffers
    bool training = false, ws_training = false, dirty = false;
    bool bwd_built = false;         // data-gradient packings + gather jobs exist (they survive set_training(0))
    std::vector<svb::BwdStage> bwd;
    float *zero_bias = nullptr;     // [max channels] zeros: the dgrad convs have no bias
    float *post_w_nat = nullptr;    // conv_post weight [C][K]
    float *post_b_dev = nullptr;
    float *grad_flat = nullptr;
    size_t grad_floats = 0;
    std::map<std::string, svb::GradBuf> grads;
    char *bws = nullptr;            // backward workspace (activation gradients)
    size_t bws_cap = 0;
    int bws_B = 0, bws_T = 0;
    int64_t bwd_launches = 0;
    std::map<std::string, svb::GradBuf> nat_dev;    // device copies of the folded tensors (svb_gen_set_weight_dev)
    std::vector<svb::PackJob> jobs;
    std::vector<void *> job_allocs;
    bool dev_dirty = false;

    // Ragged batches (svb_gen_forward_ragged).  rg_len: frames per clip of the current forward (empty: every clip has T);
    // rg_dev: its device copy [len | zero from | zero to | first frame] (4 B ints).  Rows at or past a clip's end must be zero
    // in every activation buffer (the conv's zero padding), and kernels never write them, but an earlier, longer call may
    // have: ws_live[b] = the frames of clip b's rows that may be nonzero since the last full memset, and a ragged forward
    // first zeroes each clip's rows between its length and ws_live (zero_tails in generator.cu).
    std::vector<int> rg_len, ws_live, wl_len;   // wl_len: the lengths the cached work lists were built for
    std::vector<char> ws_fused;                 // per stage: the fused layout the workspace was zeroed for
    const int *rg_dev = nullptr;                // the current forward's copy (in rg_buf or in the host call's staging)
    int *rg_buf = nullptr;
    size_t rg_cap = 0;
    int cur_T = 0;                              // frames of the current forward (T, or T_max of a ragged one)

    // host staging (spec2wav_host)
    float *pin_in = nullptr, *pin_out = nullptr, *dev_in = nullptr, *dev_out = nullptr;
    size_t pin_in_cap = 0, pin_out_cap = 0;
    float *dev_pack = nullptr;      // the clips of a ragged host call back to back (svb_gen_spec2wav_ragged_host)
    size_t pack_cap = 0;
    int16_t *dev_i16 = nullptr;      // int16 samples + per-clip peak (svb_gen_spec2wav_host_i16)
    size_t i16_cap = 0;

    int64_t last_launches = 0;
    double last_flops = 0;
    bool timing = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;

    // per-launch profile of the last forward (svb_gen_enable_timing(g, 2)): CUDA events around every launch
    struct LaunchRec {
        const char *name;
        cudaEvent_t e0, e1;
        double bytes, flops;
    };
    // the NSF source runs on this stream, overlapping conv_pre and the first upsampler
    cudaStream_t side = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_side = nullptr;

    // merged launches: the ResBlock chains of a stage step together in one persistent launch (conv_tc.cuh: TcWorkList).
    // Lists depend on the stage, the batch / length and the plan's MT; cached per (stage, chain_ordered, MT).
    bool merge = true;              // SVB_MERGE=0: one launch per convolution (round-1 schedule)
    bool fuse = true;               // SVB_FUSE=0: two launches per ResBlock1 step also where the fused launch fits (the
                                    // reference path of the bit-identity tests)
    bool epi = true;                // SVB_EPI=0: the tensor-core epilogue loads residual / running sum per thread instead
                                    // of streaming them through shared memory (the reference of its bit-identity tests)
    int fused_ctas = 0;             // SVB_TC_FUSED_CTAS=1: the fused C = 32 steps keep one CTA per SM where two fit (the
                                    // reference of the two-CTA bit-identity tests); 2 or unset: two where they fit
    std::map<int, svb::TcWorkList> worklists;

    bool profile = false;
    std::vector<LaunchRec> recs;
    std::vector<cudaEvent_t> ev_pool;
    size_t ev_used = 0;
};


namespace svb {
int gen_upload(svb_gen *g, const std::vector<float> &h, float **out);
int gen_get_w(svb_gen *g, const std::string &name, std::vector<int64_t> want, const HostTensor **out);
int gen_build_layers(svb_gen *g);
int gen_build_bwd_layers(svb_gen *g);      // generator_bwd.cu
StepBufs step_bufs(const svb_gen *g, int stage, int chain, int m);     // in the layout of the last forward (svb_gen::bf)
}  // namespace svb
