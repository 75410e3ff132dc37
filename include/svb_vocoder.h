/*
 * svb_vocoder.h -- C ABI of libsvb_vocoder.so, the H100 (sm_90a) implementation of the
 * NeuralSVB mel-to-waveform hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types, no C++ in the
 * signatures.  Every entry point names the reference interface it replaces.  The reference
 * is pure Python/PyTorch, so its "FFI" is ctypes: INTEGRATION.md shows the stub a
 * maintainer adds to vocoders/hifigan.py to bind these.
 *
 * Conventions
 *   - every function returns 0 on success and a negative svb_status otherwise; nothing
 *     throws across the ABI; svb_last_error() gives the message for the calling thread.
 *   - "dev" pointers are device pointers on the handle's device, "host" pointers are host
 *     memory; all buffers are caller-owned; scratch space is owned by the handle.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Calls are
 *     stream-ordered and do not synchronise unless documented (the *_host entry points
 *     synchronise before returning, like the reference's `.cpu()`).
 *   - one handle per (process, device); a handle is not thread-safe.
 *   - all floating-point tensors are fp32, dense, row-major in the stated shape.
 */
#ifndef SVB_VOCODER_H_
#define SVB_VOCODER_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SVB_ABI_VERSION 1

typedef enum svb_status {
    SVB_OK = 0,
    SVB_ERR_INVALID = -1,      /* bad argument / shape / config */
    SVB_ERR_CUDA = -2,         /* a CUDA runtime call or kernel failed */
    SVB_ERR_STATE = -3,        /* call order violated (e.g. forward before finalize) */
    SVB_ERR_MISSING = -4,      /* a required weight tensor was never set */
    SVB_ERR_NOMEM = -5
} svb_status;

/* arithmetic used for the dense ResBlock / upsampler contractions */
typedef enum svb_precision {
    SVB_PREC_FP32 = 0,         /* CUDA-core FFMA, fp32 everywhere                              */
    SVB_PREC_TF32 = 1,         /* wgmma tf32, operands rounded to nearest, fp32 accumulate     */
    SVB_PREC_TF32X3 = 2,       /* wgmma 3xTF32 split (hi*hi + hi*lo + lo*hi), ~fp32 accuracy   */
    SVB_PREC_BF16X3 = 3        /* wgmma bf16, operands split into bf16 hi + lo (16-bit mantissa),
                                  3 MMAs at twice the TF32 rate, fp32 accumulate -- the default      */
} svb_precision;

#define SVB_MAX_UPS 8
#define SVB_MAX_RBK 4
#define SVB_MAX_DIL 4

/* Mirrors the `h` dict given to HifiGanGenerator(h) -- modules/hifigan/hifigan.py:105-142;
 * values for the shipped model: egs/egs_bases/tts/vocoder/hifigan.yaml:3-12. */
typedef struct svb_gen_config {
    int32_t n_mel;                                 /* input channels of conv_pre (80, hifigan.py:118)   */
    int32_t upsample_initial_channel;              /* 512                                                */
    int32_t n_ups;                                 /* len(upsample_rates)                                */
    int32_t upsample_rates[SVB_MAX_UPS];           /* [8,8,2,2]                                          */
    int32_t upsample_kernel_sizes[SVB_MAX_UPS];    /* [16,16,4,4]                                        */
    int32_t resblock;                              /* 1 = ResBlock1 (:30-67), 2 = ResBlock2 (:70-91)     */
    int32_t n_resblock_kernels;                    /* len(resblock_kernel_sizes)                         */
    int32_t resblock_kernel_sizes[SVB_MAX_RBK];    /* [3,7,11]                                           */
    int32_t n_dilations;                           /* dilations per ResBlock (3 for '1', 2 for '2')      */
    int32_t resblock_dilation_sizes[SVB_MAX_RBK][SVB_MAX_DIL];
    int32_t use_pitch_embed;                       /* NSF source + noise_convs (:111-117,126-132)        */
    int32_t audio_sample_rate;                     /* 22050                                              */
    int32_t precision;                             /* svb_precision                                      */
} svb_gen_config;

typedef struct svb_gen svb_gen_t;                  /* opaque generator handle */

/* Message describing the last failure on the calling thread (never NULL). */
const char *svb_last_error(void);
int svb_abi_version(void);

/* ---- HiFi-GAN(-NSF) generator: replaces HifiGanGenerator (modules/hifigan/hifigan.py:104-178)
 *      as it is built and driven by vocoders/hifigan.py:17-33 (load_model) and :55-69 (spec2wav). */

/* HifiGanGenerator.__init__ (hifigan.py:105-142).  `device` is a CUDA ordinal. */
int svb_gen_create(const svb_gen_config *cfg, int device, svb_gen_t **out);
void svb_gen_destroy(svb_gen_t *g);

/* load_state_dict + remove_weight_norm (vocoders/hifigan.py:27-28, hifigan.py:171-178).
 * `name` is the reference state_dict key with weight norm already folded
 * ("conv_pre.weight", "ups.0.bias", "resblocks.4.convs2.1.weight", "noise_convs.2.weight",
 * "m_source.l_linear.weight", ...); `data` is a HOST fp32 tensor in the PyTorch layout
 * (Conv1d [Cout,Cin,K]; ConvTranspose1d [Cin,Cout,K]; Linear [out,in]; bias [C]). */
int svb_gen_set_weight(svb_gen_t *g, const char *name, const float *data, const int64_t *shape, int32_t ndim);
/* weight-norm folding on the device: w = g * v / ||v|| over all dims but 0
 * (torch.nn.utils.weight_norm dim=0; hifigan.py:35-50,118,124,140).  v_host [d0, inner], g_host [d0]. */
int svb_fold_weight_norm_host(const float *v_host, const float *g_host, int64_t d0, int64_t inner,
                              float *w_host, int device);
/* Packs the weights into kernel layouts and uploads them; checks every tensor is present. */
int svb_gen_finalize(svb_gen_t *g);
/* change svb_precision after finalize (repacks nothing; all layouts are kept resident) */
int svb_gen_set_precision(svb_gen_t *g, int32_t precision);

/* HifiGanGenerator.forward(x, f0) (hifigan.py:144-169), batched, device buffers.
 *   mel_dev      [B, n_mel, T]   log10-mel
 *   f0_dev       [B, T] Hz, 0 = unvoiced, or NULL for the non-NSF call model(c)
 *   rand_ini_dev [B, 9]   initial phases of SineGen (source.py:53-55; column 0 is forced to 0)
 *   noise_dev    [B, T*hop, 9] standard-normal draw of SineGen (source.py:132)
 *                both NULL -> drawn in-kernel from a Philox4x32-10 stream keyed by `seed`
 *   wav_dev      [B, T*hop]      output in (-1, 1)
 * Stream-ordered, no host synchronisation.
 * Clip length: tested up to 70 000 frames (6.8 min at hop 128) in every precision.  On the tensor-core precisions a clip
 * whose rows overflow the work-item table of one conv launch (120 items per CTA, one CTA per SM) runs that conv
 * in slices of rows on 256-row boundaries, with the same result bit for bit. */
int svb_gen_forward(svb_gen_t *g, const float *mel_dev, const float *f0_dev, const float *rand_ini_dev,
                    const float *noise_dev, uint64_t seed, int32_t B, int32_t T, float *wav_dev, void *stream);

/* HifiGAN.spec2wav(mel, f0=...) (vocoders/hifigan.py:55-69) end to end from HOST memory:
 *   mel_host [B, T, n_mel] (the reference's [T, 80] frame-major layout, B clips of equal T),
 *   f0_host [B, T] or NULL, wav_host [B, T*hop].  Copies in (pinned staging, H2D), runs the
 *   generator, copies out (D2H) and synchronises `stream` before returning. */
int svb_gen_spec2wav_host(svb_gen_t *g, const float *mel_host, const float *f0_host, uint64_t seed,
                          int32_t B, int32_t T, float *wav_host, void *stream);

/* spec2wav followed by save_wav's sample conversion (utils/audio.py:11-16: [norm: wav / max|wav| per clip,]
 * wav * 32767, float -> int16 truncation toward zero) ON THE DEVICE, so the D2H copy is 2 bytes per sample:
 * the reference moves the fp32 waveform to the host (vocoders/hifigan.py:63-66) and converts it in a CPU pool
 * (tasks/tts/tts.py:111, svb_vae_task.py:373-375).  wav_host int16 [B, T*hop]. */
int svb_gen_spec2wav_host_i16(svb_gen_t *g, const float *mel_host, const float *f0_host, uint64_t seed, int32_t B,
                              int32_t T, int32_t norm, int16_t *wav_host, void *stream);
/* the conversion alone on device buffers: wav_dev fp32 [B, n] -> out_dev int16 [B, n] (stream-ordered). */
int svb_wav_to_int16(const float *wav_dev, int32_t B, int64_t n, int32_t norm, int16_t *out_dev, void *stream);

/* Ragged batches (inference only): HifiGanGenerator.forward (hifigan.py:144-169) run on each clip alone, as the reference's
 * spec2wav (vocoders/hifigan.py:55-69) vocodes clips of different lengths one at a time, in one call.  Clip b has
 * lengths_host[b] frames, 1 <= lengths_host[b] <= T_max; the buffers are laid out as svb_gen_forward's with T = T_max, and mel /
 * f0 frames at or past a clip's length are never read (they may hold anything).  wav_dev[b, t] = 0 for t >= lengths_host[b] * hop.
 * Clip b is bit-identical to a B = 1 svb_gen_forward of that clip alone given the same draws (rand_ini row b, noise[b, :len*hop]);
 * the Philox draws stay keyed by (seed, b, t).  Lengths are checked on the host before anything touches the GPU; a training
 * handle returns SVB_ERR_STATE. */
int svb_gen_forward_ragged(svb_gen_t *g, const float *mel_dev, const float *f0_dev, const float *rand_ini_dev,
                           const float *noise_dev, uint64_t seed, int32_t B, int32_t T_max, const int32_t *lengths_host,
                           float *wav_dev, void *stream);
/* svb_gen_forward_ragged with the Philox draws of clip b keyed by (seed, first_clip + b, t): a batch vocoded in several calls
 * draws what one call over all its clips would (first_clip >= 0; 0 is svb_gen_forward_ragged). */
int svb_gen_forward_ragged_from(svb_gen_t *g, const float *mel_dev, const float *f0_dev, const float *rand_ini_dev,
                                const float *noise_dev, uint64_t seed, int32_t first_clip, int32_t B, int32_t T_max,
                                const int32_t *lengths_host, float *wav_dev, void *stream);
/* spec2wav over a ragged batch from HOST memory (vocoders/hifigan.py:55-69, clip by clip): mel_host holds the clips' [T_b, n_mel]
 * mels back to back ([sum T_b, n_mel], as svb_wav2spec_batch returns them), f0_host their [T_b] f0 back to back or NULL;
 * wav_host receives sum(T_b) * hop samples, clip after clip.  One H2D copy, one forward, one D2H copy, one synchronisation. */
int svb_gen_spec2wav_ragged_host(svb_gen_t *g, const float *mel_host, const float *f0_host, uint64_t seed, int32_t B,
                                 const int32_t *lengths_host, float *wav_host, void *stream);
/* the same followed by save_wav's int16 conversion on the device (svb_gen_spec2wav_host_i16); `norm` divides each clip by the
 * peak of its own samples.  wav_host int16 [sum T_b * hop]. */
int svb_gen_spec2wav_ragged_host_i16(svb_gen_t *g, const float *mel_host, const float *f0_host, uint64_t seed, int32_t B,
                                     const int32_t *lengths_host, int32_t norm, int16_t *wav_host, void *stream);

/* Intermediate tap for layer-level parity tests: copies a named activation of the LAST forward
 * ("har_source" [B,T*hop]; "conv_pre", "ups{i}", "stage{i}" as [B,C,T_i]) to out_dev.  shape3 receives its shape;
 * out_dev = NULL with capacity_floats = 0 only queries that shape. */
int svb_gen_get_tap(svb_gen_t *g, const char *name, float *out_dev, int64_t capacity_floats,
                    int64_t *shape3, void *stream);
int64_t svb_gen_hop(const svb_gen_t *g);
/* number of kernels launched by the last forward / their algorithmic FLOPs (for bench.py) */
int64_t svb_gen_last_launches(const svb_gen_t *g);
double svb_gen_last_flops(const svb_gen_t *g);
/* on = 1: CUDA events around the whole forward (svb_gen_last_ms, else -1).
 * on = 2: additionally CUDA events around EVERY launch of the forward, on the launching stream;
 *         svb_gen_profile_count / _get return, per launch of the last forward: the kernel family,
 *         its event time, its algorithmic HBM bytes (layer-streaming model: each conv reads its
 *         input once, writes its output once, reads the residual / running sum once) and FLOPs. */
int svb_gen_enable_timing(svb_gen_t *g, int32_t on);
float svb_gen_last_ms(svb_gen_t *g);
int32_t svb_gen_profile_count(svb_gen_t *g);
int svb_gen_profile_get(svb_gen_t *g, int32_t i, char *name, int32_t name_cap, float *ms, double *bytes, double *flops);

/* ---- training: backward of the discriminator-side operators ------------------------------------------------
 * Replaces torch autograd through the Conv1d / Conv2d((k,1)) + leaky_relu stacks of DiscriminatorP / DiscriminatorS
 * (modules/hifigan/hifigan.py:193-221, :262-286), AvgPool1d(4,2,1) (:304-306), the reflect pad (:209-212) and the
 * element-wise loss gradients of feature_loss / discriminator_loss / generator_loss (:328-365) and of
 * SpectralConvergengeLoss / LogSTFTMagnitudeLoss (modules/parallel_wavegan/losses/stft_loss.py:34-73).
 *   svb_conv_nct_backward: tensors as svb_conv_nct_forward; y = the forward's post-activation output (mask source,
 *     may be null when out_slope == 1), dy = gradient w.r.t. y.  dz_scratch [B,Cout,Tout,W] receives the masked
 *     gradient; dx (written), dw / db (ACCUMULATED with atomics; the caller zeroes them) may each be null.
 *   svb_loss_grad: da = (accumulate ? da : 0) + scale * f(a, b); kind 0 sign(a-b), 1 (a-1), 2 a, 3 (a-b),
 *     4 sign(ln a - ln b) / a. */
int svb_conv_nct_backward(const float *x_dev, const float *w_dev, const float *y_dev, const float *dy_dev, int32_t B,
                          int32_t Cin, int32_t Cout, int32_t Tin, int32_t W, int32_t K, int32_t stride, int32_t dil,
                          int32_t pad, int32_t groups, float out_slope, float *dz_scratch_dev, float *dx_dev,
                          float *dw_dev, float *db_dev, void *stream);
/* cond_net of the mel-conditioned ("use_cond") discriminators: ConvTranspose1d(C = 80, 1, K = 2*stride, stride,
 * padding = stride/2) (modules/hifigan/hifigan.py:185-189, :257-260).  mel [B, C, T] -> y [B, (T-1)*stride - 2*pad + K];
 * w [C, 1, K], bias [1] on the device.  backward ACCUMULATES dw / db (the mel is an input: no gradient). */
int svb_cond_net_forward(const float *mel_dev, const float *w_dev, const float *bias_dev, int32_t B, int32_t C, int32_t T,
                         int32_t K, int32_t stride, int32_t pad, float *y_dev, void *stream);
int svb_cond_net_backward(const float *mel_dev, const float *dy_dev, int32_t B, int32_t C, int32_t T, int32_t K, int32_t stride,
                          int32_t pad, float *dw_dev, float *db_dev, void *stream);
int svb_avgpool1d_4_2_1_backward(const float *dy_dev, float *dx_dev, int64_t rows, int32_t Tin, void *stream);
int svb_pad_reflect_right_backward(const float *dy_dev, float *dx_dev, int64_t rows, int32_t T, int32_t Tpad, void *stream);
int svb_loss_grad(const float *a_dev, const float *b_dev, int32_t kind, float scale, float *da_dev, int64_t n,
                  int32_t accumulate, void *stream);
/* same, with the factor scale * (*scale_dev) read on the device (the upstream gradient of an autograd node) */
int svb_loss_grad_dev(const float *a_dev, const float *b_dev, int32_t kind, float scale, const float *scale_dev,
                      float *da_dev, int64_t n, int32_t accumulate, void *stream);

/* ---- dense discriminator convolutions on the tensor-core kernel -------------------------------------------------
 * One handle per Conv1d / Conv2d((k,1)) layer with groups == 1 (modules/hifigan/hifigan.py:193-199, :262-271):
 * tensors are PyTorch-layout device buffers [B, C, T, W] (W = period columns, 1 for DiscriminatorS); weights
 * [Cout, Cin, K] and bias are device buffers re-packed by svb_tc_layer_set_weight_dev (cheap: call it whenever
 * they change).  forward: y = leaky_relu(conv(x) + bias, out_slope).  backward: dy is the gradient w.r.t. y;
 * dx is written, dw [Cout, Cin, K] / db [Cout] are ACCUMULATED (caller zeroes them); each may be null.
 * Shapes: stride 1 needs padding (K-1)/2; Cin*K (stride > 1) or Cin (stride 1) and Cout multiples of 32, Cout <= 1024. */
typedef struct svb_tc_layer svb_tc_layer_t;
int svb_tc_layer_create(int32_t Cin, int32_t Cout, int32_t K, int32_t stride, int32_t pad, int32_t precision, int device,
                        svb_tc_layer_t **out);
/* The GROUPED k = 41 layers of DiscriminatorS (Conv1d(128,128,41,2,groups=4) ... Conv1d(1024,1024,41,1,groups=16),
 * modules/hifigan/hifigan.py:263-267: 32 % of the discriminators' FLOPs) on the same wgmma kernel, in polyphase
 * form: a stride-s conv with K taps = a stride-1 conv with ceil(K/s) taps over Cin*s "space-to-depth" channels (a
 * permutation of the input, 1x traffic); every GEMM column block contracts only over the input channels of its own conv
 * groups.  forward / backward / set_weight_dev / out_len / destroy are the svb_tc_layer_* calls below; weights are
 * the natural [Cout, Cin/groups, K] tensor.  Needs ceil(K/stride) odd and (Cin/groups*stride, Cout/groups) to tile into
 * 32-channel chunks (pairs of narrow groups share a tile). */
int svb_tc_layer_create_grouped(int32_t Cin, int32_t Cout, int32_t K, int32_t stride, int32_t pad, int32_t groups,
                                int32_t precision, int device, svb_tc_layer_t **out);
/* 2-D convolutions: Conv2d(Cin, Cout, (KH, KW), stride (SH, SW), padding (PH, PW)) of the mel discriminator
 * (modules/fastspeech/multi_window_disc.py:16-30, 3x3 / stride 2 / padding 1 on 128 -> 128 channels).  One K = 1 GEMM over the
 * Cin*KH*KW im2col channels c*KH*KW + kh*KW + kw (the natural flatten of the [Cout, Cin, KH, KW] weight, which set_weight_dev
 * takes as is).  With this handle the svb_tc_layer_* calls below read T as the height and W as the width of x [B, Cin, T, W]
 * and write y [B, Cout, T', W'],
 *     T' = (T + 2*PH - KH) / SH + 1 (= svb_tc_layer_out_len),   W' = (W + 2*PW - KW) / SW + 1;
 * dy / y of backward are [B, Cout, T', W'], dx [B, Cin, T, W], dw [Cout, Cin, KH, KW].  Needs 2*PH <= KH, 2*PW <= KW and
 * Cin*KH*KW, Cout tensor-core shapes as svb_tc_layer_create (multiples of 32, Cin*KH*KW <= 3072, Cout <= 1024). */
int svb_tc_layer_create_2d(int32_t Cin, int32_t Cout, int32_t KH, int32_t KW, int32_t SH, int32_t SW, int32_t PH, int32_t PW,
                           int32_t precision, int device, svb_tc_layer_t **out);
void svb_tc_layer_destroy(svb_tc_layer_t *layer);
int svb_tc_layer_set_weight_dev(svb_tc_layer_t *layer, const float *w_dev, const float *bias_dev, void *stream);
int64_t svb_tc_layer_out_len(const svb_tc_layer_t *layer, int64_t T);
int svb_tc_layer_forward(svb_tc_layer_t *layer, const float *x_dev, int32_t B, int32_t T, int32_t W, float out_slope,
                         float *y_dev, void *stream);
int svb_tc_layer_backward(svb_tc_layer_t *layer, const float *x_dev, const float *y_dev, const float *dy_dev, int32_t B,
                          int32_t T, int32_t W, float out_slope, float *dx_dev, float *dw_dev, float *db_dev, void *stream);
/* Ragged batches (inference; dense stride-1 layers of svb_tc_layer_create, W = 1): clip b is x[b][:, :len[b]] (1 <= len[b] <= T),
 * its frames past len[b] read as zero whatever they hold, as the clip alone and unpadded sees its padding; y[b][:, len[b]:] is
 * written as zeros.  Only each clip's live 128-row tiles run.  A clip's result is the same bits in any batch, at any row and padded
 * length.  len_host / len_dev: the same int32 [B] on the host (checked, planned) and on the device (read by the kernels). */
int svb_tc_layer_forward_ragged(svb_tc_layer_t *layer, const float *x_dev, int32_t B, int32_t T, const int32_t *len_host,
                                const int32_t *len_dev, float out_slope, float *y_dev, void *stream);

/* ---- mel discriminator (modules/fastspeech/multi_window_disc.py): fp32 operators ------------------------------------
 * svb_conv2d_forward: y[b, co] = scale[b, co] * leaky_relu(conv2d(x, w) + bias, out_slope) on [B, C, H, W] device tensors,
 *   w [Cout, Cin, KH, KW]; H' = (H + 2*PH - KH) / SH + 1, W' likewise; bias and scale [B, Cout] (a Dropout2d mask: 0 or
 *   1/(1-p) per plane) may be NULL.  Needs 2*PH <= KH and 2*PW <= KW.
 * svb_conv2d_backward: y = the forward's output (mask source, may be NULL when out_slope == 1), same scale, dy = gradient
 *   w.r.t. y.  dz_scratch [B, Cout, H', W'] receives the masked gradient; dx is written, dw / db are ACCUMULATED (the caller
 *   zeroes them); each may be NULL.
 * svb_drop_inorm_forward: Dropout2d + InstanceNorm2d(C, affine=True) over planes of N = H*W elements:
 *   u = scale[b, c] * v (scale NULL = all ones), y = gamma[c] (u - mean) / sqrt(var + eps) + beta[c] with the biased variance
 *   of the plane; mean / rstd [B, C] are kept for the backward.  A dropped or constant plane gives beta.
 * svb_drop_inorm_backward: dv (written; may be NULL) and dgamma / dbeta [C] (ACCUMULATED; each may be NULL) from dy.
 * svb_linear1_forward: adv_layer = Linear(N, 1): y[b] = x[b, :] . w + bias[0], x [B, N].
 * svb_linear1_backward: dx [B, N] written, dw [N] / db [1] ACCUMULATED (each may be NULL); dy [B] on the device. */
int svb_conv2d_forward(const float *x_dev, const float *w_dev, const float *bias_dev, const float *scale_dev, float *y_dev, int32_t B,
                       int32_t Cin, int32_t Cout, int32_t H, int32_t W, int32_t KH, int32_t KW, int32_t SH, int32_t SW, int32_t PH,
                       int32_t PW, float out_slope, void *stream);
int svb_conv2d_backward(const float *x_dev, const float *w_dev, const float *y_dev, const float *scale_dev, const float *dy_dev,
                        int32_t B, int32_t Cin, int32_t Cout, int32_t H, int32_t W, int32_t KH, int32_t KW, int32_t SH, int32_t SW,
                        int32_t PH, int32_t PW, float out_slope, float *dz_scratch_dev, float *dx_dev, float *dw_dev, float *db_dev,
                        void *stream);
int svb_drop_inorm_forward(const float *v_dev, const float *scale_dev, const float *gamma_dev, const float *beta_dev, int32_t B,
                           int32_t C, int32_t N, float eps, float *y_dev, float *mean_dev, float *rstd_dev, void *stream);
int svb_drop_inorm_backward(const float *v_dev, const float *scale_dev, const float *gamma_dev, const float *mean_dev,
                            const float *rstd_dev, const float *dy_dev, int32_t B, int32_t C, int32_t N, float *dv_dev,
                            float *dgamma_dev, float *dbeta_dev, void *stream);
int svb_linear1_forward(const float *x_dev, const float *w_dev, const float *bias_dev, int32_t B, int32_t N, float *y_dev,
                        void *stream);
int svb_linear1_backward(const float *x_dev, const float *w_dev, const float *dy_dev, int32_t B, int32_t N, float *dx_dev,
                         float *dw_dev, float *db_dev, void *stream);

/* ---- training: backward of the generator -------------------------------------------------------------
 * Replaces torch autograd through HifiGanGenerator.forward (modules/hifigan/hifigan.py:144-169; ResBlock1/2
 * :54-61 / :81-86; weight_norm :35-50,118,124; SourceModuleHnNSF.l_linear source.py:393-394) for the
 * vocoder training step (SURVEY 8(d) cfg 3).
 *   svb_gen_set_training(g, 1): forwards keep every conv input (the tape), the flipped / transposed weight
 *     packings of the data-gradient convs are built and one gradient buffer per folded tensor is allocated.
 *   svb_gen_backward(g, dwav [B, T*hop]): ACCUMULATES d(loss)/d(folded tensor) for the last forward into those
 *     buffers (svb_gen_zero_grad clears them), in the reference's tensor names and layouts
 *     ("conv_pre.weight" [Cout,Cin,K], "ups.0.weight" [Cin,Cout,K], "noise_convs.0.weight",
 *     "resblocks.3.convs1.0.bias", "conv_post.weight", "m_source.l_linear.weight", ...).
 *   svb_gen_get_grad copies one of them to a device buffer of exactly svb_gen_grad_numel floats.
 *   After an optimizer step: svb_gen_set_weight(...) for the changed tensors, then svb_gen_update_weights(g).
 *   svb_weight_norm_backward: (dv, dg) of w = g * v / ||v|| (norm over all dims but 0) from dw. */
int svb_gen_set_training(svb_gen_t *g, int32_t on);
int svb_gen_update_weights(svb_gen_t *g);
/* Device-side variant (no host round trip): the folded tensor `name` is copied from a device buffer, then ALL
 * kernel packings (forward, data-gradient twins, wgmma tiles) are rebuilt by gather / tile kernels on `stream`.
 * svb_fold_weight_norm_dev: w = g * v / ||v|| on device buffers (hifigan.py:35-50 weight_norm, dim 0). */
int svb_gen_set_weight_dev(svb_gen_t *g, const char *name, const float *src_dev, int64_t n, void *stream);
int svb_gen_update_weights_dev(svb_gen_t *g, void *stream);
int svb_fold_weight_norm_dev(const float *v_dev, const float *g_dev, int64_t d0, int64_t inner, float *w_dev, void *stream);
int svb_gen_zero_grad(svb_gen_t *g, void *stream);
int svb_gen_backward(svb_gen_t *g, const float *dwav_dev, void *stream);
int64_t svb_gen_grad_numel(svb_gen_t *g, const char *name);
int svb_gen_get_grad(svb_gen_t *g, const char *name, float *dst_dev, int64_t n, void *stream);
int64_t svb_gen_bwd_launches(const svb_gen_t *g);
int svb_weight_norm_backward(const float *v_dev, const float *g_dev, const float *dw_dev, int64_t rows, int64_t cols,
                             float *dv_dev, float *dg_dev, void *stream);

/* One convolution layer of the generator on PyTorch-layout device tensors, through the CUDA-core
 * (precision 0) or wgmma (1, 2) kernel -- for kernel-level parity tests and per-layer timing.
 *   y = out_scale * (conv(leaky_relu(x, in_slope)) + bias [+ res])
 *   transposed_stride = 0: Conv1d(Cin, Cout, K, dilation=dil, padding=dil*(K-1)/2), w_host [Cout,Cin,K]
 *                          (F.conv1d; hifigan.py:30-61)
 *   transposed_stride = u: ConvTranspose1d(Cin, Cout, K, stride=u, padding=(K-u)/2), w_host [Cin,Cout,K]
 *                          (F.conv_transpose1d; hifigan.py:122-125)
 * x [B,Cin,T], res / y [B,Cout,T or T*u].  Runs 1 warm-up + `iters` timed launches; *avg_ms = mean
 * CUDA-event time per launch.  Synchronises `stream`. */
int svb_conv1d_run(const float *x_nct_dev, const float *w_host, const float *bias_host, const float *res_nct_dev,
                   int32_t B, int32_t Cin, int32_t Cout, int32_t T, int32_t K, int32_t dil,
                   int32_t transposed_stride, float in_slope, float out_scale, int32_t precision, int32_t iters,
                   float *y_nct_dev, float *avg_ms, void *stream);
/* Backward of the same layer (no residual, out_scale 1) through the launchers and argument mappings of the
 * generator's backward: for y = conv(leaky_relu(x, in_slope)) + bias and dy [B,Cout,T or T*u],
 *   dw_dev [Cout,Cin,K] (transposed: [Cin,Cout,K]) and db_dev [Cout] are ACCUMULATED (device buffers the caller
 *   zeroes), dx_nct_dev [B,Cin,T] is written (the leaky-relu derivative of x included).
 * Stride 1: weight gradient on the wgmma kernel in the tensor-core precisions (split bf16) when the shape allows it,
 * data gradient = the forward kernel of `precision` on the flipped, transposed weights.  Transposed: fp32 kernels.
 * w_host as svb_conv1d_run.  Synchronises `stream`. */
int svb_conv1d_backward_run(const float *x_nct_dev, const float *w_host, const float *dy_nct_dev, int32_t B, int32_t Cin,
                            int32_t Cout, int32_t T, int32_t K, int32_t dil, int32_t transposed_stride, float in_slope,
                            int32_t precision, float *dx_nct_dev, float *dw_dev, float *db_dev, void *stream);

/* ---- discriminator-side operators of the vocoder losses (forward; fp32 CUDA cores) ------------ */

/* y = leaky_relu(conv(x) + bias, out_slope) on PyTorch-layout tensors [B, C, T, W] with W independent inner
 * columns: W = 1 is F.conv1d(stride, dilation, padding, groups) (DiscriminatorS, hifigan.py:262-271);
 * W = period is the (K,1)-kernel / (stride,1)-stride Conv2d of DiscriminatorP (hifigan.py:193-200).
 * w_dev [Cout, Cin/groups, K], bias_dev [Cout] or NULL; Tout = (Tin + 2*pad - dil*(K-1) - 1)/stride + 1. */
int svb_conv_nct_forward(const float *x_dev, const float *w_dev, const float *bias_dev, float *y_dev, int32_t B,
                         int32_t Cin, int32_t Cout, int32_t Tin, int32_t W, int32_t K, int32_t stride, int32_t dil,
                         int32_t pad, int32_t groups, float out_slope, void *stream);
/* svb_conv_nct_forward on a ragged batch (inference, W = 1), with svb_tc_layer_forward_ragged's contract: clip b is
 * x[b][:, :len[b]]; its output has (len[b] + 2*pad - dil*(K-1) - 1)/stride + 1 frames (>= 1), the frames after them are zeros. */
int svb_conv_nct_forward_ragged(const float *x_dev, const float *w_dev, const float *bias_dev, float *y_dev, int32_t B, int32_t Cin,
                                int32_t Cout, int32_t Tin, int32_t K, int32_t stride, int32_t dil, int32_t pad, int32_t groups,
                                float out_slope, const int32_t *len_host, const int32_t *len_dev, void *stream);
/* AvgPool1d(4, 2, padding=1) over the last dim of [rows, Tin] (MultiScaleDiscriminator.meanpools, hifigan.py:304-307) */
int svb_avgpool1d_4_2_1(const float *x_dev, float *y_dev, int64_t rows, int32_t Tin, void *stream);
/* F.pad(x, (0, Tpad - T), 'reflect') over the last dim of [rows, T] (DiscriminatorP.forward, hifigan.py:209-212) */
int svb_pad_reflect_right(const float *x_dev, float *y_dev, int64_t rows, int32_t T, int32_t Tpad, void *stream);
/* out6_dev (double[6]) = { sum (a-b)^2, sum a^2, sum |ln a - ln b| (if want_log), sum |a-b|, sum (1-a)^2, sum b^2 }
 * -- the reductions behind feature_loss / discriminator_loss / generator_loss (hifigan.py:328-365) and the
 * spectral-convergence / log-magnitude STFT losses (losses/stft_loss.py:34-73).  b_dev may be NULL. */
int svb_pair_stats(const float *a_dev, const float *b_dev, int64_t n, int32_t want_log, double *out6_dev, void *stream);
/* sigma = u . (W v) of torch.nn.utils.spectral_norm in eval mode (no power iteration), W [rows, inner] */
int svb_spectral_sigma_host(const float *w_host, const float *u_host, const float *v_host, int64_t rows, int64_t inner,
                            int device, float *sigma);

/* ---- STFT / mel front end ------------------------------------------------------------------ */

typedef enum svb_pad_mode {
    SVB_PAD_CENTER_ZERO = 0,    /* librosa.stft(center=True, pad_mode='constant'): data_gen_utils.py:123-124 */
    SVB_PAD_CENTER_REFLECT = 1, /* torch.stft(center=True) default: losses/stft_loss.py:26                   */
    SVB_PAD_HALF_REFLECT = 2    /* reflect-pad (n_fft-hop)/2 then center=False: mel_utils.py:66-71           */
} svb_pad_mode;

typedef enum svb_spec_out {
    SVB_OUT_LOG10_MEL = 0,      /* log10(max(eps, mel_basis @ |X|))              data_gen_utils.py:125-134   */
    SVB_OUT_LN_MEL = 1,         /* ln(max(eps, mel_basis @ sqrt(|X|^2 + 1e-9)))  mel_utils.py:74-76,23-24     */
    SVB_OUT_MAG = 2,            /* sqrt(max(|X|^2, floor))                       losses/stft_loss.py:31       */
    SVB_OUT_MAG_RAW = 3,        /* |X|                                           data_gen_utils.py:125        */
    SVB_OUT_MEL_MAG = 4         /* mel_basis @ sqrt(max(|X|^2, floor)), no log   parallel_wavegan/stft_loss.py:40-47 (use_mel_loss) */
} svb_spec_out;

typedef struct svb_stft_config {
    int32_t n_fft;              /* power of two, 64..4096                         */
    int32_t hop;
    int32_t win;                /* periodic hann(win) centred in n_fft            */
    int32_t pad_mode;           /* svb_pad_mode                                   */
    int32_t out_kind;           /* svb_spec_out                                   */
    int32_t clamp_input;        /* clamp(y, -1, 1) first (mel_utils.py:59)        */
    int32_t n_mels;             /* rows of mel_basis (mel outputs only)           */
    int32_t frames_major;       /* 1: out [B, frames, n_out]; 0: out [B, n_out, frames] */
    float eps;                  /* log floor (1e-10 / 1e-5) or magnitude floor (1e-7) */
} svb_stft_config;

/* number of frames the reference produces for `n` samples under cfg (bit-exact frame indexing):
 *   CENTER_*: 1 + n / hop ; HALF_REFLECT: 1 + (n + 2*((n_fft-hop)/2) - n_fft) / hop */
int64_t svb_stft_num_frames(const svb_stft_config *cfg, int64_t n);

/* wav_dev [B, n]; mel_basis_dev [n_mels, n_fft/2+1] (NULL for magnitude outputs);
 * out_dev [B, frames, n_out] or [B, n_out, frames]  (n_out = n_mels or n_fft/2+1). */
int svb_stft_forward(const svb_stft_config *cfg, const float *wav_dev, int32_t B, int64_t n,
                     const float *mel_basis_dev, float *out_dev, void *stream);
/* Backward of svb_stft_forward (torch autograd through torch.stft + magnitude [+ mel + log] in
 * mel_spectrogram, modules/hifigan/mel_utils.py:59-76, and stft(), modules/parallel_wavegan/losses/stft_loss.py:26-31):
 * dout = gradient w.r.t. the forward's output (same layout); the gradient w.r.t. the waveform is ACCUMULATED into
 * dwav [B, n] (atomics; the caller zeroes it).  The spectrum is recomputed per frame, nothing is kept from forward. */
int svb_stft_backward(const svb_stft_config *cfg, const float *wav_dev, int32_t B, int64_t n, const float *mel_basis_dev,
                      const float *dout_dev, float *dwav_dev, void *stream);

/* Spectral-subtraction post-filter of the vocoder output (vocoders/vocoder_utils.py:7-15, applied by
 * vocoders/hifigan.py:66-69 when hparams['vocoder_denoise_c'] > 0):  librosa.stft(n_fft, hop, win, pad 'constant') ->
 * max(|X| - v, 0) with the phase kept -> librosa.istft(hop, win).  wav [B, n] -> out [B, hop * (n / hop)] (device).
 * Only n_fft / hop / win of cfg are read. */
int svb_denoise(const svb_stft_config *cfg, const float *wav_dev, int32_t B, int64_t n, float v, float *out_dev, void *stream);

/* PWG.wav2spec / process_utterance (vocoders/pwg.py:105-122, data_gen_utils.py:93-147) at the binarizer's call site
 * (data_gen/tts/base_binarizer.py:168-178, data_gen/singing/binarize_para.py:116-217 call wav2spec once per file from a CPU
 * process pool) as ONE call over a ragged batch on device memory, with no copy of the samples and no synchronisation.
 * wav_concat_dev: the clips back to back (lengths: host array); mel_basis_dev [n_mels, n_fft/2+1]; mel_concat_dev receives the
 * [frames_c, n_mels] log10-mels back to back (1 + lengths[c] / hop frames each), wav_out_dev (NULL = not wanted) every clip
 * zero-padded on the right to frames_c * hop samples (audio.librosa_pad_lr, utils/audio.py:67-76), back to back (what wav2spec
 * returns as its waveform, in the layout svb_pitch_ac_batch takes).  One kernel launch over all frames of all clips.  The only copy is the small clip table, into
 * the caller-owned workspace of svb_wav2spec_workspace_bytes bytes.  Both reject before any launch (SVB_ERR_INVALID) a bad config,
 * an empty clip, a null buffer or a short workspace; frames_out (NULL = not wanted) receives the frame counts.  svb_wav2spec_batch
 * returns the total frame count, svb_wav2spec_workspace_bytes the workspace size, or a negative status. */
int64_t svb_wav2spec_workspace_bytes(const svb_stft_config *cfg, const int64_t *lengths, int32_t n_clips, int64_t *frames_out);
int64_t svb_wav2spec_batch(const svb_stft_config *cfg, const float *wav_concat_dev, const int64_t *lengths, int32_t n_clips,
                           const float *mel_basis_dev, float *mel_concat_dev, float *wav_out_dev, int64_t *frames_out,
                           void *workspace_dev, int64_t workspace_bytes, void *stream);

/* ---- SVB acoustic step, first piece (SURVEY 8(f) N1): the WN gated dilated-conv stack of the GlobalFVAE
 * (modules/fastspeech/fs2_vae.py:19-91; built by modules/voice_conversion/vae_models.py:81-146 with hidden 192,
 * kernel 5, dilation_rate 1, 4 decoder / 8 encoder layers).  Inference (eval mode: dropout is the identity).
 * Weights are the FOLDED ones (WN.remove_weight_norm, fs2_vae.py:96-103), set by the reference's state_dict names:
 *   in_layers.{i}.weight [2H, H, K] / .bias [2H];  res_skip_layers.{i}.weight [2H (H on the last layer), H, 1] / .bias;
 *   cond_layer.weight [2*H*n_layers, gin, 1] / .bias  (when gin_channels > 0). */
typedef struct svb_wn svb_wn_t;
int svb_wn_create(int32_t hidden_channels, int32_t kernel_size, int32_t dilation_rate, int32_t n_layers, int32_t gin_channels,
                  int32_t precision, int32_t device, svb_wn_t **out);
void svb_wn_destroy(svb_wn_t *w);
int svb_wn_set_weight(svb_wn_t *w, const char *name, const float *data_host, const int64_t *shape, int32_t ndim);
int svb_wn_finalize(svb_wn_t *w);
/* WN.forward(x, x_mask, g) (fs2_vae.py:62-94) on device tensors in the reference's layout: x [B, H, T], mask [B, T]
 * (x_mask[:, 0, :], NULL = all ones), g [B, gin, T] (NULL = unconditioned) -> out [B, H, T]. */
int svb_wn_forward(svb_wn_t *w, const float *x_dev, const float *mask_dev, const float *g_dev, int32_t B, int32_t T, float *out_dev,
                   void *stream);
/* FVAEDecoder / GlobalFVAEDecoder (modules/fastspeech/fs2_vae.py:130-152, modules/voice_conversion/vae_models.py:108-128): the mel
 * decoder whose output `spec2wav` consumes -- pre_net ConvTranspose1d(latent, H, k = stride, stride) -> * mask -> WN(dilation_rate 1)
 * -> * mask -> out_proj Conv1d(H, out, 1).  Same handle type as WN; additional weights `pre_net.0.weight [latent, H, stride]`,
 * `pre_net.0.bias`, `out_proj.weight [out, H, 1]`, `out_proj.bias` (svb_wn_set_weight), WN weights under their plain names.
 * forward: z [B, latent, T / stride], mask [B, T] or NULL, g [B, gin, T] or NULL -> out [B, out_channels, T]. */
int svb_fvae_decoder_create(int32_t latent_channels, int32_t hidden_channels, int32_t out_channels, int32_t kernel_size, int32_t n_layers,
                            int32_t gin_channels, int32_t stride, int32_t precision, int32_t device, svb_wn_t **out);
int svb_fvae_decoder_forward(svb_wn_t *w, const float *z_dev, const float *mask_dev, const float *g_dev, int32_t B, int32_t T,
                             float *out_dev, void *stream);
/* Training of a WN / decoder handle (replaces torch autograd through fs2_vae.py:62-94 / :147-152).
 *   svb_wn_set_training(w, 1): builds the data-gradient packings, one gradient buffer per folded tensor (the names of
 *     svb_wn_set_weight) and a device copy of every folded tensor; set_training(w, 0) keeps them (eval forwards between steps).
 *   The tape is CALLER-OWNED, one per call, so several training forwards may run before their backwards:
 *     svb_wn_tape_bytes(w, B, T) is its size (-1 on a bad argument); svb_wn_forward_train / svb_fvae_decoder_forward_train
 *     compute what svb_wn_forward / svb_fvae_decoder_forward compute (bit for bit) and fill the tape;
 *     svb_wn_backward / svb_fvae_decoder_backward(w, tape, B, T, dout, ...) read it back.  B and T must be those of the
 *     forward that wrote the tape.  dx [B, H, T] / dz [B, latent, T / stride] / dg [B, gin, T] are written (each may be NULL;
 *     dg needs a conditioned forward); the weight / bias gradients ACCUMULATE (svb_wn_zero_grad clears them).
 *   svb_wn_get_grad copies one gradient to a device buffer of exactly svb_wn_grad_numel(w, name) floats.
 *   After an optimizer step: svb_wn_set_weight_dev(w, name, folded tensor) for the changed tensors, then
 *     svb_wn_update_weights_dev(w) rebuilds every packing (forward, data-gradient twins, wgmma tiles) on the device. */
int svb_wn_set_training(svb_wn_t *w, int32_t on);
int64_t svb_wn_tape_bytes(const svb_wn_t *w, int32_t B, int32_t T);
int svb_wn_forward_train(svb_wn_t *w, const float *x_dev, const float *mask_dev, const float *g_dev, int32_t B, int32_t T,
                         float *out_dev, void *tape_dev, void *stream);
int svb_fvae_decoder_forward_train(svb_wn_t *w, const float *z_dev, const float *mask_dev, const float *g_dev, int32_t B, int32_t T,
                                   float *out_dev, void *tape_dev, void *stream);
int svb_wn_backward(svb_wn_t *w, const void *tape_dev, int32_t B, int32_t T, const float *dout_dev, float *dx_dev, float *dg_dev,
                    void *stream);
int svb_fvae_decoder_backward(svb_wn_t *w, const void *tape_dev, int32_t B, int32_t T, const float *dout_dev, float *dz_dev,
                              float *dg_dev, void *stream);
int svb_wn_zero_grad(svb_wn_t *w, void *stream);
int64_t svb_wn_grad_numel(const svb_wn_t *w, const char *name);
int svb_wn_get_grad(svb_wn_t *w, const char *name, float *dst_dev, int64_t n, void *stream);
int svb_wn_set_weight_dev(svb_wn_t *w, const char *name, const float *src_dev, int64_t n, void *stream);
int svb_wn_update_weights_dev(svb_wn_t *w, void *stream);

/* ---- PPG extractor (VCASR, modules/voice_conversion/vc_modules.py:56-80) pieces that are not convolutions, on [B, C, T] tensors.
 * nn.LayerNorm(C) of EncoderLayer (modules/fastspeech/conformer/layers.py:167-178): statistics over the channel axis per (b, t). */
int svb_layer_norm_nct(const float *x_dev, const float *gamma_dev, const float *beta_dev, int32_t B, int32_t C, int32_t T, float eps,
                       float *y_dev, void *stream);
/* RelPositionMultiHeadedAttention.forward after its linear projections (modules/commons/espnet_transformer_attn.py:147-186, with
 * rel_shift :127-145 and forward_attention :59-88): q, k, v [B, C, T] (head h = channels [h*dk, (h+1)*dk)), p = linear_pos(pos_emb)
 * [C, T], pos_bias_u / pos_bias_v [n_head * dk], mask [B, T] (0 = padded key; NULL = none) -> context [B, C, T] (before linear_out). */
int svb_relpos_attention_nct(const float *q_dev, const float *k_dev, const float *v_dev, const float *p_dev, const float *bias_u_dev,
                             const float *bias_v_dev, const float *mask_dev, int32_t B, int32_t C, int32_t T, int32_t n_head,
                             float *out_dev, void *stream);
/* The same on a ragged batch: clip b is computed as alone at T = len[b] (1 <= len[b] <= T; its keys, queries and position rows),
 * its rows past len[b] are written as zeros.  len_host / len_dev as svb_tc_layer_forward_ragged. */
int svb_relpos_attention_nct_ragged(const float *q_dev, const float *k_dev, const float *v_dev, const float *p_dev,
                                    const float *bias_u_dev, const float *bias_v_dev, const float *mask_dev, int32_t B, int32_t C,
                                    int32_t T, int32_t n_head, const int32_t *len_host, const int32_t *len_dev, float *out_dev,
                                    void *stream);

/* ---- Length-aware reductions of the SVB acoustic model (MleSVBVAE with per-clip frame counts; csrc/acoustic_ragged.cu).  Each
 * clip is reduced over its own frames in an order that depends only on its frame count and the channel shape.
 * y = x + relu(GroupNorm(groups, C)(h)) over clip b's first len[b] frames of [B, C, T] tensors (ConvStacks' ConvBlock, norm 'gn'),
 * statistics in float32 over those frames only; y[b][:, len[b]:] = 0. */
int svb_group_norm_relu_add_ragged(const float *x_dev, const float *h_dev, const float *gamma_dev, const float *beta_dev, int32_t B,
                                   int32_t C, int32_t T, int32_t groups, float eps, const int32_t *len_host, const int32_t *len_dev,
                                   float *y_dev, void *stream);
/* The GlobalFVAEEncoder's head (vae_models.py:102-104) on the last pooling's output x [B, 2*latent, T]: per clip the mean over its
 * first n3 frames, n3 = its encoder frame count enc_len[b] through three valid k = 3 stride-2 convolutions (n -> (n - 3)/2 + 1,
 * 1 <= n3 <= T), split into m / logs [B, latent] and z = m + eps * exp(logs) (eps [B, latent]). */
int svb_global_latent_head_ragged(const float *x_dev, int32_t B, int32_t latent, int32_t T, const int32_t *enc_len_host,
                                  const int32_t *enc_len_dev, const float *eps_dev, float *m_dev, float *logs_dev, float *z_dev,
                                  void *stream);

/* ---- Mel reconstruction loss of the SVB acoustic step (the `ssim:0.5|l1:0.5` recipe: FastSpeech2Task.l1_loss and
 * ssim_loss(bias), tasks/tts/fs2.py:158-175, ssim(..., size_average=False), modules/commons/ssim.py:319-351).
 * pred / target [B, T, M] (M <= 128); a frame's weight is 1 when its target row has a non-zero element, else 0:
 *   l1 = sum w |pred - target| / sum w,   ssim = sum w (1 - SSIM(pred + bias, target + bias)) / sum w   (sums over B*T*M pixels)
 * with the 11x11 Gaussian window (sigma 1.5) over the whole [T, M] image (padding frames included), zero padding outside it.
 * svb_mel_loss_workspace_bytes: size of the caller-owned partial-sum buffer (-1 on a bad shape).
 * svb_mel_loss_forward writes out3_dev (double[3]) = {l1, ssim, sum w}; NaN for both losses when sum w = 0, like the reference.
 * svb_mel_loss_backward writes dpred = g_l1 * d l1 / d pred + g_ssim * d ssim / d pred, reading the upstream gradients from the
 * device scalars g_l1_dev / g_ssim_dev (NULL = 0) and sum w from the forward's out3_dev.  No gradient to the target. */
int64_t svb_mel_loss_workspace_bytes(int32_t B, int32_t T, int32_t M);
int svb_mel_loss_forward(const float *pred_dev, const float *target_dev, int32_t B, int32_t T, int32_t M, float bias,
                         double *workspace_dev, double *out3_dev, void *stream);
int svb_mel_loss_backward(const float *pred_dev, const float *target_dev, int32_t B, int32_t T, int32_t M, float bias,
                          const double *out3_dev, const float *g_l1_dev, const float *g_ssim_dev, float *dpred_dev, void *stream);

/* ---- Shape-aware DTW pitch alignment (csrc/sadtw.cu): SADTW (modules/voice_conversion/dtw/shape_aware_dtw.py) and EHSADTW
 * (enhance_sadtw.py) over time_warp / align_from_distances (align.py).  A batch of n pairs is ragged: the amateur f0 of every pair
 * concatenated in src_f0_dev (pair p has src_len[p] frames), the professional f0 in tgt_f0_dev (tgt_len[p] frames), float32 or
 * float64 (dtype), lengths on the host.  The professional histogram uses the scale factor tgt_scale[p] (NULL: tgt_len / src_len,
 * cal_shape_dist's), the amateur one 1.0.
 * svb_sadtw_workspace_bytes: size of the caller-owned workspace (-1 on bad lengths); offsets_host (5 entries, NULL = not wanted)
 *   receives the byte offsets of its sections: [0] per-sequence and [1] per-pair metadata, [2] histograms float32 [rows, 48] (the
 *   amateur frames of all pairs, then the professional ones), [3] costs float32 and [4] direction bytes (0 up, 1 left, 2 diagonal),
 *   pair p's R x C cells (R = tgt_len[p], C = src_len[p]) after those of the pairs before it, anti-diagonal-major: cell (i, j) at
 *   (number of cells with i' + j' < i + j) + i - max(0, i + j - C + 1).
 * svb_sadtw_align writes alignment_dev int64 [sum tgt_len] (pair p's rows after the pairs before it): for each professional frame the
 *   amateur frame align_from_distances picks; path_cost_dev (NULL = not wanted) float32 [n] = the pair's DTW value at its last cell.
 *   stage_ms_host (NULL = not wanted) receives 4 CUDA-event times (histogram, cost, DTW, backtrack) and makes the call synchronise.
 *   Rejected before any launch (SVB_ERR_INVALID): a length below 2, min(S, T) > 8192, a frame whose slope windows are all empty
 *   after scaling (the reference divides by zero), a bad dtype / variant / scale or a short workspace.  f0 must be finite (the
 *   reference exits otherwise); that is the caller's check. */
typedef enum svb_sadtw_variant { SVB_SADTW = 0, SVB_EHSADTW = 1 } svb_sadtw_variant;
typedef enum svb_sadtw_dtype { SVB_SADTW_F32 = 0, SVB_SADTW_F64 = 1 } svb_sadtw_dtype;
int64_t svb_sadtw_workspace_bytes(int32_t n_pairs, const int32_t *src_len_host, const int32_t *tgt_len_host, int64_t *offsets_host);
int svb_sadtw_align(const void *src_f0_dev, const void *tgt_f0_dev, int32_t dtype, int32_t variant, int32_t n_pairs,
                    const int32_t *src_len_host, const int32_t *tgt_len_host, const double *tgt_scale_host, void *workspace_dev,
                    int64_t workspace_bytes, int64_t *alignment_dev, float *path_cost_dev, float *stage_ms_host, void *stream);
/* Whole songs: svb_sadtw_long_workspace_bytes / svb_sadtw_align_long take the arguments of svb_sadtw_workspace_bytes /
 * svb_sadtw_align and compute the same results, with each take of a pair at most 65536 frames (6.3 min at 22.05 kHz / hop 128)
 * and no bound on min(S, T) below that.  A pair with min(S, T) <= 8192 runs on the one-CTA DTW kernel as in svb_sadtw_align; a
 * longer one on ceil(min(S, T) / 8192) CTAs (at most 8) of a thread-block cluster, each holding its share of the three live
 * anti-diagonals and reading its neighbours' edge cells through distributed shared memory.  Alignment and path cost are
 * bit-identical to the one-CTA kernel's on any pair both can run.  The workspace is the same layout, 4 B of cost plus 1 B of
 * direction per cell: 8.5 GB for a 4-minute pair (41 344 x 41 344 frames), 21.5 GB at 65536 x 65536.  A pair over 65536 frames
 * on either side is refused (SVB_ERR_INVALID, -1 from the size query) before any launch.  The environment variable
 * SVB_DTW_CTA_CELLS=<1 .. 8192>, read per call, replaces the 8192-cell share (clusters still at most 8 CTAs, so a share grows to
 * ceil(min(S, T) / 8) when it would need more): a test and measurement hook that puts shorter pairs on clusters. */
int64_t svb_sadtw_long_workspace_bytes(int32_t n_pairs, const int32_t *src_len_host, const int32_t *tgt_len_host, int64_t *offsets_host);
int svb_sadtw_align_long(const void *src_f0_dev, const void *tgt_f0_dev, int32_t dtype, int32_t variant, int32_t n_pairs,
                         const int32_t *src_len_host, const int32_t *tgt_len_host, const double *tgt_scale_host, void *workspace_dev,
                         int64_t workspace_bytes, int64_t *alignment_dev, float *path_cost_dev, float *stage_ms_host, void *stream);
/* Whole songs in bounded device memory: svb_sadtw_align_striped computes what svb_sadtw_align_long computes, bit for bit (same
 * arguments and limits, plus budget_bytes), in a workspace of at most budget_bytes.  Every pair's anti-diagonals are cut into
 * stripes of K diagonals; a stripe's cost is computed into one of two stripe buffers (K x min(S, T) floats per pair) on a side
 * stream while the DTW runs the stripe before it on the caller's stream, starting from the two diagonals before the stripe (a
 * checkpoint slot of 2 x min(S, T) floats per pair).
 *   SVB_SADTW_SINGLE_PASS: one forward pass writes every direction byte (S x T bytes per pair, the skewed layout), then the
 *     backtrack runs once.  Chosen when it fits the budget, at K = min(512, longest S + T - 1).
 *   SVB_SADTW_CHECKPOINTED: the forward pass keeps the last two diagonals of every stripe and no direction; the backward pass
 *     recomputes each stripe's cost and DTW from the last stripe to the first, with stripe-local directions (K x min(S, T) bytes
 *     per pair), and continues the backtrack over it.  About twice the work; memory linear in length.  K is the largest power of
 *     two <= 8192 that fits the budget.
 * svb_sadtw_striped_plan (host only, no CUDA call) fills *plan for these lengths and budget: the mode, K, the stripe count
 *   ceil(max(S + T - 1) / K), the section offsets [seq metas, pair metas, stripe metas, histograms, 2 stripe cost buffers,
 *   directions, checkpoint slots (ceil((S + T - 1) / K) per pair, 1 in single pass), walk states (16 B per pair)], the total
 *   (the workspace svb_sadtw_align_striped needs) and the smallest budget it would accept.  It validates the lengths as
 *   svb_sadtw_long_workspace_bytes does and refuses (SVB_ERR_INVALID) a budget below that minimum, naming it.  The environment
 *   variable SVB_DTW_STRIPE_DIAGS=<1 .. 131072>, read per call, forces the checkpointed mode at that K (a test and measurement
 *   hook); a forced K whose workspace exceeds the budget is refused.  SVB_DTW_CTA_CELLS acts as in svb_sadtw_align_long.
 * svb_sadtw_align_striped refuses a workspace smaller than the plan's total.  stage_ms_host receives (histogram, forward,
 *   backward, backtrack): forward is the caller's stream from the end of the histograms to the last stripe's DTW, which includes
 *   waiting for stripe costs not hidden under the DTW; backward is the checkpointed backward pass (costs, DTW and backtrack
 *   stripe by stripe; 0 in single pass), backtrack the single pass's backtrack (0 when checkpointed). */
typedef enum svb_sadtw_stripe_mode { SVB_SADTW_SINGLE_PASS = 0, SVB_SADTW_CHECKPOINTED = 1 } svb_sadtw_stripe_mode;
typedef struct svb_sadtw_stripe_plan {
    int32_t mode, stripe_diags, stripes, reserved;
    int64_t offsets[8];
    int64_t total_bytes, min_budget_bytes;
} svb_sadtw_stripe_plan;
int svb_sadtw_striped_plan(int32_t n_pairs, const int32_t *src_len_host, const int32_t *tgt_len_host, int64_t budget_bytes,
                           svb_sadtw_stripe_plan *plan);
int svb_sadtw_align_striped(const void *src_f0_dev, const void *tgt_f0_dev, int32_t dtype, int32_t variant, int32_t n_pairs,
                            const int32_t *src_len_host, const int32_t *tgt_len_host, const double *tgt_scale_host, void *workspace_dev,
                            int64_t workspace_bytes, int64_t budget_bytes, int64_t *alignment_dev, float *path_cost_dev,
                            float *stage_ms_host, void *stream);
/* The histogram kernel alone (cal_hist_of_f0(f, max_window=64, scale_factor=scale[k])): n_seq sequences concatenated in f0_dev,
 * hist_dev float32 [sum len, 48] = k / total (normalize_hist=True), counts_dev int32 [sum len, 48] = k (NULL = not wanted).
 * The workspace holds the per-sequence metadata (svb_sadtw_histogram_workspace_bytes). */
int64_t svb_sadtw_histogram_workspace_bytes(int32_t n_seq);
int svb_sadtw_histogram(const void *f0_dev, int32_t dtype, int32_t variant, int32_t n_seq, const int32_t *len_host, const double *scale_host,
                        void *workspace_dev, int64_t workspace_bytes, float *hist_dev, int32_t *counts_dev, void *stream);
/* cal_hist_dist(hist_a, hist_b): dist_dev float32 [n_a, n_b] row-major, sum_m 0.5 (b_m - a_m)^2 / (b_m + a_m + 1e-8) over the 48
 * bins in order.  Histograms float32 [n, 48], 16-byte aligned. */
int svb_sadtw_cost(const float *hist_a_dev, int32_t n_a, const float *hist_b_dev, int32_t n_b, float *dist_dev, void *stream);
/* time_warp / align_from_distances on an arbitrary cost [rows, cols] (row-major, float32 or float64; min(rows, cols) <= 8192):
 * alignment_dev int64 [rows] (NULL = not wanted), path_cost_dev one element of the cost's type (NULL = not wanted), dtw_dev the
 * whole DTW matrix [rows, cols] in the cost's type (NULL = not wanted).  svb_dtw_workspace_bytes: -1 on a bad shape. */
int64_t svb_dtw_workspace_bytes(int32_t dtype, int32_t rows, int32_t cols);
int svb_dtw_align(const void *cost_dev, int32_t dtype, int32_t rows, int32_t cols, void *workspace_dev, int64_t workspace_bytes,
                  int64_t *alignment_dev, void *path_cost_dev, void *dtw_dev, void *stream);

/* ---- Baseline pitch alignments of the paper's comparison (csrc/sadtw.cu): LoNDTW (modules/voice_conversion/dtw/local_norm_dtw.py),
 * NaiveDTW / ZMNaiveDTW / NNaiveDTW (naive_dtw.py) over time_warp / align_from_distances, and NInterpo (naive_interpo.py).  Batches
 * are ragged as in svb_sadtw_align: src_dev holds the amateur rows of every pair, tgt_dev the professional ones, float32 or float64
 * (dtype, svb_sadtw_dtype), each row feat_dim values (NaiveDTW: 1 .. 4096; every other method aligns 1-D f0: 1).  The cost is
 * torch.cdist's in the input's type: its matrix-product form sqrt(clamp_min(((sum_k -2 x_k y_k) + |x|^2) + |y|^2, 0)) summed in order
 * k = 0, 1, ..., or, when both sides have at most 25 frames, sqrt(sum_k (x_k - y_k)^2).  NInterpo maps professional frame i to
 * amateur frame min(floor(float(i) * (float(S) / T)), S - 1) (F.interpolate(mode='nearest')) and runs no DTW.
 * svb_dtw_baselines_workspace_bytes: size of the caller-owned workspace (-1 on a bad method, dtype or length).
 * svb_dtw_baselines_align writes alignment_dev int64 [sum tgt_len] as svb_sadtw_align does; path_cost_dev (NULL = not wanted; not
 *   written by NInterpo) [n] in the input's type = the pair's DTW value at its last cell; stage_ms_host (NULL = not wanted) receives
 *   4 CUDA-event times (per-frame features, cost, DTW, backtrack) and makes the call synchronise.
 * svb_dtw_baselines_cost writes the cost alone, pair p's cdist matrix [src_len[p], tgt_len[p]] row-major after those of the pairs
 *   before it, in the input's type (NInterpo is refused).
 * Both reject before any launch (SVB_ERR_INVALID): a null pointer, a bad dtype, method or feat_dim, a length below 2, min(S, T) >
 * 8192 for a DTW method, or a short workspace. */
typedef enum svb_dtw_baseline {
    SVB_LONDTW = 0, SVB_NAIVEDTW = 1, SVB_ZMNAIVEDTW = 2, SVB_NNAIVEDTW = 3, SVB_NINTERPO = 4
} svb_dtw_baseline;
int64_t svb_dtw_baselines_workspace_bytes(int32_t method, int32_t dtype, int32_t n_pairs, const int32_t *src_len_host,
                                          const int32_t *tgt_len_host);
int svb_dtw_baselines_align(const void *src_dev, const void *tgt_dev, int32_t dtype, int32_t method, int32_t n_pairs,
                            const int32_t *src_len_host, const int32_t *tgt_len_host, int32_t feat_dim, void *workspace_dev,
                            int64_t workspace_bytes, int64_t *alignment_dev, void *path_cost_dev, float *stage_ms_host, void *stream);
int svb_dtw_baselines_cost(const void *src_dev, const void *tgt_dev, int32_t dtype, int32_t method, int32_t n_pairs,
                           const int32_t *src_len_host, const int32_t *tgt_len_host, int32_t feat_dim, void *workspace_dev,
                           int64_t workspace_bytes, void *cost_dev, void *stream);

/* ---- Autocorrelation pitch tracker (csrc/pitch_ac.cu): the f0 of the binarizer's get_pitch (data_gen/tts/data_gen_utils.py:150-184),
 * Boersma's method as Praat's "To Pitch (ac)" describes it; oracle/pitch_ac.py states every step.  A batch is ragged: n_clips
 * float32 waveforms concatenated (clip c has lengths[c] samples, host array), each analysed on its own grid of
 * floor((N / sr - 3 / floor) / time_step) + 1 frames, and the path's f0 placed into mel_frames[c] output frames (lpad zero frames in
 * front, then cut, or extended with the last value), the clips' outputs back to back.  time_step must be hop / sr.
 * svb_pitch_ac_workspace_bytes: size of the caller-owned workspace (-1 on a bad config or length); frames_out (NULL = not wanted)
 *   receives each clip's analysis frame count.
 * svb_pitch_ac_batch (device pointers): f0_out_dev float32 [sum mel_frames]; cand_dev (NULL = not wanted) float32 [frames, 15, 2] =
 *   (frequency, strength) of the unvoiced candidate then the voiced ones strongest first (unused: (0, -inf)); count_dev int32 [frames];
 *   r_dev float32 [frames, tau_max + 2] = the normalised autocorrelation r(tau); stage_ms_host (NULL = not wanted) receives 3 CUDA-event
 *   times (clip statistics, candidates, path) and makes the call synchronise.
 * All reject before any launch (SVB_ERR_INVALID): a null pointer, a bad config, a clip shorter than one window, a short workspace. */
typedef struct svb_pitch_config {
    int32_t sr;
    int32_t hop;
    double floor;                  /* Hz (80)                                 */
    double ceiling;                /* Hz (750)                                */
    double time_step;              /* s, hop / sr                             */
    double voicing_threshold;      /* 0.6                                     */
    double silence_threshold;      /* 0.03                                    */
    double octave_cost;            /* 0.01                                    */
    double octave_jump_cost;       /* 0.35                                    */
    double voiced_unvoiced_cost;   /* 0.14                                    */
    int32_t lpad;                  /* zero frames placed in front (2 pad_size) */
    int32_t reserved;
} svb_pitch_config;
int64_t svb_pitch_ac_workspace_bytes(const svb_pitch_config *cfg, const int64_t *lengths, int32_t n_clips, int32_t *frames_out);
int svb_pitch_ac_batch(const svb_pitch_config *cfg, const float *wav_concat_dev, const int64_t *lengths, int32_t n_clips,
                       const int64_t *mel_frames, float *f0_out_dev, void *workspace_dev, int64_t workspace_bytes, float *cand_dev,
                       int32_t *count_dev, float *r_dev, float *stage_ms_host, void *stream);

/* ---- Resampling (csrc/resample.cu): librosa.core.load(path, sr=target)'s resampy kaiser_best resampler (reference
 * data_gen/tts/data_gen_utils.py:111); oracle/resample.py states every step.  A batch is ragged: n_clips float32 waveforms concatenated
 * (clip c has lengths[c] samples at src_sr[c] Hz, host arrays; rates may differ within a batch), one target rate per call.  Clip c
 * yields out_lengths[c] = ceil(lengths[c] ratio) samples (int(lengths[c] ratio) filtered ones, then fix_length zeros), the clips'
 * outputs back to back; a clip already at target_sr is copied.  win_host: the filter's float64 right wing (nwin taps, num_table per
 * zero crossing: 32769 and 512 for kaiser_best), scaled and differenced here per source rate.
 * svb_resample_plan: size of the caller-owned workspace, -1 on a bad rate, a clip that yields no sample, or a ratio below
 *   1 / num_table; res_lengths_out / out_lengths_out (NULL = not wanted) receive each clip's lengths before and after the padding.
 *   No CUDA call.
 * svb_resample_batch (device pointers): out_dev float32 [sum out_lengths]; stage_ms_host (NULL = not wanted) receives 2 CUDA-event
 *   times (time register, filter) and makes the call synchronise.
 * All reject before any launch (SVB_ERR_INVALID): a null pointer, a bad rate or length, a short workspace. */
int64_t svb_resample_plan(int32_t target_sr, const int32_t *src_sr, const int64_t *lengths, int32_t n_clips, int32_t nwin,
                          int32_t num_table, int64_t *res_lengths_out, int64_t *out_lengths_out);
int svb_resample_batch(int32_t target_sr, const int32_t *src_sr, const int64_t *lengths, int32_t n_clips, const double *win_host,
                       int32_t nwin, int32_t num_table, const float *wav_concat_dev, float *out_dev, void *workspace_dev,
                       int64_t workspace_bytes, float *stage_ms_host, void *stream);

/* ---- FLAC decoding (csrc/flac.cu): a ragged batch of native FLAC streams (RFC 9639; oracle/flac.py is the reference) to float32
 * mono, one call.  Stream s is nbytes[s] bytes of data_dev (streams back to back, normally whole files), its first frame at byte
 * first_frame[s] (where the metadata ends), with STREAMINFO's sample_rate, channels, bits and total_samples (host arrays; the
 * caller parses the metadata).  Output: total_samples[s] float32 samples per stream, back to back: sample / 2^(bits - 1), channels
 * averaged as numpy's float32 mean(axis=1) over a C-ordered [n, ch] array (in order; 8 channels pairwise, as numpy adds exactly 8
 * elements) -- bit-identical to utils.audio.read_wav of a WAV holding the same PCM.  The last frame must end where the stream does.
 * svb_flac_plan: size of the caller-owned workspace and each stream's output sample count, -1 (svb_last_error names the stream) on
 *   bits outside 4..24, total_samples 0 (unknown), more than 8 channels, or 2 GiB of input or more.  No CUDA call.
 * svb_flac_decode_batch: finds the frames (sync code, header, CRC-8; a candidate is a frame only when the CRC-16 of the span to the
 *   next accepted frame checks out and its number continues the chain), checks each frame against STREAMINFO and the chain against
 *   its total, decodes every subframe with a reader bounded by its frame, and writes out_dev.  Synchronises the stream; a damaged
 *   stream returns SVB_ERR_INVALID with the stream and byte offset in svb_last_error.  stage_ms_host (NULL = not wanted) receives
 *   the CUDA-event time of the decode launches. */
int64_t svb_flac_plan(int32_t n_streams, const int64_t *nbytes, const int64_t *first_frame, const int32_t *sample_rate,
                      const int32_t *channels, const int32_t *bits, const int64_t *total_samples, int64_t *out_samples);
int svb_flac_decode_batch(int32_t n_streams, const int64_t *nbytes, const int64_t *first_frame, const int32_t *sample_rate,
                          const int32_t *channels, const int32_t *bits, const int64_t *total_samples, const void *data_dev,
                          float *out_dev, void *workspace_dev, int64_t workspace_bytes, float *stage_ms_host, void *stream);

/* Host-only view of the schedule of a merged tensor-core launch (csrc/conv_tc.cu: tc_schedule; no CUDA call, usable without a GPU):
 * `n_layers` convolutions of one shape class (taps KS[l], residual / accumulate flags) over B clips x Tq rows, tiles of 128 rows in
 * items of up to MT tiles, `col_blocks` column blocks, `grid` CTAs.  items_out receives 5 ints per item (layer, column block, clip,
 * first row, tiles) in execution order, off_out [grid + 1] the item range of every CTA, balance_out the mean / max estimated load.
 * Returns the item count or a negative status. */
int64_t svb_tc_schedule_probe(int32_t n_layers, const int32_t *KS, const int32_t *has_res, const int32_t *accumulate, int32_t Cin, int32_t B,
                              int32_t Tq, int32_t MT, int32_t col_blocks, int32_t chain_ordered, int32_t grid, int32_t *items_out,
                              int64_t items_capacity, int32_t *off_out, double *balance_out);
/* The same for the fused ResBlock1 launches (one item = c1 and c2 of one dilation step of chain l for P output rows): c1 taps KS1[l]
 * at dilation dil1[l], c2 taps KS2[l], c2 accumulate flags, Cin channels (one column block), items of 256 c1 rows.  items_out
 * receives 7 ints per item: the 5 of svb_tc_schedule_probe, then the first padded row and the row count of the item's c1 slab copy
 * (padded rows of a clip: [0, round_up(Tq, 256) + 128)).  P_out receives P. */
int64_t svb_tc_fused_schedule_probe(int32_t n_layers, const int32_t *KS1, const int32_t *dil1, const int32_t *KS2, const int32_t *accumulate,
                                    int32_t Cin, int32_t B, int32_t Tq, int32_t chain_ordered, int32_t grid, int32_t *items_out,
                                    int64_t items_capacity, int32_t *off_out, int32_t *P_out, double *balance_out);
/* The same for a ragged batch: clip b has lengths[b] >= 1 rows.  KS2 = NULL: the items of svb_tc_schedule_probe (taps KS, MT,
 * col_blocks); else the fused items of svb_tc_fused_schedule_probe (c1 taps KS, c2 taps KS2, MT = 2, col_blocks = 1; P_out receives
 * P, else 0).  items_out receives 6 ints per item: the 5 of svb_tc_schedule_probe, then the row bound the item carries. */
int64_t svb_tc_ragged_schedule_probe(int32_t n_layers, const int32_t *KS, const int32_t *KS2, const int32_t *has_res, const int32_t *accumulate,
                                     int32_t Cin, int32_t B, const int32_t *lengths, int32_t MT, int32_t col_blocks, int32_t chain_ordered,
                                     int32_t grid, int32_t *items_out, int64_t items_capacity, int32_t *off_out, int32_t *P_out,
                                     double *balance_out);

#ifdef __cplusplus
}
#endif
#endif /* SVB_VOCODER_H_ */
