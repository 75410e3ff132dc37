"""Beautify raw singing: an amateur take and a professional take of the same song in, the a2p (amateur-to-professional) take
out, as ``SVBVAEMleTask --infer`` computes it for a binarized pair, but straight from WAV or FLAC files and for a ragged batch of pairs
in one call.

For every pair the chain is the existing route's, stage by stage: ``PopBuTFyENBinarizer.process_batch`` (``wav2spec``, the
pitch tracker, EHSADTW on the uncropped f0), ``MultiSpkEmbDataset``'s take and collate rules (``take_conditioning``,
``clip_alignment``, zero padding), ``MleSVBVAE`` with the ways a2a + p2p + a2p and the amateur take's embedding, and the vocoder on
the a2p mel with the professional take's denormalised f0.  Each stage runs once per batch on device tensors:

    decoded samples --H2D--> resampler (off-rate takes) -> front end (svb_wav2spec_batch) -> pitch tracker -> EHSADTW
        -> [host: crop, f0 normalisation, collate] -> MleSVBVAE -> ragged generator -> [denoise] --D2H--> waveforms

The takes reach the device through ``utils.audio.load_takes``, the one loading route of the package.  The samples cross PCIe once
each way; in between only the per-frame f0, pitch ids and alignments do.

The acoustic model runs on the zero-padded batch, as the task's collated batches do, and the model is not blind to padding: a
pair's a2p mel depends on the batch it is in and can differ from the same pair beautified alone, which is what ``--infer``
(batch size 1) computes.  Beautify one pair per call to get exactly that.  Every other stage is per pair: bit-identical alone and
in any batch.

``beautify_songs`` takes whole songs (up to 65536 frames a take): each song is aligned whole (within a device-memory budget,
``align_bytes``), run through the model in overlapping segments of at most max_frames and vocoded whole from the stitched mel.

``python -m neuralsvb_b200.inference.beautify --config C --exp_name X [--hparams ...] --amateur a.wav ... --prof p.wav ...
--spk_emb e.npy ... --out o.wav ... [--song [--align_gb G]]`` writes one file per pair."""
import argparse
import os

import numpy as np
import torch

from neuralsvb_b200.data_gen.tts.data_gen_utils import pitch_ac_device, pitch_frames
from neuralsvb_b200.modules.fastspeech.fs2_vae import check_frames
from neuralsvb_b200.inference.song_plan import plan_song, segment_sizes, stitch_mels
from neuralsvb_b200.modules.voice_conversion.dtw.core import LONG_MAX_FRAMES
from neuralsvb_b200.tasks.singing.dataset_utils import clip_alignment, cropped_frames, normalized_take_f0, take_conditioning
from neuralsvb_b200.utils import audio, collate_1d
from neuralsvb_b200.utils.ckpt_utils import get_all_ckpts
from neuralsvb_b200.utils.hparams import hparams, set_hparams
from neuralsvb_b200.utils.pitch_utils import denorm_f0, f0_to_coarse, norm_interp_f0

WAYS = ('a2a', 'p2p', 'a2p')
ALIGN_METHOD = 'EHSADTW'
EMB_DIM = 256
SONG_ALIGN_BYTES = 24 << 30     # beautify_songs' default budget for the alignment workspace of all songs of a call (align_songs)
SONG_VOCODE_FRAMES = 1 << 17    # and vocodes them together up to this many padded frames (songs x the longest professional take)


def newest_checkpoint(work_dir):
    """The ``model_ckpt_steps_*.ckpt`` of ``work_dir`` with the largest step."""
    paths = get_all_ckpts(work_dir)
    if not paths:
        raise FileNotFoundError(f'no model_ckpt_steps_*.ckpt under {work_dir!r}')
    return paths[0]


def load_f0_stats(hp):
    """Set hp['f0_mean'] / hp['f0_std'] from ``train_f0s_mean_std.npy`` in binary_data_dir, as MultiSpkEmbDataset does.  Without the
    file they are None, which pitch_norm 'standard' cannot use: then the error names the file."""
    fn = os.path.join(hp['binary_data_dir'], 'train_f0s_mean_std.npy')
    if os.path.exists(fn):
        hp['f0_mean'], hp['f0_std'] = (float(x) for x in np.load(fn))
    else:
        if hp.get('pitch_norm') == 'standard':
            raise FileNotFoundError(f'{fn} is missing: pitch_norm "standard" normalises f0 with the training set\'s statistics, '
                                    'which the binarizer writes there')
        hp['f0_mean'] = hp['f0_std'] = None


def _embedding(e, i):
    """The amateur take's embedding as the dataset reads it (FloatTensor of the stored array), checked to be 256 finite floats."""
    try:
        raw = np.load(e, allow_pickle=False) if isinstance(e, str) else np.asarray(e)
        ok = raw.shape == (EMB_DIM,) and bool(np.isfinite(raw.astype(np.float64)).all())
    except (ValueError, TypeError, OSError) as err:
        raise ValueError(f'pair {i}: the speaker embedding could not be read as numbers ({err})') from None
    if not ok:
        raise ValueError(f'pair {i}: the speaker embedding must be {EMB_DIM} finite floats, got shape {raw.shape}')
    return torch.FloatTensor(raw)


def condition(frames, f0s, pitches, aligns, spk, hp):
    """The collated sample of B pairs, MultiSpkEmbDataset's rules on each take (host tensors): ``frames`` / ``f0s`` / ``pitches``
    hold the B amateur takes then the B professional ones (mel frame counts, f0 in Hz, pitch ids), ``aligns`` the B uncropped a2p
    alignments, ``spk`` the B embeddings.  Also returns each take's cropped frame count."""
    B = len(aligns)
    ama = [take_conditioning(frames[i], f0s[i], pitches[i], hp, 500) for i in range(B)]
    prof = [take_conditioning(frames[B + i], f0s[B + i], pitches[B + i], hp, 900) for i in range(B)]
    align = [clip_alignment(aligns[i], prof[i][0], ama[i][0]) for i in range(B)]
    c1 = lambda xs, pad=0: collate_1d(xs, pad)
    sample = {'pitch': c1([a[1] for a in ama]), 'f0': c1([a[2] for a in ama], 0.0), 'uv': c1([a[3] for a in ama]),
              'prof_pitch': c1([p[1] for p in prof]), 'prof_f0': c1([p[2] for p in prof], 0.0), 'prof_uv': c1([p[3] for p in prof]),
              'a2p_f0_alignment': c1(align), 'spk': torch.stack(list(spk))}
    return sample, [a[0] for a in ama], [p[0] for p in prof]


class _Stages:
    """CUDA-event times of the stages of one call (``SVBBeautifier.stage_ms``), or nothing when timing is off."""

    def __init__(self, on):
        self.on, self.marks = on, []

    def mark(self, name):
        if self.on:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.marks.append((name, ev))

    def ms(self):
        if not self.on:
            return None
        torch.cuda.synchronize()
        out = {}
        for (n, a), (_, b) in zip(self.marks[:-1], self.marks[1:]):
            out[n] = out.get(n, 0.0) + a.elapsed_time(b)         # a stage marked more than once: its total
        return out


class SVBBeautifier:
    """The a2p chain of an SVB experiment.  Loads what ``SVBVAEMleTask`` loads for ``--infer``: the experiment's ``config.yaml``
    (``set_hparams``; ``hp`` replaces it), the newest ``model_ckpt_steps_*.ckpt``'s ``state_dict['model']`` into ``MleSVBVAE`` in
    eval mode, the vocoder of ``hparams['vocoder']`` / ``vocoder_ckpt`` and the f0 statistics of ``binary_data_dir``.  Like
    ``set_hparams``, it makes its hyper-parameters the package's ``hparams``, which the vocoder plugin reads."""

    def __init__(self, work_dir, hp=None, device=None):
        if hp is None:
            hp = set_hparams(config=os.path.join(work_dir, 'config.yaml'), print_hparams=False, global_hparams=False)
            hp['work_dir'] = work_dir
        if hp is not hparams:
            hparams.clear()
            hparams.update(hp)
        self.hp = hparams
        load_f0_stats(self.hp)
        ckpt = newest_checkpoint(work_dir)
        if not torch.cuda.is_available():
            raise RuntimeError('SVBBeautifier runs on CUDA: neuralsvb_b200 has no CPU fallback')
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        from neuralsvb_b200.modules.voice_conversion.svb_vae import MleSVBVAE
        from neuralsvb_b200.vocoders.base_vocoder import get_vocoder_cls
        self.model = MleSVBVAE(hp=self.hp, precision=self.hp.get('svb_precision', 'bf16x3'))
        self.model.load_state_dict(torch.load(ckpt, map_location='cpu', weights_only=False)['state_dict']['model'], strict=True)
        self.model.eval().to(self.device)
        print(f'| SVBBeautifier: model from {ckpt}')
        with torch.cuda.device(self.device):
            self.vocoder = get_vocoder_cls(self.hp)()
        self.mel_basis = torch.tensor(audio.build_mel_basis(self.hp), dtype=torch.float32, device=self.device)
        self.timing, self.stage_ms = False, None
        self._batch_invariant = False       # the current call's batch_invariant (beautify_batch / beautify_songs)

    # ------------------------------------------------------------------ host checks
    def _takes(self, amateur, professional, spk_emb, songs=False):
        """Decoded takes (B amateur, then B professional; ``audio.decode_wavs``), their rates, their lengths at audio_sample_rate
        and mel frame counts, and the B embeddings; every pair checked before any device work.  songs: takes up to LONG_MAX_FRAMES
        instead of max_frames."""
        amateur, professional, spk_emb = list(amateur), list(professional), list(spk_emb)
        B = len(amateur)
        if B == 0 or len(professional) != B or len(spk_emb) != B:
            raise ValueError(f'{B} amateur takes, {len(professional)} professional takes and {len(spk_emb)} embeddings: '
                             'one of each per pair, at least one pair')
        spk = [_embedding(e, i) for i, e in enumerate(spk_emb)]
        hp, sr, hop = self.hp, int(self.hp['audio_sample_rate']), int(self.hp['hop_size'])
        dec = audio.decode_wavs(amateur + professional, sr, self.device)
        for k, (w, _) in enumerate(dec):
            if w.ndim != 1 or len(w) == 0:
                raise ValueError(f'pair {k % B}: the {"amateur" if k < B else "professional"} take must be 1-D samples, '
                                 f'got shape {tuple(w.shape)}')
        rates = [r for _, r in dec]
        lens = np.array([len(w) for w, _ in dec], np.int64)
        off = [k for k, r in enumerate(rates) if r != sr]
        if off:
            lens[off] = audio.resample_lengths(lens[off], [rates[k] for k in off], sr)[1]
        frames = lens // hop + 1
        for k in range(2 * B):
            what = f'{"song" if songs else "pair"} {k % B}: the {"amateur" if k < B else "professional"} take'
            if songs and frames[k] > LONG_MAX_FRAMES:
                raise ValueError(f'{what} has {frames[k]} frames, more than the {LONG_MAX_FRAMES} a song may have '
                                 f'({LONG_MAX_FRAMES * hop / sr:.1f} s)')
            if not songs and frames[k] > hp['max_frames']:
                raise ValueError(f'{what} has {frames[k]} frames, more than max_frames = {hp["max_frames"]} '
                                 f'({hp["max_frames"] * hop / sr:.1f} s); beautify_songs takes whole songs')
            if pitch_frames(frames[k] * hop, hp) < 1:
                raise ValueError(f'{what} is shorter than one pitch window')
            try:
                check_frames(cropped_frames(int(frames[k]), hp))
            except ValueError as e:
                raise ValueError(f'{what} is too short: {frames[k]} frames, cropped to {cropped_frames(int(frames[k]), hp)} ({e})') from None
        return dec, rates, lens, frames, spk

    # ------------------------------------------------------------------ device stages
    def _front_end(self, dec, rates, lens, st):
        """``audio.load_takes`` of what ``_takes`` returned (``dec`` holds each take's rate; one H2D copy of the host samples, the
        resampler over the off-rate takes), then the front end on the ``lens`` samples of each take -> (mels, padded waveforms)."""
        from neuralsvb_b200.vocoders.hifigan import HifiGAN
        x, _ = audio.load_takes(dec, int(self.hp['audio_sample_rate']), self.device)
        st.mark('front_end')
        mel, wav, _ = HifiGAN.wav2spec_device(x, lens, self.hp, self.mel_basis)
        return mel, wav

    def _pitch(self, wav, frames):
        """The pitch tracker on the padded waveforms -> (device float32 f0 back to back, host float64 f0 of each take)."""
        f0 = pitch_ac_device(wav, frames * int(self.hp['hop_size']), frames, self.hp).f0
        host = f0.cpu().numpy()
        offs = np.concatenate([[0], np.cumsum(frames)])
        return f0, [host[offs[k]:offs[k + 1]].astype(np.float64) for k in range(len(frames))]

    def _align(self, f0_dev, frames):
        """EHSADTW of every pair on the device f0 (float64, as the binarizer aligns the host f0) -> host int64 alignments."""
        from neuralsvb_b200.modules.voice_conversion.dtw.core import align_batch
        B = len(frames) // 2
        t = torch.split(f0_dev.double(), [int(x) for x in frames])
        return align_batch(list(t[:B]), list(t[B:]), ALIGN_METHOD).split()

    def _acoustic(self, sample, mel, frames, Ta, Tp, eps):
        """MleSVBVAE on the collated batch -> a2p mel_out [B, max Tp, n_mel] (device)."""
        B = len(Ta)
        offs = np.concatenate([[0], np.cumsum(frames)])
        return self._model_on(sample, mel, offs[:B], offs[B:2 * B], Ta, Tp, eps)

    def _model_on(self, sample, mel, a_rows, p_rows, Ta, Tp, eps):
        """MleSVBVAE on the collated batch whose amateur take b is mel rows [a_rows[b], a_rows[b] + Ta[b]) and professional take
        b rows [p_rows[b], p_rows[b] + Tp[b]) -> a2p mel_out [B, max Tp, n_mel] (device).  With the call's batch_invariant, the
        model runs in its length-aware mode on Ta / Tp."""
        B = len(Ta)
        d = self.device

        def pad(rows, T):
            x = torch.zeros(B, max(T), mel.shape[1], device=d)
            for b, (r, t) in enumerate(zip(rows, T)):
                x[b, :t] = mel[int(r):int(r) + t]
            return x
        out = self.model(amateur_mel=pad(a_rows, Ta), prof_mel=pad(p_rows, Tp), amateur_pitch=sample['pitch'].to(d),
                         prof_pitch=sample['prof_pitch'].to(d), amateur_spk_id=sample['spk'].to(d), prof_spk_id=sample['spk'].to(d),
                         a2p_alignment=sample['a2p_f0_alignment'].to(d), infer=False, concurrent_ways=list(WAYS),
                         disable_map=self.hp['disable_map'], eps=eps,
                         **(dict(amateur_lens=Ta, prof_lens=Tp) if self._batch_invariant else {}))
        return out['a2p']['mel_out']

    def _vocode(self, mel_out, f0, Tp, seed, first_clip=0):
        """The ragged generator at the professional frame counts, the denoise post-filter per clip when vocoder_denoise_c > 0
        -> device waveforms back to back.  Clip b's NSF draws are keyed by (seed, first_clip + b)."""
        hop = int(self.hp['hop_size'])
        y = self.vocoder.model(mel_out.transpose(1, 2).contiguous(), f0=f0.to(self.device), seed=seed, lengths=Tp,
                               first_clip=first_clip)
        clips = [y[b, 0, :t * hop] for b, t in enumerate(Tp)]
        v = self.hp.get('vocoder_denoise_c', 0.0)
        if v > 0:
            from neuralsvb_b200.vocoders.vocoder_utils import denoise_device
            clips = [denoise_device(c, v, self.hp) for c in clips]
        return torch.cat(clips)

    # ------------------------------------------------------------------ public
    def beautify_batch(self, amateur, professional, spk_emb, seed=None, eps=None, batch_invariant=False):
        """The a2p take of every (amateur, professional, embedding) triple: float32 arrays of T_prof x hop samples, T_prof the
        professional take's frame count after the dataset's crop.  A take is a WAV path (any rate) or a float32 array at
        audio_sample_rate; an embedding is the amateur take's own [256] vector or a .npy path (row 0 of multi_spk_emb).

        ``seed`` keys the NSF draws as spec2wav_batch does (Philox by seed and clip index; default: the vocoder's next seed) and
        seeds the posterior noise, drawn as [B, latent, 1] on the device unless ``eps`` gives it.  ``disable_map`` and
        ``vocoder_denoise_c`` act as in the task.

        Every pair is checked before the model runs, and a bad one raises ValueError naming its index, with nothing returned:
        a take shorter than one pitch window or than 60 frames after the frames_multiple crop, a take longer than max_frames
        (the task would crop it silently), a take without voiced f0 (the binarizer's "Empty f0" skip), lists of different
        lengths, or an embedding that is not 256 finite floats.  The binarizer's ``max_mel_tech_gap`` skip is dataset curation and
        is not applied.

        ``batch_invariant``: the acoustic model runs in its length-aware mode (MleSVBVAE's amateur_lens / prof_lens), so each
        pair's a2p mel is the same bits as that pair beautified alone with batch_invariant=True and the same eps row, and its
        waveform too given the same NSF key.  The reference only ever runs one pair at a time.  The default (False) runs the model
        on the zero-padded batch, as the task's collated batches do: a pair's mel then moves with the other pairs' lengths."""
        with torch.no_grad(), torch.cuda.device(self.device):
            return self._run(amateur, professional, spk_emb, seed, eps, batch_invariant)

    def beautify(self, amateur, professional, spk_emb, **kw):
        """``beautify_batch`` of one pair -> one float32 array."""
        return self.beautify_batch([amateur], [professional], [spk_emb], **kw)[0]

    def beautify_songs(self, amateur, professional, spk_emb, seed=None, eps=None, segment_frames=None, overlap_frames=64,
                       align_bytes=None, batch_invariant=False):
        """The a2p take of whole songs: ``beautify_batch``'s inputs, with each take up to LONG_MAX_FRAMES frames (6.3 min at
        22.05 kHz / hop 128) instead of max_frames.  Returns one float32 array of Tp x hop samples per song, Tp the professional
        frame count cropped to a multiple of frames_multiple.

        All songs are aligned whole in one ``align_songs`` call (EHSADTW on the device f0 in float64, align_long's results) within
        ``align_bytes`` of device workspace (default SONG_ALIGN_BYTES; a lower budget trades about twice the alignment time for
        memory linear in the songs' lengths, with the same results), then each song is cut by ``plan_song`` into professional
        segments of at most ``segment_frames`` (default max_frames) overlapping by ``overlap_frames``, each with the amateur slice
        its alignment reads; the segments are conditioned by ``condition()``'s rules on their slices of the whole takes' f0 and
        pitch ids, with alignment a2p[s:e] - a_lo.  MleSVBVAE runs once per song on that song's segments as one batch, with the
        song's embedding and eps[b] repeated, so a song's result does not depend on the other songs of the call.  The a2p mels
        are stitched with a linear cross-fade over each overlap (``stitch_mels``) and the songs vocoded whole in one ragged
        generator call per group, with the whole professional take's f0.

        With ``normalize_pitch`` each take is normalised once over the whole take and then sliced: one key for the song, where
        per-clip conditioning would move every segment to the statistics on its own.  A song that fits one segment (Tp <=
        segment_frames and Ta <= max_frames) gives exactly ``beautify`` of the pair with the same seed and eps.

        ``seed`` keys the NSF draws by (seed, song index) as spec2wav_batch does, however the songs are grouped for the vocoder
        (consecutive songs up to SONG_VOCODE_FRAMES padded frames per generator call), and draws eps [n_songs, latent, 1]
        unless given.  Bad segment_frames / overlap_frames and an align_bytes below the smallest workable alignment budget (the
        message names it) raise before any device work; every song is checked and planned
        before the model runs: a bad take, a take over LONG_MAX_FRAMES or a song that cannot be planned raises ValueError naming
        the song.

        ``batch_invariant``: each segment runs as it would alone (``beautify_batch``'s batch_invariant), so the short tail segment
        no longer moves with the padding to the longest segment; a song that fits one segment then gives exactly
        ``beautify(..., batch_invariant=True)`` of the pair."""
        with torch.no_grad(), torch.cuda.device(self.device):
            return self._run_songs(amateur, professional, spk_emb, seed, eps, segment_frames, overlap_frames, align_bytes,
                                   batch_invariant)

    def _song_conditioning(self, frames, f0s, B):
        """Per take (B amateur, then B professional): the cropped frame count, the f0 the segments are conditioned on (moved by
        normalize_pitch over the whole take) and its pitch ids."""
        hp, fm = self.hp, int(self.hp['frames_multiple'])
        out = []
        for k, f in enumerate(f0s):
            if hp.get('normalize_pitch', False):
                f = normalized_take_f0(f, hp, 500 if k < B else 900)
            out.append((int(frames[k]) // fm * fm, f, f0_to_coarse(f)))
        return out

    def _align_songs(self, f0_dev, frames, st):
        """EHSADTW of every song on the device f0 (float64, as _align) in one align_songs call within the call's alignment budget
        -> host int64 alignments.  With timing on, align_ms holds the call's (histogram, forward, backward, backtrack) times."""
        from neuralsvb_b200.modules.voice_conversion.dtw.core import align_songs
        B = len(frames) // 2
        t = torch.split(f0_dev.double(), [int(x) for x in frames])
        st.mark('alignment')
        r = align_songs(list(t[:B]), list(t[B:]), ALIGN_METHOD, workspace_bytes=self._align_bytes, stage_ms=self.timing)
        self.align_ms = [r.stage_ms] if self.timing else []
        return r.split()

    def _run_songs(self, amateur, professional, spk_emb, seed, eps, segment_frames, overlap_frames, align_bytes=None,
                   batch_invariant=False):
        from neuralsvb_b200.modules.voice_conversion.dtw.core import striped_plan
        hp = self.hp
        segment_sizes(hp, segment_frames, overlap_frames, 'beautify_songs')         # before any device work
        dec, rates, lens, frames, spk = self._takes(amateur, professional, spk_emb, songs=True)
        B = len(spk)
        self._batch_invariant = bool(batch_invariant)
        self._align_bytes = SONG_ALIGN_BYTES if align_bytes is None else int(align_bytes)
        try:
            striped_plan(frames[:B], frames[B:], self._align_bytes)                  # a budget below the minimum: before any device work
        except ValueError as e:
            raise ValueError(f'beautify_songs: align_bytes = {self._align_bytes}: {e}') from None
        if eps is not None:
            eps = torch.as_tensor(eps, dtype=torch.float32)
            if tuple(eps.shape) != (B, hp['latent_size'], 1):
                raise ValueError(f'eps must be [{B}, {hp["latent_size"]}, 1], got {tuple(eps.shape)}')
        st = _Stages(self.timing)
        st.mark('load')
        mel, wav = self._front_end(dec, rates, lens, st)
        st.mark('pitch')
        f0_dev, f0s = self._pitch(wav, frames)
        for k, f in enumerate(f0s):
            if sum(f) == 0:
                raise ValueError(f'song {k % B}: the {"amateur" if k < B else "professional"} take has no voiced f0 '
                                 '(the alignment is undefined)')
        aligns = self._align_songs(f0_dev, frames, st)
        torch.cuda.empty_cache()        # the DTW workspace's cached blocks: the generator allocates its workspace outside torch
        st.mark('plan_conditioning')
        takes = self._song_conditioning(frames, f0s, B)
        hp_seg = dict(hp, normalize_pitch=False)        # the segments' f0 is already the whole take's normalised one
        songs = []
        for b in range(B):
            (Ta, fa, pa), (Tp, fp, pp) = takes[b], takes[B + b]
            a2p = clip_alignment(aligns[b], Tp, Ta).numpy()
            pf0, puv = norm_interp_f0(fp[:Tp], hp)
            plan = plan_song(Tp, Ta, a2p, puv.numpy(), hp, segment_frames, overlap_frames, name=f'song {b}')
            K = len(plan)
            sample, sa, sp = condition([a1 - a0 for _, _, a0, a1 in plan] + [e - s for s, e, _, _ in plan],
                                       [fa[a0:a1] for _, _, a0, a1 in plan] + [fp[s:e] for s, e, _, _ in plan],
                                       [pa[a0:a1] for _, _, a0, a1 in plan] + [pp[s:e] for s, e, _, _ in plan],
                                       [a2p[s:e] - a0 for s, e, a0, _ in plan], [spk[b]] * K, hp_seg)
            songs.append((plan, sample, sa, sp, denorm_f0(pf0, puv, hp)))
        if seed is None:
            self.vocoder.model.seed += 1
            seed = self.vocoder.model.seed
        if eps is None:
            eps = torch.randn(B, hp['latent_size'], 1, device=self.device, generator=torch.Generator(self.device).manual_seed(seed))
        eps = eps.to(self.device)
        offs = np.concatenate([[0], np.cumsum(frames)])
        song_mels = []
        for b, (plan, sample, sa, sp, _) in enumerate(songs):
            st.mark('acoustic_model')
            K = len(plan)
            out = self._model_on(sample, mel, [offs[b] + a0 for _, _, a0, _ in plan], [offs[B + b] + s for s, _, _, _ in plan],
                                 sa, sp, eps[b:b + 1].expand(K, -1, -1).contiguous())
            st.mark('stitch')
            song_mels.append(stitch_mels([out[k] for k in range(K)], plan, overlap_frames))
        clips = []
        Tps = [songs[b][0][-1][1] for b in range(B)]
        for g0, g1 in _groups([1] * B, SONG_VOCODE_FRAMES, lambda a, b: (b - a) * max(Tps[a:b])):
            st.mark('vocoder')
            x = torch.zeros(g1 - g0, max(Tps[g0:g1]), mel.shape[1], device=self.device)
            f0 = torch.zeros(g1 - g0, max(Tps[g0:g1]))
            for q, b in enumerate(range(g0, g1)):
                x[q, :Tps[b]] = song_mels[b]
                f0[q, :Tps[b]] = songs[b][4]
            clips.append(self._vocode(x, f0, Tps[g0:g1], seed, first_clip=g0))
        st.mark('d2h')
        out = torch.cat(clips).cpu().numpy()
        st.mark('end')
        self.stage_ms = st.ms()
        self.song_mels, self.song_plans = song_mels, [s[0] for s in songs]
        hop = int(hp['hop_size'])
        return np.split(out, np.cumsum([t * hop for t in Tps])[:-1])

    def _run(self, amateur, professional, spk_emb, seed, eps, batch_invariant=False):
        hp = self.hp
        dec, rates, lens, frames, spk = self._takes(amateur, professional, spk_emb)
        B = len(spk)
        self._batch_invariant = bool(batch_invariant)
        if eps is not None:
            eps = torch.as_tensor(eps, dtype=torch.float32)
            if tuple(eps.shape) != (B, hp['latent_size'], 1):
                raise ValueError(f'eps must be [{B}, {hp["latent_size"]}, 1], got {tuple(eps.shape)}')
        st = _Stages(self.timing)
        st.mark('load')
        mel, wav = self._front_end(dec, rates, lens, st)
        st.mark('pitch')
        f0_dev, f0s = self._pitch(wav, frames)
        for k, f in enumerate(f0s):
            if sum(f) == 0:
                raise ValueError(f'pair {k % B}: the {"amateur" if k < B else "professional"} take has no voiced f0 '
                                 '(the binarizer skips such a pair as "Empty f0"; the alignment is undefined)')
        st.mark('alignment')
        aligns = self._align(f0_dev, frames)
        st.mark('conditioning')
        sample, Ta, Tp = condition(frames, f0s, [f0_to_coarse(f) for f in f0s], aligns, spk, hp)
        if seed is None:
            self.vocoder.model.seed += 1
            seed = self.vocoder.model.seed
        if eps is None:
            eps = torch.randn(B, hp['latent_size'], 1, device=self.device, generator=torch.Generator(self.device).manual_seed(seed))
        st.mark('acoustic_model')
        mel_out = self._acoustic(sample, mel, frames, Ta, Tp, eps.to(self.device))
        st.mark('vocoder')
        f0 = denorm_f0(sample['prof_f0'], sample['prof_uv'], hp)
        wav = self._vocode(mel_out, f0, Tp, seed)
        st.mark('d2h')
        out = wav.cpu().numpy()
        st.mark('end')
        self.stage_ms = st.ms()
        hop = int(hp['hop_size'])
        return np.split(out, np.cumsum([t * hop for t in Tp])[:-1])


def _groups(sizes, limit, size_of=None):
    """Consecutive [g0, g1) ranges of items whose size (size_of(g0, g1), default the sum of sizes) stays within limit; an item
    over the limit alone is a group."""
    size_of = size_of or (lambda a, b: sum(sizes[a:b]))
    out, g0 = [], 0
    for g1 in range(1, len(sizes) + 1):
        if g1 - g0 > 1 and size_of(g0, g1) > limit:
            out.append((g0, g1 - 1))
            g0 = g1 - 1
    return out + [(g0, len(sizes))]


def parse_args(argv=None):
    p = argparse.ArgumentParser(description='Beautify amateur singing with an SVB experiment: one output WAV per '
                                            '(amateur, professional, embedding) triple.')
    p.add_argument('--config', type=str, default='')
    p.add_argument('--exp_name', type=str, required=True)
    p.add_argument('--hparams', type=str, default='')
    p.add_argument('--amateur', nargs='+', required=True)
    p.add_argument('--prof', nargs='+', required=True)
    p.add_argument('--spk_emb', nargs='+', required=True)
    p.add_argument('--out', nargs='+', required=True)
    p.add_argument('--song', action='store_true', help='whole songs (beautify_songs): takes longer than max_frames are aligned '
                                                       'whole, run through the model in overlapping segments and vocoded whole')
    p.add_argument('--align_gb', type=float, default=None,
                   help='with --song: device memory budget of the alignment in GiB (default 24); a lower one aligns in about '
                        'twice the time with the same results')
    p.add_argument('--batch_invariant', action='store_true',
                   help='run the acoustic model on each pair\'s (or song segment\'s) own frames only: every output is then the same '
                        'as that pair beautified alone, whatever else is in the call')
    args = p.parse_args(argv)
    counts = {k: len(getattr(args, k)) for k in ('amateur', 'prof', 'spk_emb', 'out')}
    if len(set(counts.values())) != 1:
        p.error(f'--amateur, --prof, --spk_emb and --out take one value per pair each, got {counts}')
    return args


def main(argv=None):
    args = parse_args(argv)
    work_dir = f'checkpoints/{args.exp_name}'
    newest_checkpoint(work_dir)                       # before set_hparams, which would write a config.yaml into a new work_dir
    hp = set_hparams(config=args.config, exp_name=args.exp_name, hparams_str=args.hparams, print_hparams=False)
    hp['infer'] = True
    b = SVBBeautifier(work_dir, hp=hparams)
    if args.song:
        align_bytes = None if args.align_gb is None else int(args.align_gb * (1 << 30))
        wavs = b.beautify_songs(args.amateur, args.prof, args.spk_emb, align_bytes=align_bytes, batch_invariant=args.batch_invariant)
    else:
        wavs = b.beautify_batch(args.amateur, args.prof, args.spk_emb, batch_invariant=args.batch_invariant)
    for w, fn in zip(wavs, args.out):
        if os.path.dirname(fn):
            os.makedirs(os.path.dirname(fn), exist_ok=True)
        audio.save_wav(w, fn, hparams['audio_sample_rate'], norm=hparams['out_wav_norm'])
        print(f'| {fn}: {len(w) / hparams["audio_sample_rate"]:.2f} s')


if __name__ == '__main__':
    main()
