"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, and
exports every symbol include/svb_vocoder.h declares.  No compute calls (no GPU here)."""
import ctypes
import os

import pytest

from neuralsvb_b200 import _native


@pytest.fixture(scope='module')
def built():
    try:
        return _native.build()
    except RuntimeError as e:          # no nvcc on this box: the prebuilt library must already be there
        if os.path.exists(_native.LIB_PATH):
            return _native.LIB_PATH
        pytest.fail(str(e))


def test_library_exports_every_declared_symbol(built):
    l = ctypes.CDLL(built)
    declared = _native.declared_symbols()
    assert len(declared) >= 15
    missing = [s for s in declared if not hasattr(l, s)]
    assert not missing, f'declared in include/svb_vocoder.h but not exported: {missing}'


def test_binding_covers_every_declared_symbol():
    declared = set(_native.declared_symbols())
    bound = set(_native._PROTOS)
    assert declared <= bound, f'no ctypes prototype for {sorted(declared - bound)}'


def test_abi_version_and_error_string(built):
    l = _native.lib()
    assert l.svb_abi_version() == 1
    assert isinstance(l.svb_last_error(), bytes)


def test_struct_layout_matches_header():
    # 3 + 8 + 8 + 2 + 4 + 1 + 16 + 3 int32 fields
    assert ctypes.sizeof(_native.GenConfig) == 4 * (3 + 8 + 8 + 2 + 4 + 1 + 16 + 3)
    assert ctypes.sizeof(_native.StftConfig) == 4 * 9


def test_argument_validation_without_gpu(built):
    l = _native.lib()
    # null config -> SVB_ERR_INVALID before any CUDA call
    assert l.svb_stft_num_frames(None, 100) < 0
    c = _native.StftConfig(1024, 256, 512, _native.PAD_CENTER_ZERO, _native.OUT_LOG10_MEL, 0, 80, 1, 1e-10)
    assert l.svb_stft_num_frames(ctypes.byref(c), 44100) == 173          # 1 + n // hop
    assert l.svb_stft_num_frames(ctypes.byref(c), 1000) == 4
    c.pad_mode = _native.PAD_HALF_REFLECT
    assert l.svb_stft_num_frames(ctypes.byref(c), 32768) == 128          # T_wav / hop exactly
    c.n_fft = 1000                                                      # not a power of two
    rc = l.svb_stft_forward(ctypes.byref(c), None, 1, 100, None, None, None)
    assert rc == -1 and b'power of two' in l.svb_last_error()


def test_product_fails_loudly_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from neuralsvb_b200.modules.hifigan.hifigan import HifiGanGenerator
    from neuralsvb_b200.utils import synthetic as S
    h = S.small_config()
    m = HifiGanGenerator(h)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        m(torch.zeros(1, 80, 8))
    from neuralsvb_b200.vocoders.hifigan import HifiGAN
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        HifiGAN.wav2spec(S.make_clip(2048), hp=S.hifigan_config())


def test_training_entry_points_validate_arguments_without_gpu(built):
    """The backward / training half of the ABI rejects bad arguments before any CUDA call (negative svb_status, message set)."""
    l = _native.lib()
    f = ctypes.c_float
    assert l.svb_gen_set_training(None, 1) < 0 and b'not finalized' in l.svb_last_error()
    assert l.svb_gen_backward(None, None, None) < 0
    assert l.svb_gen_grad_numel(None, b'conv_pre.weight') == -1
    assert l.svb_weight_norm_backward(None, None, None, 4, 4, None, None, None) < 0
    assert l.svb_conv_nct_backward(None, None, None, None, 1, 1, 1, 8, 1, 3, 1, 1, 1, 1, f(0.1), None, None, None, None, None) < 0
    assert l.svb_loss_grad_dev(None, None, 0, f(1.0), None, None, 8, 0, None) < 0
    assert l.svb_cond_net_forward(None, None, None, 1, 80, 8, 512, 256, 128, None, None) < 0
    # single-layer backward: (x, w, dy, B, Cin, Cout, T, K, dil, u, slope, precision, dx, dw, db, stream); host buffers
    # stand in for every pointer, the call must refuse before it touches one
    import numpy as np
    buf = np.zeros(1 << 16, np.float32)
    p = ctypes.c_void_p(buf.ctypes.data)
    bwd = lambda Cin, Cout, K, dil, u, prec, x=p, db=p: l.svb_conv1d_backward_run(x, p, p, 2, Cin, Cout, 16, K, dil, u, f(0.1), prec,
                                                                                  p, p, db, None)
    assert bwd(32, 32, 3, 1, 0, 3, x=None) < 0 and b'bad argument' in l.svb_last_error()
    assert bwd(32, 32, 3, 1, 0, 3, db=None) < 0 and b'bad argument' in l.svb_last_error()
    assert bwd(32, 32, 3, 1, -1, 3) < 0 and b'bad argument' in l.svb_last_error()
    assert bwd(32, 32, 3, 1, 0, 4) < 0 and b'bad precision' in l.svb_last_error()
    assert bwd(30, 32, 3, 1, 0, 0) < 0 and b'multiples of 4' in l.svb_last_error()
    assert bwd(32, 32, 4, 1, 0, 0) < 0 and b'odd kernel' in l.svb_last_error()
    assert bwd(32, 32, 3, 0, 0, 0) < 0 and b'odd kernel' in l.svb_last_error()          # dilation 0
    assert bwd(32, 32, 11, 13, 0, 3) < 0 and b'halo' in l.svb_last_error()             # 5 * 13 = 65 rows > 64
    assert bwd(32, 32, 4, 0, 8, 0) < 0 and b'transposed kernel' in l.svb_last_error()  # K < u
    assert bwd(32, 32, 15, 0, 8, 0) < 0 and b'transposed kernel' in l.svb_last_error() # odd K - u
    # discriminator conv backward: (x, w, y, dy, B, Cin, Cout, Tin, W, K, stride, dil, pad, groups, slope, dz, dx, dw, db, stream);
    # every reject comes before the first launch, so dz / dx / dw / db are never written
    nct = lambda K, stride, dx=p, dw=p: l.svb_conv_nct_backward(p, p, p, p, 1, 4, 4, 64, 1, K, stride, 1, 0, 1, f(0.1), p, dx, dw, p, None)
    assert nct(3, 5) < 0 and b'stride 5 unsupported' in l.svb_last_error()
    assert nct(9, 1) < 0 and b'kernel size 9 has no weight-gradient instance' in l.svb_last_error()
    assert nct(9, 5, dw=None) < 0 and b'stride 5 unsupported' in l.svb_last_error()
    assert nct(9, 5, dx=None) < 0 and b'kernel size 9' in l.svb_last_error()
    # cond_net backward with an empty output: (T - 1) * stride - 2 * pad + K = 0
    assert l.svb_cond_net_backward(p, p, 1, 80, 1, 2, 1, 1, p, p, None) < 0 and b'empty output' in l.svb_last_error()
    h = ctypes.c_void_p()
    # 33 -> 64 channels is not a tensor-core shape; a stride-1 layer needs 'same' padding
    assert l.svb_tc_layer_create(33, 64, 5, 1, 2, 3, 0, ctypes.byref(h)) < 0 and b'tensor-core shape' in l.svb_last_error()
    assert l.svb_tc_layer_create(64, 64, 5, 1, 1, 3, 0, ctypes.byref(h)) < 0 and b"'same' padding" in l.svb_last_error()
    assert l.svb_tc_layer_create(64, 64, 5, 3, 2, 0, 0, ctypes.byref(h)) < 0          # fp32 is not a tensor-core mode
    assert l.svb_tc_layer_out_len(None, 100) == -1
    c = _native.StftConfig(1024, 256, 512, _native.PAD_CENTER_ZERO, _native.OUT_MAG_RAW, 0, 0, 1, 0.0)
    assert l.svb_denoise(ctypes.byref(c), None, 1, 4096, f(0.1), None, None) < 0
    c.n_fft = 1000
    assert l.svb_stft_backward(ctypes.byref(c), None, 1, 4096, None, None, None, None) < 0 and b'power of two' in l.svb_last_error()


def _schedule(KS, has_res, accum, B, Tq, MT, col_blocks, chain_ordered, grid=132, Cin=128):
    import ctypes

    import numpy as np
    from neuralsvb_b200 import _native
    n = len(KS)
    arr = lambda v: np.ascontiguousarray(v, dtype=np.int32)
    ks, hr, ac = arr(KS), arr(has_res), arr(accum)
    cap = 200000
    items, off, bal = np.zeros((cap, 5), np.int32), np.zeros(grid + 1, np.int32), ctypes.c_double()
    cnt = _native.check(_native.lib().svb_tc_schedule_probe(n, ks.ctypes.data, hr.ctypes.data, ac.ctypes.data, Cin, B, Tq, MT, col_blocks,
                                                            int(chain_ordered), grid, items.ctypes.data, cap, off.ctypes.data, ctypes.byref(bal)),
                        'tc_schedule_probe')
    return items[:cnt], off, bal.value


def test_merged_launch_schedule_covers_every_tile_once():
    """Host logic of the merged ResBlock-chain launches (csrc/conv_tc.cu:tc_schedule), no GPU needed: the three chains of stage 1 of
    config 2 (C = 128: k 3 / 7 / 11, 16 clips x 8192 rows)."""
    import numpy as np
    items, off, bal = _schedule([3, 7, 11], [0, 0, 0], [0, 0, 0], 16, 8192, 2, 1, False)
    assert len(items) == 3 * 16 * 32 and off[0] == 0 and off[-1] == len(items)
    seen = set(map(tuple, items[:, :4]))
    assert len(seen) == len(items)                                           # no (layer, block, clip, row) twice
    for l in range(3):
        rows = items[items[:, 0] == l]
        assert sorted(map(tuple, rows[:, 2:4])) == [(b, t) for b in range(16) for t in range(0, 8192, 256)]
    assert (items[:, 4] == 2).all() and bal > 0.95
    assert (np.diff(off) <= 120).all()
    # a CTA alternates its layers instead of running them one after the other
    first = items[off[0]:off[1], 0]
    assert len(set(first[:3].tolist())) > 1


def test_chain_ordered_schedule_keeps_the_layers_of_a_tile_together():
    """The step that accumulates the three ResBlocks into the stage output: every CTA runs layers 0, 1, 2 of a tile back to back."""
    items, off, bal = _schedule([3, 7, 11], [1, 1, 1], [0, 1, 1], 16, 1024, 2, 2, True, Cin=256)
    assert len(items) == 3 * 16 * 4 * 2
    for c in range(len(off) - 1):
        mine = items[off[c]:off[c + 1]]
        assert len(mine) % 3 == 0
        for i in range(0, len(mine), 3):
            assert mine[i:i + 3, 0].tolist() == [0, 1, 2]
            assert (mine[i:i + 3, 1:] == mine[i, 1:]).all()                    # same column block, clip, row, tiles
    assert 0.8 < bal <= 1.0


def test_schedule_handles_an_odd_tile_count():
    items, off, bal = _schedule([3, 11], [0, 0], [0, 0], 3, 5 * 128 - 7, 2, 1, False, grid=8)
    tiles = items[:, 4]
    assert set(tiles.tolist()) == {1, 2}                                      # the last item of a clip has one tile
    assert int(tiles.sum()) == 2 * 3 * 5


# ---- autocorrelation pitch tracker (csrc/pitch_ac.cu): host-side planning and refusals
PITCH_CONFIGS = [(22050, 128, 8), (22050, 256, 4), (22880, 128, 8), (22881, 128, 8), (24000, 128, 8), (44100, 256, 4),
                 (45920, 256, 4), (16000, 110, 0)]


def _pitch_cfg(sr, hop, lpad):
    from neuralsvb_b200.data_gen.tts import data_gen_utils as DG
    return DG.pitch_config({'audio_sample_rate': sr, 'hop_size': hop}, lpad)


def _pitch_frames(l, cfg, lengths):
    import numpy as np
    lens = np.ascontiguousarray(lengths, dtype=np.int64)
    out = np.full(len(lens), -7, np.int32)
    ws = l.svb_pitch_ac_workspace_bytes(ctypes.byref(cfg), lens.ctypes.data, len(lens), out.ctypes.data)
    return ws, out


@pytest.mark.parametrize('sr,hop,lpad', PITCH_CONFIGS, ids=[f'{s}-{h}-{p}' for s, h, p in PITCH_CONFIGS])
def test_pitch_frame_counts_match_the_oracle_grid(built, sr, hop, lpad):
    """frames_out of svb_pitch_ac_workspace_bytes equals oracle.pitch_ac.grid and data_gen_utils.pitch_frames for clips around one
    window (L), one window plus a hop, and random lengths; a clip with no analysis frame is refused by all three."""
    import numpy as np

    from neuralsvb_b200.data_gen.tts import data_gen_utils as DG
    from oracle import pitch_ac as P
    l = _native.lib()
    cfg = _pitch_cfg(sr, hop, lpad)
    hp = {'audio_sample_rate': sr, 'hop_size': hop}
    L = 2 * int(np.floor(3.0 / 80.0 * sr / 2.0)) + 1
    rs = np.random.RandomState(sr + hop)
    Ns = list(range(L - 4, L + 5)) + list(range(L + hop - 4, L + hop + 5)) + rs.randint(L, 40 * sr, 40).tolist()
    refused = 0
    for N in Ns:
        try:
            n = P.grid(N, sr, hop / sr)[0]
        except ValueError:
            n = 0
        ws, out = _pitch_frames(l, cfg, [N])
        if n == 0:
            refused += 1
            assert ws < 0 and b'shorter than one pitch window' in l.svb_last_error(), N
            assert DG.pitch_frames(N, hp) < 1, N
            continue
        assert ws > 0 and out[0] == n == DG.pitch_frames(N, hp), (N, ws, out[0], n, DG.pitch_frames(N, hp))
    assert 0 < refused < len(Ns)
    # the same lengths in one ragged call
    good = [N for N in Ns if DG.pitch_frames(N, hp) >= 1]
    ws, out = _pitch_frames(l, cfg, good)
    assert ws > 0 and out.tolist() == [P.grid(N, sr, hop / sr)[0] for N in good]


def test_pitch_refuses_bad_arguments_without_gpu(built):
    """svb_pitch_ac_workspace_bytes and svb_pitch_ac_batch refuse before any CUDA call (negative status, message set).  Host buffers
    stand in for the device pointers: a refusal must come before one is touched."""
    import numpy as np

    from oracle import pitch_ac as P
    l = _native.lib()
    buf = np.zeros(1 << 16, np.float32)
    p = ctypes.c_void_p(buf.ctypes.data)
    ok = [22050, 30000]
    mel = np.array([200, 240, 100], np.int64)

    def refuse(c, lens, msg, n=None):
        lens = np.ascontiguousarray(lens, dtype=np.int64)
        n = len(lens) if n is None else n
        frames = np.zeros(max(len(lens), 1), np.int32)
        assert l.svb_pitch_ac_workspace_bytes(c, lens.ctypes.data, n, frames.ctypes.data) < 0, msg
        assert msg in l.svb_last_error(), (msg, l.svb_last_error())
        l.svb_pitch_ac_workspace_bytes(cfg(hop=0), lens.ctypes.data, n, None)    # another message in between
        assert msg not in l.svb_last_error()
        assert l.svb_pitch_ac_batch(c, p, lens.ctypes.data, n, mel.ctypes.data, p, p, 1 << 30, None, None, None, None, None) < 0
        assert msg in l.svb_last_error(), (msg, l.svb_last_error())

    def cfg(**kw):
        c = _pitch_cfg(22050, 128, 8)
        for k, v in kw.items():
            setattr(c, k, v)
        return ctypes.byref(c)

    assert l.svb_pitch_ac_workspace_bytes(cfg(), np.array(ok, np.int64).ctypes.data, 2, None) > 0    # the refusals below are not vacuous
    refuse(None, ok, b'null config')
    big = _pitch_cfg(45920, 256, 4)
    assert l.svb_pitch_ac_workspace_bytes(ctypes.byref(big), np.array(ok, np.int64).ctypes.data, 2, None) > 0   # 576 lags: the widest
    big.sr, big.time_step = 45921, 256 / 45921                              # ceil(45921 / 80) + 2 = 577 lags
    refuse(ctypes.byref(big), ok, b'needs 577 lags, more than 576')
    big.sr, big.time_step = 48000, 256 / 48000
    refuse(ctypes.byref(big), ok, b'more than 576')
    refuse(cfg(ceiling=11025.5), ok, b'above sr / 2')
    assert l.svb_pitch_ac_workspace_bytes(cfg(ceiling=11025.0), np.array(ok, np.int64).ctypes.data, 2, None) > 0
    refuse(cfg(time_step=0.0058), ok, b'is not hop / sr')
    refuse(cfg(time_step=256 / 22050), ok, b'is not hop / sr')
    refuse(cfg(lpad=-1), ok, b'negative lpad')
    for k in ('voicing_threshold', 'octave_cost', 'octave_jump_cost', 'voiced_unvoiced_cost'):
        refuse(cfg(**{k: -0.01}), ok, b'negative threshold or cost')
    refuse(cfg(silence_threshold=0.0), ok, b'negative threshold or cost')
    refuse(cfg(), [22050, 0, 30000], b'clip 1 has 0 samples')
    longest = next(N for N in range(900, 700, -1) if _no_frame(P, N, 22050, 128))
    assert not _no_frame(P, longest + 1, 22050, 128)
    refuse(cfg(), [22050, 30000, longest], b'clip 2 has %d samples' % longest)
    refuse(cfg(), ok, b'no clips', n=0)
    # null buffers and a short workspace: svb_pitch_ac_batch only (the planner takes no buffers)
    lens = np.array(ok, np.int64)
    need = l.svb_pitch_ac_workspace_bytes(cfg(), lens.ctypes.data, 2, None)
    batch = lambda wav=p, m=mel.ctypes.data, f0=p, ws=p, nb=need: l.svb_pitch_ac_batch(cfg(), wav, lens.ctypes.data, 2, m, f0, ws, nb,
                                                                                        None, None, None, None, None)
    for k in ('wav', 'm', 'f0', 'ws'):
        assert batch(**{k: None}) < 0 and b'null buffer' in l.svb_last_error(), k
    assert batch(nb=need - 1) < 0 and b'workspace of %d bytes, %d needed' % (need - 1, need) in l.svb_last_error()
    assert l.svb_pitch_ac_workspace_bytes(cfg(), None, 2, None) < 0 and b'null lengths' in l.svb_last_error()
    assert (buf == 0).all()


def _no_frame(P, N, sr, hop):
    try:
        P.grid(N, sr, hop / sr)
        return False
    except ValueError:
        return True
