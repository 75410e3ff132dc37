"""Host-side checks of the GlobalFVAE training path (no GPU needed): the new C entry points reject bad arguments before any
CUDA call, and the Python modules keep refusing what they cannot do (training when not opted in, CPU tensors, dropout)."""
import ctypes
import os

import pytest
import torch

from neuralsvb_b200 import _native


@pytest.fixture(scope='module')
def lib():
    try:
        _native.build()
    except RuntimeError as e:          # no nvcc on this box: the prebuilt library must already be there
        if not os.path.exists(_native.LIB_PATH):
            pytest.fail(str(e))
    return _native.lib()


def test_wn_training_entry_points_reject_a_null_handle(lib):
    import numpy as np
    buf = np.zeros(1 << 12, np.float32)
    p = ctypes.c_void_p(buf.ctypes.data)           # host memory stands in for every buffer: the call must refuse first
    err = lambda: lib.svb_last_error()
    assert lib.svb_wn_set_training(None, 1) < 0 and b'not finalized' in err()
    assert lib.svb_wn_tape_bytes(None, 2, 64) == -1
    assert lib.svb_wn_forward_train(None, p, p, p, 2, 64, p, p, None) < 0 and b'not finalized' in err()
    assert lib.svb_fvae_decoder_forward_train(None, p, p, p, 2, 64, p, p, None) < 0 and b'not a finalized decoder' in err()
    assert lib.svb_wn_backward(None, p, 2, 64, p, p, p, None) < 0 and b'not a training handle' in err()
    assert lib.svb_fvae_decoder_backward(None, p, 2, 64, p, p, p, None) < 0 and b'not a training handle' in err()
    assert lib.svb_wn_zero_grad(None, None) < 0 and b'not a training handle' in err()
    assert lib.svb_wn_grad_numel(None, b'in_layers.0.weight') == -1
    assert lib.svb_wn_get_grad(None, b'in_layers.0.weight', p, 4, None) < 0 and b'null argument' in err()
    assert lib.svb_wn_set_weight_dev(None, b'in_layers.0.weight', p, 4, None) < 0 and b'null argument' in err()
    assert lib.svb_wn_update_weights_dev(None, None) < 0 and b'not a training handle' in err()


def test_conv_nct_backward_admits_k8_and_still_rejects_k9(lib):
    """K = 8 (the GlobalFVAE's pre_net / g_pre_net) has a weight-gradient instance now; K = 9 still has none."""
    import numpy as np
    buf = np.zeros(1 << 16, np.float32)
    p = ctypes.c_void_p(buf.ctypes.data)
    f = ctypes.c_float
    nct = lambda K, stride: lib.svb_conv_nct_backward(p, p, p, p, 1, 4, 4, 64, 1, K, stride, 1, 0, 1, f(0.1), p, p, p, p, None)
    assert nct(9, 1) < 0 and b'kernel size 9 has no weight-gradient instance' in lib.svb_last_error()
    assert nct(8, 5) < 0 and b'stride 5 unsupported' in lib.svb_last_error()      # a K = 8 call reaches the later checks


def _modules(trainable, p_dropout=0):
    from neuralsvb_b200.modules.fastspeech.fs2_vae import WN, FVAEDecoder, GlobalFVAEEncoder
    return (WN(64, 3, 1, 2, p_dropout=p_dropout, trainable=trainable), FVAEDecoder(16, 64, 80, 3, 2, p_dropout=p_dropout, trainable=trainable),
            GlobalFVAEEncoder(80, 64, 16, 3, 2, 0, p_dropout=p_dropout, trainable=trainable))


def _call(m, i):
    if i == 0:
        return m(torch.zeros(1, 64, 16))
    if i == 1:
        return m(torch.zeros(1, 16, 4), torch.ones(1, 1, 16), None)
    return m(torch.zeros(1, 80, 16), torch.ones(1, 1, 16), None)


def test_default_modules_still_refuse_training():
    for i, m in enumerate(_modules(False)):
        with pytest.raises(RuntimeError, match='inference only'):
            _call(m.train(), i)


def test_trainable_modules_have_no_cpu_path():
    for i, m in enumerate(_modules(True)):
        with pytest.raises(RuntimeError, match='no CPU path'):
            _call(m.train(), i)
        with pytest.raises(RuntimeError, match='no CPU path'):
            with torch.no_grad():
                _call(m.eval(), i) if i < 2 else m.wn(torch.zeros(1, 64, 4))


def test_dropout_is_refused_in_training():
    wn, dec, enc = _modules(True, p_dropout=0.1)
    with pytest.raises(NotImplementedError, match='p_dropout'):
        _call(wn.train(), 0)
    with pytest.raises(NotImplementedError, match='p_dropout'):
        _call(dec.train(), 1)
    with pytest.raises(NotImplementedError, match='p_dropout'):
        enc.wn.train()(torch.zeros(1, 64, 4))


def test_trainable_is_passed_down():
    from neuralsvb_b200.modules.fastspeech.fs2_vae import GlobalFVAE
    m = GlobalFVAE(80, 64, 16, 3, 2, 2, 32, [4], trainable=True)
    assert m.encoder.trainable and m.encoder.wn.trainable and m.decoder.trainable and m.decoder.wn.trainable
    m = GlobalFVAE(80, 64, 16, 3, 2, 2, 32, [4])
    assert not (m.encoder.trainable or m.decoder.trainable or m.encoder.wn.trainable)
