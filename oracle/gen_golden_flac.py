"""Write tests/golden/flac/: small FLAC files made by an encoder this project did not write (FFmpeg's native FLAC encoder in
libavcodec, driven through its C API with ctypes), each next to the PCM it encodes (``<name>.npz``: pcm int32 [n, channels], sr,
bits).  The tests decode every file with oracle/flac.py and csrc/flac.cu and compare with that PCM, so a misreading of the
specification shared by the project's own encoder and decoder shows up here.

    LD_LIBRARY_PATH=<its directory> python oracle/gen_golden_flac.py /path/to/libavcodec.so.NN

(any FFmpeg 5.1+ build of libavcodec with the native flac encoder; libavutil is loaded from the same directory)

FFmpeg's encoder writes 16- and 24-bit streams only; the 8-bit case is 8-bit PCM in a 16-bit stream (its samples are multiples of
256, so the encoder codes them with 8 wasted bits).  The 8-bit header code itself is covered by the test encoder."""
import ctypes
import os
import sys

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden', 'flac')
EAGAIN, EOF = -11, -0x20464F45
AV_PKT_DATA_NEW_EXTRADATA = 1

# name, sample rate, bits, channel layout, samples, compression level
CASES = [
    ('l0_s16_stereo', 44100, 16, 'stereo', 20000, 0),
    ('l5_s16_stereo', 44100, 16, 'stereo', 20000, 5),
    ('l12_s16_stereo', 44100, 16, 'stereo', 20000, 12),
    ('l5_s24_mono', 48000, 24, 'mono', 15000, 5),
    ('l12_s24_mono', 22050, 24, 'mono', 9000, 12),
    ('l5_u8_mono', 16000, 8, 'mono', 8000, 5),
    ('l5_s16_6ch', 48000, 16, '5.1', 6000, 5),
    ('l8_s16_odd', 32000, 16, 'stereo', 4608 * 2 + 777, 8),
]


def pcm_for(n, chans, bits, seed):
    """Tones with vibrato and a little noise, different per channel, plus a silent stretch (a CONSTANT subframe for the encoder)."""
    rng = np.random.default_rng(seed)
    t = np.arange(n)[:, None] / 8000.0
    f = 180.0 * (1 + np.arange(chans))[None, :]
    x = 0.5 * np.sin(2 * np.pi * f * t + 3 * np.sin(2 * np.pi * 5 * t)) + 0.02 * rng.standard_normal((n, chans))
    x[n // 3:n // 3 + 1500] = 0.0
    q = 1 << (bits - 1)
    return np.clip(np.round(x * q), -q, q - 1).astype(np.int32)


class AvCodec:
    def __init__(self, path):
        self.c = ctypes.CDLL(path)
        util = [f for f in os.listdir(os.path.dirname(path)) if f.startswith('libavutil')]
        self.u = ctypes.CDLL(os.path.join(os.path.dirname(path), util[0])) if util else self.c
        for lib, name, res, args in [
            (self.c, 'avcodec_find_encoder_by_name', ctypes.c_void_p, [ctypes.c_char_p]),
            (self.c, 'avcodec_find_decoder_by_name', ctypes.c_void_p, [ctypes.c_char_p]),
            (self.c, 'avcodec_alloc_context3', ctypes.c_void_p, [ctypes.c_void_p]),
            (self.c, 'avcodec_open2', ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
            (self.c, 'avcodec_send_packet', ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
            (self.c, 'avcodec_receive_frame', ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
            (self.c, 'avcodec_send_frame', ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
            (self.c, 'avcodec_receive_packet', ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
            (self.c, 'avcodec_free_context', None, [ctypes.c_void_p]),
            (self.c, 'av_packet_alloc', ctypes.c_void_p, []),
            (self.c, 'av_new_packet', ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
            (self.c, 'av_packet_unref', None, [ctypes.c_void_p]),
            (self.c, 'av_packet_get_side_data', ctypes.c_void_p, [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_size_t)]),
            (self.u, 'av_frame_alloc', ctypes.c_void_p, []),
            (self.u, 'av_frame_unref', None, [ctypes.c_void_p]),
            (self.u, 'av_opt_set', ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int]),
            (self.u, 'av_opt_set_int', ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int64, ctypes.c_int]),
            (self.u, 'av_opt_get_int', ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int64)]),
            (self.u, 'av_opt_next', ctypes.c_void_p, [ctypes.c_void_p, ctypes.c_void_p]),
        ]:
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args

    def field_offset(self, ctx, name):
        o = None
        while True:
            o = self.u.av_opt_next(ctx, o)
            assert o, name
            if ctypes.string_at(ctypes.c_void_p.from_address(o).value) == name:
                return ctypes.c_int.from_address(o + 16).value          # AVOption { name, help, int offset, ... }

    def context(self, codec, sr, layout, fmt, **opts):
        ctx = self.c.avcodec_alloc_context3(codec)
        # sample_fmt has no AVOption: it is the int between sample_rate ("ar") and ch_layout in AVCodecContext
        at = self.field_offset(ctx, b'ar') + 4
        assert at == self.field_offset(ctx, b'ch_layout') - 4
        ctypes.c_int.from_address(ctx + at).value = {'s16': 1, 's32': 2}[fmt]
        ok = [self.u.av_opt_set_int(ctx, b'ar', sr, 0), self.u.av_opt_set(ctx, b'ch_layout', layout.encode(), 0)]
        ok += [self.u.av_opt_set_int(ctx, k.encode(), v, 1) for k, v in opts.items()]
        assert all(r == 0 for r in ok), ok
        assert self.c.avcodec_open2(ctx, codec, None) == 0
        return ctx

    @staticmethod
    def packet_bytes(pkt):
        # AVPacket starts { AVBufferRef *buf; int64_t pts, dts; uint8_t *data; int size; ... } in every FFmpeg since 4.0
        data = ctypes.c_void_p.from_address(pkt + 24).value
        size = ctypes.c_int.from_address(pkt + 32).value
        return ctypes.string_at(data, size) if size else b''

    def encode(self, pcm, sr, bits, layout, level):
        n, chans = pcm.shape
        fmt, dec_name = ('s16', b'pcm_s16le') if bits <= 16 else ('s32', b'pcm_s32le')
        raw = (pcm.astype('<i2') if bits <= 16 else (pcm.astype(np.int64) << 8).astype('<i4'))
        enc = self.context(self.c.avcodec_find_encoder_by_name(b'flac'), sr, layout, fmt, compression_level=level,
                           bits_per_raw_sample=16 if bits <= 16 else 24)
        dec = self.context(self.c.avcodec_find_decoder_by_name(dec_name), sr, layout, fmt)
        fs = ctypes.c_int64()
        assert self.u.av_opt_get_int(enc, b'frame_size', 0, ctypes.byref(fs)) == 0 and fs.value > 0
        pkt, opkt, frame = self.c.av_packet_alloc(), self.c.av_packet_alloc(), self.u.av_frame_alloc()
        frames, streaminfo = [], None

        def drain():
            nonlocal streaminfo
            while True:
                r = self.c.avcodec_receive_packet(enc, opkt)
                if r in (EAGAIN, EOF):
                    return
                assert r == 0, r
                frames.append(self.packet_bytes(opkt))
                sz = ctypes.c_size_t()
                sd = self.c.av_packet_get_side_data(opkt, AV_PKT_DATA_NEW_EXTRADATA, ctypes.byref(sz))
                if sd:
                    streaminfo = ctypes.string_at(sd, sz.value)
                self.c.av_packet_unref(opkt)

        # PCM -> AVFrame through FFmpeg's own PCM decoder, so that no AVFrame field is set by hand
        for i in range(0, n, fs.value):
            chunk = raw[i:i + fs.value].tobytes()
            assert self.c.av_new_packet(pkt, len(chunk)) == 0
            ctypes.memmove(ctypes.c_void_p.from_address(pkt + 24).value, chunk, len(chunk))
            assert self.c.avcodec_send_packet(dec, pkt) == 0
            self.c.av_packet_unref(pkt)
            assert self.c.avcodec_receive_frame(dec, frame) == 0
            assert self.c.avcodec_send_frame(enc, frame) == 0
            self.u.av_frame_unref(frame)
            drain()
        assert self.c.avcodec_send_frame(enc, None) == 0
        drain()
        for ctx in (enc, dec):
            self.c.avcodec_free_context(ctypes.byref(ctypes.c_void_p(ctx)))
        assert streaminfo is not None and len(streaminfo) == 34, 'no final STREAMINFO from the encoder'
        return b'fLaC' + bytes([0x80, 0, 0, 34]) + streaminfo + b''.join(frames)


def main(path):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from oracle import flac as F
    av = AvCodec(path)
    os.makedirs(OUT, exist_ok=True)
    for k, (name, sr, bits, layout, n, level) in enumerate(CASES):
        chans = {'mono': 1, 'stereo': 2, '5.1': 6}[layout]
        pcm = pcm_for(n, chans, bits, 100 + k)
        stored = (pcm.astype(np.int32) << 8) if bits == 8 else pcm        # 8-bit PCM as 16-bit samples
        data = av.encode(stored, sr, bits if bits != 8 else 16, layout, level)
        got, si = F.decode(data, name, check_md5=True)
        assert np.array_equal(got, stored) and si['sample_rate'] == sr, name
        with open(os.path.join(OUT, name + '.flac'), 'wb') as f:
            f.write(data)
        np.savez_compressed(os.path.join(OUT, name + '.npz'), pcm=stored.astype(np.int32), sr=sr, bits=si['bits'], level=level)
        print(f'{name}: {len(data)} bytes, {n} samples x {chans} at {si["bits"]} bits, level {level}')


if __name__ == '__main__':
    main(sys.argv[1])
