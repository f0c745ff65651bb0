"""FLAC without a GPU: the numpy encoder round-trips every coding tool through the plain decoder (tests/flac_oracle.py), the host
STREAMINFO parser (data/audio.py: FlacStream) skips every metadata block it need not read and refuses malformed or unsupported
files by name, ttsb_flac_decode_batch refuses bad tables before any CUDA call, and the corpus scans find .flac files."""
import re

import numpy as np
import pytest

import flac_oracle as fo

CASES = fo.tool_matrix()


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_oracle_round_trips_the_tool_matrix(case):
    name, x, rate, bps, kw = case
    y, info = fo.decode(fo.encode(x, rate, bps, **kw))
    assert np.array_equal(x, y)
    assert (info['rate'], info['bps'], info['channels'], info['total']) == (rate, bps, x.shape[1], len(x))


def test_crc16_batch_equals_the_plain_crc():
    rng = np.random.default_rng(0)
    blobs = [rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in (0, 1, 2, 3, 17, 1000, 4097)]
    assert fo.crc16_batch(blobs) == [fo.crc16(b) for b in blobs]
    assert fo.crc16(b'123456789') == 0xFEE8 and fo.crc8(b'123456789') == 0xF4       # the published check values


def _stream(data, name='x.flac'):
    from transformertts_b200.data.audio import FlacStream
    return FlacStream(name, data)


def _file(blocks=(), bps=16, total=1000, min_block=4096, max_block=4096):
    return fo.flac_file(fo.streaminfo(min_block, max_block, 22050, 1, bps, total), blocks) + b'\xff\xf8'


@pytest.mark.parametrize('kind', [fo.PADDING, fo.APPLICATION, fo.SEEKTABLE, fo.VORBIS_COMMENT, fo.CUESHEET, fo.PICTURE, 9])
def test_metadata_blocks_are_skipped(kind):
    x = fo.speech_like(3000, 2, 16, 22050, 5)
    body = bytes(range(256)) * 3
    data = fo.encode(x, 22050, 16, metadata=[(kind, body), (fo.PADDING, bytes(10))])
    st = _stream(data)
    assert st.frame_offset == 4 + 38 + 4 + len(body) + 4 + 10
    assert st.stream_info() == (2, 16, 22050, 3000, 3000, 3000)
    assert data[st.frame_offset:st.frame_offset + 2] == b'\xff\xf8'


def test_the_default_metadata_is_skipped():
    x = fo.speech_like(9000, 1, 24, 48000, 6)
    data = fo.encode(x, 48000, 24)
    st = _stream(data)
    assert st.stream_info() == (1, 24, 48000, 4096, 4096, 9000)
    assert st.frame_offset > 8192 and data[st.frame_offset:st.frame_offset + 2] == b'\xff\xf8'


@pytest.mark.parametrize('data, what', [
    (b'RIFF\x00\x00\x00\x00WAVE', 'no fLaC magic'),
    (b'fL', 'truncated metadata'),
    (b'fLaC' + bytes([0x80 | fo.PADDING, 0, 0, 4]) + bytes(4), 'not a 34-byte STREAMINFO'),
    (_file()[:20], 'truncated metadata'),
    (fo.flac_file(fo.streaminfo(4096, 4096, 22050, 1, 16, 1000), [(fo.PADDING, bytes(100))])[:60], 'truncated metadata'),
    (_file(total=0), 'unknown (0) total'),
    (_file(bps=25), '25-bit FLAC is not supported'),
    (_file(bps=32), '32-bit FLAC is not supported'),
    (_file(bps=3), '3 bits per sample is not supported'),
    (_file(min_block=8, max_block=4096), 'block sizes'),
    (_file(blocks=[(127, b'')]), 'type 127'),
], ids=lambda v: v if isinstance(v, str) else None)
def test_malformed_or_unsupported_files_are_refused_by_name(data, what):
    with pytest.raises(ValueError, match=re.escape(what)) as e:
        _stream(data, 'corpus/LJ001-0001.flac')
    assert 'corpus/LJ001-0001.flac' in str(e.value)


def test_read_for_batch_refuses_by_name(tmp_path):
    from transformertts_b200.data.audio import Audio
    audio = Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                  normalizer='MelGAN', device='cpu')
    p = tmp_path / 'bad.flac'
    p.write_bytes(_file(bps=28))
    with pytest.raises(ValueError, match='bad.flac: 28-bit FLAC is not supported'):
        audio.read_for_batch(p)
    good = tmp_path / 'good.flac'
    good.write_bytes(fo.encode(fo.speech_like(3000, 1, 16, 48000, 1), 48000, 16))
    st, sr = audio.read_for_batch(good)
    assert sr is None and st.total_samples == 3000 and st.sample_rate == 48000


def test_the_entry_point_refuses_bad_tables_before_any_cuda_call():
    import ctypes as C
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    cdll = lib.load()
    p = C.c_void_p(256)

    def call(offsets, info, n=1):        # only tables that are refused reach the decode call: fake pointers, nothing launches
        bo = (C.c_int64 * len(offsets))(*offsets)
        si = (C.c_int64 * len(info))(*info)
        ws = cdll.ttsb_flac_decode_workspace_bytes(bo, si, n)
        rc = cdll.ttsb_flac_decode_batch(p, bo, si, n, p, None, p, p, C.c_int64(1 << 40), None) if ws < 0 else None
        return ws, rc, cdll.ttsb_last_error().decode()

    ws, rc, _ = call([0, 1000], [2, 16, 22050, 4096, 4096, 10000])
    assert ws >= 4 * 2 * 10000 + 1000 // 5 * 12
    for info, what in (([2, 25, 22050, 4096, 4096, 10], '25- to 32-bit FLAC is not supported'),
                       ([2, 32, 22050, 4096, 4096, 10], '25- to 32-bit FLAC is not supported'),
                       ([9, 16, 22050, 4096, 4096, 10], 'channels'), ([2, 3, 22050, 4096, 4096, 10], 'bits per sample'),
                       ([2, 16, 22050, 8, 4096, 10], 'min block size'), ([2, 16, 22050, 4096, 70000, 10], 'max block size'),
                       ([2, 16, 22050, 4096, 4096, 0], 'total_samples'), ([2, 16, 0, 4096, 4096, 10], 'sample rate')):
        ws, rc, err = call([0, 1000], info)
        assert ws == -1 and rc == -1 and what in err, (info, err)
    for offsets, what in (([5, 1000], 'start at 0'), ([0, 1000, 500], 'decrease')):
        ws, rc, err = call(offsets, [1, 16, 22050, 4096, 4096, 10] * (len(offsets) - 1), len(offsets) - 1)
        assert ws == -1 and rc == -1 and what in err, (offsets, err)
    bo = (C.c_int64 * 2)(0, 1000)
    si = (C.c_int64 * 6)(1, 16, 22050, 4096, 4096, 10)
    need = cdll.ttsb_flac_decode_workspace_bytes(bo, si, 1)
    assert cdll.ttsb_flac_decode_batch(p, bo, si, 1, p, None, p, p, C.c_int64(need - 1), None) == -1
    assert 'workspace too small' in cdll.ttsb_last_error().decode()


def _touch(path):
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_bytes(b'')


def test_scans_find_flac_and_refuse_stem_collisions(tmp_path):
    from transformertts_b200.data.datasets import DataReader, scan_recordings
    wav_only = tmp_path / 'wav_only'
    for name in ('a.wav', 'sub/b.wav', 'sub/deeper/c.wav', 'notes.txt', 'd.WAV.bak'):
        _touch(wav_only / name)
    want = {w.with_suffix('').name: w for w in wav_only.resolve().rglob('*.wav')}
    got = scan_recordings(wav_only)
    assert got == want and list(got) == list(want)
    (tmp_path / 'meta.csv').write_text('a|x|x\n', encoding='utf-8')
    reader = DataReader(tmp_path / 'meta.csv', wav_directory=wav_only, scan_wavs=True)
    assert reader.wav_paths == want and list(reader.wav_paths) == list(want)
    mixed = tmp_path / 'mixed'
    for name in ('a.wav', 'b.flac', 'sub/c.flac', 'sub/d.wav'):
        _touch(mixed / name)
    got = DataReader(tmp_path / 'meta.csv', wav_directory=mixed, scan_wavs=True).wav_paths
    assert {k: v.name for k, v in got.items()} == {'a': 'a.wav', 'b': 'b.flac', 'c': 'c.flac', 'd': 'd.wav'}
    _touch(mixed / 'other' / 'c.wav')
    with pytest.raises(ValueError, match='^c exists as both'):
        scan_recordings(mixed)
    with pytest.raises(ValueError, match='c exists as both'):
        DataReader(tmp_path / 'meta.csv', wav_directory=mixed, scan_wavs=True)
