"""FLAC decoding on the GPU (ttsb_flac_decode_batch through data/audio.py): every coding tool of the numpy encoder
(tests/flac_oracle.py) decodes to the encoded PCM bit for bit and to read_wav's float32 mono of the same PCM as WAV; a ragged
batch equals each file alone; a sync lookalike inside subframe data is ignored; malformed streams are refused by file and frame
while the rest of the call decodes; create_training_data.py writes byte-identical files for a corpus stored as WAV and as FLAC."""
import pickle
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import yaml

import flac_oracle as fo

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
CASES = fo.tool_matrix()


def _audio(**kw):
    from transformertts_b200.data.audio import Audio
    s = dict(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
             normalizer='MelGAN')
    s.update(kw)
    return Audio(**s)


def _decode(blobs, pcm=True):
    from transformertts_b200.data.audio import FlacStream, flac_decode_streams
    return flac_decode_streams([FlacStream(f'f{i}.flac', b) for i, b in enumerate(blobs)], 'cuda:0', pcm=pcm)


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_tool_matrix_decodes_bit_exactly(case, tmp_path):
    name, x, rate, bps, kw = case
    r = _decode([fo.encode(x, rate, bps, **kw)])[0]
    assert r['error'] is None
    assert r['pcm'].shape == x.shape and np.array_equal(r['pcm'], x)
    fo.write_wav(tmp_path / 'x.wav', x, rate, bps)
    want, sr = _audio().read_wav(tmp_path / 'x.wav')
    assert sr == rate == r['rate'] and r['mono'].dtype == np.float32 and np.array_equal(r['mono'], want)


def _ragged_corpus():
    rng = np.random.default_rng(7)
    out = []
    for i in range(64):
        C = int(rng.choice([1, 2, 2, 3, 6, 8]))
        bps = int(rng.choice([8, 12, 16, 20, 24]))
        rate = int(rng.choice([16000, 22050, 44100, 48000]))
        n = int(rng.integers(50, 30000))
        x = fo.speech_like(n, C, bps, rate, 1000 + i)
        kw = dict(block_size=int(rng.choice([576, 1152, 4096])))
        if i % 5 == 0 and n >= 48:
            kw = dict(variable=True, blocks=[n // 3, n // 3, n - 2 * (n // 3)])
        out.append((x, rate, bps, fo.encode(x, rate, bps, **kw)))
    return out


def test_ragged_batch_equals_each_file_alone():
    from transformertts_b200.data.audio import FlacStream, flac_decode_streams
    corpus = _ragged_corpus()
    alone = [_decode([blob])[0] for _, _, _, blob in corpus]
    poison = bytes([0xFF, 0xF8, 0xC9, 0x18, 0x00, 0xC2]) * 50 + bytes(range(256))
    streams = [FlacStream(f'f{i}.flac', blob + poison) for i, (_, _, _, blob) in enumerate(corpus)]   # trailing bytes after the
    batch = flac_decode_streams(streams, 'cuda:0', pcm=True)                                             # total are never read
    for i, ((x, rate, _, _), a, b) in enumerate(zip(corpus, alone, batch)):
        assert a['error'] is None and b['error'] is None, i
        assert np.array_equal(a['pcm'], x) and np.array_equal(b['pcm'], x), i
        assert np.array_equal(a['mono'], b['mono']), i


def test_a_sync_lookalike_in_subframe_data_is_ignored():
    x = fo.speech_like(3 * 4096, 1, 16, 22050, 11)
    clean = fo.encode(x, 22050, 16, spec=dict(type='verbatim'), metadata=None)
    hdr = fo.frame_header(4096, 22050, 0, 16, 1, False)            # frame 1's header, with a correct CRC-8
    assert clean.find(hdr) > 0
    raw = hdr + bytes(len(hdr) % 2)
    words = np.frombuffer(raw, '>i2').astype(np.int64)
    y = x.copy()
    y[100:100 + len(words), 0] = words                              # a VERBATIM 16-bit subframe stores these bytes as they are
    blob = fo.encode(y, 22050, 16, spec=dict(type='verbatim'))
    st_off = blob.find(hdr)
    assert 0 < st_off < blob.find(hdr, st_off + 1)                  # the lookalike lies inside frame 0, before the real frame 1
    r = _decode([blob])[0]
    assert r['error'] is None and np.array_equal(r['pcm'], y)


def test_malformed_streams_are_refused_by_file_and_frame():
    from transformertts_b200.data.audio import Audio, FlacDecodeError, FlacStream
    good = [fo.speech_like(20000, 1, 16, 22050, 20 + i) for i in range(3)]
    spec = dict(type='fixed', order=2, escape=True)         # fixed-width residuals: a flipped bit leaves the frame's layout
    blobs = [fo.encode(x, 22050, 16, spec=spec) for x in good]
    # flip a residual bit in the middle of frame 2: its CRC-16 fails
    hdr2 = fo.frame_header(4096, 22050, 0, 16, 2, False)
    hdr3 = fo.frame_header(4096, 22050, 0, 16, 3, False)
    a, b = blobs[1].index(hdr2), blobs[1].index(hdr3)
    flipped = bytearray(blobs[1])
    flipped[(a + b) // 2] ^= 0x10
    truncated = blobs[2][:(blobs[2].index(hdr2) + blobs[2].index(hdr3)) // 2]
    res = _decode([blobs[0], bytes(flipped), truncated])
    assert res[0]['error'] is None and np.array_equal(res[0]['pcm'], good[0])
    assert res[1]['error'] == 'CRC-16 mismatch (frame 2)', res[1]['error']
    assert res[2]['error'].startswith('the data ends inside a frame') and res[2]['error'].endswith('(frame 2)'), res[2]['error']
    assert not res[1]['mono'].any() and not res[2]['mono'].any()
    with pytest.raises(FlacDecodeError, match=r'bad\.flac: CRC-16 mismatch \(frame 2\)') as e:
        Audio.read_flac_batch(_audio(), [FlacStream('ok.flac', blobs[0]), FlacStream('bad.flac', bytes(flipped)),
                                         FlacStream('cut.flac', truncated)])
    assert set(e.value.failed) == {'bad.flac', 'cut.flac'}


def _corpus(root: Path, fmt: str):
    """Eight files: 22050 and 48000 Hz, mono and stereo, 16 and 24-bit, in `fmt` ('wav' or 'flac'), with a metadata file."""
    wav_dir = root / 'wavs'
    wav_dir.mkdir(parents=True)
    rng = np.random.default_rng(3)
    names, texts = [], []
    for i, (rate, C, bps) in enumerate([(22050, 1, 16), (48000, 2, 24), (22050, 2, 16), (48000, 1, 16), (22050, 1, 24),
                                        (48000, 2, 16), (22050, 2, 24), (48000, 1, 24)]):
        n = int(rng.integers(int(1.2 * rate), int(2.5 * rate)))
        x = fo.speech_like(n, C, bps, rate, 300 + i)
        name = f'LJ{i:03d}-{rate}-{C}-{bps}'
        if fmt == 'wav':
            fo.write_wav(wav_dir / f'{name}.wav', x, rate, bps)
        else:
            (wav_dir / f'{name}.flac').write_bytes(fo.encode(x, rate, bps))
        names.append(name)
        texts.append(''.join(rng.choice(list('abdefhijklmnoprstuvwz'), int(rng.integers(5, 30)))))
    (root / 'metadata.csv').write_text(''.join(f'{n}|raw text|{t}\n' for n, t in zip(names, texts)), encoding='utf-8')
    return names


@pytest.mark.parametrize('trim', [False, True])
def test_create_training_data_is_byte_identical_for_wav_and_flac(tmp_path, trim):
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    outputs = {}
    for fmt in ('wav', 'flac'):
        root = tmp_path / fmt
        _corpus(root, fmt)
        cfg = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
        cfg['paths'].update(log_directory=str(root / 'logs'), train_data_directory=str(root / 'data'),
                            metadata_path=str(root / 'metadata.csv'), wav_directory=str(root / 'wavs'))
        cfg['training_data_settings'].update(n_test=2, min_mel_len=30, max_mel_len=400)
        if trim:
            cfg['audio_settings'] = dict(cfg.get('audio_settings') or {}, trim_silence=True, trim_silence_top_db=60,
                                         trim_long_silences=False)
        (root / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
        r = subprocess.run([sys.executable, str(ROOT / 'create_training_data.py'), '--config', str(root / 'cfg.yaml')],
                           cwd=root, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout + r.stderr
        data = TrainingConfigManager(root / 'cfg.yaml', aligner=True).data_dir
        outputs[fmt] = {str(p.relative_to(data)): p.read_bytes() for p in sorted(data.rglob('*')) if p.is_file()}
    wav, flac = outputs['wav'], outputs['flac']
    assert set(wav) == set(flac)
    assert sum(k.endswith('.npy') for k in wav) >= 12 and any(k.endswith('pitch_stats.pkl') for k in wav)
    assert any(k.endswith('mel_len.pkl') for k in wav)
    for k in wav:
        assert wav[k] == flac[k], k
    lens = pickle.loads(next(v for k, v in wav.items() if k.endswith('mel_len.pkl')))
    assert len(lens) == 8


def test_load_wav_of_flac_equals_load_wav_of_wav(tmp_path):
    audio = _audio(norm_wav=True, target_dBFS=-30, int16_max=32767)
    for i, (C, bps) in enumerate([(1, 16), (2, 24), (3, 12)]):
        x = fo.speech_like(30000, C, bps, 22050, 40 + i)
        fo.write_wav(tmp_path / f'{i}.wav', x, 22050, bps)
        (tmp_path / f'{i}.flac').write_bytes(fo.encode(x, 22050, bps))
        a, sa = audio.load_wav(tmp_path / f'{i}.wav')
        b, sb = audio.load_wav(tmp_path / f'{i}.flac')
        assert sa == sb == 22050 and a.dtype == b.dtype and np.array_equal(a, b)
    paths = [tmp_path / '0.flac', tmp_path / '1.wav', tmp_path / '2.flac']
    assert all(np.array_equal(a, b) for a, b in zip(audio.load_wavs(paths), audio.load_wavs([p.with_suffix('.wav') for p in paths])))
