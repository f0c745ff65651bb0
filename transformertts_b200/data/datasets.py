"""On-disk training-data formats and batching of the reference (SURVEY.md section 8(f) row 3), host side.

Mirrors ``data/datasets.py`` and ``data/metadata_readers.py`` of the reference:
  * metadata ``name|text`` files (``ljspeech`` reader :21-32, ``post_processed_reader`` :35-50 with the x10 upsampling
    of utterances containing ``?`` or ``!``), ``DataReader`` (datasets.py:19-73);
  * per-utterance ``.npy`` files: mel ``(T, mel_channels)`` float32, durations ``int32 (Tp,)``, per-character pitch
    ``(Tp,)`` (datasets.py:187-193), Aligner samples = start vector + mel + end vector with stop targets 1,..,1,2
    (datasets.py:88-93);
  * ``Dataset``: shuffle once per pass with ``Random(42)`` (datasets.py:241,285-291) and
    ``tf.data.experimental.bucket_by_sequence_length`` (datasets.py:256-269; TensorFlow, restated from its documented
    behaviour): bucket i takes lengths in ``[boundaries[i-1], boundaries[i])``, a bucket emits a zero-padded batch as soon
    as it holds ``bucket_batch_sizes[i]`` samples, the partial buckets are flushed in ascending bucket order at the end of a
    pass unless ``drop_remainder``; ``next_batch`` iterates over endless passes.
  * ``pitch_per_char`` (extract_durations.py:108-115).

What is GPU-specific: batches are assembled directly into PINNED host tensors and a background thread keeps
``prefetch`` batches ahead (``PrefetchLoader``), optionally already copied to the device on a side stream, so that the
training step's H2D copy (10 MB per LJ256 batch) overlaps the previous step; with ``rank`` / ``world_size`` every rank
takes a disjoint slice of each emitted batch (data-parallel training, one process per GPU).

Tokenisation is a callable ``text -> list[int]`` (the espeak phonemizer is outside the hot path); no TensorFlow.
"""
from __future__ import annotations

import queue
import threading
from pathlib import Path
from random import Random
from typing import Callable, Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch


# ----------------------------------------------------------------------------------------------------------------------
# metadata (data/metadata_readers.py)
# ----------------------------------------------------------------------------------------------------------------------
def ljspeech(metadata_path, column_sep: str = '|') -> Dict[str, str]:
    """metadata_readers.py:21-32: first column = file name (a ``.wav`` suffix is dropped), LAST column = text."""
    text_dict = {}
    with open(metadata_path, 'r', encoding='utf-8') as f:
        for line in f.readlines():
            parts = line.split(column_sep)
            filename, text = parts[0], parts[-1]
            if filename.endswith('.wav'):
                filename = filename.split('.')[0]
            text_dict[filename] = text.replace('\n', '')
    return text_dict


def post_processed_reader(metadata_path, column_sep: str = '|', upsample_indicators: str = '?!', upsample_factor: int = 10):
    """metadata_readers.py:35-50: SECOND column = text; names whose text holds one of the indicators are listed
    ``upsample_factor`` extra times (appended to the training file list by DataReader)."""
    text_dict, upsample = {}, []
    with open(metadata_path, 'r', encoding='utf-8') as f:
        for line in f.readlines():
            parts = line.split(column_sep)
            filename, text = parts[0], parts[1].replace('\n', '')
            if any(el in text for el in list(upsample_indicators)):
                upsample.extend([filename] * upsample_factor)
            text_dict[filename] = text
    return text_dict, upsample


def get_preprocessor_by_name(name: str) -> Callable:
    """metadata_readers.py:13-19."""
    return {'ljspeech': ljspeech, 'post_processed_reader': post_processed_reader}[name.lower()]


class DataReader:
    """datasets.py:19-73 (the wav scan is outside the path)."""

    def __init__(self, metadata_path, metadata_reading_function: Callable = None, training: bool = False, is_processed: bool = False,
                 wav_directory=None):
        self.metadata_reading_function = metadata_reading_function or (post_processed_reader if is_processed else ljspeech)
        self.metadata_path = Path(metadata_path)
        self.wav_directory = Path(wav_directory) if wav_directory is not None else None
        self.upsample: List[str] = []
        if not is_processed:
            self.text_dict = self.metadata_reading_function(self.metadata_path)
            self.filenames = list(self.text_dict.keys())
        else:
            self.text_dict, self.upsample = self.metadata_reading_function(self.metadata_path)
            self.filenames = list(self.text_dict.keys())
            if training:
                self.filenames += self.upsample

    KINDS = ('original', 'phonemized', 'train', 'valid')

    @classmethod
    def from_config(cls, config_manager, kind: str):
        """datasets.py:47-72: ``original`` reads the corpus metadata with the reader named by ``data_name``; ``phonemized``,
        ``train`` and ``valid`` read the processed ``name|phonemes`` files, the training list with its upsampled names."""
        if kind not in cls.KINDS:
            raise ValueError(f'Invalid kind type. Expected one of: {list(cls.KINDS)}')
        reader, training, is_processed = post_processed_reader, False, True
        if kind == 'train':
            metadata, training = config_manager.train_metadata_path, True
        elif kind == 'original':
            metadata = config_manager.metadata_path
            reader = get_preprocessor_by_name(config_manager.config['data_name'])
            is_processed = False
        elif kind == 'valid':
            metadata = config_manager.valid_metadata_path
        else:
            metadata = config_manager.phonemized_metadata_path
        return cls(metadata_path=metadata, metadata_reading_function=reader, training=training, is_processed=is_processed,
                   wav_directory=config_manager.wav_directory)


# ----------------------------------------------------------------------------------------------------------------------
# per-sample preprocessors (datasets.py:76-161)
# ----------------------------------------------------------------------------------------------------------------------
class AlignerPreprocessor:
    """datasets.py:76-104 -> (norm_mel (T+2, C), tokens, stop_probs (T+2), name)."""
    fields = ('mel', 'tokens', 'stop_prob', 'name')
    dtypes = (np.float32, np.int32, np.int32, None)

    def __init__(self, mel_channels: int, mel_start_value: float, mel_end_value: float, tokenizer: Callable):
        self.start_vec = np.ones((1, mel_channels), dtype=np.float32) * mel_start_value
        self.end_vec = np.ones((1, mel_channels), dtype=np.float32) * mel_end_value
        self.tokenizer = tokenizer

    def __call__(self, mel, text, sample_name):
        norm_mel = np.concatenate([self.start_vec, mel, self.end_vec], axis=0)
        stop_probs = np.ones((norm_mel.shape[0],))
        stop_probs[-1] = 2
        return norm_mel, self.tokenizer(text), stop_probs, sample_name

    @staticmethod
    def get_sample_length(norm_mel, *_):
        return norm_mel.shape[0]

    @classmethod
    def from_config(cls, config_manager, tokenizer: Callable):
        """datasets.py:98-103."""
        c = config_manager.config
        return cls(mel_channels=int(c['mel_channels']), mel_start_value=float(c['mel_start_value']),
                   mel_end_value=float(c['mel_end_value']), tokenizer=tokenizer)


class TTSPreprocessor:
    """datasets.py:143-161 -> (mel, tokens, durations, pitch, name)."""
    fields = ('mel', 'tokens', 'durations', 'pitch', 'name')
    dtypes = (np.float32, np.int32, np.int32, np.float32, None)

    def __init__(self, mel_channels: int, tokenizer: Callable):
        self.mel_channels = mel_channels
        self.tokenizer = tokenizer

    def __call__(self, text, mel, durations, pitch, sample_name):
        return mel, self.tokenizer(text), durations, pitch, sample_name

    @staticmethod
    def get_sample_length(mel, *_):
        return mel.shape[0]


# ----------------------------------------------------------------------------------------------------------------------
# bucketed, padded batches (datasets.py:233-291)
# ----------------------------------------------------------------------------------------------------------------------
def bucket_index(length: int, boundaries: Sequence[int]) -> int:
    """bucket_by_sequence_length: bucket i holds boundaries[i-1] <= length < boundaries[i]; the last bucket is open."""
    i = 0
    while i < len(boundaries) and length >= boundaries[i]:
        i += 1
    return i


def _pad_stack(items: List[np.ndarray], dtype, pin: bool, lead: Optional[int] = None) -> torch.Tensor:
    arrs = [np.asarray(a) for a in items]
    lead = max([a.shape[0] for a in arrs] + [lead or 0])
    shape = (len(arrs), lead) + tuple(arrs[0].shape[1:])
    out = torch.zeros(shape, dtype=torch.from_numpy(np.zeros(0, dtype=dtype)).dtype)
    if pin and torch.cuda.is_available():
        out = out.pin_memory()
    view = out.numpy()
    for i, a in enumerate(arrs):
        view[i, :a.shape[0]] = a
    return out


class Dataset:
    """datasets.py:233-291.  ``samples``: names; ``preprocessor(name)`` -> tuple described by ``fields`` / ``dtypes``
    (``dtype None`` = passed through as a python list, e.g. the sample names)."""

    def __init__(self, samples: list, preprocessor: Callable, len_function: Callable, fields: Tuple[str, ...], dtypes: tuple,
                 bucket_boundaries: list, bucket_batch_sizes: list, shuffle: bool = True, drop_remainder: bool = True, seed: int = 42,
                 pin_memory: bool = True, rank: int = 0, world_size: int = 1):
        if len(bucket_batch_sizes) != len(bucket_boundaries) + 1:
            raise ValueError('bucket_batch_sizes must have one more entry than bucket_boundaries')
        self._random = Random(seed)
        self._samples = samples[:]
        self.preprocessor = preprocessor
        self.len_function = len_function
        self.fields, self.dtypes = fields, dtypes
        self.boundaries, self.batch_sizes = list(bucket_boundaries), list(bucket_batch_sizes)
        self.shuffle, self.drop_remainder = shuffle, drop_remainder
        self.pin_memory = pin_memory
        self.rank, self.world_size = int(rank), int(world_size)
        if self.world_size > 1:
            # data parallel: every emitted (global) batch is split into equal row slices, so that all ranks walk the same
            # stream of batches, see shards of the same padded shape and the mean of the shard losses IS the loss of the
            # global batch (the reference loss is a mean over the padded batch tensor, utils/losses.py:41-49)
            bad = [b for b in self.batch_sizes if b % self.world_size]
            if bad:
                raise ValueError(f'data-parallel batching needs bucket batch sizes divisible by world_size={self.world_size}; got {bad} '
                                 f'(round them with datasets.round_batch_sizes)')
        self._endless: Optional[Iterator] = None

    def _datagen(self, shuffle: bool):
        """Shuffle once per pass (the Random instance persists, so every pass has a new order; datasets.py:285-291)."""
        samples = self._samples[:]
        if shuffle:
            self._random.shuffle(samples)
        return (self.preprocessor(s) for s in samples)

    def _emit(self, rows: list) -> dict:
        # padded lengths come from the GLOBAL batch, so every rank's shard has the same shape
        leads = [None if dt is None else max(np.asarray(r[k]).shape[0] for r in rows) for k, dt in enumerate(self.dtypes)]
        if self.world_size > 1:  # data parallel: rank r takes rows r, r + W, ... of every global batch
            rows = rows[self.rank::self.world_size]
        batch = {}
        for k, (name, dt) in enumerate(zip(self.fields, self.dtypes)):
            col = [r[k] for r in rows]
            batch[name] = col if dt is None else _pad_stack(col, dt, self.pin_memory, leads[k])
        return batch

    def _one_pass(self) -> Iterator[dict]:
        buckets: List[list] = [[] for _ in self.batch_sizes]
        for sample in self._datagen(self.shuffle):
            b = bucket_index(int(self.len_function(*sample)), self.boundaries)
            buckets[b].append(sample)
            if len(buckets[b]) == self.batch_sizes[b]:
                rows, buckets[b] = buckets[b], []
                yield self._emit(rows)
        if not self.drop_remainder:
            for rows in buckets:
                # data parallel: the tail is cut to a multiple of world_size (identical on every rank), never skipped by
                # some ranks only
                rows = rows[:len(rows) - len(rows) % self.world_size]
                if rows:
                    yield self._emit(rows)

    def all_batches(self) -> Iterator[dict]:
        return self._one_pass()

    def next_batch(self) -> dict:
        if self._endless is None:
            def forever():
                while True:
                    empty = True
                    for b in self._one_pass():
                        empty = False
                        yield b
                    if empty:
                        raise RuntimeError('the dataset yields no batch (every bucket is smaller than its batch size)')
            self._endless = forever()
        return next(self._endless)


def round_batch_sizes(batch_sizes: Sequence[int], world_size: int) -> List[int]:
    """Bucket batch sizes of the single-process config (training_config.yaml:22-23) rounded DOWN to multiples of the
    data-parallel world size (at least one row per rank)."""
    return [max(world_size, b - b % world_size) for b in batch_sizes]


class _FileDataset:
    def get_dataset(self, bucket_batch_sizes, bucket_boundaries, shuffle=True, drop_remainder=False, **kw) -> Dataset:
        return Dataset(samples=self.metadata_reader.filenames, preprocessor=self._process_sample,
                       len_function=self.preprocessor.get_sample_length, fields=self.preprocessor.fields,
                       dtypes=self.preprocessor.dtypes, shuffle=shuffle, drop_remainder=drop_remainder,
                       bucket_batch_sizes=bucket_batch_sizes, bucket_boundaries=bucket_boundaries, **kw)


class AlignerDataset(_FileDataset):
    """datasets.py:106-140."""

    def __init__(self, data_reader: DataReader, preprocessor: AlignerPreprocessor, mel_directory):
        self.metadata_reader = data_reader
        self.preprocessor = preprocessor
        self.mel_directory = Path(mel_directory)

    def _read_sample(self, sample_name):
        text = self.metadata_reader.text_dict[sample_name]
        mel = np.load((self.mel_directory / sample_name).with_suffix('.npy').as_posix())
        return mel, text

    def _process_sample(self, sample_name):
        mel, text = self._read_sample(sample_name)
        return self.preprocessor(mel=mel, text=text, sample_name=sample_name)

    @classmethod
    def from_config(cls, config_manager, preprocessor: AlignerPreprocessor, kind: str, mel_directory=None):
        """datasets.py:136-150."""
        if kind not in DataReader.KINDS:
            raise ValueError(f'Invalid kind type. Expected one of: {list(DataReader.KINDS)}')
        return cls(data_reader=DataReader.from_config(config_manager, kind=kind), preprocessor=preprocessor,
                   mel_directory=config_manager.mel_dir if mel_directory is None else mel_directory)


class TTSDataset(_FileDataset):
    """datasets.py:164-230: mel, durations and per-character pitch of one utterance are three ``.npy`` files."""

    def __init__(self, data_reader: DataReader, preprocessor: TTSPreprocessor, mel_directory, duration_directory,
                 pitch_per_char_directory, pitch_directory=None):
        self.metadata_reader = data_reader
        self.preprocessor = preprocessor
        self.mel_directory = Path(mel_directory)
        self.duration_directory = Path(duration_directory)
        self.pitch_directory = Path(pitch_directory) if pitch_directory is not None else None
        self.pitch_per_char_directory = Path(pitch_per_char_directory)

    def _read_sample(self, sample_name: str):
        text = self.metadata_reader.text_dict[sample_name]
        mel = np.load((self.mel_directory / sample_name).with_suffix('.npy').as_posix())
        durations = np.load((self.duration_directory / sample_name).with_suffix('.npy').as_posix())
        char_wise_pitch = np.load((self.pitch_per_char_directory / sample_name).with_suffix('.npy').as_posix())
        return mel, text, durations, char_wise_pitch

    def _process_sample(self, sample_name: str):
        mel, text, durations, pitch = self._read_sample(sample_name)
        return self.preprocessor(mel=mel, text=text, durations=durations, pitch=pitch, sample_name=sample_name)


# ----------------------------------------------------------------------------------------------------------------------
# extract_durations.py:108-115
# ----------------------------------------------------------------------------------------------------------------------
def pitch_per_char(pitch: np.ndarray, durations: np.ndarray, mel_len: int, pitch_mean: float, pitch_std: float) -> np.ndarray:
    """Mean of the non-zero, < 400 Hz (after de-normalisation) frame pitches under each character; 0 where none.
    As in the reference the loop runs over ``min(mel_len, len(durations))`` characters."""
    durs_cum = np.cumsum(np.pad(durations, (1, 0)))
    pitch_char = np.zeros((durations.shape[0],), dtype=np.float64)
    for idx, a, b in zip(range(mel_len), durs_cum[:-1], durs_cum[1:]):
        values = pitch[a:b][np.where(pitch[a:b] != 0.0)[0]]
        values = values[np.where((values * pitch_std + pitch_mean) < 400)[0]]
        pitch_char[idx] = np.mean(values) if len(values) > 0 else 0.0
    return pitch_char


# ----------------------------------------------------------------------------------------------------------------------
# background prefetch into pinned memory / onto the device
# ----------------------------------------------------------------------------------------------------------------------
class PrefetchLoader:
    """Keeps ``prefetch`` batches of ``dataset.next_batch()`` ready.  With ``device`` set the tensors are copied on a side
    CUDA stream from their pinned buffers; ``next()`` makes the consumer's current stream wait for that copy only."""

    def __init__(self, dataset: Dataset, prefetch: int = 4, device: Optional[torch.device] = None):
        self.dataset = dataset
        self.device = torch.device(device) if device is not None else None
        self._q: 'queue.Queue' = queue.Queue(maxsize=max(1, prefetch))
        self._stop = threading.Event()
        self._stream = torch.cuda.Stream(self.device) if self.device is not None and self.device.type == 'cuda' else None
        self._error: Optional[BaseException] = None
        self._thread = threading.Thread(target=self._work, daemon=True)
        self._thread.start()

    def _work(self):
        try:
            while not self._stop.is_set():
                batch = self.dataset.next_batch()
                event = None
                if self._stream is not None:
                    with torch.cuda.stream(self._stream):
                        batch = {k: (v.to(self.device, non_blocking=True) if torch.is_tensor(v) else v) for k, v in batch.items()}
                        event = torch.cuda.Event()
                        event.record(self._stream)
                while not self._stop.is_set():
                    try:
                        self._q.put((batch, event), timeout=0.1)
                        break
                    except queue.Full:
                        continue
        except BaseException as e:  # surfaced to the consumer
            self._error = e
            self._q.put((None, None))

    def next(self) -> dict:
        batch, event = self._q.get()
        if batch is None:
            raise RuntimeError('prefetch thread failed') from self._error
        if event is not None:
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(event)
            # the tensors were allocated on the side stream: tell the caching allocator that the consumer's stream uses them,
            # or their blocks could be handed to the next prefetch copy while training kernels still read them
            for v in batch.values():
                if torch.is_tensor(v) and v.is_cuda:
                    v.record_stream(cur)
        return batch

    __next__ = next

    def __iter__(self):
        return self

    def close(self):
        self._stop.set()
        self._thread.join(timeout=2.0)
