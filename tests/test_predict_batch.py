"""ForwardTransformer.predict_batch without a device: the batch plan (sort, split, padding, rounded shapes) and every input
refusal, which happens before anything is placed on the GPU."""
import numpy as np
import pytest
import torch

from oracle import forward_oracle as fo
from transformertts_b200.model.models import (GRAPH_TM_MULTIPLE, GRAPH_TP_MULTIPLE, ForwardTransformer, _round_len, padded_batch,
                                              plan_batches)


def test_plan_sorts_by_length_and_splits():
    lengths = [5, 2, 9, 2, 7, 1, 9]
    plan = plan_batches(lengths, 3)
    assert plan == [[5, 1, 3], [0, 4, 2], [6]]          # stable: equal lengths keep input order
    flat = [i for b in plan for i in b]
    assert sorted(flat) == list(range(len(lengths)))     # a permutation: every line exactly once
    inverse = np.argsort(flat)                            # where each input line sits in the plan
    assert [flat[j] for j in inverse] == list(range(len(lengths)))
    assert [lengths[i] for i in flat] == sorted(lengths)
    assert plan_batches(lengths, 64) == [flat]
    assert plan_batches(lengths, 1) == [[i] for i in flat]


def test_padded_batch_and_rounded_shapes():
    lines = [np.array([3, 4, 5]), np.array([7]), np.array([1, 2])]
    tok = padded_batch(lines, [1, 2, 0], 4)
    assert tok.dtype == np.int32
    assert tok.tolist() == [[7, 0, 0, 0], [1, 2, 0, 0], [3, 4, 5, 0]]
    f = padded_batch([np.array([0.5, 1.5])], [0], 3, np.float32)
    assert f.dtype == np.float32 and f.tolist() == [[0.5, 1.5, 0.0]]
    assert GRAPH_TP_MULTIPLE == 16 and GRAPH_TM_MULTIPLE == 64
    assert _round_len(1, 16, 2000) == 16
    assert _round_len(16, 16, 2000) == 16
    assert _round_len(17, 16, 2000) == 32
    assert _round_len(130, 64, 10000) == 192
    assert _round_len(9990, 64, 10000) == 10000       # never past the positional-encoding table ...
    assert _round_len(10000, 64, 10000) == 10000
    assert _round_len(10001, 64, 10000) == 10001      # ... unless the length itself is


@pytest.fixture(scope='module')
def model():
    return ForwardTransformer(**fo.CONFIGS['C1'], device='cpu')


LINES = [np.array([3, 9, 4]), np.array([12, 5])]


@pytest.mark.parametrize('inputs, match', [
    ([], 'non-empty list'),
    ('abc', 'non-empty list'),
    ([np.array([3, 4]), np.array([], dtype=np.int64)], 'line 1: expected a non-empty'),
    ([np.array([[3, 4]])], 'line 0: expected a non-empty 1-D'),
    ([np.array([3, 0, 4])], 'line 0: pad id 0'),
    ([np.array([3, 4, 0])], 'line 0: pad id 0'),
])
def test_refuses_bad_lines(model, inputs, match):
    with pytest.raises(ValueError, match=match):
        model.predict_batch(inputs)


@pytest.mark.parametrize('kw', ['phoneme_durations', 'phoneme_pitch'])
def test_refuses_bad_per_line_arrays(model, kw):
    with pytest.raises(ValueError, match=f'{kw}: 1 arrays for 2 lines'):
        model.predict_batch(LINES, **{kw: [np.ones(3)]})
    with pytest.raises(ValueError, match=fr'{kw}\[1\]: 3 values for a line of 2 tokens'):
        model.predict_batch(LINES, **{kw: [np.ones(3), np.ones(3)]})
    with pytest.raises(ValueError, match=fr'{kw}\[0\]: 2 values for a line of 3 tokens'):
        model.predict_batch(LINES, **{kw: [torch.ones(2), torch.ones(2)]})


def test_refuses_attention_weights_and_batch_size():
    m = ForwardTransformer(**fo.CONFIGS['C1'], device='cpu', return_attention_weights=True)
    with pytest.raises(ValueError, match='no attention weights'):
        m.predict_batch(LINES)
    m = ForwardTransformer(**fo.CONFIGS['C1'], device='cpu')
    with pytest.raises(ValueError, match='batch_size must be positive'):
        m.predict_batch(LINES, batch_size=0)
