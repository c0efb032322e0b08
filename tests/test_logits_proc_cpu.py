"""CPU checks of the logits processors: the parallel (Z-function / prefix-max) form of the n-gram levels equals the
reference's KMP restatement, and LlamaDecoder's argument checks refuse bad input before anything reaches the library."""
import types

import numpy as np
import pytest

from tests import ngram_oracle as ng
from zhilight_b200 import llama


def _fibonacci_word(n):
    a, b = [0], [0, 1]
    while len(b) < n:
        a, b = b, b + a
    return b[:n]


def test_levels_by_hand():
    # seq 1 2 1 2 -> r = 2 1 2 1: next = -1 -1 0 1, so ngrams[1] = 2 and token 1 (which would continue the loop) gets
    # level 2, token 2 level 0
    assert ng.kmp_levels([2, 1, 2, 1]) == [0, 2, 0, 0]
    f = ng.ngram_factors([1, 2, 1, 2], 2.0, 1.0)
    assert f == {1: np.float32(8.0), 2: np.float32(2.0)}


def test_z_form_equals_kmp_on_random_sequences():
    rng = np.random.default_rng(0)
    for _ in range(10000):
        alphabet = int(rng.integers(1, 51))
        r = rng.integers(0, alphabet, size=int(rng.integers(0, 81))).tolist()
        assert ng.z_levels(r) == ng.kmp_levels(r), r


@pytest.mark.parametrize("name", ["empty", "one", "constant", "period", "fibonacci", "period_tail"])
def test_z_form_equals_kmp_on_adversarial_sequences(name):
    cases = {
        "empty": [[]],
        "one": [[7]],
        "constant": [[3] * n for n in (2, 3, 64, 513, 1500)],
        "period": [[k % p for k in range(n)] for p in range(2, 8) for n in (p, 2 * p + 1, 300)],
        "fibonacci": [_fibonacci_word(n) for n in (1, 2, 5, 13, 100, 987)],
        "period_tail": [[k % p for k in range(200)] + [9, 9, 1, 2, 1] for p in range(2, 8)],
    }[name]
    for r in cases:
        assert ng.z_levels(r) == ng.kmp_levels(r), (name, len(r))


def test_process_order_penalty_then_bias():
    l = np.array([2.0, -2.0, 1.0, 0.5], dtype=np.float32)
    out = ng.process(l, [0, 1, 0, 1], repetition_penalty=1.0, ngram_penalty=2.0, bias={0: 1.0, 3: -np.inf})
    f = ng.ngram_factors([0, 1, 0, 1], 2.0, 1.0)
    assert out[0] == np.float32(2.0 / f[0] + 1.0)
    assert out[1] == np.float32(-2.0 * f[1])
    assert out[2] == np.float32(1.0) and out[3] == -np.inf
    # n-gram off: the bitmap rule over the sequence's distinct tokens; presence_penalty applies there
    out = ng.process(l, [0, 0], presence_penalty=0.5, bias={2: 0.25})
    np.testing.assert_array_equal(out, np.array([1.5, -2.0, 1.25, 0.5], dtype=np.float32))


def test_logit_bias_arrays_accepts_ints_and_strings():
    toks, vals = llama.logit_bias_arrays({"5": 1.5, 7: -np.inf}, 10)
    assert toks.tolist() == [5, 7] and toks.dtype == np.int32
    assert vals.dtype == np.float32 and vals[0] == 1.5 and vals[1] == -np.inf
    toks, vals = llama.logit_bias_arrays(None, 10)
    assert toks.size == 0 and vals.size == 0
    toks, _ = llama.logit_bias_arrays({t: 0.0 for t in range(1024)}, 2000)
    assert toks.size == 1024


@pytest.mark.parametrize("bias", [
    {5: 1.0, "5": 2.0},               # one token twice
    {-1: 1.0},                        # id out of range
    {10: 1.0},
    {3: float("nan")},
    {3: float("inf")},
    {t: 0.0 for t in range(1025)},    # more than 1024 entries
], ids=["duplicate", "negative", "too_large", "nan", "plus_inf", "too_many"])
def test_logit_bias_arrays_refuses(bias):
    vocab = 10 if len(bias) < 1000 else 4096
    with pytest.raises(ValueError):
        llama.logit_bias_arrays(bias, vocab)


@pytest.mark.parametrize("value", [0.0, -1.0, float("nan"), float("inf")])
def test_ngram_penalty_refused(value):
    with pytest.raises(ValueError):
        llama.check_ngram_penalty(value)
    llama.check_ngram_penalty(1.0)
    llama.check_ngram_penalty(0.5)


@pytest.mark.parametrize("value", [float("nan"), float("inf"), -1.0])
def test_set_sampling_checks_ngram_penalty_before_the_presence_override(value):
    # GeneratorArg turns the n-gram penalty off under a presence penalty; a bad value is still refused, before anything
    # reaches the library (the stand-in decoder has no handle)
    with pytest.raises(ValueError):
        llama.LlamaDecoder.set_sampling(types.SimpleNamespace(), 0, presence_penalty=0.5, ngram_penalty=value)
