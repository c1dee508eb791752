"""ContinuousDecoder's host logic against a fake engine (no GPU): admission, step order, retirement, compaction, validation.

The fake `decode_step` records every image's schedule rows and returns a deterministic function of them, so a request's output
tells which rows it saw and in which order.
"""
import numpy as np
import pytest
import torch

from selftoktokenizer_b200 import config as C
from selftoktokenizer_b200.continuous import ContinuousDecoder


class _Tables:
    def __init__(self, k):
        self.k = torch.as_tensor(k)


class FakeEngine:
    """x_out[b] = x[b] * 2 + (step_b + 1) on every element; records (request tag, step) per image, the tag being x[b, 0, 0, 0]
    of the admitted noise carried along in element [0, 0, 0, 1]."""

    def __init__(self, dims, steps=50):
        self.dims = dims
        self.steps = steps
        self.device = "cpu"
        self.tables = _Tables(np.maximum(dims.K - 1 - np.arange(steps) * (dims.K // steps + 1), 1))
        self.calls = []

    def decode_step(self, tokens, x, step, *, token_range=None, cfg_scale=None, out=None):
        step = np.asarray(step)
        assert tokens.shape[0] == x.shape[0] == step.shape[0] and out is x
        self.calls.append((x[:, 0, 0, 1].tolist(), step.tolist(), None if cfg_scale is None else np.asarray(cfg_scale).tolist(),
                           np.asarray(token_range).tolist()))
        body = x.clone()
        body[:, 0, 0, 0] = x[:, 0, 0, 0] * 2 + torch.as_tensor(step, dtype=torch.float32) + 1
        out.copy_(body)
        return out


D = C.TINY


def _expected(tag_noise, n):
    v = tag_noise
    for s in range(n):
        v = v * 2 + s + 1
    return v


def _ids(seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, D.codebook_size, D.K))


def _noise(tag):
    x = torch.zeros(1, D.in_channels, D.latent, D.latent)
    x[0, 0, 0, 0] = 0.25 * tag
    x[0, 0, 0, 1] = tag
    return x


def test_fifo_admission_and_max_batch():
    eng = FakeEngine(D, steps=6)
    dec = ContinuousDecoder(eng, 3)
    rids = [dec.submit(_ids(i), _noise(i), steps=2 + i % 4) for i in range(8)]
    assert dec.pending == 8 and dec.active == 0
    seen_order = []
    while dec.pending or dec.active:
        dec.step()
        assert dec.active <= 3
        for tag in eng.calls[-1][0]:
            if tag not in seen_order:
                seen_order.append(tag)
        assert len(eng.calls[-1][0]) <= 3
    assert seen_order == [float(i) for i in range(8)]                  # admitted in submission order
    assert rids == list(range(8))


def test_every_request_sees_its_rows_once_in_order_and_returns_once():
    eng = FakeEngine(D, steps=7)
    dec = ContinuousDecoder(eng, 3)
    steps = [7, 1, 3, 7, 2, 5, 1, 4]
    results = {}
    for i, n in enumerate(steps):
        dec.submit(_ids(i), _noise(i), steps=n)
        if i % 2:                                                      # staggered arrivals between steps
            for rid, out in dec.step():
                assert rid not in results
                results[rid] = out
    for rid, out in dec.drain():
        assert rid not in results
        results[rid] = out
    assert sorted(results) == list(range(len(steps)))
    rows = {}
    for tags, st, _, _ in eng.calls:
        for t, s in zip(tags, st):
            rows.setdefault(int(t), []).append(s)
    for i, n in enumerate(steps):
        assert rows[i] == list(range(n)), (i, rows[i])
        out = results[i]
        assert tuple(out.shape) == (1, D.in_channels, D.latent, D.latent)
        assert float(out[0, 0, 0, 0]) == _expected(0.25 * i, n)
        assert float(out[0, 0, 0, 1]) == i


def test_outputs_are_not_views_of_the_state():
    eng = FakeEngine(D, steps=3)
    dec = ContinuousDecoder(eng, 2)
    dec.submit(_ids(0), _noise(0), steps=1)
    dec.submit(_ids(1), _noise(1), steps=3)
    (rid, out), = dec.step()
    before = out.clone()
    dec.submit(_ids(2), _noise(2), steps=3)
    dec.drain()
    assert rid == 0 and torch.equal(out, before)
    assert out.untyped_storage().data_ptr() != dec._x.untyped_storage().data_ptr()


def test_drain_and_postprocess():
    eng = FakeEngine(D, steps=4)
    batches = []
    dec = ContinuousDecoder(eng, 4, postprocess=lambda x: (batches.append(x.shape[0]), x * 10)[1])
    for i in range(5):
        dec.submit(_ids(i), _noise(i), steps=4)
    res = dict(dec.drain())
    assert dec.pending == 0 and dec.active == 0 and dec.step() == []
    assert sorted(res) == list(range(5)) and batches == [4, 1]
    assert float(res[3][0, 0, 0, 0]) == 10 * _expected(0.75, 4)


def test_default_noise_is_the_cpu_global_draw():
    eng = FakeEngine(D, steps=2)
    dec = ContinuousDecoder(eng, 1)
    torch.manual_seed(1234)
    want = torch.randn(1, D.in_channels, D.latent, D.latent)
    torch.manual_seed(1234)
    dec.submit(_ids(0), steps=1)
    assert torch.equal(dec._queue[0][2], want[0])


def test_guided_scales_and_windows_reach_the_engine():
    eng = FakeEngine(D, steps=3)
    dec = ContinuousDecoder(eng, 2, guided=True)
    dec.submit(_ids(0), _noise(0), cfg_scale=2.5, token_range=(0, 9), steps=3)
    dec.submit(_ids(1), _noise(1), cfg_scale=1.5, steps=3)
    dec.step()
    _, _, scales, ranges = eng.calls[-1]
    assert scales == [2.5, 1.5] and ranges == [[0, 9], [0, D.K]]


def test_submit_errors():
    eng = FakeEngine(D, steps=50)
    k_last = int(eng.tables.k[-1])
    dec = ContinuousDecoder(eng, 2)
    gdec = ContinuousDecoder(eng, 2, guided=True)
    ids = _ids(0)
    for bad in [(-1, 5), (5, 5), (0, D.K + 1), (9, 3)]:
        with pytest.raises(ValueError, match="token_range"):
            dec.submit(ids, token_range=bad)
    with pytest.raises(ValueError, match="visible token"):
        gdec.submit(ids, cfg_scale=2.5, token_range=(k_last + 1, D.K))
    gdec.submit(ids, cfg_scale=2.5, token_range=(k_last + 1, D.K), steps=1)   # visible at step 0
    with pytest.raises(ValueError, match="cfg_scale"):
        gdec.submit(ids)
    with pytest.raises(ValueError, match="cfg_scale"):
        dec.submit(ids, cfg_scale=2.0)
    bad_ids = ids.clone()
    bad_ids[12] = D.codebook_size
    with pytest.raises(ValueError, match="token id"):
        dec.submit(bad_ids, token_range=(10, 20))
    with pytest.raises(ValueError, match="ids"):
        dec.submit(ids[:-1])
    with pytest.raises(ValueError, match="ids"):
        dec.submit(ids[None])
    with pytest.raises(ValueError, match="noise"):
        dec.submit(ids, torch.zeros(2, D.in_channels, D.latent, D.latent))
    with pytest.raises(ValueError, match="steps"):
        dec.submit(ids, steps=51)
    assert dec.pending == 0 and gdec.pending == 1


def test_padding_outside_the_window_is_accepted():
    eng = FakeEngine(D, steps=2)
    dec = ContinuousDecoder(eng, 2)
    ids = _ids(3)
    ids[:10] = -1
    ids[20:] = D.codebook_size + 7
    dec.submit(ids, _noise(0), token_range=(10, 20), steps=2)
    (rid, _), = dec.drain()
    assert rid == 0

