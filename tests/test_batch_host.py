"""Host logic of the packed batch loop (generators/batch.py): request validation, the global step schedule and the split of a
sequence set into packed forwards. No GPU needed: validation raises before anything touches the device."""
import pytest
import torch

from mmada_parallel_b200.generators.batch import batch_schedule, generate_ti2ti_batch, packed_chunks
from mmada_parallel_b200.schedule import image_generation_step_indices


class _HostModel:
    """Just the attributes the request checks read; any device work would fail (no forward methods that run)."""
    max_seq_len, max_batch = 64, 2

    def forward_rows(self, *a, **k):
        raise AssertionError("validation must fail before any forward")

    forward_rows_packed = forward_rows


def _req(L=40, seed=0, **kw):
    r = dict(input_ids=torch.zeros((1, L), dtype=torch.int64), text_start=1, text_end=5, image_start=6, seq_len=4,
             newline_every=2, generator=torch.Generator().manual_seed(seed))
    r.update(kw)
    return r


def test_rejects_empty_list():
    with pytest.raises(ValueError):
        generate_ti2ti_batch(_HostModel(), [])


def test_rejects_missing_and_shared_generators():
    m = _HostModel()
    with pytest.raises(ValueError):
        generate_ti2ti_batch(m, [_req(), _req(generator=None)])
    g = torch.Generator().manual_seed(3)
    with pytest.raises(ValueError):
        generate_ti2ti_batch(m, [_req(generator=g), _req(L=30, generator=g)])


def test_rejects_mismatched_lengths_and_shapes():
    m = _HostModel()
    with pytest.raises(ValueError):  # longer than the model's max_seq_len
        generate_ti2ti_batch(m, [_req(), _req(L=65, seed=1)])
    with pytest.raises(ValueError):  # B != 1
        generate_ti2ti_batch(m, [_req(input_ids=torch.zeros((2, 40), dtype=torch.int64))])
    with pytest.raises(ValueError):  # an unconditional prefix longer than its sequence
        generate_ti2ti_batch(m, [_req(L=20, uncon_text=torch.zeros((1, 21), dtype=torch.int64))])
    with pytest.raises(ValueError):  # one vocabulary per batch
        generate_ti2ti_batch(m, [_req(), _req(seed=1, codebook_size=4096)])


def test_rejects_models_without_packed_forward_and_bad_requests():
    class NoPacked:
        max_seq_len, max_batch = 64, 2

        def forward_rows(self, *a, **k):
            raise AssertionError

    with pytest.raises(TypeError):
        generate_ti2ti_batch(NoPacked(), [_req()])
    with pytest.raises(NotImplementedError):  # generate_ti2ti's own checks, in its order
        generate_ti2ti_batch(_HostModel(), [_req(), _req(seed=1, remasking="random")])
    with pytest.raises(TypeError):
        generate_ti2ti_batch(_HostModel(), [_req(bogus=1)])


@pytest.mark.parametrize("steps", [[(8, 3), (5, 5), (12, 4)], [(16, 16), (4, 1)], [(3, 2)], [(10, 7), (10, 3), (6, 6), (1, 1)]])
def test_schedule_visits_each_requests_own_steps(steps):
    sched = batch_schedule([t for t, _ in steps], [ts for _, ts in steps])
    assert len(sched) == max(t for t, _ in steps)
    for i, (t, ts) in enumerate(steps):
        visited = [g for g, (active, _) in enumerate(sched) if i in active]
        images = [g for g, (_, img) in enumerate(sched) if i in img]
        assert visited == list(range(t))
        assert images == sorted(set(image_generation_step_indices(t, ts)))
        for active, img in sched:
            assert set(img) <= set(active) and active == sorted(active)


def test_uncond_set_split_over_max_batch():
    assert packed_chunks(3, 3) == [range(0, 3)]
    assert packed_chunks(4, 3) == [range(0, 3), range(3, 4)]
    assert packed_chunks(7, 2) == [range(0, 2), range(2, 4), range(4, 6), range(6, 7)]
    for n in range(1, 12):
        for mb in range(1, 5):
            ch = packed_chunks(n, mb)
            assert [i for c in ch for i in c] == list(range(n)) and all(1 <= len(c) <= mb for c in ch)
