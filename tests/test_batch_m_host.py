"""Host logic of the variant-M batch loop (generators/batch.py::interleave_generate_batch): request validation, the global step
schedule and the split of the [cond; uncond] sequence set into packed forwards. No GPU needed: validation raises before anything
touches the device."""
from types import SimpleNamespace

import pytest
import torch

from mmada_parallel_b200.generators.batch import batch_schedule, interleave_generate_batch, packed_chunks
from mmada_parallel_b200.schedule import image_generation_step_indices


class _HostModel:
    """Just the attributes the request checks read; any device work would fail."""
    max_seq_len, max_batch = 128, 4

    def forward_rows(self, *a, **k):
        raise AssertionError("validation must fail before any forward")

    forward_rows_packed = forward_rows

    @property
    def device(self):
        raise AssertionError("validation must fail before anything touches the device")


class _Tok:
    bos_token_id = 5

    def __init__(self, n=1000):
        self.n = n

    def __len__(self):
        return self.n


def _conf(n_vq=16, max_seq=32, codebook=64):
    return SimpleNamespace(model=SimpleNamespace(mmada=SimpleNamespace(num_vq_tokens=n_vq, codebook_size=codebook)),
                           dataset=SimpleNamespace(preprocessing=SimpleNamespace(max_seq_length=max_seq)))


def _req(P=10, seed=0, **kw):
    """A request of L = P + 16 + 32 + 2 tokens."""
    r = dict(input_ids=torch.zeros(P, dtype=torch.int64), uncond_input_ids=torch.zeros(P, dtype=torch.int64),
             reserved_token_mapping={"<|soi|>": 1, "<|eoi|>": 2}, generator=torch.Generator().manual_seed(seed), config=_conf(),
             uni_prompting=SimpleNamespace(text_tokenizer=_Tok()), text_steps=8, image_steps=4)
    r.update(kw)
    return r


def test_rejects_empty_list():
    with pytest.raises(ValueError):
        interleave_generate_batch(_HostModel(), [])


def test_rejects_missing_and_shared_generators():
    m = _HostModel()
    with pytest.raises(ValueError):
        interleave_generate_batch(m, [_req(), _req(generator=None)])
    g = torch.Generator().manual_seed(3)
    with pytest.raises(ValueError):
        interleave_generate_batch(m, [_req(generator=g), _req(P=12, generator=g)])


def test_rejects_text_gumbel():
    with pytest.raises(ValueError):
        interleave_generate_batch(_HostModel(), [_req(), _req(seed=1, text_temperature=0.5)])


def test_rejects_mixed_vocabularies():
    m = _HostModel()
    with pytest.raises(ValueError):
        interleave_generate_batch(m, [_req(), _req(seed=1, uni_prompting=SimpleNamespace(text_tokenizer=_Tok(999)))])
    with pytest.raises(ValueError):
        interleave_generate_batch(m, [_req(), _req(seed=1, config=_conf(codebook=128))])


def test_rejects_unequal_prompts_and_long_sequences():
    m = _HostModel()
    with pytest.raises(ValueError):
        interleave_generate_batch(m, [_req(), _req(seed=1, uncond_input_ids=torch.zeros(11, dtype=torch.int64))])
    with pytest.raises(ValueError):  # L = 79 + 50 = 129 > max_seq_len
        interleave_generate_batch(m, [_req(), _req(P=79, seed=1)])
    with pytest.raises(RuntimeError):  # L = 78 + 50 = 128 fits: the next check is what fails
        interleave_generate_batch(m, [_req(P=78), _req(seed=1, image_steps=0)])


def test_rejects_requests_without_image_step_and_bad_arguments():
    m = _HostModel()
    with pytest.raises(RuntimeError):  # interleave_generate raises this after its loop; the batch before any forward
        interleave_generate_batch(m, [_req(), _req(seed=1, image_steps=0)])
    with pytest.raises(ValueError):  # interleave_generate's own check
        interleave_generate_batch(m, [_req(text_cfg=0.0, image_cfg=0.0)])
    with pytest.raises(NotImplementedError):
        interleave_generate_batch(m, [_req(remasking="random")])


def test_rejects_models_without_packed_forward():
    class NoPacked:
        max_seq_len, max_batch = 128, 4

    with pytest.raises(TypeError):
        interleave_generate_batch(NoPacked(), [_req()])


@pytest.mark.parametrize("steps", [[(8, 4), (5, 5), (12, 3)], [(16, 16), (4, 1)], [(10, 7), (10, 3), (6, 6), (2, 1)]])
def test_schedule_visits_each_requests_own_text_and_image_steps(steps):
    """interleave_generate runs text steps 0 .. text_steps - 1 and its image steps at image_generation_step_indices(text_steps,
    image_steps); the batch runs request i's step g at global step g."""
    sched = batch_schedule([t for t, _ in steps], [ts for _, ts in steps])
    assert len(sched) == max(t for t, _ in steps)
    for i, (t, ts) in enumerate(steps):
        assert [g for g, (active, _) in enumerate(sched) if i in active] == list(range(t))
        assert [g for g, (_, img) in enumerate(sched) if i in img] == sorted(set(image_generation_step_indices(t, ts)))


def test_cond_uncond_sequences_split_over_max_batch():
    """N requests give 2N sequences, [cond_0, uncond_0, cond_1, ...]; max_batch = 2 puts each request in its own forward."""
    for n_req in range(1, 6):
        assert packed_chunks(2 * n_req, 2) == [range(2 * i, 2 * i + 2) for i in range(n_req)]
        for mb in (3, 4, 7, 64):
            ch = packed_chunks(2 * n_req, mb)
            assert [i for c in ch for i in c] == list(range(2 * n_req)) and all(1 <= len(c) <= mb for c in ch)
    assert packed_chunks(6, 4) == [range(0, 4), range(4, 6)]


class _RecordingModel:
    """A host stand-in whose packed forward records its sequences and windows and returns zero logits."""
    max_seq_len = 4096

    def __init__(self, max_batch):
        self.max_batch, self.calls = max_batch, []

    def forward_rows_packed(self, ids, lens, rows_a=None, rows_b=None, col0_b=0, ncols_b=0, row_windows=None):
        self.calls.append((list(lens), row_windows))
        return (torch.zeros((rows_a.numel(), 3)) if rows_a is not None else None,
                torch.zeros((rows_b.numel(), ncols_b)) if rows_b is not None else None)


@pytest.mark.parametrize("max_batch", [2, 3, 64])
def test_loop_runs_each_requests_own_steps_with_its_windows(monkeypatch, max_batch):
    """Through interleave_generate_batch with the device work stubbed: request i's text step g and image step g run at global
    step g exactly for its own schedule, each packed forward holds at most max_batch of the [cond; uncond] sequences, and every
    sequence carries the window interleave_generate would use (text rows, or from the image rows on image steps)."""
    from mmada_parallel_b200 import mmada

    class State:
        def __init__(self, model, **a):
            lay = mmada.interleave_layout(a["config"], a["uni_prompting"], a["input_ids"], a["uncond_input_ids"], a["text_steps"],
                                          a["image_steps"])
            self.L, self.P, self.max_seq, self.img_idx = lay["L"], lay["P"], lay["max_seq"], lay["img_idx"]
            self.both = torch.zeros((2, self.L), dtype=torch.int64)
            self.rows_text = torch.arange(self.L - self.max_seq, self.L, dtype=torch.int32).repeat(2)
            self.pos = torch.arange(self.P + 1, self.P + 1 + lay["n_vq"], dtype=torch.int32)
            self.tag = a["input_ids"].numel()
            self.window = lambda g: (self.P + 1, self.L) if g in self.img_idx else (self.L - self.max_seq, self.L)

        def results(self):
            return self.tag

    log = []
    monkeypatch.setattr(mmada, "InterleaveState", State)
    monkeypatch.setattr(mmada, "interleave_text_step", lambda st, g, c, u: log.append(("text", st.tag, g, c.shape[0], u.shape[0])))
    monkeypatch.setattr(mmada, "interleave_image_step", lambda st, g, c, u: log.append(("image", st.tag, g, c.shape, u.shape)))
    steps = [(8, 4), (5, 5), (12, 3)]
    reqs = [_req(P=10 + i, seed=i, text_steps=t, image_steps=ts) for i, (t, ts) in enumerate(steps)]
    model = _RecordingModel(max_batch)
    assert interleave_generate_batch(model, reqs) == [10, 11, 12]
    for i, (t, ts) in enumerate(steps):
        img = sorted(set(image_generation_step_indices(t, ts)))
        assert [e[2] for e in log if e[0] == "text" and e[1] == 10 + i] == list(range(t))
        assert [e[2] for e in log if e[0] == "image" and e[1] == 10 + i] == img
        assert all(e[3:] == (32, 32) for e in log if e[0] == "text")
        assert all(e[3:] == ((16, 64), (16, 64)) for e in log if e[0] == "image")
    # forwards: per global step the active requests' [cond; uncond] sequences, chunked by max_batch, each with its window
    k = 0
    for g in range(12):
        active = [i for i, (t, _) in enumerate(steps) if g < t]
        lens = [reqs[i]["input_ids"].numel() + 50 for i in active for _ in range(2)]
        wins = []
        for i in active:
            L, P = lens[2 * active.index(i)], 10 + i
            w = (P + 1, L) if g in set(image_generation_step_indices(*steps[i])) else (L - 32, L)
            wins += [w, w]
        for c in packed_chunks(len(lens), max_batch):
            assert model.calls[k] == ([lens[j] for j in c], [wins[j] for j in c]), (g, k)
            k += 1
    assert k == len(model.calls)
