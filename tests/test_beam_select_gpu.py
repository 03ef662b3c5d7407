"""GPU tests of ``ops.beam_select`` / ``ops.kv_beam_reorder`` (csrc/beam_select_sm100.cu) and of the graphed beam
search built on them: the kernel against a restatement of one eager ``beam_search`` step (``torch.log_softmax``,
``torch.topk`` over ``max(2, 1 + n_eos) * num_beams`` candidates, ``_BeamHyps`` for the hypotheses), the in-place
reorder against ``index_select``, and ``generate_texts(num_beams > 1)`` under ``enable_decode_graphs`` against the
eager loop."""
import itertools

import pytest
import torch

pytestmark = pytest.mark.gpu

MARGIN = 1e-4            # the restatement's decisions must not hinge on score differences below this


class _State:
    """Beam state of B sequences of nb rows, as the eager loop keeps it."""

    def __init__(self, B, nb, lp):
        from tests.test_generate_gpu import _BeamHyps
        self.B, self.nb = B, nb
        self.seqs = [[] for _ in range(B * nb)]
        self.scores = torch.tensor([[0.0] + [-1e9] * (nb - 1)] * B, dtype=torch.float32).view(-1)
        self.hyps = [_BeamHyps(nb, lp) for _ in range(B)]
        self.done = [False] * B


def _restated_step(st, logits, step, eos, pad, min_length, penalty, lp):
    """One iteration of the eager loop of generation.beam_search, written out again; returns (tokens, parents, margins)."""
    B, nb = st.B, st.nb
    scores = torch.log_softmax(logits.float(), dim=-1)
    if penalty != 1.0 and step > 0:
        seqs = torch.tensor(st.seqs, dtype=torch.long, device=logits.device)
        picked = scores.gather(1, seqs)
        scores = scores.scatter(1, seqs, torch.where(picked < 0, picked * penalty, picked / penalty))
    if step < min_length and eos:
        scores[:, eos] = float("-inf")
    V = scores.shape[-1]
    K = max(2, 1 + len(eos)) * nb
    cand = (scores + st.scores.to(logits.device)[:, None]).view(B, nb * V)
    top_s, top_i = cand.topk(K + 1, dim=1)
    top_s, top_i = top_s.tolist(), top_i.tolist()
    margins = []
    toks, pars, new_seqs, new_scores = [], [], [], []
    for b in range(B):
        if st.done[b]:
            toks += [pad] * nb; pars += [b * nb] * nb
            new_seqs += [st.seqs[b * nb] + [pad]] * nb; new_scores += [0.0] * nb
            continue
        finite = [s for s in top_s[b] if s > -1e8]
        margins += [finite[i] - finite[i + 1] for i in range(len(finite) - 1)]
        h = st.hyps[b]
        k = 0
        for rank in range(K):
            sc, idx = top_s[b][rank], top_i[b][rank]
            row, tok = b * nb + idx // V, idx % V
            if tok in eos:
                if rank < nb:
                    if len(h.beams) >= nb:
                        margins.append(abs(sc / (max(step, 1) ** lp) - h.worst_score))
                    h.add(list(st.seqs[row]), sc)
            else:
                toks.append(tok); pars.append(row); new_seqs.append(st.seqs[row] + [tok]); new_scores.append(sc)
                k += 1
            if k == nb:
                break
        while k < nb:
            toks.append(pad); pars.append(b * nb); new_seqs.append(st.seqs[b * nb] + [pad]); new_scores.append(0.0)
            k += 1
        if len(h.beams) >= nb:
            margins.append(abs(h.worst_score - top_s[b][0] / (step + 1) ** lp))
        st.done[b] = st.done[b] or h.is_done(top_s[b][0], step + 1)
    st.seqs, st.scores = new_seqs, torch.tensor(new_scores, dtype=torch.float32)
    return toks, pars, margins


class _Device:
    """The buffers ``ops.beam_select`` reads and writes."""

    def __init__(self, B, nb, V, max_new, eos, penalty, lp):
        from mm_interleaved_b200 import ops
        R, d = B * nb, "cuda"
        self.nb = nb
        self.params = torch.tensor([penalty, lp], dtype=torch.float64, device=d)
        self.beam_scores = torch.tensor([[0.0] + [-1e9] * (nb - 1)] * B, dtype=torch.float32, device=d).view(-1)
        self.history = torch.full((R, max_new), -5, dtype=torch.long, device=d)
        self.next_ids = torch.zeros((R, 1), dtype=torch.long, device=d)
        self.parent = torch.zeros((R,), dtype=torch.long, device=d)
        self.done = torch.zeros((B,), dtype=torch.bool, device=d)
        self.hyp_scores = torch.zeros((B, nb), dtype=torch.float64, device=d)
        self.hyp_ids = torch.zeros((B, nb, max_new), dtype=torch.long, device=d)
        self.hyp_meta = torch.full((B, nb, 2), -1, dtype=torch.long, device=d)
        self.scratch = torch.zeros((R * ops.beam_candidates(nb, len(eos)),), dtype=torch.long, device=d)
        self.eos = torch.tensor(eos, dtype=torch.long, device=d) if eos else None

    def step(self, logits, step, pad, min_length):
        from mm_interleaved_b200 import ops
        ops.beam_select(logits, torch.tensor([step], device="cuda"), self.params, self.beam_scores, self.history,
                        self.next_ids, self.parent, self.done, self.hyp_scores, self.hyp_ids, self.hyp_meta, self.scratch,
                        self.nb, eos=self.eos, pad_id=pad, min_length=min_length)

    def hyps(self, b):
        meta, ids, sc = self.hyp_meta[b].tolist(), self.hyp_ids[b].tolist(), self.hyp_scores[b].tolist()
        slots = sorted((m[1], j) for j, m in enumerate(meta) if m[0] >= 0)
        return [(sc[j], ids[j][:meta[j][0]]) for _, j in slots]


def _logits_stream(R, V, eos, seed, eos_boost):
    """Logits per step around a fixed base (so ids recur and the repetition penalty bites), eos ids placed near the
    top of every row (``eos_boost`` above the row's maximum, minus 2)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn((R, V), generator=g) * 4.0
    top = base.max(dim=1).values
    for i, e in enumerate(eos):
        base[:, e] = top + eos_boost - 2.0 - 0.3 * i
    while True:
        yield (base + torch.randn((R, V), generator=g) * 0.7).cuda()


def _drive(B, nb, V, eos, lp, penalty, seed, eos_boost=2.0, min_length=2, n_steps=6, pad=0):
    dev = _Device(B, nb, V, n_steps, eos, penalty, lp)
    st = _State(B, nb, lp)
    stream = _logits_stream(B * nb, V, eos, seed, eos_boost)
    margins = []
    for step in range(n_steps):
        logits = next(stream)
        dev.step(logits, step, pad, min_length)
        toks, pars, m = _restated_step(st, logits, step, eos, pad, min_length, penalty, lp)
        margins += m
        assert min(margins, default=1.0) > MARGIN, "near-tie in the restatement: pick another seed"
        assert dev.next_ids[:, 0].tolist() == toks, (step, dev.next_ids[:, 0].tolist(), toks)
        assert dev.parent.tolist() == pars, (step, dev.parent.tolist(), pars)
        assert dev.done.tolist() == st.done, (step, dev.done.tolist(), st.done)
        assert dev.history[:, :step + 1].tolist() == st.seqs, step
        torch.testing.assert_close(dev.beam_scores.cpu(), st.scores, atol=1e-5, rtol=1e-6)
        for b in range(B):
            got, want = dev.hyps(b), st.hyps[b].beams
            assert [x[1] for x in got] == [x[1] for x in want], (step, b, got, want)
            torch.testing.assert_close(torch.tensor([x[0] for x in got], dtype=torch.float64),
                                       torch.tensor([x[0] for x in want], dtype=torch.float64), atol=1e-5, rtol=1e-6)
    return st


@pytest.mark.parametrize("V,nb,n_eos,lp,penalty", list(itertools.product((64, 32002), (3, 5), (1, 2), (0.7, 1.0, 1.3),
                                                                           (1.0, 1.4))))
def test_beam_select_matches_the_restated_eager_step(V, nb, n_eos, lp, penalty):
    eos = [7, 11][:n_eos]
    st = _drive(2, nb, V, eos, lp, penalty, seed=1000 * nb + 10 * n_eos + V % 97)
    assert any(h.beams for h in st.hyps)                               # the hypothesis path was taken


@pytest.mark.parametrize("V", [64, 32002])
def test_beam_select_takes_enough_candidates_when_eos_ids_dominate(V):
    """Both eos ids outscore everything in every row: the top 2 * nb hold 2 * nb eos candidates, so only the
    (1 + n_eos) * nb candidates of the reference leave room for nb continuing beams."""
    st = _drive(2, 3, V, [7, 11], 1.0, 1.0, seed=5, eos_boost=30.0, min_length=0, n_steps=4)
    assert all(len(h.beams) == 3 for h in st.hyps)


@pytest.mark.parametrize("parents", ["identity", "one_row", "cyclic", "random"])
def test_kv_beam_reorder_moves_generated_positions_only(parents):
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(2)
    n, B, nb, T, H, hd = 6, 3, 5, 40, 3, 8
    R = B * nb
    kv = torch.randn((n, R, T, H, hd), generator=g).to(torch.bfloat16).cuda()
    local = {"identity": [list(range(nb))] * B, "one_row": [[2] * nb, [0] * nb, [4] * nb],
             "cyclic": [[(j + 1) % nb for j in range(nb)]] * B,
             "random": [torch.randint(0, nb, (nb,), generator=g).tolist() for _ in range(B)]}[parents]
    parent = torch.tensor([b * nb + p for b in range(B) for p in local[b]], dtype=torch.long).cuda()
    cur, step = 30, 7
    for done in (None, torch.tensor([False, True, False]).cuda()):
        got = kv.clone()
        ops.kv_beam_reorder(got, parent, torch.tensor([cur]).cuda(), torch.tensor([step]).cuda(), nb, 10, done=done)
        want = kv.clone()
        want[:, :, cur - step:cur] = kv[:, :, cur - step:cur].index_select(1, parent)
        if done is not None:
            want[:, nb:2 * nb] = kv[:, nb:2 * nb]                      # a finished group is left alone
        assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def _second_call(ids, vis):
    g = torch.Generator().manual_seed(123)
    vis2_d = {"vis_embed": (torch.randn(vis["vis_embed"].shape, generator=g) * 0.5).cuda(),
              "multiscale_features": [(torch.randn(f.shape, generator=g) * 2).cuda() for f in vis["multiscale_features"]]}
    mask2 = torch.ones_like(ids)
    mask2[1, :2] = 0
    return vis2_d, mask2.cuda()


@pytest.mark.parametrize("nb", [3, 5])
def test_graphed_beam_search_equals_eager_with_one_graph(nb):
    from tests.test_generate_gpu import _setup
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    vis2_d, mask2 = _second_call(ids, vis)
    args, args2 = (ids.cuda(), vis_d, nimg.cuda(), 2), (ids.cuda(), vis2_d, nimg.cuda(), 2)
    free = dev.generate_texts(*args, max_new_tokens=8, eos_token_id=None).cpu()
    kw = dict(max_new_tokens=8, eos_token_id=[int(free[0, 3]), int(free[1, 2])], min_length=2, num_beams=nb,
              length_penalty=1.3, num_return_sequences=2, pad_token_id=0)
    calls = [(args, {}), (args2, dict(attention_mask=mask2)), (args, dict(length_penalty=0.7))]
    eager = [dev.generate_texts(*a, **dict(kw, **extra)).cpu() for a, extra in calls]
    dev.enable_decode_graphs()
    try:
        graphed = [dev.generate_texts(*a, **dict(kw, **extra)).cpu() for a, extra in calls]
        assert len(dev._decode_graphs) == 1 and next(iter(dev._decode_graphs))[-1] == "beam"
        for e, g in zip(eager, graphed):
            assert torch.equal(e, g), (e, g)
        assert not torch.equal(eager[0], eager[1])
    finally:
        dev.enable_decode_graphs(False)


def test_graphed_beam_search_stops_within_two_replays_and_adds_two_launches():
    from tests.test_generate_gpu import _setup
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    with torch.no_grad():
        dev.text_decoder.head.bias[5] += 20.0                          # id 5 (an eos id below) dominates every row
    args = (ids.cuda(), vis_d, nimg.cuda(), 2)
    n_new = 16
    kw = dict(max_new_tokens=n_new, eos_token_id=[5, 9], min_length=0, num_beams=3, length_penalty=0.0)
    calls = [0]
    hook = dev.mm_decoder.register_forward_pre_hook(lambda *_: calls.__setitem__(0, calls[0] + 1))
    eager = dev.generate_texts(*args, **kw).cpu()
    hook.remove()
    eager_steps = calls[0]                                             # prefill + one forward per step but the last
    assert eager_steps < n_new
    dev.enable_decode_graphs()
    try:
        graphed = dev.generate_texts(*args, **kw).cpu()
        dec = next(iter(dev._decode_graphs.values()))
        assert torch.equal(eager, graphed), (eager, graphed)
        assert eager_steps <= dec.replays <= eager_steps + 2, (dec.replays, eager_steps)
        dev.generate_texts(*args, max_new_tokens=n_new, eos_token_id=[5, 9])        # greedy graph of the same shape
        greedy = [d for k, d in dev._decode_graphs.items() if k[-1] == "greedy"][0]
        assert dec.launches == greedy.launches + 2                     # beam_select (2 kernels) + kv_beam_reorder - decode_select
    finally:
        dev.enable_decode_graphs(False)


def test_reference_defaults_take_the_beam_graph_through_mm_interleaved_generate():
    from tests.test_mm_interleaved_gpu import DEV, _batch, _build
    model, _ = _build()
    ids, images, nimg, mask = _batch()
    batch = dict(text_ids=ids.to(DEV), image_tensors=images.to(DEV), num_image_per_seq=nimg.to(DEV),
                 attention_mask=mask.to(DEV), meta=None)
    eager = model.generate(mode="generate_texts", **batch)["text_ids"]                # 5 beams, min 8, eos [eos, soi]
    model.enable_decode_graphs()
    try:
        graphed = model.generate(mode="generate_texts", **batch)["text_ids"]
        assert len(model._decode_graphs) == 1 and next(iter(model._decode_graphs))[-2:] == (5, "beam")
        assert torch.equal(eager, graphed), (eager, graphed)
    finally:
        model.enable_decode_graphs(False)
