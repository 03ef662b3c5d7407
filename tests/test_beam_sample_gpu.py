"""GPU tests of beam sample (HF transformers 4.31 ``GenerationMixin.beam_sample``): ``ops.beam_sample``
(csrc/beam_select_sm100.cu) with injected uniforms against a float64 restatement of the step that draws by the same
Gumbel race, its tie handling and error flag, the statistics of its Philox draws, the eager beam-sample loop against a
plain-Python 4.31 loop over the oracle decoder, and the graphed beam-sample decode."""
import itertools

import pytest
import torch

pytestmark = pytest.mark.gpu

MARGIN = 1e-4            # the restatement's decisions must not hinge on differences below this
NEG = float("-inf")


class _State:
    """Beam-sample state of B sequences of nb rows (every beam starts at score 0)."""

    def __init__(self, B, nb, lp):
        from tests.test_generate_gpu import _BeamHyps
        self.B, self.nb = B, nb
        self.seqs = [[] for _ in range(B * nb)]
        self.scores = torch.zeros(B * nb, dtype=torch.float64)
        self.hyps = [_BeamHyps(nb, lp) for _ in range(B)]
        self.done = [False] * B
        self.error = False


def _gaps(v):
    """Differences between neighbours of the sorted finite values of v, exact ties excluded."""
    v = sorted(x for x in v if x > NEG)
    return [b - a for a, b in zip(v, v[1:]) if b != a]


def _restated_step(st, logits, step, eos, pad, min_length, penalty, lp, T, top_p, top_k, u):
    """Steps 1-7 of one 4.31 beam_sample step in float64, the top-p cut stated as the kernel keeps ties (every token
    whose weight is >= the smallest weight at which the ascending mass exceeds (1 - top_p) * Z, which is HF's set when
    no weights tie), and the multinomial draw as the race key = s - log(-log u).  Returns (tokens, parents, margins)."""
    B, nb = st.B, st.nb
    V = logits.shape[1]
    scores = torch.log_softmax(logits.double(), dim=-1)
    if penalty != 1.0 and step > 0:
        seqs = torch.tensor(st.seqs, dtype=torch.long, device=logits.device)
        picked = scores.gather(1, seqs)
        scores = scores.scatter(1, seqs, torch.where(picked < 0, picked * penalty, picked / penalty))
    if step < min_length and eos:
        scores[:, eos] = NEG
    s = (scores + st.scores.to(logits.device)[:, None]) / T
    margins = []
    k = min(max(top_k, 2), V) if top_k > 0 else V
    kth = s.topk(k, dim=-1).values[:, -1:]
    d = (s - kth).abs()
    d = d[(d > 0) & (d < 1)]                                               # the k-th value is not a near-tie
    margins += [float(d.min())] if d.numel() else []
    s = s.masked_fill(s < kth, NEG)
    if top_p < 1.0:
        w = (s - s.max(dim=-1, keepdim=True).values).exp()
        srt = w.sort(dim=-1).values
        cum = srt.cumsum(-1)
        thr = (1.0 - top_p) * cum[:, -1:]
        margins.append(float((cum - thr).abs().min()))
        first = (cum > thr).int().argmax(dim=-1, keepdim=True)
        tau = torch.minimum(srt.gather(1, first), srt[:, -2:-1])           # min_tokens_to_keep = 2
        s = s.masked_fill(w < tau, NEG)
    key = (s - (-u.double().log()).log()).view(B, nb * V)
    s = s.view(B, nb * V)
    M = 2 * nb
    top_g, top_i = key.topk(M + 1, dim=1)
    toks, pars, new_seqs, new_scores = [], [], [], []
    for b in range(B):
        if st.done[b]:
            toks += [pad] * nb; pars += [b * nb] * nb
            new_seqs += [st.seqs[b * nb] + [pad]] * nb; new_scores += [0.0] * nb
            continue
        g = top_g[b].tolist()
        margins += _gaps(g)
        drawn = [(float(s[b, i]), i) for i, gi in zip(top_i[b, :M].tolist(), g[:M]) if gi > NEG]
        margins += _gaps([x[0] for x in drawn])
        drawn.sort(key=lambda c: (-c[0], c[1]))                           # higher score first, then lower flat index
        h = st.hyps[b]
        kept = 0
        for rank, (sc, idx) in enumerate(drawn):
            row, tok = b * nb + idx // V, idx % V
            if tok in eos:
                if rank < nb:
                    if len(h.beams) >= nb:
                        margins.append(abs(sc / (max(step, 1) ** lp) - h.worst_score))
                    h.add(list(st.seqs[row]), sc)
            else:
                toks.append(tok); pars.append(row); new_seqs.append(st.seqs[row] + [tok]); new_scores.append(sc)
                kept += 1
            if kept == nb:
                break
        st.error |= kept < nb
        while kept < nb:
            toks.append(pad); pars.append(b * nb); new_seqs.append(st.seqs[b * nb] + [pad]); new_scores.append(0.0)
            kept += 1
        if drawn:
            if len(h.beams) >= nb:
                margins.append(abs(h.worst_score - drawn[0][0] / (step + 1) ** lp))
            st.done[b] = st.done[b] or h.is_done(drawn[0][0], step + 1)
    st.seqs, st.scores = new_seqs, torch.tensor(new_scores, dtype=torch.float64)
    return toks, pars, margins


class _Device:
    """The buffers ``ops.beam_sample`` reads and writes."""

    def __init__(self, B, nb, V, max_new, eos, penalty, lp, T, top_p):
        from mm_interleaved_b200 import ops
        R, d = B * nb, "cuda"
        self.nb = nb
        self.params = torch.tensor([penalty, lp, T, top_p], dtype=torch.float64, device=d)
        self.beam_scores = torch.zeros((R,), dtype=torch.float32, device=d)
        self.history = torch.full((R, max_new), -5, dtype=torch.long, device=d)
        self.next_ids = torch.zeros((R, 1), dtype=torch.long, device=d)
        self.parent = torch.zeros((R,), dtype=torch.long, device=d)
        self.done = torch.zeros((B,), dtype=torch.bool, device=d)
        self.hyp_scores = torch.zeros((B, nb), dtype=torch.float64, device=d)
        self.hyp_ids = torch.zeros((B, nb, max_new), dtype=torch.long, device=d)
        self.hyp_meta = torch.full((B, nb, 2), -1, dtype=torch.long, device=d)
        self.error = torch.zeros((1,), dtype=torch.int32, device=d)
        self.scratch = torch.zeros((ops.beam_sample_scratch(nb, R),), dtype=torch.long, device=d)
        self.eos = torch.tensor(eos, dtype=torch.long, device=d) if eos else None

    def step(self, logits, step, pad, min_length, top_k, uniforms=None, seed=None):
        from mm_interleaved_b200 import ops
        ops.beam_sample(logits, torch.tensor([step], device="cuda"), self.params, self.beam_scores, self.history,
                        self.next_ids, self.parent, self.done, self.hyp_scores, self.hyp_ids, self.hyp_meta, self.error,
                        self.scratch, self.nb, eos=self.eos, pad_id=pad, min_length=min_length, top_k=top_k,
                        uniforms=uniforms, seed=seed)

    def hyps(self, b):
        meta, ids, sc = self.hyp_meta[b].tolist(), self.hyp_ids[b].tolist(), self.hyp_scores[b].tolist()
        slots = sorted((m[1], j) for j, m in enumerate(meta) if m[0] >= 0)
        return [(sc[j], ids[j][:meta[j][0]]) for _, j in slots]


def _uniforms(R, V, g):
    return torch.rand((R, V), generator=g).clamp(1e-6, 1 - 1e-6).cuda()


def _drive(B, nb, V, eos, lp, penalty, T, top_p, top_k, seed, logits_fn, min_length=2, n_steps=6, pad=0):
    """Kernel and restatement over n_steps; returns the restated state, or None where a decision of the restatement
    lies within MARGIN of flipping (the caller then takes another seed)."""
    dev = _Device(B, nb, V, n_steps, eos, penalty, lp, T, top_p)
    st = _State(B, nb, lp)
    g = torch.Generator().manual_seed(seed)
    for step in range(n_steps):
        logits = logits_fn(g, step)
        u = _uniforms(B * nb, V, g)
        dev.step(logits, step, pad, min_length, top_k, uniforms=u)
        toks, pars, m = _restated_step(st, logits, step, eos, pad, min_length, penalty, lp, T, top_p, top_k, u)
        if min(m, default=1.0) <= MARGIN:
            return None
        assert dev.next_ids[:, 0].tolist() == toks, (step, dev.next_ids[:, 0].tolist(), toks)
        assert dev.parent.tolist() == pars, (step, dev.parent.tolist(), pars)
        assert dev.done.tolist() == st.done, (step, dev.done.tolist(), st.done)
        assert bool(dev.error.item()) == st.error, step
        assert dev.history[:, :step + 1].tolist() == st.seqs, step
        torch.testing.assert_close(dev.beam_scores.double().cpu(), st.scores, atol=1e-4, rtol=1e-5)
        for b in range(B):
            got, want = dev.hyps(b), st.hyps[b].beams
            assert [x[1] for x in got] == [x[1] for x in want], (step, b, got, want)
            torch.testing.assert_close(torch.tensor([x[0] for x in got], dtype=torch.float64),
                                       torch.tensor([x[0] for x in want], dtype=torch.float64), atol=1e-4, rtol=1e-5)
    return st


def _random_logits(R, V, eos, seed, eos_boost=0.0):
    """Logits per step around a fixed base (so ids recur and the repetition penalty bites), eos ids placed
    ``eos_boost - 2`` above each row's maximum."""
    base = torch.randn((R, V), generator=torch.Generator().manual_seed(seed)) * 4.0
    top = base.max(dim=1).values
    for i, e in enumerate(eos):
        base[:, e] = top + eos_boost - 2.0 - 0.3 * i
    return lambda g, step: (base + torch.randn((R, V), generator=g) * 0.7).cuda()


def _drive_some_seed(B, nb, V, eos, lp, penalty, T, top_p, top_k, make_logits, **kw):
    for seed in range(8):
        st = _drive(B, nb, V, eos, lp, penalty, T, top_p, top_k, seed, make_logits(seed), **kw)
        if st is not None:
            return st
    pytest.fail("every seed tried puts a decision within MARGIN of a tie")


@pytest.mark.parametrize("V,nb,n_eos,T,top_p,top_k,penalty",
                         list(itertools.product((64, 32002), (3, 5), (1, 2), (1.0, 0.7), (0.9, 1.0), (2, 50), (1.0, 1.4))))
def test_beam_sample_matches_the_restated_step(V, nb, n_eos, T, top_p, top_k, penalty):
    eos = [7, 11][:n_eos]
    B = 2
    _drive_some_seed(B, nb, V, eos, 1.3, penalty, T, top_p, top_k,
                     lambda seed: _random_logits(B * nb, V, eos, 1000 * nb + 10 * n_eos + V % 97 + seed))


@pytest.mark.parametrize("top_p", [0.9, 1.0])
def test_constant_rows_keep_every_tied_token(top_p):
    """Every logit equal: every token ties at the k-th value and at the top-p threshold, so all stay drawable; the
    drawn candidates then tie on score and are ordered by flat index."""
    B, nb, V = 2, 3, 64
    st = _drive(B, nb, V, [7], 1.0, 1.0, 1.0, top_p, 50, 3, lambda g, step: torch.zeros((B * nb, V)).cuda(),
                n_steps=3)
    assert st is not None


def test_rows_tied_at_the_kth_value_keep_all_ties():
    """Twelve tokens share the row's 45th largest logit: top-k 50 keeps all of them (56 tokens)."""
    B, nb, V = 2, 3, 256

    def logits(g, step):
        x = torch.randn((B * nb, V), generator=g) * 3.0
        srt = x.sort(dim=-1, descending=True)
        x.scatter_(1, srt.indices[:, 44:56], srt.values[:, 44:45].expand(-1, 12).contiguous())
        return x.cuda()

    for seed in range(8):
        if _drive(B, nb, V, [7], 1.0, 1.0, 1.0, 1.0, 50, seed, logits, n_steps=4) is not None:
            return
    pytest.fail("every seed tried puts a decision within MARGIN of a tie")


def test_eos_dominated_rows_set_the_error_flag_and_exactly_nb_eos_do_not():
    B, nb, V = 2, 3, 64
    # ids 7 and 11 hold practically all the mass of every row, so the 2 * nb drawn are their 2 * nb entries: all eos
    # when both are eos ids, exactly nb eos when only 7 is
    for eos, want in (([7, 11], True), ([7], False)):
        st = _drive_some_seed(B, nb, V, eos, 1.0, 1.0, 1.0, 1.0, 50,
                              lambda seed: _random_logits(B * nb, V, [7, 11], seed, eos_boost=40.0), min_length=0,
                              n_steps=1)
        assert st.error == want
        if want:                                                       # every drawn candidate is eos: ranks < nb are kept
            assert all(len(h.beams) == nb for h in st.hyps)


def _draws(dev, B, nb, V):
    """The draw itself, read from the row stage's candidate lists: per sequence, the flat indices of the 2 * nb
    largest Gumbel keys, largest first."""
    M = 2 * nb
    w = dev.scratch.view(B * nb * M, 2)[:, 0].cpu().view(B, nb * M)       # (key << 32) | (2^32 - 1 - flat)
    key = (w >> 32) & 0xffffffff
    flat = 0xffffffff - (w & 0xffffffff)
    order = key.argsort(dim=1, descending=True, stable=True)[:, :M]
    return flat.gather(1, order)


def _stat_setup(B, seed=None):
    nb, V = 2, 4
    row = torch.tensor([[0.0, 0.5, 1.0, 1.5], [1.2, -0.3, 0.7, 0.2]])
    logits = row.repeat(B, 1).cuda()
    dev = _Device(B, nb, V, 1, [], 1.0, 1.0, 1.0, 1.0)
    dev.step(logits, 0, 0, 0, 0, seed=torch.tensor([seed], device="cuda"))
    probs = torch.log_softmax(row.double(), -1).view(-1).softmax(0)   # the sequence's 8 entries, beam scores 0
    return dev, nb, V, probs


def test_philox_draws_follow_the_softmax_without_replacement():
    from scipy import stats
    B = 20000
    dev, nb, V, probs = _stat_setup(B, seed=1234)
    d = _draws(dev, B, nb, V)
    assert (d >= 0).all() and (d < nb * V).all()
    assert all(len(set(x)) == 2 * nb for x in d.tolist())                  # no index twice within a sequence
    first = torch.bincount(d[:, 0], minlength=nb * V).double()
    assert stats.chisquare(first.numpy(), (probs * B).numpy()).pvalue > 1e-4
    # the unordered pair of the first two picks, against torch.multinomial without replacement
    ref = torch.multinomial(probs.float().expand(B, -1), 2 * nb, replacement=False,
                            generator=torch.Generator().manual_seed(5))
    pair = lambda x: (x[:, :2].min(dim=1).values * (nb * V) + x[:, :2].max(dim=1).values)
    a, b = (torch.bincount(pair(x), minlength=(nb * V) ** 2) for x in (d, ref))
    keep = (a + b) > 0
    table = torch.stack([a[keep], b[keep]]).numpy()
    assert stats.chi2_contingency(table).pvalue > 1e-4
    # the drawn set is what the scorer saw: the best two of it by score became the beams
    assert dev.error.item() == 0


def test_philox_draws_are_keyed_by_the_seed():
    B = 512
    d1 = _draws(_stat_setup(B, seed=77)[0], B, 2, 4)
    d2 = _draws(_stat_setup(B, seed=77)[0], B, 2, 4)
    d3 = _draws(_stat_setup(B, seed=78)[0], B, 2, 4)
    assert torch.equal(d1, d2) and not torch.equal(d1, d3)


class _Race:
    """A deterministic stand-in for ``torch.multinomial(probs, n)`` without replacement: the n largest keys
    log p - log(-log u), u from a CPU generator seeded by the call count (the same law as the real draw)."""

    def __init__(self):
        self.calls = 0

    def __call__(self, probs, num_samples, replacement=False, generator=None):
        assert not replacement
        g = torch.Generator().manual_seed(100 + self.calls)
        self.calls += 1
        u = torch.rand(probs.shape, generator=g, dtype=torch.float64).clamp(1e-12, 1 - 1e-12)
        key = probs.detach().double().cpu().log() - (-u.log()).log()
        return key.topk(num_samples, dim=-1).indices.to(probs.device)


@pytest.mark.parametrize("n_ret", [1, 2])
def test_eager_beam_sample_matches_the_hf_algorithm_on_the_oracle_decoder(monkeypatch, n_ret):
    """nb = 3, two eos ids, min_length, length_penalty != 1, T != 1: the eager beam sample (prefill once, replicated and
    re-gathered caches) against 4.31's beam_sample written out in plain Python over the oracle decoder, the draw
    replaced by the same deterministic race on both sides."""
    from tests.test_generate_gpu import _BeamHyps, _oracle_step_logits, _setup
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    nb, n_new, min_len, lp, pad, T, top_p = 3, 6, 2, 1.3, 0, 0.7, 0.9
    free = dev.generate_texts(ids.cuda(), vis_d, nimg.cuda(), 2, max_new_tokens=n_new, eos_token_id=None).cpu()
    eos = [int(free[0, 3]), int(free[1, 2])]
    race = _Race()
    monkeypatch.setattr(torch, "multinomial", race)
    got = dev.generate_texts(ids.cuda(), vis_d, nimg.cuda(), 2, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=pad,
                             min_length=min_len, num_beams=nb, length_penalty=lp, use_nucleus_sampling=True,
                             temperature=T, top_p=top_p, num_return_sequences=n_ret).cpu()
    n_eager = race.calls
    race.calls = 0

    B = ids.shape[0]
    G = B * n_ret
    first = [0, int(nimg[0])]
    rows = [b for b in range(B) for _ in range(n_ret * nb)]
    img_rows = [i for b in rows for i in range(first[b], first[b] + int(nimg[b]))]
    ids_r, nimg_r = ids[rows], nimg[rows]
    vis_r = {"vis_embed": vis["vis_embed"][img_rows], "multiscale_features": [f[img_rows] for f in vis["multiscale_features"]]}
    seqs = [[] for _ in range(G * nb)]
    beam_scores = torch.zeros(G * nb)
    hyps = [_BeamHyps(nb, lp) for _ in range(G)]
    done = [False] * G
    for step in range(n_new):
        cur = torch.cat([ids_r, torch.tensor(seqs, dtype=torch.long).view(G * nb, -1)], dim=1)
        logp = torch.log_softmax(_oracle_step_logits(cfg, sd, cur, ids_r, nimg_r, vis_r, step).float(), -1)
        if step < min_len:
            logp[:, eos] = NEG
        V = logp.shape[-1]
        s = (logp + beam_scores[:, None]) / T                                  # TemperatureLogitsWarper
        s = s.masked_fill(s < s.topk(min(50, V), dim=-1).values[:, -1:], NEG)  # TopKLogitsWarper
        srt, idx = s.sort(dim=-1)                                               # TopPLogitsWarper, 2 kept
        drop = srt.softmax(-1).cumsum(-1) <= 1 - top_p
        drop[:, -2:] = False
        s = s.masked_fill(drop.scatter(1, idx, drop), NEG).view(G, nb * V)
        nxt = torch.multinomial(s.softmax(-1), 2 * nb)
        sc_all, order = s.gather(1, nxt).sort(dim=1, descending=True, stable=True)
        nxt = nxt.gather(1, order)
        new_seqs, new_scores = [], []
        for b in range(G):
            if done[b]:
                new_seqs += [seqs[b * nb] + [pad]] * nb; new_scores += [0.0] * nb
                continue
            kept = 0
            for rank in range(2 * nb):
                sc, i = float(sc_all[b, rank]), int(nxt[b, rank])
                row, tok = b * nb + i // V, i % V
                if tok in eos:
                    if rank < nb:
                        hyps[b].add(list(seqs[row]), sc)
                else:
                    new_seqs.append(seqs[row] + [tok]); new_scores.append(sc); kept += 1
                if kept == nb:
                    break
            assert kept == nb
            done[b] = done[b] or hyps[b].is_done(float(sc_all[b].max()), len(seqs[b * nb]) + 1)
        seqs, beam_scores = new_seqs, torch.tensor(new_scores)
        if all(done):
            break
    assert race.calls == n_eager
    for b in range(G):
        if not done[b]:
            for j in range(nb):
                hyps[b].add(list(seqs[b * nb + j]), float(beam_scores[b * nb + j]))
    best = [sorted(h.beams, key=lambda x: x[0])[-1][1] for h in hyps]
    width = min(max(len(x) for x in best) + 1, n_new)
    want = torch.full((G, width), pad, dtype=torch.long)
    for i, x in enumerate(best):
        want[i, :len(x)] = torch.tensor(x, dtype=torch.long)
        if len(x) < width:
            want[i, len(x)] = eos[0]
    assert torch.equal(got, want), (got, want)


def test_eos_dominated_model_raises_value_error_eager_and_graphed():
    from tests.test_generate_gpu import _setup
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    with torch.no_grad():
        dev.text_decoder.head.bias[[5, 9]] += 40.0                     # both eos ids outweigh everything
    args = (ids.cuda(), vis_d, nimg.cuda(), 2)
    kw = dict(max_new_tokens=4, eos_token_id=[5, 9], min_length=0, num_beams=3, use_nucleus_sampling=True)
    with pytest.raises(ValueError, match="At most 3 tokens"):
        dev.generate_texts(*args, **kw)
    dev.enable_decode_graphs(True, sampling=True)
    try:
        with pytest.raises(ValueError, match="At most 3 tokens"):
            dev.generate_texts(*args, generator=torch.Generator(device="cuda").manual_seed(1), **kw)
    finally:
        dev.enable_decode_graphs(False)


class _Uncaptured:
    """Stands in for a graphed decoder's captured graph: each "replay" runs the step's kernels directly."""

    def __init__(self, dec):
        self.replay = dec._step


def test_graphed_beam_sample_is_seeded_reuses_one_graph_equals_uncaptured_steps_and_adds_two_launches():
    from tests.test_beam_select_gpu import _second_call
    from tests.test_generate_gpu import _setup
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    vis2_d, mask2 = _second_call(ids, vis)
    args, args2 = (ids.cuda(), vis_d, nimg.cuda(), 2), (ids.cuda(), vis2_d, nimg.cuda(), 2)
    kw = dict(max_new_tokens=8, eos_token_id=[int(x) for x in (7, 11)], min_length=2, num_beams=3, length_penalty=1.3,
              num_return_sequences=2, use_nucleus_sampling=True, temperature=0.7, top_p=0.9)
    gen = lambda a, seed, **extra: dev.generate_texts(*a, generator=torch.Generator(device="cuda").manual_seed(seed),
                                                      **dict(kw, **extra)).cpu()
    dev.enable_decode_graphs(True, sampling=True)
    try:
        first = gen(args, 7)
        other = gen(args2, 7, attention_mask=mask2)
        again = gen(args, 7)
        assert len(dev._decode_graphs) == 1 and next(iter(dev._decode_graphs))[-2:] == (3, "beam_sample")
        assert torch.equal(first, again), (first, again)
        assert first.shape[0] == 4 and other.shape[0] == 4 and int(first.max()) < 64
        dec = next(iter(dev._decode_graphs.values()))
        graph, dec.graph = dec.graph, _Uncaptured(dec)
        try:
            uncaptured = gen(args, 7)
        finally:
            dec.graph = graph
        assert torch.equal(first, uncaptured), (first, uncaptured)
        dev.enable_decode_graphs(True)                                 # a greedy graph of the same shape
        dev.generate_texts(*args, max_new_tokens=8, eos_token_id=[7, 11])
        greedy = next(iter(dev._decode_graphs.values()))
        dev.enable_decode_graphs(True, sampling=True)
        gen(args, 7)
        sample = next(iter(dev._decode_graphs.values()))
        assert sample.launches == greedy.launches + 2                  # beam_sample (2 kernels) + kv_beam_reorder - decode_select
    finally:
        dev.enable_decode_graphs(False)


def test_reference_defaults_with_nucleus_sampling_through_mm_interleaved_generate():
    from tests.test_mm_interleaved_gpu import DEV, _batch, _build
    model, _ = _build()
    ids, images, nimg, mask = _batch()
    batch = dict(text_ids=ids.to(DEV), image_tensors=images.to(DEV), num_image_per_seq=nimg.to(DEV),
                 attention_mask=mask.to(DEV), meta=None, use_nucleus_sampling=True)
    for graphed in (False, True):
        model.enable_decode_graphs(graphed, sampling=True)
        try:
            g = torch.Generator(device=DEV).manual_seed(3)
            out = model.generate(mode="generate_texts", generator=g, **batch)["text_ids"]   # 5 beams, min 8, eos [eos, soi]
            assert out.dtype == torch.long and out.shape[0] == ids.shape[0] and 1 <= out.shape[1] <= 30, out.shape
            if graphed:
                assert next(iter(model._decode_graphs))[-2:] == (5, "beam_sample")
        finally:
            model.enable_decode_graphs(False)
