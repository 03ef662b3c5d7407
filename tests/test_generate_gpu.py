"""GPU test: greedy generate_texts (prefill + KV-cache decode with the decode-kernel path) produces the same tokens
as a CPU oracle greedy loop built from the restatement of the reference decoder (tiny config, fp32)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.glue import cross_attention_mask_ref, pack_mmfs_features_ref, prepare_mm_embeds_ref, text_head_ref  # noqa: E402
from oracle.llama import llama_model_ref  # noqa: E402
from tests.golden.make_golden import LLAMA_TINY, seeded_state_dict  # noqa: E402


def test_greedy_generation_matches_oracle_loop():
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.mm_interleaved import InterleavedForward
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = m.LlamaMMFSConfig(**LLAMA_TINY)
    BOS, IMG, SOI = 1, 62, 63
    model = InterleavedForward(cfg, special_tokens=dict(bos_token_id=BOS, image_token_id=IMG, soi_token_id=SOI), orig_vocab_size=62)
    sd = seeded_state_dict(model.state_dict(), seed=31337)
    sd["text_decoder.head.weight"][60:] = 0        # never emit the special ids: their logits stay 0 < max of 60 random logits
    sd["text_decoder.head_new.weight"].zero_()
    sd["text_decoder.head.bias"][60:] = 0
    sd["text_decoder.head_new.bias"].zero_()
    model.load_state_dict(sd)
    g = torch.Generator().manual_seed(3)
    L, n_tok = 20, 3
    ids = torch.randint(3, 60, (2, L), generator=g)
    ids[:, 0] = BOS
    ids[0, 2] = SOI; ids[0, 3:3 + n_tok] = IMG
    ids[0, 10] = SOI; ids[0, 11:11 + n_tok] = IMG
    ids[1, 5] = SOI; ids[1, 6:6 + n_tok] = IMG
    nimg = torch.tensor([2, 1])
    vis = {"vis_embed": torch.randn((3, n_tok, cfg.hidden_size), generator=g) * 0.5,
           "multiscale_features": [torch.randn((3, cfg.image_embed_dim, s, s), generator=g) for s in (8, 4, 2)]}
    n_new = 6
    dev = model.cuda().eval()
    got = dev.generate_texts(ids.cuda(), {"vis_embed": vis["vis_embed"].cuda(),
                                          "multiscale_features": [f.cuda() for f in vis["multiscale_features"]]},
                             nimg.cuda(), 2, max_new_tokens=n_new, eos_token_id=None).cpu()

    # oracle loop (recomputes the full prefix every step: no cache, same arithmetic as the reference forward)
    dec = {k[len("mm_decoder."):]: v for k, v in sd.items() if k.startswith("mm_decoder.")}
    ocfg = dict(eps=cfg.rms_norm_eps, n_heads=cfg.num_attention_heads, n_layers=cfg.num_hidden_layers,
                spatial_shapes=[(s, s) for s in cfg.spatial_shapes])
    feats = pack_mmfs_features_ref(vis["multiscale_features"], cfg.spatial_shapes, nimg)
    cur = ids.clone()
    want = []
    cross0 = cross_attention_mask_ref(ids, nimg, BOS, SOI)
    for step in range(n_new):
        emb = torch.nn.functional.embedding(cur, dec["embed_tokens.weight"])
        emb = prepare_mm_embeds_ref(emb, cur, vis["vis_embed"], sd["soi_token"], IMG, SOI)
        cross = torch.cat([cross0] + [cross0[:, -1:]] * step, dim=1)      # new tokens reuse the last mask row
        hid, _ = llama_model_ref(dec, emb, torch.ones_like(cur), None, feats, cross, ocfg)
        logits = text_head_ref(sd, hid[:, -1], 62)
        nxt = logits.argmax(-1)
        want.append(nxt)
        cur = torch.cat([cur, nxt[:, None]], dim=1)
    want = torch.stack(want, 1)
    assert torch.equal(got, want), (got, want)
    # the reference-style growing (cat) cache gives the same tokens as the pre-allocated in-place cache used above
    got_cat = dev.generate_texts(ids.cuda(), {"vis_embed": vis["vis_embed"].cuda(),
                                              "multiscale_features": [f.cuda() for f in vis["multiscale_features"]]},
                                 nimg.cuda(), 2, max_new_tokens=n_new, eos_token_id=None, static_cache=False).cpu()
    assert torch.equal(got_cat, want)


def _setup(seed_weights=31337):
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.mm_interleaved import InterleavedForward
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = m.LlamaMMFSConfig(**LLAMA_TINY)
    BOS, IMG, SOI = 1, 62, 63
    model = InterleavedForward(cfg, special_tokens=dict(bos_token_id=BOS, image_token_id=IMG, soi_token_id=SOI), orig_vocab_size=62)
    sd = seeded_state_dict(model.state_dict(), seed=seed_weights)
    sd["text_decoder.head.weight"][60:] = 0
    sd["text_decoder.head_new.weight"].zero_()
    sd["text_decoder.head.bias"][60:] = 0
    sd["text_decoder.head_new.bias"].zero_()
    model.load_state_dict(sd)
    g = torch.Generator().manual_seed(3)
    L, n_tok = 20, 3
    ids = torch.randint(3, 60, (2, L), generator=g)
    ids[:, 0] = BOS
    ids[0, 2] = SOI; ids[0, 3:3 + n_tok] = IMG
    ids[0, 10] = SOI; ids[0, 11:11 + n_tok] = IMG
    ids[1, 5] = SOI; ids[1, 6:6 + n_tok] = IMG
    nimg = torch.tensor([2, 1])
    vis = {"vis_embed": torch.randn((3, n_tok, cfg.hidden_size), generator=g) * 0.5,
           "multiscale_features": [torch.randn((3, cfg.image_embed_dim, s, s), generator=g) for s in (8, 4, 2)]}
    vis_d = {"vis_embed": vis["vis_embed"].cuda(), "multiscale_features": [f.cuda() for f in vis["multiscale_features"]]}
    return cfg, model.cuda().eval(), sd, ids, nimg, vis, vis_d


def _oracle_step_logits(cfg, sd, cur, ids, nimg, vis, step):
    dec = {k[len("mm_decoder."):]: v for k, v in sd.items() if k.startswith("mm_decoder.")}
    ocfg = dict(eps=cfg.rms_norm_eps, n_heads=cfg.num_attention_heads, n_layers=cfg.num_hidden_layers,
                spatial_shapes=[(s, s) for s in cfg.spatial_shapes])
    feats = pack_mmfs_features_ref(vis["multiscale_features"], cfg.spatial_shapes, nimg)
    cross0 = cross_attention_mask_ref(ids, nimg, 1, 63)
    emb = torch.nn.functional.embedding(cur, dec["embed_tokens.weight"])
    emb = prepare_mm_embeds_ref(emb, cur, vis["vis_embed"], sd["soi_token"], 62, 63)
    cross = torch.cat([cross0] + [cross0[:, -1:]] * step, dim=1)
    hid, _ = llama_model_ref(dec, emb, torch.ones_like(cur), None, feats, cross, ocfg)
    return text_head_ref(sd, hid[:, -1], 62)


def test_min_length_eos_list_and_repetition_penalty_follow_hf_semantics():
    """Greedy decoding with HF's RepetitionPenalty / MinLength processors and a list of eos ids, against the oracle
    decoder loop with the same processors written out in plain PyTorch."""
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    n_new, min_len, pen, pad = 7, 3, 1.7, 0
    free = dev.generate_texts(ids.cuda(), vis_d, nimg.cuda(), 2, max_new_tokens=n_new, eos_token_id=None).cpu()
    eos = [int(free[0, 1]), int(free[1, 4])]          # ids the unconstrained run emits: they become end-of-sequence ids
    got = dev.generate_texts(ids.cuda(), vis_d, nimg.cuda(), 2, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=pad,
                             min_length=min_len, repetition_penalty=pen).cpu()
    cur, want, fin = ids.clone(), [], torch.zeros(2, dtype=torch.bool)
    for step in range(n_new):
        sc = _oracle_step_logits(cfg, sd, cur, ids, nimg, vis, step)
        for b in range(2):
            for t in set(int(x[b]) for x in want):                                   # repetition penalty on generated ids
                sc[b, t] = sc[b, t] * pen if sc[b, t] < 0 else sc[b, t] / pen
        if step < min_len:
            sc[:, eos] = float("-inf")
        nxt = sc.argmax(-1)
        nxt = torch.where(fin, torch.full_like(nxt, pad), nxt)
        for e in eos:
            fin = fin | (nxt == e)
        want.append(nxt)
        cur = torch.cat([cur, nxt[:, None]], dim=1)
    want = torch.stack(want, 1)
    assert torch.equal(got, want), (got, want)
    assert not torch.equal(got, free)                 # the processors changed the continuation


def test_nucleus_sampling_limits_and_determinism():
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    args = (ids.cuda(), vis_d, nimg.cuda(), 2)
    greedy = dev.generate_texts(*args, max_new_tokens=5, eos_token_id=None)
    # top_p -> 0 keeps only the most likely token; temperature -> 0 concentrates all mass on it
    a = dev.generate_texts(*args, max_new_tokens=5, eos_token_id=None, use_nucleus_sampling=True, top_p=1e-6)
    b = dev.generate_texts(*args, max_new_tokens=5, eos_token_id=None, use_nucleus_sampling=True, top_p=1.0, temperature=1e-4)
    assert torch.equal(a, greedy) and torch.equal(b, greedy)
    g1 = torch.Generator(device="cuda").manual_seed(5)
    g2 = torch.Generator(device="cuda").manual_seed(5)
    s1 = dev.generate_texts(*args, max_new_tokens=6, eos_token_id=None, use_nucleus_sampling=True, top_p=0.95, temperature=2.0, generator=g1)
    s2 = dev.generate_texts(*args, max_new_tokens=6, eos_token_id=None, use_nucleus_sampling=True, top_p=0.95, temperature=2.0, generator=g2)
    assert torch.equal(s1, s2) and int(s1.max()) < 64 and not torch.equal(s1[:, :5], greedy)


class _BeamHyps:
    """BeamHypotheses of transformers 4.31 (generation/beam_search.py), early_stopping=False."""

    def __init__(self, num_beams, length_penalty):
        self.num_beams, self.length_penalty, self.beams, self.worst_score = num_beams, length_penalty, [], 1e9

    def add(self, hyp, sum_logprobs):
        score = sum_logprobs / (max(len(hyp), 1) ** self.length_penalty)
        if len(self.beams) < self.num_beams or score > self.worst_score:
            self.beams.append((score, hyp))
            if len(self.beams) > self.num_beams:
                srt = sorted((s, i) for i, (s, _) in enumerate(self.beams))
                del self.beams[srt[0][1]]
                self.worst_score = srt[1][0]
            else:
                self.worst_score = min(score, self.worst_score)

    def is_done(self, best_sum_logprobs, cur_len):
        if len(self.beams) < self.num_beams:
            return False
        return self.worst_score >= best_sum_logprobs / cur_len ** self.length_penalty


def test_beam_search_matches_the_hf_algorithm_on_the_oracle_decoder():
    """num_beams = 3 with min_length / eos list / length penalty: the GPU path (prefill once, replicated + re-gathered
    in-place caches, split-KV decode attention) against HF's beam_search + BeamSearchScorer written out in plain
    Python over the oracle decoder (full-prefix recompute per beam, no cache)."""
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    nb, n_new, min_len, lp, pad = 3, 6, 2, 1.3, 0
    free = dev.generate_texts(ids.cuda(), vis_d, nimg.cuda(), 2, max_new_tokens=n_new, eos_token_id=None).cpu()
    eos = [int(free[0, 3]), int(free[1, 2])]
    got = dev.generate_texts(ids.cuda(), vis_d, nimg.cuda(), 2, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=pad,
                             min_length=min_len, num_beams=nb, length_penalty=lp).cpu()

    B = ids.shape[0]
    first = [0, int(nimg[0])]
    rows = [b for b in range(B) for _ in range(nb)]
    img_rows = [i for b in rows for i in range(first[b], first[b] + int(nimg[b]))]
    ids_r, nimg_r = ids[rows], nimg[rows]
    vis_r = {"vis_embed": vis["vis_embed"][img_rows], "multiscale_features": [f[img_rows] for f in vis["multiscale_features"]]}
    seqs = [[] for _ in range(B * nb)]
    beam_scores = torch.tensor([[0.0] + [-1e9] * (nb - 1)] * B).view(-1)
    hyps = [_BeamHyps(nb, lp) for _ in range(B)]
    done = [False] * B
    for step in range(n_new):
        cur = torch.cat([ids_r, torch.tensor(seqs, dtype=torch.long).view(B * nb, -1)], dim=1)
        logp = torch.log_softmax(_oracle_step_logits(cfg, sd, cur, ids_r, nimg_r, vis_r, step).float(), -1)
        if step < min_len:
            logp[:, eos] = float("-inf")
        V = logp.shape[-1]
        top_s, top_i = (logp + beam_scores[:, None]).view(B, nb * V).topk(2 * nb, dim=1)
        new_seqs, new_scores = [], []
        for b in range(B):
            if done[b]:
                new_seqs += [seqs[b * nb] + [pad]] * nb; new_scores += [0.0] * nb
                continue
            kept = 0
            for rank in range(2 * nb):
                sc, idx = float(top_s[b, rank]), int(top_i[b, rank])
                row, tok = b * nb + idx // V, idx % V
                if tok in eos:
                    if rank < nb:
                        hyps[b].add(list(seqs[row]), sc)
                else:
                    new_seqs.append(seqs[row] + [tok]); new_scores.append(sc); kept += 1
                if kept == nb:
                    break
            done[b] = done[b] or hyps[b].is_done(float(top_s[b].max()), len(seqs[b * nb]) + 1)
        seqs, beam_scores = new_seqs, torch.tensor(new_scores)
        if all(done):
            break
    for b in range(B):
        if not done[b]:
            for j in range(nb):
                hyps[b].add(list(seqs[b * nb + j]), float(beam_scores[b * nb + j]))
    best = [sorted(h.beams, key=lambda x: x[0])[-1][1] for h in hyps]
    width = min(max(len(x) for x in best) + 1, n_new)
    want = torch.full((B, width), pad, dtype=torch.long)
    for i, x in enumerate(best):
        want[i, :len(x)] = torch.tensor(x, dtype=torch.long)
        if len(x) < width:
            want[i, len(x)] = eos[0]
    assert torch.equal(got, want), (got, want)


def test_graphed_greedy_decode_matches_eager_across_calls_with_new_images():
    """``enable_decode_graphs()``: one CUDA graph per generated token, static KV cache / masks / PreparedVision buffers
    reused by later calls.  Tokens must equal the eager loop's (which equals the oracle loop, first test) -- also on the
    SECOND call with different images and a different prompt mask, which replays the graph captured by the first."""
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    g = torch.Generator().manual_seed(123)
    vis2_d = {"vis_embed": (torch.randn(vis["vis_embed"].shape, generator=g) * 0.5).cuda(),
              "multiscale_features": [(torch.randn(f.shape, generator=g) * 2).cuda() for f in vis["multiscale_features"]]}
    mask2 = torch.ones_like(ids)
    mask2[1, :2] = 0                                                   # left padding on the second sequence
    kw = dict(max_new_tokens=7, eos_token_id=[2, 17], min_length=3)
    eager_a = dev.generate_texts(ids.cuda(), vis_d, nimg.cuda(), 2, **kw).cpu()
    eager_b = dev.generate_texts(ids.cuda(), vis2_d, nimg.cuda(), 2, attention_mask=mask2.cuda(), **kw).cpu()
    assert not torch.equal(eager_a, eager_b)
    dev.enable_decode_graphs()
    graph_a = dev.generate_texts(ids.cuda(), vis_d, nimg.cuda(), 2, **kw).cpu()
    graph_b = dev.generate_texts(ids.cuda(), vis2_d, nimg.cuda(), 2, attention_mask=mask2.cuda(), **kw).cpu()
    graph_a2 = dev.generate_texts(ids.cuda(), vis_d, nimg.cuda(), 2, **kw).cpu()
    assert len(dev._decode_graphs) == 1                                # one captured graph served all three calls
    assert torch.equal(graph_a, eager_a), (graph_a, eager_a)
    assert torch.equal(graph_b, eager_b), (graph_b, eager_b)
    assert torch.equal(graph_a2, eager_a)
    dev.generate_texts(ids.cuda(), vis_d, nimg.cuda(), 2, repetition_penalty=1.7, **kw)
    assert len(dev._decode_graphs) == 1                                # plain and penalised greedy share one graph
    dev.enable_decode_graphs(False)
