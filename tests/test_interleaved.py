"""CPU tests of the host logic of ``generate_interleaved`` (interleaved.py): ``update_texts`` against a restatement of
the reference's tensor version (inference.py:118-185), the static cache's length budget against every turn outcome,
and the refusals made before any work."""
import itertools
from types import SimpleNamespace

import pytest
import torch

ST = dict(bos_token_id=1, eos_token_id=2, pad_token_id=31999, soi_token_id=32000, image_token_id=32001)


def reference_update_texts(text_ids, num_img_token, force_gen_image_next):
    """inference.py's update_texts on a (1, W) tensor, without the inputs dict: (appended ids, gen_image_next, stopped)."""
    gen_image_next, stopped = False, False
    text_ids = text_ids[0][1:]
    if text_ids[-1] == ST["eos_token_id"]:
        text_ids = text_ids[:-1]
        stopped = True
    if force_gen_image_next and text_ids[-1] != ST["soi_token_id"]:
        text_ids = torch.cat((text_ids, torch.tensor([ST["soi_token_id"]]).type_as(text_ids)), dim=-1)
    if text_ids[-1] == ST["soi_token_id"]:
        text_ids = torch.cat((text_ids, torch.tensor([ST["image_token_id"]] * num_img_token).type_as(text_ids)), dim=-1)
        gen_image_next = True
    return text_ids.tolist(), gen_image_next, stopped


def _sequences():
    body = [[5, 6], [5, ST["pad_token_id"]], [ST["soi_token_id"]], [7, ST["soi_token_id"]], [ST["eos_token_id"]],
            [8, ST["eos_token_id"]], [ST["soi_token_id"], ST["eos_token_id"]], [9, ST["eos_token_id"], ST["pad_token_id"]],
            [ST["eos_token_id"], ST["soi_token_id"]], [4, 4, 4, 4]]
    for first in (ST["bos_token_id"], 11):
        for b in body:
            yield [first] + b


@pytest.mark.parametrize("force", [False, True])
def test_update_texts_matches_the_reference(force):
    from mm_interleaved_b200.interleaved import update_texts
    for seq in _sequences():
        try:
            want = reference_update_texts(torch.tensor([seq]), 64, force)
        except IndexError:                          # the reference indexes an empty tensor: so does the session
            with pytest.raises(IndexError):
                update_texts(seq, ST, 64, force)
            continue
        assert update_texts(seq, ST, 64, force) == want, seq


def _worst_length(length, mode, num_iter, max_length, n_tok):
    """The largest cache length any run can need: every text turn's outcome (generated width, eos or not, <soi> or
    not) enumerated; a text turn needs its prompt plus max_length positions while decoding."""
    best = length

    def turn(L, mode, left):
        nonlocal best
        if left == 0:
            best = max(best, L)
            return
        if mode == "generate_images":
            turn(L, "generate_texts", left - 1)
            return
        best = max(best, L + max_length)
        for width in range(2, max_length + 1):
            turn(L + width - 1, "generate_texts", left - 1)                     # no <soi>
            turn(L + width - 1 + n_tok, "generate_images", left - 1)            # ends with <soi>
            turn(L + width + n_tok, "generate_images", left - 1)                # a forced <soi>

    turn(length, mode, num_iter)
    return best


@pytest.mark.parametrize("mode,num_iter,max_length", list(itertools.product(
    ("generate_texts", "generate_images"), (1, 2, 4), (2, 5))))
def test_cache_budget_covers_every_run(mode, num_iter, max_length):
    from mm_interleaved_b200.interleaved import cache_budget
    budget = cache_budget(20, mode, num_iter, max_length, 3)
    worst = _worst_length(20, mode, num_iter, max_length, 3)
    assert budget == worst


def _stub_model(vae=True):
    sd = SimpleNamespace(vae_decode=(lambda x: x) if vae else None)
    return SimpleNamespace(special_token_dict=ST, num_img_token=64, image_decoder=SimpleNamespace(decoder=sd))


def _inputs(batch=1):
    ids = torch.ones((batch, 70), dtype=torch.long)
    return dict(text_ids=ids, image_tensors=torch.zeros((1, 3, 224, 224)), num_image_per_seq=torch.tensor([1] * batch),
                attention_mask=torch.ones_like(ids))


def test_refusals():
    from mm_interleaved_b200.interleaved import generate_interleaved
    with pytest.raises(ValueError, match="one sample"):
        generate_interleaved(_stub_model(), **_inputs(batch=2))
    with pytest.raises(NotImplementedError, match="tokenizer"):
        generate_interleaved(_stub_model(), **_inputs(), force_replace_gen_text=True)
    with pytest.raises(RuntimeError, match="VAE decoder"):
        generate_interleaved(_stub_model(vae=False), **_inputs())
    with pytest.raises(RuntimeError, match="VAE decoder"):
        generate_interleaved(SimpleNamespace(special_token_dict=ST, num_img_token=64, image_decoder=None), **_inputs())
    with pytest.raises(ValueError, match="generate_mode"):
        generate_interleaved(_stub_model(), **_inputs(), generate_mode="generate_scores")
    with pytest.raises(TypeError, match="unexpected"):
        generate_interleaved(_stub_model(), **_inputs(), beam_width=3)
    with pytest.raises(ValueError, match="max_cache_length"):                   # 70 + 421 > 490
        generate_interleaved(_stub_model(), **_inputs(), num_iter=4, max_length=90, max_cache_length=490)


def test_model_method_refuses_without_image_decoder():
    from mm_interleaved_b200 import LlamaMMFSConfig
    from mm_interleaved_b200.mm_interleaved import MMInterleaved
    from tests.golden.make_golden import LLAMA_TINY

    class Tok(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.proj = torch.nn.Linear(3, 4)

    cfg = LlamaMMFSConfig(**LLAMA_TINY)
    model = MMInterleaved(llm_config=cfg, txt_vocab_size=cfg.vocab_size, visual_tokenizer=Tok(),
                          image_embed_dim=cfg.image_embed_dim, spatial_shapes=cfg.spatial_shapes)
    with pytest.raises(RuntimeError, match="VAE decoder"):
        model.generate_interleaved(**_inputs())
