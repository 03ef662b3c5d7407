"""CPU test of ``MMInterleaved.freeze_like_reference()``: the trainable parameters of the LLM, the text head and
``soi_token`` are exactly those the reference's constructor leaves trainable (mm_interleaved.py:74-78: the LLM frozen
except names containing ``llama_cross_attn``; decoder_text.py:50-51: the text head frozen except ``head_new``), applied
here by name; the visual tokenizer and image decoder are left as they were."""


def test_trainable_set_matches_the_reference_rule():
    import mm_interleaved_b200 as m
    from tests.golden.make_golden import LLAMA_TINY
    vt_cfg = dict(clip_config=m.visual_tokenizer.CLIPVisionConfigLite(hidden_size=64, intermediate_size=64, num_hidden_layers=4,
                                                                     num_attention_heads=2, image_size=28, patch_size=14),
                  perceiver_config=dict(num_queries=2, hidden_size=64, encoder_hidden_size=64, cross_attention_frequency=2,
                                        num_hidden_layers=2, num_attention_heads=2, intermediate_size=64,
                                        qk_normalization=True), grid_size=2)
    st = dict(bos_token_id=1, eos_token_id=2, pad_token_id=0, soi_token_id=62, image_token_id=63)
    model = m.MMInterleaved(llm_config=dict(LLAMA_TINY, vocab_size=62), txt_vocab_size=64, seq_len=32, special_token_dict=st,
                            visual_tokenizer_config=vt_cfg, image_embed_dim=LLAMA_TINY["image_embed_dim"],
                            cross_attention_frequency=2, spatial_shapes=LLAMA_TINY["spatial_shapes"])
    model.visual_tokenizer.requires_grad_(False)
    before = {n: p.requires_grad for n, p in model.named_parameters() if n.startswith("visual_tokenizer.")}
    assert model.freeze_like_reference() is model

    def reference_rule(name):
        if name.startswith("mm_decoder."):
            return "llama_cross_attn" in name
        if name.startswith("text_decoder."):
            return name.startswith("text_decoder.head_new.")
        return name == "soi_token"

    names = [n for n, _ in model.named_parameters() if n.split(".")[0] in ("mm_decoder", "text_decoder", "soi_token")]
    got = {n for n, p in model.named_parameters() if n in names and p.requires_grad}
    want = {n for n in names if reference_rule(n)}
    assert got == want
    assert any("llama_cross_attn.attn.sampling_offsets" in n for n in got) and "text_decoder.head_new.weight" in got
    assert any(n.endswith("llama_cross_attn.gate") for n in got) and "soi_token" in got
    assert before == {n: p.requires_grad for n, p in model.named_parameters() if n.startswith("visual_tokenizer.")}
