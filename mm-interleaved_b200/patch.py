"""``replace_*_b200()`` -- the reference's own start-up patch mechanism (inference.py:10-24,
mm_interleaved/models/utils/monkey_patch/__init__.py:1-5), pointed at this repository's classes.

Call them where ``inference.py`` / ``evaluate.py`` call ``replace_blip2_attn_with_qknorm_attn()`` etc., i.e. after
``import mm_interleaved...`` and BEFORE ``MMInterleaved(**config.model)`` is constructed (inference.py:291).  Every
function rebinds the reference class objects wherever a reference module already holds them (``from ..x import MMFS``
creates a second binding in the importer's namespace), so construction afterwards builds the H100 modules while the
reference's own ``MMInterleaved`` / ``LlamaModel`` / ``ImageDecoder`` glue, state-dict names and checkpoints stay as
they are.  Nothing here imports the reference: the functions look the modules up in ``sys.modules`` / by name and raise
if the reference package is not importable.
"""
from __future__ import annotations

import importlib
import sys
from typing import Dict

_REF = "mm_interleaved"
_UNDO = []          # (module, attribute, previous value) in application order


def _set(mod, attr, new):
    _UNDO.append((mod, attr, getattr(mod, attr, None)))
    setattr(mod, attr, new)


def restore_reference() -> None:
    """Undo every rebinding made by the replace_*_b200() calls of this process (tests; A/B runs)."""
    while _UNDO:
        mod, attr, old = _UNDO.pop()
        if old is None:
            if hasattr(mod, attr):
                delattr(mod, attr)
        else:
            setattr(mod, attr, old)
    if getattr(sys.modules.get("MultiScaleDeformableAttention"), "_b200_dropin", False):
        del sys.modules["MultiScaleDeformableAttention"]


def _module(name: str):
    """The already-imported reference module ``name`` or a fresh import of it."""
    if name in sys.modules:
        return sys.modules[name]
    try:
        return importlib.import_module(name)
    except Exception as e:      # transformers / diffusers drift makes some parents unimportable: say which
        raise RuntimeError(f"cannot import reference module {name!r} ({type(e).__name__}: {e}); import the reference "
                           "package (or its leaf modules) before calling replace_*_b200()") from e


def _rebind(replacements: Dict[type, type]) -> int:
    """Replace every attribute of every loaded ``mm_interleaved.*`` module that IS one of the old classes."""
    n = 0
    for name, mod in list(sys.modules.items()):
        if mod is None or not (name == _REF or name.startswith(_REF + ".")):
            continue
        for attr, val in list(vars(mod).items()):
            new = replacements.get(val) if isinstance(val, type) else None
            if new is not None:
                _set(mod, attr, new)
                n += 1
    return n


def replace_msda_b200() -> None:
    """The native op: both ``ms_deform_attn_func.py`` twins do ``import MultiScaleDeformableAttention as MSDA`` inside a
    try/except (ops/functions/ms_deform_attn_func.py:18-21, encoders/vit_adapter/ops/functions/ms_deform_attn_func.py:19-22).
    Register this repo's drop-in module under that name and rebind ``MSDA`` in twins that were imported earlier."""
    from . import msda as _msda
    import types
    mod = sys.modules.get("MultiScaleDeformableAttention")
    if mod is None or getattr(mod, "ms_deform_attn_forward", None) is not _msda.ms_deform_attn_forward:
        mod = types.ModuleType("MultiScaleDeformableAttention")
        mod.ms_deform_attn_forward = _msda.ms_deform_attn_forward
        mod.ms_deform_attn_backward = _msda.ms_deform_attn_backward
        mod._b200_dropin = True
        mod.__doc__ = "H100 drop-in for the reference's compiled extension (libmmfs_b200.so behind ctypes)"
        sys.modules["MultiScaleDeformableAttention"] = mod
    for name in (f"{_REF}.models.utils.ops.functions.ms_deform_attn_func",
                 f"{_REF}.models.encoders.vit_adapter.ops.functions.ms_deform_attn_func"):
        if name in sys.modules:
            _set(sys.modules[name], "MSDA", mod)


def replace_mmfs_b200() -> None:
    """``MMFS`` (ops/modules/mmfs.py:25) -> this repo's fused-sampler module (same ctor args, state-dict keys, forward
    signature); also installs the native op."""
    from .mmfs import MMFS
    replace_msda_b200()
    ref = _module(f"{_REF}.models.utils.ops.modules.mmfs")
    old = ref.MMFS
    if old is not MMFS:
        _set(ref, "MMFS", MMFS)
        _rebind({old: MMFS})


def replace_llama_b200() -> None:
    """The decoder building blocks of decoders/modeling_llama_mmfs.py (LlamaRMSNorm :53, LlamaMLP :175, LlamaAttention
    :192, LlamaMMFSAttention :311, LlamaDecoderLayer :370): parameter names are identical, so the reference's
    ``LlamaModel`` / ``LlamaForCausalLM`` construct and load checkpoints unchanged and run the H100 layer."""
    from . import llama_mmfs as b
    replace_mmfs_b200()
    ref = _module(f"{_REF}.models.decoders.modeling_llama_mmfs")
    repl = {}
    for name in ("LlamaRMSNorm", "LlamaMLP", "LlamaAttention", "LlamaMMFSAttention", "LlamaDecoderLayer"):
        old, new = getattr(ref, name), getattr(b, name)
        if old is not new:
            _set(ref, name, new)
            repl[old] = new
    if repl:
        _rebind(repl)


def replace_visual_b200() -> None:
    """``VisualTokenizer`` (encoders/visual_tokenizer.py:11), ``MMFSNet`` / ``MMFSBlock`` (decoders/sd_mmfs.py:44,154) and
    ``PerceiverResampler`` (decoders/perceiver.py) -> this repo's modules.  Modules of the reference that cannot be
    imported in this environment (diffusers / xformers / timm missing) are skipped: there is nothing to rebind in them."""
    from .sd_mmfs import MMFSBlock, MMFSNet
    from .visual_tokenizer import PerceiverResampler, VisualTokenizer
    replace_mmfs_b200()
    repl = {}
    for modname, names in ((f"{_REF}.models.decoders.sd_mmfs", {"MMFSNet": MMFSNet, "MMFSBlock": MMFSBlock}),
                           (f"{_REF}.models.encoders.visual_tokenizer", {"VisualTokenizer": VisualTokenizer}),
                           (f"{_REF}.models.decoders.perceiver", {"PerceiverResampler": PerceiverResampler})):
        try:
            ref = _module(modname)
        except RuntimeError:
            continue
        for name, new in names.items():
            old = getattr(ref, name, None)
            if old is not None and old is not new:
                _set(ref, name, new)
                repl[old] = new
    if repl:
        _rebind(repl)


def replace_all_b200() -> None:
    """Everything above, in dependency order."""
    replace_msda_b200()
    replace_mmfs_b200()
    replace_llama_b200()
    replace_visual_b200()
