"""mm_interleaved_b200 -- H100-native (sm_90a) kernels for MM-Interleaved's interleaved
image-text forward hot path, behind the reference's own operator / module API.

Import name ``mm_interleaved_b200`` (via the shim ``mm_interleaved_b200.py`` at the repo
root); the directory carries the project's hyphenated name.
"""
from . import _lib  # noqa: F401
from .msda import (  # noqa: F401
    ms_deform_attn_backward,
    ms_deform_attn_forward,
    ms_deform_attn_forward_host,
    msda_index_stream,
)
from .functions import MSDeformAttnFunction  # noqa: F401
from .sampler import mmfs_sampler_forward, mmfs_sampler_locw  # noqa: F401
from .mmfs import MMFS  # noqa: F401
from . import ops  # noqa: F401
from . import autograd_ops  # noqa: F401
from .sd_mmfs import MMFSBlock, MMFSNet, PreparedSDFeatures  # noqa: F401
from . import unet_sd, visual_tokenizer  # noqa: F401
from .llama_mmfs import (LlamaAttention, LlamaDecoderLayer, LlamaMLP, LlamaMMFSAttention, LlamaMMFSConfig,  # noqa: F401
                         LlamaModel, LlamaRMSNorm)

from .mm_interleaved import ImageDecoder, InterleavedForward, MMInterleaved, StableDiffusion, TextDecoder  # noqa: F401
from .patch import (replace_all_b200, replace_llama_b200, replace_mmfs_b200, replace_msda_b200,  # noqa: F401
                    replace_visual_b200)
from ._cache import clear_activation_caches  # noqa: F401

__version__ = "0.2.0"
