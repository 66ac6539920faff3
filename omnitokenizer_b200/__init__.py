"""omnitokenizer_b200: H100 (sm_90a) implementation of OmniTokenizer_VQGAN.encode/decode.

Drop-in for the reference's ``from OmniTokenizer import OmniTokenizer_VQGAN``
(/root/reference/OmniTokenizer/__init__.py:7); see INTEGRATION.md.
"""
from .vqgan import OmniTokenizer_VQGAN, VQGAN, canonical_args  # noqa: F401
from . import consumers, dist  # noqa: F401

__all__ = ["OmniTokenizer_VQGAN", "VQGAN", "canonical_args", "consumers", "dist"]
