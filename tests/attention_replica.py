"""Host replica of the attention-probability dropout layout of vtx_attn_fwd / _bwd at every shape they take.

The kernels hash element ((b * heads + h) * Qs + i) * Ks + j for query i and key j, with Qs = Tq rounded up to a
multiple of 32 and Ks = Tk rounded up to a multiple of 64; the LSE row of (b, h, i) is (b * heads + h) * Qs + i.  For
Tq <= 32 and Tk <= 64 that is ((b * heads + h) * 32 + i) * 64 + j, the layout tests/dropout_replica.py's attn_index
states for those shapes.  The hash itself is tests/dropout_replica.py's keep_scale.
"""
import numpy as np

from tests import dropout_replica as R


def attn_rows(Tq, Tk):
    """(Qs, Ks): the query and key extents of the layout, Tq rounded up to 32 and Tk rounded up to 64."""
    return -(-Tq // 32) * 32, -(-Tk // 64) * 64


def attn_index(B, heads, Tq, Tk):
    """[B, heads, Tq, Tk] element indices of the attention-probability site."""
    Qs, Ks = attn_rows(Tq, Tk)
    b = np.arange(B, dtype=np.uint64)[:, None, None, None]
    h = np.arange(heads, dtype=np.uint64)[None, :, None, None]
    i = np.arange(Tq, dtype=np.uint64)[None, None, :, None]
    j = np.arange(Tk, dtype=np.uint64)[None, None, None, :]
    return ((b * np.uint64(heads) + h) * np.uint64(Qs) + i) * np.uint64(Ks) + j


def attn_scale(seed, site, B, heads, Tq, Tk, p):
    """[B, heads, Tq, Tk] scale of the attention probabilities (query i, key j)."""
    return R.keep_scale(seed, site, attn_index(B, heads, Tq, Tk), p)
