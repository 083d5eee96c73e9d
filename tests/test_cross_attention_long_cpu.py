"""CPU: the C-ABI argument contract of the long-memory cross-attention hook.  Every refusal happens before the library
touches the device, so the calls below pass placeholder addresses that must never be dereferenced."""
import ctypes

import pytest

from b200mdm import _lib as L

FAKE = ctypes.c_void_p(0x1000)   # never dereferenced: each call below is refused by the argument check


def _call(q=FAKE, kv=FAKE, mask=FAKE, out=FAKE, n=2, S=60, n_tokens=100, ld_kv=1024):
    lib = L.load()
    return lib.b200mdm_test_cross_attention(q, kv, mask, out, n, S, n_tokens, ld_kv, None)


@pytest.mark.parametrize("n_tokens", [0, -1, 513, 1 << 20])
def test_token_count_out_of_range(n_tokens):
    """A memory holds 1..512 tokens (DistilBERT's position limit): anything else is EINVAL."""
    assert _call(n_tokens=n_tokens) == L.EINVAL


@pytest.mark.parametrize("which", ["q", "kv", "mask", "out"])
def test_null_pointer(which):
    assert _call(**{which: None}) == L.EINVAL
    assert _call(**{which: None}, n_tokens=512) == L.EINVAL


@pytest.mark.parametrize("kw", [dict(n=0), dict(S=0), dict(ld_kv=1023), dict(ld_kv=1028)])
def test_bad_shape_long_memory(kw):
    assert _call(n_tokens=300, **kw) == L.EINVAL
