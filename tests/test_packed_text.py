"""CPU tests of the host plumbing the packed text encoders share: the kept-range rows the readout averages, the
over-long sentence refusal, and the tokens-per-launch budget of the text extractors."""
import types

import numpy as np
import pytest
import torch

from mertools_b200.extract import albert_text as A
from mertools_b200.extract import text
from mertools_b200.extract.packed_text import kept_ranges

LENS = [1, 2, 3, 4, 17, 1, 40, 2]


@pytest.mark.parametrize("start", [0, 1, 2])
@pytest.mark.parametrize("end", [None, -1, -2])
def test_kept_ranges_are_the_packed_rows_of_each_slice(start, end):
    """Row s of the result is [begin, end) of sentence s's ids[start:end] in the packed buffer; a sentence with
    nothing left gets begin == end (a zero mean, which TextExtractor replaces by its zero vector)."""
    seg = kept_ranges(LENS, start, end)
    assert seg.dtype == np.int32 and seg.shape == (2, len(LENS))
    o = 0
    for s, n in enumerate(LENS):
        want = list(range(o, o + n))[start:end]
        begin, stop = int(seg[0, s]), int(seg[1, s])
        if want:
            assert list(range(begin, stop)) == want, (s, n, start, end)
        else:
            assert begin == stop, (s, n, start, end)
        o += n


def test_over_long_sentence_is_refused_with_value_error():
    """ALBERT refuses a sentence longer than its position table as the decoders do: a ValueError before any launch."""
    enc = A.AlbertTextEncoder.__new__(A.AlbertTextEncoder)
    enc.max_pos, enc.vocab_size = 4, 10
    with pytest.raises(ValueError, match="5 tokens exceeds max_position_embeddings 4"):
        enc.forward([[1, 2, 3], [1, 2, 3, 4, 5]])


# The budget each extractor used to compute in place, with its row length: LLaMA / DeBERTa / ALBERT
# max_position_embeddings, BLOOM / OPT / Falcon max_pos or 2048, GPT-2 n_positions, XLNet MAX_LEN.
@pytest.mark.parametrize("row_len", [512, 1024, 2048, 4096])
@pytest.mark.parametrize("bytes_per_token", [2560 * 4 * 11 + 10240 * 4, 4096 * 20 + 11008 * 10, 312 * 44])
@pytest.mark.parametrize("free", [0, 1 << 20, 3 << 30, 70 << 30])
def test_tokens_per_launch_matches_the_budget_expression(monkeypatch, row_len, bytes_per_token, free):
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device: (free, 80 << 30))
    enc = types.SimpleNamespace(device="cuda:0", bytes_per_token=bytes_per_token)
    got = text._tokens_per_launch(enc, row_len)
    assert got == int(min(16384, max(row_len, free // 2 // bytes_per_token)))
    assert isinstance(got, int) and min(row_len, 16384) <= got <= 16384
