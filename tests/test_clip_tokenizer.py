"""The package's CLIP tokenizer against token rows produced by the reference's own tokenizer
(tests/golden/clip_tokens.npz, written by tests/golden/make_clip_tokens_golden.py).  The BPE vocabulary is a
data file of a CoDA checkout, not of this package; tests/golden/clip_bpe_merges_48894.txt.gz holds the part of
CLIP's bpe_simple_vocab_16e6.txt.gz the tokenizer reads (the header line and the first 49152 - 256 - 2 merges)."""
import os
from pathlib import Path

import numpy as np
import pytest
import torch

from coda_neurips2023_b200.clip import tokenizer

GOLDEN = Path(__file__).parent / "golden" / "clip_tokens.npz"
CANDIDATES = [os.environ.get("CODA_CLIP_BPE", ""), str(Path(__file__).parent / "golden" / "clip_bpe_merges_48894.txt.gz")]


def _vocab():
    for c in CANDIDATES:
        if c and os.path.isfile(c):
            return c
    return None


def test_missing_vocabulary_is_a_file_not_found_error(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("CODA_CLIP_BPE", raising=False)
    with pytest.raises(FileNotFoundError):
        tokenizer.find_vocab()


@pytest.mark.skipif(_vocab() is None, reason="no CoDA checkout (BPE vocabulary file) reachable")
def test_tokenize_matches_reference_tokenizer_rows():
    g = np.load(GOLDEN)
    prompts = [str(p) for p in g["prompts"]]
    rows = tokenizer.tokenize(prompts, vocab_path=_vocab())
    assert rows.dtype == torch.int32 and tuple(rows.shape) == g["tokens"].shape
    assert np.array_equal(rows.numpy(), g["tokens"])
    assert len(tokenizer.ByteBPE(_vocab()).ids) == int(g["vocab_size"])


@pytest.mark.skipif(_vocab() is None, reason="no CoDA checkout (BPE vocabulary file) reachable")
def test_truncation_and_overflow():
    long = "chair " * 100
    with pytest.raises(RuntimeError):
        tokenizer.tokenize(long, vocab_path=_vocab())
    row = tokenizer.tokenize(long, truncate=True, vocab_path=_vocab())[0]
    assert row[0].item() == 49406 and row[-1].item() == 49407
