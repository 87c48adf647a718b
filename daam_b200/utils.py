"""Small helpers kept from the reference's API surface (``daam/utils.py``): seeding, device/autocast
shims and the word -> token-row lookup (``compute_token_merge_indices``, utils.py:73-91). spaCy and plotting helpers
are out of scope (SURVEY.md section 2, rows 4)."""
from __future__ import annotations

import os
import random
import sys
from pathlib import Path
from typing import List, Optional, Tuple, TypeVar

import numpy as np
import torch

__all__ = ['set_seed', 'compute_token_merge_indices', 'cache_dir', 'auto_device', 'auto_autocast', 'context_rows',
           't5_rows', 'T5Pieces']

T = TypeVar('T')


def auto_device(obj: T = torch.device('cpu')) -> T:
    """``torch.device`` -> the best device; anything else -> moved to CUDA when there is one (utils.py:22-29)."""
    has_cuda = torch.cuda.is_available()
    if isinstance(obj, torch.device):
        return torch.device('cuda' if has_cuda else 'cpu')
    return obj.to('cuda') if has_cuda else obj


def auto_autocast(*args, **kwargs):
    """``torch.autocast('cuda', ...)`` that switches itself off without a GPU (utils.py:32-36)."""
    if not torch.cuda.is_available():
        kwargs['enabled'] = False
    return torch.autocast('cuda', *args, **kwargs)


def set_seed(seed: int) -> torch.Generator:
    """Seeds python, numpy and torch (all devices) and returns a seeded generator on the auto device (utils.py:46-55)."""
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)
    gen = torch.Generator(device=auto_device())
    gen.manual_seed(seed)
    return gen


def cache_dir() -> Path:
    """Per-user cache folder, honouring XDG_CACHE_HOME on Linux (utils.py:58-70)."""
    if sys.platform == 'darwin':
        return Path(os.path.expanduser('~'), 'Library/Caches/daam')
    if os.name == 'posix':
        return Path(os.environ.get('XDG_CACHE_HOME', os.path.expanduser('~/.cache')), 'daam')
    return Path(os.environ.get('LOCALAPPDATA') or os.path.expanduser('~\\AppData\\Local'), 'daam')


CHUNK_TOKENS = 77          # one CLIP window: BOS, 75 prompt tokens, EOS
CHUNK_PROMPT_TOKENS = 75


def context_rows(n_tokens: int, tokens: int = CHUNK_TOKENS) -> List[int]:
    """The context rows a heat map of a ``n_tokens``-token prompt reads from a ``tokens``-row context (77, 154 or 231:
    one to three CLIP chunks), in the order of its rows: the SOS row 0, the row of every prompt token, the EOS row.

    A context of ``c`` chunks is ``c x 77`` rows, chunk ``i`` being BOS, prompt tokens ``75i .. 75i + 74``, EOS, padding
    (the layout of compel and of the long-prompt-weighting pipelines). Prompt token ``j`` sits at row
    ``77 (j // 75) + 1 + j % 75`` and the EOS row follows the last token. ``n_tokens`` is capped at ``75 c``; for one
    chunk the rows are ``[0, n_tokens + 2)``, the reference's truncation to 77."""
    chunks = tokens // CHUNK_TOKENS
    if tokens not in (CHUNK_TOKENS, 2 * CHUNK_TOKENS, 3 * CHUNK_TOKENS):
        raise ValueError(f'a context of {tokens} tokens is not 1-3 chunks of {CHUNK_TOKENS}')
    n = max(0, min(int(n_tokens), CHUNK_PROMPT_TOKENS * chunks))
    rows = [CHUNK_TOKENS * (j // CHUNK_PROMPT_TOKENS) + 1 + j % CHUNK_PROMPT_TOKENS for j in range(n)]
    return [0] + rows + [rows[-1] + 1 if rows else 1]


SENTENCEPIECE_MARK = '\u2581'   # '▁': the word-start marker of sentencepiece pieces (T5)


def t5_rows(n_pieces: int, tokens: int, clip_tokens: int = CHUNK_TOKENS) -> int:
    """How many T5 pieces of a prompt a joint-attention map has rows for: the ``tokens``-row context is ``clip_tokens``
    CLIP rows and then the T5 rows, and the pieces are capped so that the T5 EOS row after them still fits."""
    return max(0, min(int(n_pieces), tokens - clip_tokens - 1))


class T5Pieces:
    """The tokenizer of a T5 heat map: ``tokenizer.tokenize`` cut to the ``n`` pieces the map has rows for, so that
    the word lookup never names a row past the map."""

    def __init__(self, tokenizer, n: int):
        self.tokenizer, self.n = tokenizer, n

    def tokenize(self, text: str) -> List[str]:
        return list(self.tokenizer.tokenize(text))[:self.n]


def _pieces(tokenizer, text: str) -> List[str]:
    return [tok.replace('</w>', '') for tok in tokenizer.tokenize(text)]


def compute_token_merge_indices(tokenizer, prompt: str, word: str, word_idx: Optional[int] = None,
                                offset_idx: int = 0) -> Tuple[List[int], Optional[int]]:
    """Rows of the global heat map that belong to ``word``: every occurrence of the word's token pieces in the
    lower-cased prompt, shifted by one for the SOS row. With ``word_idx`` the lookup is skipped and ``[word_idx + 1]``
    returned. Raises ``ValueError('Search word ... not found in prompt!')`` like utils.py:86-87.

    A sentencepiece tokenizer (T5: a word's first piece starts with ``▁``) keeps the case, since its vocabulary does:
    the word's pieces are searched in the pieces of the prompt as written."""
    if word_idx is not None:
        return [word_idx + 1], word_idx
    needle = _pieces(tokenizer, word)
    if needle and needle[0].startswith(SENTENCEPIECE_MARK):
        haystack = _pieces(tokenizer, prompt)
    else:
        haystack = _pieces(tokenizer, prompt.lower())
        word = word.lower()
        needle = _pieces(tokenizer, word)
    n = len(needle)
    rows: List[int] = []
    for start in range(len(haystack)):
        if haystack[start:start + n] == needle:
            rows.extend(start + offset_idx + 1 + j for j in range(n))
    if not rows:
        raise ValueError(f'Search word {word} not found in prompt!')
    return rows, word_idx
