"""Text segmentation for long-form synthesis (``python -m tacotron_b200.test --long-form``).

A prompt line is split into chunks the model can say in one decoder run: at most CHUNK_CHARS characters each, counted
after the vocabulary filter of ``data_input.load_prompts`` (that is the count its 140-character limit applies to).
Break points, best first: a sentence end (``.``, ``!`` or ``?`` followed by whitespace or the end of the line), a
clause break (``,``, ``;`` or ``:`` followed by whitespace, or `` - ``), a space, and a hard cut only inside a single word longer than the budget.
Packing is greedy: each chunk takes the most text that fits and ends at the best-ranked break inside the budget.

A line that fits in one chunk is passed on unchanged, so its ids and ``text_length`` (the raw line length, newline
included) are those of the plain path.  A chunk cut out of a longer line is passed on as ``chunk + "\\n"``, so its
``text_length`` is ``len(chunk) + 1``: what it would have as a stdin line of its own.

Each chunk records the kind of break that ended it; that kind sets the pause before the next chunk (PAUSE_S).
CHUNK_CHARS and the pauses are choices, not measurements: no trained checkpoint was available to measure a speaking
rate.  A chunk whose speech runs to the last decoder frame is split again by the driver at the break nearest its middle
(``resplit``), so a budget that is too large costs synthesis rounds, not speech.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

CHUNK_CHARS = 100
SENTENCE, CLAUSE, SPACE, CUT = "sentence", "clause", "space", "cut"
PAUSE_S = {SENTENCE: 0.25, CLAUSE: 0.1, SPACE: 0.02, CUT: 0.02}
_RANK = {SENTENCE: 0, CLAUSE: 1, SPACE: 2}


@dataclass
class Chunk:
    """prompt: the line given to load_prompts; text: the chunk's text (stripped); brk: the kind of break that ends it;
    line: index of the stdin line it comes from"""
    prompt: str
    text: str
    brk: str
    line: int


def breaks(s):
    """break points of s, in order: (end, next, kind) -- the chunk before it is s[:end], the text after it starts at
    s[next:] (leading whitespace skipped by the caller)"""
    out = []
    n = len(s)
    for p in range(1, n + 1):
        c = s[p - 1]
        at_gap = p == n or s[p].isspace()
        if c in ".!?" and at_gap:
            out.append((p, p, SENTENCE))
        elif c in ",;:" and at_gap:
            out.append((p, p, CLAUSE))
        elif p < n and c.isspace() and s[p - 1:p + 2] == " - ":
            out.append((p - 1, p + 2, CLAUSE))
        elif p < n and s[p].isspace() and not c.isspace():
            out.append((p, p + 1, SPACE))
    return [b for b in out if 0 < b[0] and s[:b[0]].strip() and s[b[1]:].strip()]


def _count(s, vocab):
    return sum(1 for ch in s if ch in vocab)


def split_line(line, vocab, line_index=0, budget=None):
    """chunks of one stdin line (vocab: the characters of the model's vocabulary).  A line whose stripped text has at
    most `budget` vocabulary characters -- empty and whitespace-only lines included -- is one chunk, passed unchanged."""
    budget = CHUNK_CHARS if budget is None else budget
    s = line.strip()
    if _count(s, vocab) <= budget:
        return [Chunk(line, s, SENTENCE, line_index)]
    chunks = []
    while s:
        if _count(s, vocab) <= budget:
            chunks.append(Chunk(s + "\n", s, SENTENCE, line_index))
            break
        cnt, lim = 0, len(s)                                   # lim: the longest prefix within the budget
        for i, ch in enumerate(s):
            if ch in vocab:
                if cnt == budget:
                    lim = i
                    break
                cnt += 1
        cand = [b for b in breaks(s) if b[0] <= lim]
        if cand:
            best = min(_RANK[k] for _, _, k in cand)
            end, nxt, kind = [b for b in cand if _RANK[b[2]] == best][-1]
        else:
            end = nxt = lim
            kind = CUT
        text = s[:end].strip()
        chunks.append(Chunk(text + "\n", text, kind, line_index))
        s = s[nxt:].strip()
    return chunks


def resplit(chunk):
    """the two halves of a chunk, split at its break nearest the middle of its text (the earlier one on a tie), or None
    when it has no break.  The first half ends with that break's kind, the second with the chunk's own."""
    bs = breaks(chunk.text)
    if not bs:
        return None
    mid = len(chunk.text) / 2
    end, nxt, kind = min(bs, key=lambda b: abs(b[0] - mid))
    a, b = chunk.text[:end].strip(), chunk.text[nxt:].strip()
    return Chunk(a + "\n", a, kind, chunk.line), Chunk(b + "\n", b, chunk.brk, chunk.line)


def pause_samples(kind, sr):
    return int(round(PAUSE_S[kind] * sr))


def layout(kept, kinds, sr):
    """destinations of one line's chunks in its joined waveform: kept[i] samples of chunk i, then the pause its break
    kind sets (none after the last).  Returns (dst starts, total length)."""
    dst, pos = [], 0
    for i, n in enumerate(kept):
        dst.append(pos)
        pos += n
        if i + 1 < len(kept):
            pos += pause_samples(kinds[i], sr)
    return dst, pos


def block_diagonal(blocks, dtype=None):
    """the block-diagonal stack of 2-D arrays (a line's chunk alignments: decoder steps x encoder columns)"""
    rows = sum(b.shape[0] for b in blocks)
    cols = sum(b.shape[1] for b in blocks)
    out = np.zeros((rows, cols), dtype=dtype or (blocks[0].dtype if blocks else np.float32))
    i = j = 0
    for b in blocks:
        out[i:i + b.shape[0], j:j + b.shape[1]] = b
        i += b.shape[0]
        j += b.shape[1]
    return out
