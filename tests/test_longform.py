"""Long-form synthesis on the CPU: the text splitter (tacotron_b200/longform.py), the float64 statement of
taco_speech_bounds against trim_oracle's end of speech, the float64 statement of taco_join_segments and the sample range
each chunk keeps, the host checks of the segments, the layout of a joined line and its block-diagonal alignment."""
import numpy as np
import pytest

from tacotron_b200 import audio, data_input, kernels, longform as LF
from tests import longform_oracle as LO
from tests import trim_oracle as TO

VOCAB = set("abcdefghijklmnopqrstuvwxyz'")            # no space, punctuation or digits: they are filtered out


def _filtered(s):
    return "".join(ch for ch in s if ch in VOCAB)


def _ok(chunks, line, budget):
    for c in chunks:
        assert sum(ch in VOCAB for ch in c.text) <= budget, c
        assert c.prompt == c.text + "\n" and c.text == c.text.strip() and c.text
    assert "".join(_filtered(c.text) for c in chunks) == _filtered(line)


def test_sentence_end_beats_clause_and_space():
    line = "one two. three, four five six seven\n"
    ch = LF.split_line(line, VOCAB, budget=20)
    assert [c.text for c in ch] == ["one two.", "three,", "four five six seven"]      # 21 letters after the period
    assert [c.brk for c in ch] == [LF.SENTENCE, LF.CLAUSE, LF.SENTENCE]
    _ok(ch, line, 20)


def test_clause_beats_space_and_takes_the_furthest_of_its_rank():
    line = "one, two; three four five six seven eight\n"
    ch = LF.split_line(line, VOCAB, budget=20)
    assert ch[0].text == "one, two;" and ch[0].brk == LF.CLAUSE
    line = "alpha beta - gamma delta epsilon zeta eta\n"
    ch = LF.split_line(line, VOCAB, budget=20)
    assert ch[0].text == "alpha beta" and ch[0].brk == LF.CLAUSE and ch[1].text.startswith("gamma")
    ch = LF.split_line("aa bb cc dd ee ff gg hh ii jj kk\n", VOCAB, budget=9)
    assert [c.text for c in ch] == ["aa bb cc dd", "ee ff gg hh", "ii jj kk"] and ch[0].brk == LF.SPACE


def test_a_period_inside_a_word_is_not_a_sentence_end():
    ch = LF.split_line("see e.g.this and that then more words\n", VOCAB, budget=15)
    assert all(c.brk != LF.SENTENCE for c in ch[:-1])


def test_budget_counts_characters_after_the_vocabulary_filter():
    line = "ABC DEF GHI JKL MNO PQR STU VWX 123 456 789, abcdefghij\n"      # 56 characters, 10 in the vocabulary
    ch = LF.split_line(line, VOCAB, budget=10)
    assert len(ch) == 1 and ch[0].prompt is line
    ch = LF.split_line(line, VOCAB, budget=9)
    assert [c.text for c in ch] == [line[:44], "abcdefghi", "j"] and ch[0].brk == LF.CLAUSE
    _ok(ch, line, 9)


def test_a_line_that_fits_is_returned_unchanged():
    for line in ("  hello there, friend.  \n", "x" * 100 + "\n", "no newline"):
        ch = LF.split_line(line, VOCAB)
        assert len(ch) == 1 and ch[0].prompt is line and ch[0].text == line.strip()


def test_hard_cut_only_inside_an_over_long_word():
    word = "abcdefghijklmnopqrstuvwxyzabcd"
    line = f"hi {word} yo\n"
    ch = LF.split_line(line, VOCAB, budget=10)
    assert [c.text for c in ch] == ["hi", "abcdefghij", "klmnopqrst", "uvwxyzabcd", "yo"]
    assert [c.brk for c in ch] == [LF.SPACE, LF.CUT, LF.CUT, LF.SPACE, LF.SENTENCE]
    _ok(ch, line, 10)


@pytest.mark.parametrize("line", ["\n", "", "   \t \n", " \n"])
def test_empty_and_whitespace_lines_are_one_unchanged_chunk(line):
    ch = LF.split_line(line, VOCAB)
    assert len(ch) == 1 and ch[0].prompt is line and ch[0].text == ""
    assert LF.resplit(ch[0]) is None


def test_long_paragraph_property():
    rng = np.random.RandomState(0)
    words = ["".join(rng.choice(list("abcdefghij"), rng.randint(1, 9))) for _ in range(400)]
    punct = rng.choice(["", "", "", ",", ".", ";", "!", " -"], len(words))
    line = " ".join(w + p for w, p in zip(words, punct)) + "\n"
    for budget in (100, 37, 12):
        _ok(LF.split_line(line, VOCAB, budget=budget), line.replace(" - ", " "), budget)


def test_resplit_at_the_break_nearest_the_middle():
    c = LF.Chunk("one two three four five six\n", "one two three four five six", LF.CLAUSE, 3)
    a, b = LF.resplit(c)
    assert (a.text, b.text) == ("one two three", "four five six")
    assert (a.brk, b.brk, a.line, b.line) == (LF.SPACE, LF.CLAUSE, 3, 3)
    assert (a.prompt, b.prompt) == ("one two three\n", "four five six\n")
    c = LF.Chunk("", "aaaa bb, cccccccccc dddddddddd", LF.SENTENCE, 0)       # middle at 15: the space at 19 is nearer than ','
    a, b = LF.resplit(c)
    assert (a.text, a.brk) == ("aaaa bb, cccccccccc", LF.SPACE)
    assert LF.resplit(LF.Chunk("", "abcdefghijklmnop", LF.SPACE, 0)) is None
    assert LF.resplit(LF.Chunk("", "abc.", LF.SPACE, 0)) is None


def test_text_length_of_chunks():
    ivocab = {i: ch for i, ch in enumerate(sorted(VOCAB))}
    line = "first sentence here. second one is a bit longer, with a clause\n"
    ch = LF.split_line(line, VOCAB, budget=30)
    assert len(ch) > 1
    batch = next(data_input.load_prompts([c.prompt for c in ch], ivocab, device="cpu"))
    assert batch["text_length"].tolist() == [len(c.text) + 1 for c in ch]
    one = LF.split_line(" short line \n", VOCAB)
    plain = next(data_input.load_prompts([" short line \n"], ivocab, device="cpu"))
    got = next(data_input.load_prompts([one[0].prompt], ivocab, device="cpu"))
    assert got["text_length"].tolist() == plain["text_length"].tolist() == [13]
    assert got["text"].tolist() == plain["text"].tolist()


@pytest.mark.parametrize("r", [1, 2, 5])
def test_speech_bounds_oracle(r):
    T = {1: 24, 2: 16, 5: 8}[r]
    n = 4 * r * (T // 4)
    rng = np.random.RandomState(r)
    scale, shift = (rng.rand(1025 * r) * 2 + 1).astype(np.float32), (rng.randn(1025 * r) * 2 - 5).astype(np.float32)
    starts, ends = [0, 3, n // 2, 0, n - 2], [n // 2, n, n // 2 + 1, n, n - 1]
    for sc, sh in ((None, None), (scale, shift)):
        spec = LO.speech_span_like(len(ends), T, r, starts, ends, seed=r, scale=sc, shift=sh)
        assert TO.margin_db(spec, r, sc, sh) >= 0.5
        got = LO.speech_bounds(spec, r, sc, sh)
        assert got[:, 0].tolist() == starts and got[:, 1].tolist() == ends
        assert got[:, 2].tolist() == TO.speech_frames(spec, r, sc, sh).tolist()
        assert got[3].tolist() == [0, n, n]                                        # fully voiced
    spec = LO.speech_span_like(3, T, r, [2, 2, 2], [n // 2] * 3, seed=1)
    spec[0, 1, 5] = np.nan
    spec[1, T - 1, 7] = np.inf
    got = LO.speech_bounds(spec, r)
    assert got[:2].tolist() == [[0, n, n]] * 2 and got[2, :2].tolist() == [2, n // 2]
    assert got[:, 2].tolist() == TO.speech_frames(spec, r).tolist()


def test_kept_sample_range():
    for f0, f1, frames in ((0, 5, 8), (1, 8, 8), (3, 40, 40), (7, 9, 16), (0, 360, 360)):
        a, b = audio.kept_samples(f0, f1, frames)
        assert (a, b) == LO.kept_samples(f0, f1, frames)
        assert 0 <= a < b <= audio.hop_length * (frames - 1)
    assert audio.kept_samples(3, 9, 16) == (600, 2700)
    assert audio.kept_samples(0, 16, 16) == (0, 4500)


def test_join_mirror():
    f = LO.fade(1000, 160)
    assert np.all(f > 0) and np.all(f <= 1) and np.array_equal(f, f[::-1])
    assert np.all(f[160:840] == 1.0) and np.all(np.diff(f[:161]) > 0)
    assert abs(f[0] / np.sin(np.pi * 0.5 / 320) ** 2 - 1) < 1e-12       # 1 - cos cancels to ~1e-13 in float64
    short = LO.fade(50, 160)                                       # shorter than two fades: the two ramps meet
    assert np.array_equal(short, short[::-1]) and short.max() < 0.1
    src = np.arange(1, 101, dtype=np.float32)
    out = np.full(120, -1.0)
    LO.join_segments(out, src, [[10, 0, 30], [50, 40, 50]], 4)
    assert np.all(out[30:40] == -1) and np.all(out[90:] == -1)
    np.testing.assert_array_equal(out[4:26], src[14:36])
    np.testing.assert_allclose(out[:4], src[10:14] * (0.5 - 0.5 * np.cos(np.pi * (np.arange(4) + 0.5) / 4)))


@pytest.mark.parametrize("seg", [[[-1, 0, 5]], [[0, -1, 5]], [[0, 0, -1]], [[96, 0, 5]], [[0, 46, 5]],
                                 [[0, 0, 10], [20, 9, 10]], [[0, 20, 10], [20, 0, 21]]])
def test_segment_checks(seg):
    with pytest.raises(ValueError):
        kernels.check_segments(np.array(seg), 100, 50)


def test_segment_checks_accept_touching_segments():
    kernels.check_segments(np.array([[0, 10, 10], [50, 0, 10], [90, 20, 10]]), 100, 30)


def test_line_layout_and_pauses():
    sr = 16000
    kinds = [LF.SENTENCE, LF.CLAUSE, LF.SPACE, LF.CUT]
    dst, total = LF.layout([1000, 2000, 300, 400], kinds, sr)
    assert dst == [0, 1000 + 4000, 1000 + 4000 + 2000 + 1600, 1000 + 4000 + 2000 + 1600 + 300 + 320]
    assert total == 1000 + 2000 + 300 + 400 + 4000 + 1600 + 320
    assert LF.layout([7], [LF.SENTENCE], sr) == ([0], 7)
    assert LF.pause_samples(LF.SENTENCE, 24000) == 6000


def test_block_diagonal_alignment():
    a = np.arange(6, dtype=np.float32).reshape(2, 3) + 1
    b = np.arange(4, dtype=np.float32).reshape(4, 1) + 10
    d = LF.block_diagonal([a, b])
    assert d.shape == (6, 4) and d.dtype == np.float32
    np.testing.assert_array_equal(d[:2, :3], a)
    np.testing.assert_array_equal(d[2:, 3:], b)
    assert not d[:2, 3:].any() and not d[2:, :3].any()
