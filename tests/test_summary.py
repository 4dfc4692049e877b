"""Summaries without a GPU: TF's default histogram table and EncodeToProto as restated in tests/summary_oracle.py, the
torch-CPU mirror of taco_histogram (tests/mirror_kernels_summary.py) against the oracle on the float32 neighbours of every
limit and the other edge values, the kernel source of csrc/summary.cu under the host emulation, and the event file, tag,
WAV and PNG encoders of tacotron_b200/summary.py (read back by tensorboard where it is importable)."""
import ctypes as C
import math
import os
import struct
import sys
import zlib

import numpy as np
import pytest
import torch

from tacotron_b200 import summary as S
from tests import mirror_kernels_summary as MKS
from tests import summary_oracle as SO
from tests.emulator import emu  # noqa: F401  (the emulated library, built once per process)

NLIM = 1551
FLT_MAX = float(np.finfo(np.float32).max)


def edge_values():
    """float32: the nearest value to every nonzero finite limit and its two neighbours, +-0, denormals, +-FLT_MAX, values
    below 1e-12, NaN and +-Inf"""
    lim = np.array(SO.default_limits())
    mids = lim[1:-1][lim[1:-1] != 0.0]
    f = mids.astype(np.float32)
    special = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, FLT_MAX, -FLT_MAX, 1e-13, -5e-13, 9.9e-13, 1.0, -1.0,
                        np.nan, np.inf, -np.inf, np.nan], dtype=np.float32)
    return np.concatenate([f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf)), special])


def oracle_result(x):
    """the oracle's histogram of the finite values of x in the kernel's result layout (sums via fsum)"""
    h = SO.Histogram()
    vals = [float(v) for v in np.asarray(x, dtype=np.float32).reshape(-1) if math.isfinite(v)]
    for v in vals:
        h.add(v)
    return h, len(np.asarray(x).reshape(-1)) - len(vals), math.fsum(vals), math.fsum(v * v for v in vals)


def check_result(res, x, sums_exact=True):
    """res (int64 [nlim + 5]) against the oracle: counts, min, max and the non-finite count exact, sums to the bound"""
    res = torch.as_tensor(res).cpu()
    h, nonfinite, fs, fsq = oracle_result(x)
    assert res[:NLIM].tolist() == [int(c) for c in h.buckets]
    assert int(res[NLIM]) == nonfinite
    mn, mx, s, sq = res[NLIM + 1:].view(torch.float64).tolist()
    assert mn == h.min and mx == h.max
    xf = np.asarray(x, dtype=np.float64).reshape(-1)
    xf = xf[np.isfinite(xf)]
    if sums_exact:
        assert s == fs and sq == fsq
    else:
        assert abs(s - fs) <= 1e-12 * float(np.abs(xf).sum()) and abs(sq - fsq) <= 1e-12 * float((xf * xf).sum())


# ---- the table and the encoding ----
def test_default_limits():
    lim = S.histogram_limits()
    assert lim.dtype == np.float64 and lim.shape == (NLIM,)
    assert lim.tolist() == SO.default_limits()
    assert lim[0] == -sys.float_info.max and lim[775] == 0.0 and lim[-1] == sys.float_info.max
    assert np.all(np.diff(lim) > 0) and np.array_equal(lim[:775], -lim[776:][::-1])
    pos = lim[776:1550]
    assert pos[0] == 1e-12 and pos[-1] < 1e20 <= pos[-1] * 1.1
    # repeated multiplication, not 1e-12 * 1.1**k
    assert sum(pos[k] != 1e-12 * 1.1 ** k for k in range(774)) == 731
    # no nonzero finite limit is a float32 value: only 0.0 can be met exactly
    mids = lim[1:-1][lim[1:-1] != 0.0]
    assert not np.any(mids.astype(np.float32).astype(np.float64) == mids)


def _proto_lists(buf):
    from tacotron_b200.tf_checkpoint import _parse_proto
    m = _parse_proto(buf)
    dbl = lambda f: struct.unpack("<d", struct.pack("<Q", m[f][0]))[0] if f in m else 0.0
    arr = lambda f: np.frombuffer(m[f][0], dtype="<f8").tolist()
    return dbl(1), dbl(2), dbl(3), dbl(4), dbl(5), arr(6), arr(7)


@pytest.mark.parametrize("case", ["empty", "one", "ends", "runs", "random"])
def test_encode_collapses_empty_runs(case):
    lim = S.histogram_limits()
    counts = np.zeros(NLIM)
    if case == "one":
        counts[776] = 3
    elif case == "ends":
        counts[0] = counts[-1] = 1
    elif case == "runs":
        counts[[5, 6, 9, 700, 1549]] = [1, 2, 1, 7, 4]
    elif case == "random":
        counts = np.random.RandomState(0).poisson(0.3, NLIM).astype(np.float64)
    h = SO.Histogram()
    h.buckets = counts.tolist()
    want_l, want_c = h.encode()
    mn, mx, num, s, sq, bl, bc = _proto_lists(S.histogram_proto(counts, lim, -1.5, 2.0, counts.sum(), 0.25, 3.0))
    assert (bl, bc) == (want_l, want_c)
    assert (mn, mx, num, s, sq) == (-1.5, 2.0, counts.sum(), 0.25, 3.0)
    if case == "empty":
        assert (bl, bc) == ([sys.float_info.max], [0.0])
    if case == "runs":
        assert bl[:4] == [lim[4], lim[5], lim[6], lim[8]] and bc[:4] == [0.0, 1.0, 2.0, 0.0]


def test_oracle_add_hand_cases():
    h = SO.Histogram()
    for v in (0.0, -0.0, 1e-13, -1e-13, 1.0):
        h.add(v)
    # +-0 go to the bucket after the 0.0 limit, |x| < 1e-12 next to it
    assert h.buckets[776] == 3 and h.buckets[775] == 1 and h.buckets[776 + 1 + 289] == 1
    assert h.min == -1e-13 and h.max == 1.0 and h.num == 5


# ---- the mirror against the oracle ----
def _mirror(x):
    res = torch.empty(NLIM + 5, dtype=torch.int64)
    MKS.histogram(res, torch.from_numpy(np.asarray(x, dtype=np.float32)), torch.from_numpy(S.histogram_limits()))
    return res


def test_mirror_equals_oracle_on_edge_values():
    x = edge_values()
    check_result(_mirror(x), x)


@pytest.mark.parametrize("n", [0, 1, 3, 4097])
def test_mirror_equals_oracle_random(n):
    rng = np.random.RandomState(n)
    x = (rng.randn(n) * np.exp(rng.randn(n) * 8)).astype(np.float32)
    check_result(_mirror(x), x)


def test_mirror_all_nonfinite():
    x = np.array([np.nan, np.inf], dtype=np.float32)
    res = _mirror(x)
    check_result(res, x)
    assert res[NLIM + 1:].view(torch.float64).tolist() == [sys.float_info.max, -sys.float_info.max, 0.0, 0.0]


# ---- the kernel source under the host emulation ----
def _emu_run(emu, x):
    """the entry point with host pointers, NaN-poisoned workspace and outputs -> res int64 [nlim + 5]"""
    xt = torch.from_numpy(np.asarray(x, dtype=np.float32).copy())
    lim = torch.from_numpy(S.histogram_limits())
    ws = torch.full((emu.taco_histogram_workspace_bytes() // 8,), float("nan"), dtype=torch.float64)
    res = torch.full((NLIM + 5,), float("nan"), dtype=torch.float64).view(torch.int64)
    p = lambda t, off=0: C.c_void_p(t.data_ptr() + off)
    rc = emu.taco_histogram(p(xt), xt.numel(), p(lim), NLIM, p(ws), p(res), p(res, 8 * (NLIM + 1)), p(res, 8 * NLIM), None)
    assert rc == 0, emu.taco_last_error().decode()
    return res


def test_histogram_kernel_under_emulation(emu):
    x = edge_values()
    res = _emu_run(emu, x)
    check_result(res, x, sums_exact=False)
    assert torch.equal(res[:NLIM + 3], _mirror(x)[:NLIM + 3])
    for n in (1, 3, 4097):                     # below one float4, the n % 4 tail, several chunks of a CTA
        rng = np.random.RandomState(n)
        xr = (rng.randn(n) * np.exp(rng.randn(n) * 8)).astype(np.float32)
        check_result(_emu_run(emu, xr), xr, sums_exact=False)


def test_histogram_kernel_argument_checks(emu):
    x = torch.zeros(8)
    lim = torch.from_numpy(S.histogram_limits())
    res = torch.zeros(NLIM + 5, dtype=torch.int64)
    ws = torch.zeros(emu.taco_histogram_workspace_bytes() // 8, dtype=torch.float64)
    p = lambda t, off=0: C.c_void_p(t.data_ptr() + off)
    assert emu.taco_histogram(p(x), 8, p(lim), 100, p(ws), p(res), p(res, 8 * 1552), p(res, 8 * 1551), None) != 0
    assert b"nlim" in emu.taco_last_error()
    assert emu.taco_histogram(p(x, 4), 7, p(lim), NLIM, p(ws), p(res), p(res, 8 * 1552), p(res, 8 * 1551), None) != 0
    assert b"aligned" in emu.taco_last_error()
    assert emu.taco_histogram(None, 8, p(lim), NLIM, p(ws), p(res), p(res, 8 * 1552), p(res, 8 * 1551), None) != 0


# ---- tags ----
def test_clean_tag_and_name_scopes():
    assert S.clean_tag("seq2seq loss") == "seq2seq_loss"
    assert S.clean_tag("output loss") == "output_loss" and S.clean_tag("loss") == "loss"
    assert S.clean_tag("//a/b c") == "a/b_c"
    assert S.clean_tag("Hello, world! it's 3.5-ish?") == "Hello__world__it_s_3.5-ish_"
    sc = S.NameScopes()
    assert [sc.unique(n) for n in ("abc", "abc", "xy", "xy", "abc", "abc")] == ["abc", "abc_1", "xy", "xy_1", "abc_2", "abc_3"]
    sc = S.NameScopes()
    assert [sc.unique(n) for n in ("a_1", "a", "a")] == ["a_1", "a", "a_2"]


# ---- encoders ----
def test_wav_encoding():
    from scipy.io import wavfile
    import io
    x = np.array([0.0, 0.5, -0.5, 1.0, -1.0, 1.5, -1.5, 1 / 65536, -1 / 65536, 3 / 65536, 0.99999, -0.99999], dtype=np.float32)
    want = np.array([0, 16384, -16384, 32767, -32768, 32767, -32768, 1, -1, 2, 32768 * 0.99999, -32768 * 0.99999], dtype=np.float64)
    want = np.clip(np.sign(want) * np.floor(np.abs(want) + 0.5), -32768, 32767).astype(np.int16)
    assert want[7] == 1 and want[8] == -1 and want[9] == 2              # roundf: halves away from zero
    sr, got = wavfile.read(io.BytesIO(S.wav_bytes(x, 16000)))
    assert sr == 16000 and got.dtype == np.int16 and np.array_equal(got, want)


def _read_png(buf):
    """a minimal PNG reader (8-bit RGBA, filter 0, as png_bytes writes) on zlib"""
    assert buf[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, hdr = 8, b"", None
    while pos < len(buf):
        n = struct.unpack(">I", buf[pos:pos + 4])[0]
        kind, data = buf[pos + 4:pos + 8], buf[pos + 8:pos + 8 + n]
        assert struct.unpack(">I", buf[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(kind + data) & 0xffffffff
        if kind == b"IHDR":
            hdr = struct.unpack(">IIBBBBB", data)
        elif kind == b"IDAT":
            idat += data
        pos += 12 + n
    w, h, depth, ctype = hdr[:4]
    assert depth == 8 and ctype == 6
    raw = np.frombuffer(zlib.decompress(idat), dtype=np.uint8).reshape(h, 1 + 4 * w)
    assert not raw[:, 0].any()
    return raw[:, 1:].reshape(h, w, 4)


def test_hot_colormap():
    lut = S.HOT_LUT
    assert lut.shape == (256, 4) and (lut[:, 3] == 255).all()
    assert tuple(lut[0]) == (10, 0, 0, 255) and tuple(lut[-1]) == (255, 255, 255, 255)
    for c in range(3):
        assert np.all(np.diff(lut[:, c].astype(int)) >= 0)
    # red saturates at x = .365079 (i ~ 93), green starts there and saturates at .746032 (i ~ 190), blue after that
    assert lut[94, 0] == 255 and lut[92, 0] < 255 and lut[93, 1] == 0 and lut[191, 1] == 255 and lut[190, 2] == 0


def test_attention_image():
    rng = np.random.RandomState(0)
    a = rng.rand(37, 23).astype(np.float32)
    img = S.attention_rgba(a)
    f = 13                                                            # ceil(480 / 37)
    assert img.shape == (37 * f, 23 * f, 4)
    v = (a - a.min()) / (a.max() - a.min())
    want = S.HOT_LUT[np.clip((v * 256).astype(int), 0, 255)]
    assert np.array_equal(img[::f, ::f], want) and np.array_equal(img[f - 1::f, f - 1::f], want)
    assert tuple(img[0, 0]) == tuple(want[0, 0]) and tuple(want[np.unravel_index(a.argmax(), a.shape)]) == (255, 255, 255, 255)
    png = S.png_bytes(img)
    assert np.array_equal(_read_png(png), img)
    try:
        from PIL import Image
    except ImportError:
        return
    import io
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(png)).convert("RGBA")), img)
    assert S.attention_rgba(np.zeros((600, 4), np.float32)).shape == (600, 4, 4)


# ---- the event file ----
def _events(logdir):
    """[(step, wall_time, file_version, {tag: Summary.Value})] read with tensorboard (CRCs checked)"""
    tb = pytest.importorskip("tensorboard.backend.event_processing.event_file_loader")
    files = [f for f in os.listdir(logdir) if f.startswith("events.out.tfevents.")]
    assert len(files) == 1
    out = []
    for e in tb.LegacyEventFileLoader(os.path.join(logdir, files[0])).Load():
        out.append((e.step, e.wall_time, e.file_version, [(v.tag, v) for v in e.summary.value]))
    return out


def test_event_file_round_trip(tmp_path):
    import socket
    w = S.EventWriter(str(tmp_path))
    name = os.path.basename(w.path)
    assert name.startswith("events.out.tfevents.") and name.endswith("." + socket.gethostname())
    assert len(name.split(".")[3]) == 10
    lim = S.histogram_limits()
    x = edge_values()
    res = _mirror(x).numpy()
    counts = res[:NLIM]
    mn, mx, s, sq = res[NLIM + 1:].view(np.float64)
    wave = np.sin(np.arange(800) / 7.0).astype(np.float32) * 1.2
    align = np.random.RandomState(1).rand(20, 9).astype(np.float32)
    w.add(7, [S.histo_value("post-process/output", S.histogram_proto(counts, lim, mn, mx, float(counts.sum()), s, sq)),
              S.scalar_value("loss", 1.25), S.scalar_value("zero", 0.0)])
    w.add(8, [S.audio_value("ideal_8/audio/0", wave, 16000), S.image_value("attention_8/image/0", S.attention_rgba(align))])
    w.close()
    ev = _events(str(tmp_path))
    assert ev[0][2] == "brain.Event:2" and ev[0][0] == 0 and not ev[0][3] and ev[0][1] > 1e9
    (st1, _, _, v1), (st2, _, _, v2) = ev[1], ev[2]
    assert st1 == 7 and st2 == 8 and len(ev) == 3
    d1 = dict(v1)
    hp = d1["post-process/output"].histo
    h, _, _, _ = oracle_result(x)
    bl, bc = h.encode()
    assert list(hp.bucket_limit) == bl and list(hp.bucket) == bc
    assert (hp.min, hp.max, hp.num, hp.sum, hp.sum_squares) == (h.min, h.max, h.num, s, sq)
    assert d1["loss"].simple_value == 1.25 and d1["zero"].simple_value == 0.0
    d2 = dict(v2)
    au = d2["ideal_8/audio/0"].audio
    assert (au.sample_rate, au.num_channels, au.length_frames, au.content_type) == (16000.0, 1, 800, "audio/wav")
    assert au.encoded_audio_string == S.wav_bytes(wave, 16000)
    im = d2["attention_8/image/0"].image
    assert (im.height, im.width, im.colorspace) == (480, 216, 4)
    assert np.array_equal(_read_png(im.encoded_image_string), S.attention_rgba(align))


def test_event_record_framing(tmp_path):
    """the records by hand: length, masked CRC-32C of the length, payload, masked CRC-32C of the payload"""
    from tacotron_b200.tf_checkpoint import crc32c, mask_crc
    w = S.EventWriter(str(tmp_path))
    w.add(3, [S.scalar_value("loss", 2.0)])
    w.close()
    buf = open(w.path, "rb").read()
    pos, n_rec = 0, 0
    while pos < len(buf):
        n = struct.unpack_from("<Q", buf, pos)[0]
        assert struct.unpack_from("<I", buf, pos + 8)[0] == mask_crc(crc32c(buf[pos:pos + 8]))
        data = buf[pos + 12:pos + 12 + n]
        assert struct.unpack_from("<I", buf, pos + 12 + n)[0] == mask_crc(crc32c(data))
        pos += 16 + n
        n_rec += 1
    assert pos == len(buf) and n_rec == 2


def test_histogram_values_skip_nonfinite():
    lim = S.histogram_limits()
    res = np.zeros((3, NLIM + 5), dtype=np.int64)
    res[:, NLIM + 1:] = np.array([0.0, 1.0, 2.0, 3.0]).view(np.int64)
    res[:, 780] = 2
    res[1, NLIM] = 1
    logs = []
    vals = S.histogram_values(res, lim, logs.append)
    assert logs == ["Nan in summary histogram for: decoder/seq2seq_output"] and len(vals) == 2
