"""Text ingest (sb_text_parse, SURVEY 8f rank 1): the parsing state machine against Python's float() - on the CPU through
the host test hook (identical code, text_parse.cuh), on the GPU through the product entry point, and end to end against
the oracle's load_data restatement."""
import gzip
import random

import numpy as np
import pytest

from oracle import shifu_oracle as so


def _f32(s):
    return np.float32(float(s))


FAST = ["0", "-0", "0.0", "1", "-1", "+1.5", "3.14159", "-2.718281828", "1e5", "1E-5", "-4.25e+3", "000123.4500", ".5", "5.",
        "0.000001234", "123456789012345", "9007199254740992", "1e22", "1e-22", "  7.5  ", "7.5\r",
        "0.1", "0.2", "16777217", "33554433.0", "1e0", "-0e5", "1234567.890123", "-0.000000000000001"]
SLOW = ["4.9406564584124654", "1.17549435e-38", "3.4028235e38", "0.30000000000000004", "12345678901234567890123", "1e23", "1e-23", "nan", "inf", "-inf", "1_000", "0x10", "", ".", "e5", "1e", "--1", "1 2",
        "9007199254740993", "1.7976931348623157e308", "123456789.123456789123456789"]


def _parse_cells(sb, cells, host_debug, **kw):
    text = ("|".join(["1"] + cells) + "\n").encode()
    col_map = [sb.capi.COL_TARGET] + list(range(len(cells)))
    return sb.capi.text_parse(text, col_map, len(cells), host_debug=host_debug, **kw)


def test_number_parser_fast_path_is_bit_exact_vs_python_float(sb):
    X, y, w, flags, _ = _parse_cells(sb, FAST, True)
    assert flags == []
    want = np.array([_f32(c) for c in FAST], np.float32)
    np.testing.assert_array_equal(X[0].view(np.uint32), want.view(np.uint32))
    assert y[0] == 1.0 and w[0] == 1.0


def test_number_parser_declines_what_it_cannot_do_exactly(sb):
    X, y, w, flags, text = _parse_cells(sb, SLOW, True)
    assert sorted(f[1] for f in flags) == list(range(len(SLOW)))          # every slow cell flagged, none guessed
    for row, slot, off, ln in flags:
        assert text[off:off + ln].decode() == SLOW[slot]                 # and the flag points at exactly that cell


def test_number_parser_random_decimals_bit_exact(sb):
    rnd = random.Random(5)
    cells = []
    for _ in range(4000):
        kind = rnd.randrange(4)
        if kind == 0:
            cells.append(repr(rnd.gauss(0, 1)))                          # 17 significant digits -> mostly slow path
        elif kind == 1:
            cells.append("%.6f" % rnd.gauss(0, 3))
        elif kind == 2:
            cells.append("%.8e" % rnd.uniform(-1e6, 1e6))
        else:
            cells.append(str(rnd.randrange(-10 ** 9, 10 ** 9)))
    X, y, w, flags, text = _parse_cells(sb, cells, True)
    flagged = {f[1] for f in flags}
    assert 0 < len(flagged) < len(cells)
    for j, c in enumerate(cells):
        if j not in flagged:
            assert X[0, j].view(np.uint32) == _f32(c).view(np.uint32), c


def _make_text(n_rows, F, seed, with_weight):
    rnd = np.random.RandomState(seed)
    lines = []
    for i in range(n_rows):
        feats = ["%.6f" % v for v in rnd.randn(F)]
        if i % 7 == 3:
            feats[1] = repr(float(rnd.randn()))                          # long decimal: slow path through the flag list
        cols = [str(int(rnd.rand() < 0.3))] + feats + ["extra%d" % i]
        if with_weight:
            cols.append("%.3f" % (rnd.rand() * 4 - 1))                   # some negative weights -> 1.0
        lines.append("|".join(cols))
    return ("\n".join(lines) + "\n").encode()


def test_host_hook_full_lines_match_oracle_load_data(sb, tmp_path):
    F = 9
    raw = _make_text(301, F, 2, True)
    p = str(tmp_path / "part.gz")
    with gzip.open(p, "wb") as f:
        f.write(raw)
    want = so.load_data([p], list(range(1, F + 1)), 0, F + 2, 0.0, rng=random.Random(1))
    col_map = [sb.capi.COL_TARGET] + list(range(F)) + [sb.capi.COL_SKIP, sb.capi.COL_WEIGHT]
    X, y, w, flags, text = sb.capi.text_parse(raw, col_map, F, host_debug=True)
    for row, slot, off, ln in flags:
        assert slot == 1
        X[row, slot] = float(text[off:off + ln])
    np.testing.assert_array_equal(X, np.asarray(want["train_data"], np.float32))
    np.testing.assert_array_equal(y, np.asarray(want["train_target"], np.float32).ravel())
    np.testing.assert_array_equal(w, np.asarray(want["train_data_sample_weight"], np.float32).ravel())
    assert (w == 1.0).sum() > 40                                          # the negative ones were clamped


def test_short_line_is_reported_not_guessed(sb):
    col_map = [sb.capi.COL_TARGET, 0, 1, 2]
    X, y, w, flags, _ = sb.capi.text_parse(b"1|0.5|0.25|2\n0|0.5\n", col_map, 3, host_debug=True)
    assert [(f[0], f[1]) for f in flags] == [(1, -100)]


@pytest.mark.gpu
def test_gpu_parser_equals_host_hook_and_python(sb):
    F = 37
    raw = _make_text(5000, F, 3, True) + ("|".join(["1"] + (FAST + SLOW)[:F] + ["x", "2.5"]) + "\n").encode()
    col_map = [sb.capi.COL_TARGET] + list(range(F)) + [sb.capi.COL_SKIP, sb.capi.COL_WEIGHT]
    Xh, yh, wh, fh, _ = sb.capi.text_parse(raw, col_map, F, host_debug=True)
    Xg, yg, wg, fg, _ = sb.capi.text_parse(raw, col_map, F)
    np.testing.assert_array_equal(Xg.view(np.uint32), Xh.view(np.uint32))
    np.testing.assert_array_equal(yg, yh); np.testing.assert_array_equal(wg, wh)
    assert sorted(fg) == sorted(fh)
    assert Xg.shape == (5001, F) and yg[-1] == 1.0 and wg[-1] == 2.5


@pytest.mark.gpu
def test_load_data_gpu_equals_load_data(sb, tmp_path):
    from shifu_tensorflow_b200 import trainer as tr
    F = 12
    files = []
    for k in range(2):
        p = str(tmp_path / ("part-%d.gz" % k))
        with gzip.open(p, "wb") as f:
            f.write(_make_text(400 + 31 * k, F, 10 + k, True))
        files.append(p)
    a = tr.load_data(",".join(files), list(range(1, F + 1)), 0, F + 2, 0.25, rng=random.Random(9))
    b = tr.load_data_gpu(",".join(files), list(range(1, F + 1)), 0, F + 2, 0.25, rng=random.Random(9))
    for k in ("train_data", "valid_data", "train_target", "valid_target", "train_data_sample_weight", "valid_data_sample_weight"):
        assert isinstance(b[k], sb.capi.DeviceArray)                  # the parsed set stays on the device ...
        got = b[k].numpy()
        np.testing.assert_array_equal(np.asarray(a[k], np.float32).reshape(got.shape), got, err_msg=k)   # ... with the same bits
    assert a["feature_count"] == b["feature_count"] == F


@pytest.mark.gpu
def test_device_resident_set_feeds_the_trainer_without_a_host_copy(sb):
    """sb_text_parse_device -> device gather (split) -> sb_trainer_load_dataset / eval_loss on DEVICE pointers: same losses as
    the host-array path"""
    from oracle import shifu_oracle as so
    F = 12
    text = _make_text(600, F, 3, True)
    col_map = [sb.capi.COL_TARGET] + list(range(F)) + [sb.capi.COL_SKIP, sb.capi.COL_WEIGHT]
    Xh, yh, wh, fl_h, _ = sb.capi.text_parse(text, col_map, F)
    Xd, yd, wd, fl_d, _, kms = sb.capi.text_parse_device(text, col_map, F)
    assert sorted(fl_h) == sorted(fl_d) and kms > 0          # (the flag list is appended with an atomic counter: order varies)
    np.testing.assert_array_equal(Xd.numpy(), Xh); np.testing.assert_array_equal(yd.numpy(), yh); np.testing.assert_array_equal(wd.numpy(), wh)
    rows = np.arange(0, 600, 3)
    np.testing.assert_array_equal(Xd.take_rows(rows).numpy(), Xh[rows])
    desc = sb.make_desc(F, [16, 8], [so.ACT_RELU, so.ACT_TANH], optimizer=so.OPT_SGD, learning_rate=0.1, max_batch=128, precision=sb.PREC_BF16)
    with sb.Trainer(desc) as a, sb.Trainer(desc) as b:
        for t in (a, b):
            t.init_xavier(5)
        a.load_dataset(Xh, yh, wh)
        b.load_dataset(Xd, yd, wd)
        for k in range(4):
            assert a.step_resident(k * 128, 128) == b.step_resident(k * 128, 128)
        # (the evaluation loss is summed with fp32 atomics across CTAs: equal up to the summation order)
        assert abs(a.eval_loss(Xh, yh, wh) - b.eval_loss(Xd, yd, wd)) <= 1e-6


# ---------------------------------------------------------------------------------------------------- col_map validation
# parse_line stores a feature cell at X[row * n_feat + role] without a check of its own, so every map is checked before
# anything is parsed: on the host hook, sb_text_parse and sb_text_parse_device alike (a CPU-only machine reaches the check
# before the device lookup).
T, W, S = -2, -3, -1
BAD_MAPS = {
    "feature_past_n_feat": ([T, 0, 1, 3], 3, "outside"),
    "feature_at_n_feat": ([T, 0, 1, 2, 3], 3, "outside"),
    "below_weight": ([T, 0, 1, -4], 2, "outside"),
    "repeated_feature": ([T, 0, 1, 1, 2], 3, "mapped twice"),
    "fewer_features": ([T, 0, 1, S], 3, "maps 2 of n_feat=3"),
    "map_shorter_than_n_feat": ([T, 0], 3, "fewer than n_feat"),
    "no_target": ([0, 1, 2, W], 3, "0 target columns"),
    "two_targets": ([T, 0, 1, 2, T], 3, "2 target columns"),
    "two_weights": ([T, 0, 1, 2, W, W], 3, "2 weight columns"),
}


def _parse_raw(sb, text, col_map, n_feat, entry):
    import ctypes as C
    cm = (C.c_int32 * len(col_map))(*col_map)
    X, y, w = (np.zeros(64, np.float32) for _ in range(3))
    flags = (sb.capi.CellFlag * 4)()
    n_rows, n_flags = C.c_int64(0), C.c_int64(0)
    lib, p = sb.capi.lib(), sb.capi._ptr
    if entry == "device":
        dX, dy, dw = (sb.capi._f32p() for _ in range(3))
        return lib.sb_text_parse_device(text, len(text), b"|", cm, len(col_map), n_feat, C.byref(dX), C.byref(dy), C.byref(dw),
                                        C.byref(n_rows), flags, 4, C.byref(n_flags), 0, None)
    args = [text, len(text), b"|", cm, len(col_map), n_feat, p(X), p(y), p(w), 4, C.byref(n_rows), flags, 4, C.byref(n_flags)]
    return lib.sb_debug_text_parse_host(*args) if entry == "host" else lib.sb_text_parse(*args, 0)


@pytest.mark.parametrize("entry", ["host", "parse", "device"])
@pytest.mark.parametrize("case", sorted(BAD_MAPS))
def test_col_map_is_rejected_before_any_parsing(sb, case, entry):
    col_map, n_feat, msg = BAD_MAPS[case]
    text = b"1|0.5|0.25|2|3|4|5\n"
    assert _parse_raw(sb, text, col_map, n_feat, entry) == sb.capi.SB_ERR_INVALID
    assert msg in sb.capi.lib().sb_last_error().decode()


def test_valid_col_maps_still_parse(sb):
    for col_map, n_feat in (([T, 2, S, 0, 1, W], 3), ([1, 0, T], 2), ([T, 0], 1)):
        X, y, w, flags, _ = sb.capi.text_parse(b"1|0.5|0.25|2|3|4\n", col_map, n_feat, host_debug=True)
        assert X.shape == (1, n_feat)


# ---------------------------------------------------------------------------------------------------- GPU chunk edges
CHUNK = 16384


def _python_parse(text, col_map, n_feat):
    """float() per cell: X, y, w and the rows whose feature / target cells are missing"""
    lines = text.split(b"\n")
    if lines and lines[-1] == b"":
        lines = lines[:-1]
    X = np.zeros((len(lines), n_feat), np.float32)
    y = np.zeros(len(lines), np.float32)
    w = np.ones(len(lines), np.float32)
    bad = []
    for r, ln in enumerate(lines):
        cells = ln.split(b"|")
        seen, tgt = 0, False
        for c, role in enumerate(col_map):
            if c >= len(cells) or role == COL_SKIP or cells[c] == b"":
                continue
            if role >= 0:
                X[r, role] = float(cells[c]); seen += 1
            elif role == COL_TARGET:
                y[r] = float(cells[c]); tgt = True
            else:
                v = float(cells[c])
                w[r] = 1.0 if v < 0.0 else v
        if seen != n_feat or not tgt:
            bad.append(r)
    return X, y, w, bad


COL_SKIP, COL_TARGET, COL_WEIGHT = -1, -2, -3


def _resolve(X, y, w, flags, text):
    X, y, w = X.copy(), y.copy(), w.copy()
    bad = sorted(row for row, slot, _, _ in flags if slot == -100)
    for row, slot, off, ln in flags:
        if row in bad:
            continue
        v = float(text[off:off + ln])
        if slot >= 0:
            X[row, slot] = v
        elif slot == COL_TARGET:
            y[row] = v
        else:
            w[row] = 1.0 if v < 0.0 else v
    return X, y, w, bad


def _check_gpu_text(sb, text, col_map, n_feat, want_bad=()):
    """GPU parse == host hook (bits and sorted flags) == float() per cell, flags resolved; -> the appended text"""
    Xg, yg, wg, fg, tx = sb.capi.text_parse(text, col_map, n_feat)
    Xh, yh, wh, fh, _ = sb.capi.text_parse(text, col_map, n_feat, host_debug=True)
    np.testing.assert_array_equal(Xg.view(np.uint32), Xh.view(np.uint32))
    np.testing.assert_array_equal(yg.view(np.uint32), yh.view(np.uint32))
    np.testing.assert_array_equal(wg.view(np.uint32), wh.view(np.uint32))
    assert sorted(fg) == sorted(fh)
    X, y, w, bad = _resolve(Xg, yg, wg, fg, tx)
    Xp, yp, wp, badp = _python_parse(tx, col_map, n_feat)
    assert bad == badp == sorted(want_bad)
    ok = np.setdiff1d(np.arange(len(y)), bad)
    np.testing.assert_array_equal(X[ok].view(np.uint32), Xp[ok].view(np.uint32))
    np.testing.assert_array_equal(y[ok].view(np.uint32), yp[ok].view(np.uint32))
    np.testing.assert_array_equal(w.view(np.uint32), wp.view(np.uint32))
    return tx


def _check_load_data_gpu(sb, tmp_path, text, feats, target, weight):
    from shifu_tensorflow_b200 import trainer as tr
    p = str(tmp_path / "part.gz")
    with gzip.open(p, "wb") as f:
        f.write(text)
    a = so.load_data([p], feats, target, weight, 0.0, rng=random.Random(1))
    b = tr.load_data_gpu(p, feats, target, weight, 0.0, rng=random.Random(1))
    for k in ("train_data", "train_target", "train_data_sample_weight"):
        got = b[k].numpy()
        np.testing.assert_array_equal(np.asarray(a[k], np.float32).reshape(got.shape).view(np.uint32), got.view(np.uint32),
                                      err_msg=k)


def _edge_text(rnd, targets, F=3):
    """lines 'y|f0..f{F-1}|pad|w' whose newlines land exactly at the absolute byte offsets `targets` (the skipped pad
    column takes up the difference)"""
    out = b""
    for pos in targets:
        head = ("%d|" % rnd.randrange(2) + "|".join("%.6f" % rnd.gauss(0, 1) for _ in range(F)) + "|").encode()
        tail = ("|%.3f" % rnd.uniform(-1, 3)).encode()
        pad = pos - len(out) - len(head) - len(tail)
        assert pad >= 0, (pos, len(out))
        out += head + b"x" * pad + tail + b"\n"
        assert len(out) - 1 == pos
    return out


EDGE_MAP = [COL_TARGET, 0, 1, 2, COL_SKIP, COL_WEIGHT]


@pytest.mark.gpu
def test_gpu_cfg2_width_lines_cross_every_chunk(sb, tmp_path):
    """2000 features at %.6f: ~18 KB lines, longer than a 16 KB chunk, so some chunks hold no newline at all"""
    F, rows = 2000, 24
    rng = np.random.RandomState(7)
    lines = []
    for i in range(rows):
        cells = ["%d" % (i & 1)] + ["%.6f" % v for v in rng.randn(F) * 10] + ["%.2f" % (rng.rand() * 4 - 1)]
        lines.append("|".join(cells))
    text = ("\n".join(lines) + "\n").encode()
    assert min(len(l) for l in lines) > CHUNK
    col_map = [COL_TARGET] + list(range(F)) + [COL_WEIGHT]
    _check_gpu_text(sb, text, col_map, F)
    _check_load_data_gpu(sb, tmp_path, text, list(range(1, F + 1)), 0, F + 1)


@pytest.mark.gpu
def test_gpu_newlines_on_chunk_and_window_edges(sb, tmp_path):
    rnd = random.Random(11)
    targets = [CHUNK - 1, 2 * CHUNK, 3 * CHUNK + 1, 4 * CHUNK + 64 * 5 - 1, 4 * CHUNK + 64 * 6, 4 * CHUNK + 64 * 7 + 1,
               5 * CHUNK + 63, 6 * CHUNK - 1]
    text = _edge_text(rnd, targets)
    assert len(text) == 6 * CHUNK                              # ends exactly on a chunk boundary
    _check_gpu_text(sb, text, EDGE_MAP, 3)
    _check_load_data_gpu(sb, tmp_path, text, [1, 2, 3], 0, 5)


@pytest.mark.gpu
def test_gpu_text_of_exact_chunk_multiple(sb):
    rnd = random.Random(12)
    for n in (1, 2):
        text = _edge_text(rnd, [CHUNK * k // 4 - 1 for k in range(1, 4 * n + 1)])
        assert len(text) == n * CHUNK
        _check_gpu_text(sb, text, EDGE_MAP, 3)


@pytest.mark.gpu
def test_gpu_four_byte_lines(sb):
    """'d|d\\n': 16 lines per 64-byte thread window, 4096 per chunk"""
    rnd = random.Random(13)
    text = b"".join(b"%d|%d\n" % (rnd.randrange(2), rnd.randrange(10)) for _ in range(3 * 4096 + 5))
    assert len(text) == 4 * (3 * 4096 + 5)
    _check_gpu_text(sb, text, [COL_TARGET, 0], 1)


@pytest.mark.gpu
def test_gpu_crlf_last_line_without_newline_and_weights(sb, tmp_path):
    """CRLF endings; a last line without '\\n'; a weight column with zeros, -0, negatives (-> 1) and missing (-> 1)"""
    rnd = random.Random(14)
    wcells = ["0", "-0", "-2.5", "0.75", "3", None]
    lines = []
    for i in range(3000):
        cells = ["%d" % (i & 1)] + ["%.5f" % rnd.gauss(0, 1) for _ in range(4)]
        wc = wcells[i % len(wcells)]
        if wc is not None:
            cells.append(wc)
        lines.append("|".join(cells))
    col_map = [COL_TARGET, 0, 1, 2, 3, COL_WEIGHT]
    text = "\r\n".join(lines).encode()                       # CRLF, and no newline after the last line
    tx = _check_gpu_text(sb, text, col_map, 4)
    assert tx == text + b"\n"
    _, _, w, _, _ = sb.capi.text_parse(text, col_map, 4)
    want = np.array([[0.0, -0.0, 1.0, 0.75, 3.0, 1.0][i % 6] for i in range(3000)], np.float32)
    np.testing.assert_array_equal(w.view(np.uint32), want.view(np.uint32))
    _check_load_data_gpu(sb, tmp_path, text, [1, 2, 3, 4], 0, 5)


@pytest.mark.gpu
def test_gpu_empty_line_is_flagged_at_its_row(sb, tmp_path):
    from shifu_tensorflow_b200 import trainer as tr
    rnd = random.Random(15)
    lines = ["%d|%.4f|%.4f" % (i & 1, rnd.gauss(0, 1), rnd.gauss(0, 1)) for i in range(900)]
    lines[517] = ""
    text = ("\n".join(lines) + "\n").encode()
    _check_gpu_text(sb, text, [COL_TARGET, 0, 1], 2, want_bad=[517])
    X, y, w, flags, _ = sb.capi.text_parse(text, [COL_TARGET, 0, 1], 2)
    assert sorted((f[0], f[1]) for f in flags) == [(517, -100), (517, COL_TARGET)]   # the empty target cell, and the line
    for r in (516, 518):                                      # the neighbours are intact
        c = lines[r].split("|")
        assert (y[r], X[r, 0], X[r, 1]) == (np.float32(float(c[0])), np.float32(float(c[1])), np.float32(float(c[2])))
    p = str(tmp_path / "part.gz")
    with gzip.open(p, "wb") as f:
        f.write(text)
    with pytest.raises(ValueError, match="line 517 "):
        tr.load_data_gpu(p, [1, 2], 0, -1, 0.0, rng=random.Random(1))
