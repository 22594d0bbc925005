"""CPU suite for the play-JSON parser through its host twin (rz_ingest_json_host, the same csrc/rz_json_parse.cuh the
device parser runs): the reference trainer's arrays for the reference's own files, float32(float64(text)) bit for bit
on a corpus built to reach every conversion path, any JSON whitespace, the malformed inputs it refuses with a byte
offset, and the ``opt`` worker reading JSON with ``b200.train_from_json``."""
import decimal
import json
import logging
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ingest as oi
from reversi_zero_b200.worker import ingest as I
from reversi_zero_b200.worker import optimize as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden_optimize as G  # noqa: E402
from test_optimize_host import Clock, StandInTrainer, host_tensors, make_config  # noqa: E402

REF_CASES = ("tau1", "tau_rule", "one_hot")


def f32_bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def expected_f32(tokens):
    """what the reference trainer feeds the model: np.float32 of json.load's float64"""
    with np.errstate(over="ignore"):   # 1e400 and the doubles above float32's range become inf, as in numpy's cast
        return np.array([np.float32(json.loads(t)) for t in tokens], np.float32)


# ---- the generated corpus -----------------------------------------------------------------------------------------
def _double_of_bits(b):
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def corpus(seed=20261016):
    """>= 100 k number tokens: random doubles over the whole exponent range in repr form, subnormals and the smallest
    normals, 17-digit and > 19-digit decimals, doubles on a float32 rounding midpoint, integers and long decimals on or
    next to a double midpoint (the inputs Eisel-Lemire cannot decide), and the special tokens."""
    rng = random.Random(seed)
    toks = []
    while len(toks) < 40000:  # random bit patterns: every exponent, both signs
        d = _double_of_bits(rng.getrandbits(64))
        if d == d and abs(d) != float("inf"):
            toks.append(repr(d))
    for _ in range(8000):  # subnormals
        toks.append(repr(_double_of_bits(rng.getrandbits(52) >> rng.randrange(52))))
    toks += ["5e-324", "2.2250738585072011e-308", "2.2250738585072014e-308", "2.225073858507201e-308", "4.9406564584124654e-324",
             "2.4703282292062327e-324", "2.4703282292062328e-324", "1.7976931348623157e308", "1.7976931348623158e308",
             "1.7976931348623159e308", "3.4028235677973366e38", "3.4028235677973362e38", "1.401298464324817e-45", "7e-46",
             "7.006492321624086e-46", "7.006492321624085e-46"]
    for _ in range(12000):  # 17-digit decimals in fixed and exponent form
        m = rng.randrange(10 ** 16, 10 ** 17)
        e = rng.randrange(-340, 300)
        toks.append(f"{m // 10 ** 16}.{m % 10 ** 16:016d}e{e}" if rng.random() < 0.5 else f"0.{m}")
    for _ in range(8000):  # more than 19 significant digits
        nd = rng.randrange(20, 60)
        digits = str(rng.randrange(10 ** (nd - 1), 10 ** nd))
        k = rng.randrange(0, nd)
        toks.append(f"{digits[:k] or '0'}.{digits[k:]}e{rng.randrange(-330, 300)}")
    for _ in range(12000):  # doubles exactly on a float32 rounding midpoint: ties to even after the double rounding
        f = np.float32(rng.uniform(-1e30, 1e30) * 10.0 ** rng.randrange(-30, 8))
        if not np.isfinite(f):
            continue
        g = np.nextafter(f, np.float32(np.inf), dtype=np.float32)
        mid = (float(f) + float(g)) / 2
        toks.append(repr(mid))
    for _ in range(8000):  # integers on a double midpoint: 2^53 + odd, 2^54 + 2 (mod 4), ...
        sh = rng.randrange(0, 10)
        base = 1 << (53 + sh)
        v = base + (2 * rng.randrange(0, base >> (sh + 1)) + 1) * (1 << sh)
        if v < 10 ** 19:
            toks.append(str(v))
    toks += ["9007199254740993", "9007199254740992", "9007199254740994", "18014398509481986", "9223372036854775807",
             "9223372036854775808", "18446744073709551615", "18446744073709551616", "123456789012345678901234567890"]
    decimal.getcontext().prec = 800
    for _ in range(8000):  # decimals exactly on, and just either side of, a double midpoint
        d = abs(_double_of_bits(rng.getrandbits(64)))
        if not (0 < d < 1e300):
            continue
        nxt = np.nextafter(d, np.inf)
        mid = (decimal.Decimal(d) + decimal.Decimal(float(nxt))) / 2
        eps = decimal.Decimal(10) ** (mid.adjusted() - 40)
        for x in (mid, mid + eps, mid - eps):
            toks.append(format(x, "e").replace("E", "e").replace("e+", "e"))
    for _ in range(6000):  # short decimals in the fast path, as repr writes visit fractions
        toks.append(repr(rng.randrange(1, 800) / rng.randrange(1, 800)))
    toks += ["-0.0", "0.0", "0", "-0", "0e999", "1e400", "-1e400", "1e-400", "-1e-400", "NaN", "Infinity", "-Infinity",
             "1E5", "1e+5", "1.5E-5", "2.5e-05", "1e22", "1e23", "1.7976931348623157e308", "123456789012345678", "0.1", "-0.1"]
    return toks


def corpus_text(tokens, seed=7):
    """the tokens as records of 64 policies + z, random bitboards (0 and 2^64 - 1 included)"""
    rng = random.Random(seed)
    toks = list(tokens) + ["0"] * (-len(tokens) % 65)
    recs, boards = [], []
    for i in range(0, len(toks), 65):
        own, enemy = rng.getrandbits(64), rng.getrandbits(64)
        if i == 0:
            own, enemy = 0, 2 ** 64 - 1
        boards.append((own, enemy))
        recs.append(f"[[{own}, {enemy}], [{', '.join(toks[i:i + 64])}], {toks[i + 64]}]")
    return ("[" + ", ".join(recs) + "]").encode(), toks, boards


@pytest.fixture(scope="module")
def tokens():
    return corpus()


def planes_of(boards):
    b = np.array(boards, np.uint64)
    bits = (b[:, :, None] >> np.arange(64, dtype=np.uint64)) & np.uint64(1)
    return bits.astype(np.uint8).reshape(-1, 2, 8, 8)


def test_corpus_matches_python_float_then_float32(tokens):
    assert len(tokens) >= 100_000
    text, toks, boards = corpus_text(tokens)
    states, policy, z = I.parse_play_json_host(text)
    exp = expected_f32(toks).reshape(-1, 65)
    assert np.array_equal(f32_bits(policy), f32_bits(exp[:, :64]))
    assert np.array_equal(f32_bits(z), f32_bits(exp[:, 64]))
    assert np.array_equal(states, planes_of(boards))


@pytest.mark.parametrize("name", REF_CASES)
def test_reference_files_give_the_reference_trainers_arrays(golden_dir, name):
    g = np.load(os.path.join(golden_dir, "play_json_ref.npz"))
    states, policy, z = I.parse_play_json_host(g[name + "_text"].tobytes())
    ref_states = np.unpackbits(g[name + "_states_packed"], axis=1, bitorder="little").reshape(-1, 2, 8, 8)
    assert np.array_equal(states, ref_states)
    assert np.array_equal(f32_bits(policy), f32_bits(g[name + "_policy"].astype(np.float32)))
    assert np.array_equal(f32_bits(z), f32_bits(g[name + "_z"].astype(np.float32)))


def test_any_json_whitespace_gives_the_same_arrays(golden_dir):
    g = np.load(os.path.join(golden_dir, "play_json_ref.npz"))
    text = g["one_hot_text"].tobytes()
    recs = json.loads(text)
    base = I.parse_play_json_host(text)
    for variant in (json.dumps(recs, indent=1), json.dumps(recs, separators=(",", ":")), json.dumps(recs, indent="\t"),
                    "\r\n " + json.dumps(recs).replace(", ", " ,\n") + " \n"):
        got = I.parse_play_json_host(variant.encode())
        for a, b in zip(got, base):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_engine_json_equals_its_rows_twin(tmp_path):
    """this engine's own play_*.json and its play_*.rzrows twin give the same arrays (the rows through the oracle)"""
    path = G.write_play_files(str(tmp_path), "c")
    got = I.read_play_json_host(path)
    rows, tau1, ctt = I.read_play_rows(I.rows_path_of(path))
    ref = oi.rows_to_training_arrays(rows["own"], rows["enemy"], rows["n_visit"], rows["z"], tau1, ctt)
    for a, b in zip(got, ref):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.ascontiguousarray(b, a.dtype).view(np.uint8))


def test_empty_array_and_single_record():
    for text in (b"[]", b" [ ] \n", b"\t[\n]"):
        s, p, z = I.parse_play_json_host(text)
        assert s.shape == (0, 2, 8, 8) and p.shape == (0, 64) and z.shape == (0,)
    one = b"[[[1, 9223372036854775808], [" + b", ".join([b"0.015625"] * 64) + b"], -1]]"
    s, p, z = I.parse_play_json_host(one)
    assert s.shape == (1, 2, 8, 8) and s[0, 0].reshape(-1)[0] == 1 and s[0, 1].reshape(-1)[63] == 1 and s.sum() == 2
    assert (p == np.float32(0.015625)).all() and z[0] == -1


def _offset(text):
    with pytest.raises(I.PlayJsonError) as e:
        I.parse_play_json_host(text)
    assert "malformed play JSON at byte" in str(e.value)
    return e.value.offset


def small_text():
    recs = json.loads(np.load(os.path.join(ROOT, "tests", "golden", "play_json_ref.npz"))["tau1_text"].tobytes())[:2]
    return json.dumps(recs).encode()


def test_every_truncation_is_refused_with_an_offset():
    text = small_text()
    for k in range(len(text)):
        off = _offset(text[:k])
        assert 0 <= off <= k, k


def test_malformed_records_are_refused_at_the_first_bad_byte():
    rec = "[[1, 2], [" + ", ".join(["0.5"] * 64) + "], 1]"
    good = "[" + rec + ", " + rec + "]"
    I.parse_play_json_host(good.encode())
    cases = {
        "trailing garbage": (good + "x", len(good)),
        "trailing array": (good + "[]", len(good)),
        "trailing comma": (good[:-1] + ",]", len(good) - 1),
        "63 policies": ("[[[1, 2], [" + ", ".join(["0.5"] * 63) + "], 1]]", None),
        "65 policies": ("[[[1, 2], [" + ", ".join(["0.5"] * 65) + "], 1]]", None),
        "three bitboards": ("[[[1, 2, 3], [" + ", ".join(["0.5"] * 64) + "], 1]]", len("[[[1, 2")),
        "no z": ("[[[1, 2], [" + ", ".join(["0.5"] * 64) + "]]]", None),
        "string policy": (good.replace("0.5", '"0.5"', 1), good.index("0.5")),
        "string anywhere": (good.replace("1]", '1, "x"]', 1), None),
        "bitboard 2^64": (good.replace("[[1, 2]", "[[18446744073709551616, 2]", 1), 3),
        "negative bitboard": (good.replace("[[1, 2]", "[[-1, 2]", 1), 3),
        "fractional bitboard": (good.replace("[[1, 2]", "[[1.0, 2]", 1), 3),
        "leading zero": (good.replace("0.5", "00.5", 1), good.index("0.5")),
        "bare exponent": (good.replace("0.5", "1e", 1), good.index("0.5")),
        "plus sign": (good.replace("0.5", "+1", 1), good.index("0.5")),
        "-NaN": (good.replace("0.5", "-NaN", 1), good.index("0.5")),
        "object": ('{"a": 1}', 0),
        "not an array": ("1", 0),
        "empty": ("", 0),
        "two arrays": ("[] []", 3),
    }
    for name, (text, at) in cases.items():
        off = _offset(text.encode())
        assert 0 <= off <= len(text), name
        if at is not None:
            assert off == at, (name, off, at)


def test_pow10_table_is_what_the_generator_writes():
    assert subprocess.call([sys.executable, os.path.join(ROOT, "tools", "gen_pow10_table.py"), "--check"]) == 0


# ---- the opt worker ------------------------------------------------------------------------------------------------
def json_host_tensors(path):
    return tuple(torch.from_numpy(a) for a in I.read_play_json_host(path))


def json_worker(cfg, clock=None):
    cfg.b200.train_from_json = True
    clock = clock or Clock()
    return O.OptimizeWorker(cfg, trainer=StandInTrainer(), to_tensors=host_tensors, read_json=json_host_tensors,
                            sleep=clock.sleep, clock=clock)


def write_json_only(play_dir, key):
    path = G.write_play_files(play_dir, key)
    os.remove(I.rows_path_of(path))
    return path


def test_opt_worker_loads_unloads_and_deletes_json_files(tmp_path):
    cfg = make_config(tmp_path, delete_self_play_after_number_of_training=2)
    play_dir = cfg.resource.play_data_dir
    w = json_worker(cfg)
    a, b = write_json_only(play_dir, "a"), write_json_only(play_dir, "b")
    w.load_play_data()
    assert w.loaded_filenames == {a, b} and w.dataset_size == 480 + 480
    states, policy, z = w.dataset
    ref = [json_host_tensors(p) for p in (a, b)]
    assert torch.equal(z, torch.cat([r[2] for r in ref])) and torch.equal(states, torch.cat([r[0] for r in ref]))
    os.remove(a)
    w.load_play_data()
    assert w.loaded_filenames == {b} and w.dataset_size == 480
    w.count_up_training_count_and_delete_self_play_data_files()
    w.count_up_training_count_and_delete_self_play_data_files()
    assert not os.path.exists(b)
    w.load_play_data()
    assert w.loaded_filenames == set() and w.dataset is None


def test_opt_worker_retries_a_half_written_json_file(tmp_path, caplog):
    cfg = make_config(tmp_path)
    w = json_worker(cfg)
    path = write_json_only(cfg.resource.play_data_dir, "b")
    full = open(path, "rb").read()
    with open(path, "wb") as f:
        f.write(full[: len(full) // 2])                 # the reference's self-play writes in place
    with caplog.at_level(logging.WARNING, logger=O.__name__):
        w.load_play_data()
    assert w.loaded_filenames == set() and w.dataset_size == 0
    assert any("malformed play JSON" in r.getMessage() for r in caplog.records)
    with open(path, "wb") as f:
        f.write(full)
    w.load_play_data()
    assert w.loaded_filenames == {path} and w.dataset_size == 480


def test_opt_worker_with_json_ignores_rows_twins(tmp_path):
    cfg = make_config(tmp_path)
    w = json_worker(cfg)
    path = G.write_play_files(cfg.resource.play_data_dir, "a")
    with open(I.rows_path_of(path), "wb") as f:
        f.write(b"not a row file")
    w.load_play_data()
    assert w.loaded_filenames == {path} and w.dataset_size == 480
    assert O.OptimizeWorker(make_config(tmp_path / "x")).train_from_json is False   # the default reads the rows twins
