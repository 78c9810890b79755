"""Branch-level GPU tests of the MATCH kernels, on every kernel variant of tests/test_match_gpu.KERNELS.

Final match lists are compared bit-exactly with the C port (oracle/match_oracle.c).  The tensor-core variants must also
report exactly the candidate and hard-row counts of the integer restatement (tests/match_restatement.py): a bound that is
too loose still gives correct matches but sends rows to the full scan, and only the counts show it."""
import ctypes
import os
import re

import numpy as np
import pytest

from bundler_sfm_b200 import bundle, keymatch, synth
from tests import match_restatement as R
from tests import match_scenes
from tests.test_match_gpu import KERNELS, kernel  # noqa: F401  (the kernel-variant fixture)

pytestmark = pytest.mark.gpu
GOLD_TIES = os.path.join(os.path.dirname(__file__), "golden", "match_ties_golden.npz")
RATIOS = [(0, 0.6), (0, 0.8), (0, 0.95), (0, 0.999), (1, 0.6), (1, 0.8), (1, 0.95), (1, 0.999), (1, 1.0)]
VERBOSE = re.compile(r"\[bsfm_match_run\] candidates (\d+), hard rows (\d+), matches (\d+)")
_restated = {}


@pytest.fixture
def verbose(monkeypatch):
    """the library prints the run's candidate and hard-row counts; it reads the variable on every run"""
    monkeypatch.setenv("BSFM_MATCH_VERBOSE", "1")


def match_pair(q, db, ratio, mode, capfd):
    """bsfm_match_pair_test -> (matches, (candidates, hard rows) of the run)"""
    lib = bundle.load_library()
    fn = lib.bsfm_match_pair_test
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    fn.restype = ctypes.c_int
    q, db = np.ascontiguousarray(q, np.uint8), np.ascontiguousarray(db, np.uint8)
    out = np.zeros((max(q.shape[0], 1), 2), np.int32)
    capfd.readouterr()
    n = fn(q.ctypes.data, q.shape[0], db.ctypes.data, db.shape[0], float(ratio), int(mode), out.ctypes.data, out.shape[0])
    assert n >= 0
    return out[:n].copy(), run_counts(capfd)


def run_counts(capfd):
    lines = VERBOSE.findall(capfd.readouterr().err)
    assert lines, "no [bsfm_match_run] line"
    return int(lines[-1][0]), int(lines[-1][1])


def restated(key, q, db, ratio, mode, epilogue):
    k = (key, ratio, mode, epilogue)
    if k not in _restated:
        _restated[k] = R.restate(q, db, ratio, mode, epilogue)
    return _restated[k]


def check_counts(kernel, name, q, db, ratio, mode, got_counts, sizes=None):
    """tensor-core variants: (candidates, hard rows) equal the restatement's -> the restatement's counts"""
    if kernel == "dp4a":
        return None
    epi = R.library_epilogue(sizes or [q.shape[0], db.shape[0]], kernel)
    _, c = restated(name, q, db, ratio, mode, epi)
    assert got_counts == (c["candidates"], c["hard"]), (kernel, name, mode, ratio, epi, c)
    if epi == "exact" and not R.ties_pass(ratio, mode):
        assert got_counts[1] == 0
    return c


@pytest.fixture(scope="module")
def scenes():
    return match_scenes.all_scenes(seed=0)


def test_scenes_bit_exact_and_branch_counts(kernel, oracle, scenes, verbose, capfd):
    branches = dict.fromkeys(("verify_match", "verify_reject", "scan_match", "scan_reject"), 0)
    for name, q, db in scenes:
        for mode, ratio in RATIOS:
            got, counts = match_pair(q, db, ratio, mode, capfd)
            want = oracle.match_pair_port_test(q, db, ratio, mode)
            assert np.array_equal(got, want), (kernel, name, mode, ratio)
            c = check_counts(kernel, name, q, db, ratio, mode, counts)
            if c is not None:
                for k in branches:
                    branches[k] += c[k]
    if kernel in ("tc", "tc_quad", "tc_pair"):      # the suite reaches every branch of the bound epilogue
        assert all(v > 0 for v in branches.values()), branches


_sized = {}


def _sized_pair(nq, ndb, swap):
    k = (nq, ndb, swap)
    if k not in _sized:
        q, db = match_scenes.norm_spread(nq, ndb, seed=nq * 10007 + ndb)
        _sized[k] = (db, q) if swap else (q, db)
    return _sized[k]


@pytest.mark.parametrize("swap", [False, True], ids=["q_small", "q_large"])
@pytest.mark.parametrize("nq", [127, 128, 129])
@pytest.mark.parametrize("ndb", [63, 64, 65, 255, 256, 257, 7937, 8192, 8193])
def test_size_edges(kernel, oracle, verbose, capfd, nq, ndb, swap):
    """chunk (64 / 32 columns), tile (256 rows) and query-unit (128 rows) edges, and the norm staging buffer: 7937-8192 keys
    fill it, 8193 switch the tensor-core variants to the exact epilogue"""
    q, db = _sized_pair(nq, ndb, swap)
    for mode, ratio in ((0, 0.8), (1, 1.0)):
        got, counts = match_pair(q, db, ratio, mode, capfd)
        assert np.array_equal(got, oracle.match_pair_port_test(q, db, ratio, mode)), (kernel, mode, ratio)
        c = check_counts(kernel, ("sized", nq, ndb, swap), q, db, ratio, mode, counts)
        if c is not None and ndb == 8192 and not swap and kernel != "tc_exact":
            assert c["hard"] > 0 and R.library_epilogue([nq, ndb], kernel) == "bound"


def test_oversized_image_switches_run_to_exact_epilogue(kernel, oracle, verbose, capfd):
    sizes = [700, 8193, 900]
    imgs = synth.sift_like_descriptors(len(sizes), sizes, seed=31)
    pairs, counts, matches = keymatch.key_match_full(imgs, -1, 0.6)
    got = run_counts(capfd)
    want_txt, want_counts = oracle.match_all_pairs_port(imgs, -1, 0.6, 1)
    assert [want_counts[i, j] for j, i in pairs] == counts.tolist()
    assert keymatch.format_match_table(pairs, counts, matches, 1) == want_txt
    if kernel != "dp4a":
        assert R.library_epilogue(sizes, kernel) == "exact"
        tot = [0, 0]
        for j, i in pairs:
            _, c = restated(("run3", j, i), imgs[j], imgs[i], 0.6, 0, "exact")
            tot[0] += c["candidates"]; tot[1] += c["hard"]
        assert got == tuple(tot) and got[1] == 0


def test_window_radii_and_window_shards(kernel, oracle):
    sizes = [600, 0, 300, 17, 513, 256, 1, 700]
    N = len(sizes)
    imgs = synth.sift_like_descriptors(N, sizes, seed=41)
    for window in (0, 1, N, N + 3):
        pairs, counts, matches = keymatch.key_match_full(imgs, window, 0.6)
        want_txt, want_counts = oracle.match_all_pairs_port(imgs, window, 0.6, 1)
        assert keymatch.format_match_table(pairs, counts, matches, 1) == want_txt, window
        assert [want_counts[i, j] for j, i in pairs] == counts.tolist(), window
    keys, key_off = keymatch.concat_keys(imgs)
    db = keymatch.KeyDatabase(keys, key_off)
    try:
        for window in (1, 3):
            db.run(0, N, window, 0.6)
            c_all, m_all = db.fetch()
            parts_c, parts_m = [], []
            for b, e in keymatch.shard_images(sizes, window, 3):
                db.run(b, e, window, 0.6)
                c, m = db.fetch()
                parts_c.append(c); parts_m.append(m)
            assert np.array_equal(np.concatenate(parts_c), c_all), window
            assert np.array_equal(np.concatenate(parts_m), m_all), window
            assert c_all.shape[0] == len(keymatch.pair_list(N, window))
    finally:
        db.close()


def test_database_image_larger_than_a_launch_chunk(oracle, monkeypatch):
    """BSFM_MATCH_CHUNK_MSLOTS=1 allows 2^20 query rows (8192 units) per launch.  1040 images of 1024 keys (8 units of 128
    rows, no padding): image i has 8 i units, so images 1025-1039 each need more units than a chunk holds and get a launch
    of their own.  At ratio 1.0 almost every one of their more than 2^20 query rows is a candidate and a match, so the
    launch's buffers must be sized for the whole image.  Every kernel's chunked table equals its default one and the tc
    table; 30 pairs at ratio 0.6 and 3 at ratio 1.0 are compared with the port."""
    N, K = 1040, 1024
    imgs = synth.sift_like_descriptors(N, K, seed=43)
    keys, key_off = keymatch.concat_keys(imgs)
    tables = {}
    for name, env in KERNELS.items():
        for k in ("BSFM_MATCH_KERNEL", "BSFM_MATCH_EPILOGUE", "BSFM_MATCH_PAIR", "BSFM_MATCH_QUAD", "BSFM_MATCH_CHUNK_MSLOTS"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        db = keymatch.KeyDatabase(keys, key_off)
        try:
            got = {}
            for chunked in (False, True):
                if chunked:
                    monkeypatch.setenv("BSFM_MATCH_CHUNK_MSLOTS", "1")
                db.run(0, N, -1, 0.6)
                got[chunked, 0.6] = db.fetch() + (db.timing()["launches"],)
                db.run(1030, N, -1, 1.0)
                got[chunked, 1.0] = db.fetch() + (db.timing()["launches"],)
        finally:
            db.close()
        for ratio in (0.6, 1.0):
            (c0, m0, l0), (c1, m1, l1) = got[False, ratio], got[True, ratio]
            assert np.array_equal(c0, c1) and np.array_equal(m0, m1), (name, ratio)
            assert l1 > l0, (name, ratio, l0, l1)
        tables[name] = got[False, 0.6][:2], got[False, 1.0][:2]
    for name, t in tables.items():
        for a, b in zip(t, tables["tc"]):
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), name
    (counts, matches), (counts1, matches1) = tables["tc"]
    assert counts1[-(N - 1):].sum() > 1 << 20          # matches of the last image alone
    pairs = keymatch.pair_list(N)
    starts = np.concatenate([[0], np.cumsum(counts)])
    rng = np.random.default_rng(7)
    late = [q for q, (j, i) in enumerate(pairs) if i >= 1025]
    picked = np.concatenate([rng.choice(late, 15, replace=False), rng.choice(len(pairs), 15, replace=False)])
    picked = np.concatenate([picked, [q for q, (j, i) in enumerate(pairs) if (j, i) == (1038, 1039)]])   # consecutive: rich
    for q in picked:
        j, i = pairs[q]
        assert np.array_equal(matches[starts[q]:starts[q + 1]], oracle.match_pair_port(imgs[j], imgs[i], 0.6)), (j, i)
    assert counts[picked[-1]] > 100
    pairs1 = keymatch.pair_list(N, -1, 1030, N)
    starts1 = np.concatenate([[0], np.cumsum(counts1)])
    for q in (0, len(pairs1) // 2, len(pairs1) - 1):
        j, i = pairs1[q]
        assert np.array_equal(matches1[starts1[q]:starts1[q + 1]], oracle.match_pair_port(imgs[j], imgs[i], 1.0)), (j, i)


def test_reference_ties_golden(kernel, oracle):
    """MatchKeysExhaustive of the unmodified reference at ratio 1.0 and 0.75 (tests/golden/make_match_ties_golden.py): equal
    on every row without a passing tie; on a row with one the GPU returns the smallest caller index among the tied keys"""
    from tests.golden import make_match_ties_golden as mk
    g = np.load(GOLD_TIES)
    lib = bundle.load_library()
    fn = lib.bsfm_match_pair_test
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    fn.restype = ctypes.c_int
    tie_rows = 0
    for name, q, db in mk.tie_scenes() + mk.kermit_pairs():
        assert g[f"{name}_digest"] == mk.digest(q, db), name
        q, db = np.ascontiguousarray(q), np.ascontiguousarray(db)
        for tag, ratio in mk.RATIOS.items():
            out = np.zeros((q.shape[0], 2), np.int32)
            n = fn(q.ctypes.data, q.shape[0], db.ctypes.data, db.shape[0], ratio, 1, out.ctypes.data, q.shape[0])
            assert n >= 0
            got = mk.nearest_per_row(out[:n], q.shape[0])
            assert np.array_equal(got, mk.nearest_per_row(oracle.match_pair_port_test(q, db, ratio, 1), q.shape[0])), (kernel, name, tag)
            tied = R.passing_tie_rows(q, db, ratio, 1)
            off = np.ones(q.shape[0], bool)
            off[tied] = False
            assert np.array_equal(got[off], g[f"{name}_{tag}"][off]), (kernel, name, tag)
            if len(tied):
                d = R.sqdist(q[tied], db)
                is_tied = d == d.min(1)[:, None]
                assert np.all(got[tied] == is_tied.argmax(1)), (kernel, name, tag)   # first tied caller index
            tie_rows += len(tied)
    assert tie_rows > 100
