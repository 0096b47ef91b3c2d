"""Index parts (-I) and the -f occurrence threshold on the host, no GPU: the library's part plan against the per-part
sequence counts the reference printed (tests/golden/parts_manifest.json), and the plain-C restatement of
mm_idx_cal_max_occ (oracle/wm_oracle_occ.c) against the reference's own function on every part of the parts inputs."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]
import make_golden  # noqa: E402

MAN = json.load(open(os.path.join(ROOT, "tests", "golden", "parts_manifest.json")))
_occ = None


def occ_oracle():
    global _occ
    if _occ is None:
        so = os.path.join(tempfile.mkdtemp(prefix="wm_occ_oracle_"), "libwm_oracle_occ.so")
        subprocess.check_call(["/usr/bin/gcc", "-O2", "-fPIC", "-shared", os.path.join(ROOT, "oracle", "wm_oracle_occ.c"), "-o", so])
        _occ = C.CDLL(so)
        _occ.wm_oracle_cal_max_occ.restype = C.c_int32
        _occ.wm_oracle_cal_max_occ.argtypes = [C.c_void_p, C.c_int64, C.c_float]
    return _occ


def cal_max_occ(counts, f):
    counts = np.ascontiguousarray(counts, np.uint32)
    return occ_oracle().wm_oracle_cal_max_occ(counts.ctypes.data, len(counts), f)


@pytest.mark.parametrize("name", sorted(MAN["plan"]))
def test_part_plan_matches_reference(name, tmp_path):
    from winnowmap_b200.mapper import part_plan
    m = MAN["plan"][name]
    fa = make_golden.make_plan_input(name, str(tmp_path))
    assert make_golden.md5(fa) == m["fa_md5"], "plan input generator drifted"
    assert part_plan(fa, m["I"]) == m["n_seq"]


@pytest.mark.parametrize("name", sorted(MAN["cases"]))
def test_part_plan_of_mapping_goldens(name, tmp_path):
    from winnowmap_b200.mapper import part_plan
    m = MAN["cases"][name]
    ref, _, _ = make_golden.make_parts_inputs(m["inputs"], str(tmp_path))
    assert part_plan(ref, m["lib"].get("part_bases", 4_000_000_000)) == m["n_seq"]


def test_part_plan_rules():
    """The edges of the rule on one crafted file: mini-batch of 50 bases, part size 100."""
    from winnowmap_b200.mapper import part_plan
    with tempfile.TemporaryDirectory() as td:
        fa = os.path.join(td, "x.fa")
        lens = [60, 40, 0, 100, 1, 0, 30, 30, 30, 200, 0]
        with open(fa, "w") as f:
            for i, L in enumerate(lens):
                f.write(f">s{i}\n{'A' * L}\n")
        # mini-batches [60] [40 0 100]: the part holds 60, not > 100, so the second mini-batch is read; 200 ends the part.
        # [1 0 30 30] [30 200] ends the second; the trailing empty sequence is a part of its own
        assert part_plan(fa, 100, 50) == [4, 6, 1]
        assert part_plan(fa, 10 ** 12, 50) == [len(lens)]
        # mini-batches of min(mini_batch_size, -I) = 99 bases: [60 40] [0 100] [1 0 30 30 30 200] [0]
        assert part_plan(fa, 99, 10 ** 9) == [2, 2, 6, 1]


@pytest.mark.parametrize("key", sorted(MAN["occ"]))
def test_cal_max_occ_restatement_matches_reference(key, tmp_path):
    """The restatement on each part's occurrence counts equals mm_idx_cal_max_occ of the reference on that part, for every
    recorded f including 0 (INT32_MAX); where the reference can be built the counts and values come from it directly.  With the
    reference absent the test still pins the restatement to the recorded values."""
    rec = MAN["occ"][key]
    if make_golden.ref_parts_lib() is not None:
        ref, _, wfile = make_golden.make_parts_inputs(rec["inputs"], str(tmp_path))
        parts = make_golden.ref_parts(ref, wfile, rec["k"], rec["w"], rec["flag"], rec["I"])
        assert [p[0] for p in parts] == [p["n_seq"] for p in rec["parts"]]
        for (_, cnt, occ), p in zip(parts, rec["parts"]):
            assert {str(f): v for f, v in occ.items()} == p["max_occ"]
            h = dict(zip(*np.unique(cnt, return_counts=True)))
            assert {str(v): int(c) for v, c in h.items()} == p["hist"]
    for p in rec["parts"]:
        counts = np.repeat(np.array([int(v) for v in p["hist"]], np.uint32), [p["hist"][v] for v in p["hist"]])
        np.random.default_rng(len(counts)).shuffle(counts)
        for f, want in p["max_occ"].items():
            assert cal_max_occ(counts, float(f)) == want, (key, f)
        assert cal_max_occ(counts, 1e-30) == -1  # the rank reaches n: refused, where the reference reads past its array


def test_cal_max_occ_restatement_edges():
    assert cal_max_occ(np.array([5], np.uint32), 0.5) == 6
    assert cal_max_occ(np.array([5], np.uint32), 0.0) == 2 ** 31 - 1
    assert cal_max_occ(np.array([5], np.uint32), -1.0) == 2 ** 31 - 1
    assert cal_max_occ(np.zeros(0, np.uint32), 0.5) == -1
    c = np.array([3, 1, 2, 2, 9, 1 << 20], np.uint32)
    assert cal_max_occ(c, 0.99) == 2             # rank (uint32)(0.01 * 6) = 0
    assert cal_max_occ(c, 0.25) == 10            # rank 4
    assert cal_max_occ(c, 0.1) == (1 << 20) + 1  # rank 5 = n - 1
