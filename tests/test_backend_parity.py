"""The CUDA backend against the oracle backend call by call (tests/hostsim/tee_backend.cpp): every seed_chain, run_dp and
run_ll call of whole mapping runs, and crafted batches at the edges of the device kernels, compared field by field.  A
divergence is reported as "seed_chain call 1 #37: u[2] expected ... got ...", with the task or job that produced it.

Each case runs in a child process: the CUDA backend's thread-local allocator state and any exit() of the library stay
out of the test session."""
import gzip
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, TESTS)
import make_golden  # noqa: E402
import tee_lib as T  # noqa: E402

pytestmark = pytest.mark.gpu
MANIFEST = json.load(open(os.path.join(TESTS, "golden", "manifest.json")))
HPC_MANIFEST = json.load(open(os.path.join(TESTS, "golden", "hpc_manifest.json")))
BUDGET = 4 << 20  # backtrack bytes per DP launch: every golden run's big rounds split into several chunks

# Shapes each golden run holds, beyond those every run has (Z-drop walks, rounds of three or more DP chunks).  What a
# golden lacks is noted beside it; the crafted batches below reach every shape in every kernel class.
SHAPES = {
    "ont_sv": ["seed.pre", "seed.masked", "sort3.le2048", "seed.mixed_set_calls", "ll.jobs", "dp.coop_jobs"],  # no chaining task > 2048
    "ont_single_gap": ["seed.pre", "seed.masked", "sort3.le2048", "seed.mixed_set_calls", "ll.jobs", "dp.extz2_jobs"],  # one gap pair: no coop
    "ont_highocc": ["seed.pre", "seed.mixed_set_calls", "chain.gt4096", "dp.coop_jobs"],  # no masked task, no sort #3, no ll
    "ont_small": ["seed.pre", "seed.mixed_set_calls"],   # no masked task, no sort #3, no ll, no coop job
    "hifi_small": ["seed.pre", "seed.mixed_set_calls"],  # no masked task, no sort #3, no ll, no coop job
    "ont_tandem": ["seed.pre", "seed.mixed_set_calls"],  # no masked task, no sort #3, no ll, no coop job
    "asm20_small": ["seed.pre"],                         # every read has stage-1 anchors: one chain set; no mask, sort #3, ll, coop
    "asm5_small": ["seed.pre", "ll.jobs"],               # one chain set; no mask, sort #3, coop
    "asm10_small": ["seed.pre", "ll.jobs"],              # one chain set; no mask, sort #3, coop
    "ont_sv_long_inc": ["seed.pre", "seed.masked", "sort3.le2048", "seed.mixed_set_calls", "ll.jobs", "dp.coop_jobs"],  # as ont_sv
    "hpc_clr": ["dp.coop_jobs"],                         # one pass: no stage-1 anchors, so no mask, sort #3 or second set; no ll
    "hpc_ont_small": ["seed.pre", "seed.mixed_set_calls", "dp.coop_jobs"],  # no masked task, no sort #3, no ll
}

_CHILD = r'''
import json, sys
sys.path.insert(0, %r)
import numpy as np
import oracle_lib as ol
import tee_lib as T
so, case, rep = sys.argv[1], json.loads(sys.argv[2]), sys.argv[3]
L = T.load(so)
kind = case.pop("kind")
if kind == "map":
    L.wmt_set_scoring(*case["scoring"])
    rc = L.wmt_tee_map_file(case["ref"].encode(), case["w"].encode() if case["w"] else None, case["preset"].encode(), case["reads"].encode(),
                            case["out"].encode(), 8, case["hpc"], case["budget"], T.DEV_GPU, 0, rep.encode())
    sys.exit(0 if rc == 0 else 3)
ref = case["ref"]
contigs = T.crafted_reference(ref)
reads, origin = T.crafted_reads_with_origin(contigs)
if kind == "seed":
    k, w = case["k"], case["w"]
    rows, reads2 = T.crafted_seed_tasks(reads, k, w)
    T.seed_chain(L, rep, ref, k, w, reads, rows, reads2, T.CHAIN_SETS, T.max_occ_with_neighbours(contigs, k, w, hpc=case["hpc"]), hpc=case["hpc"])
else:
    rng = np.random.default_rng(11)
    wins = T.crafted_dp_windows(reads)
    a, b, q, e, q2, e2, sc_ambi = T.SCORINGS[case["scoring"]]
    T.align(L, rep, ref, 15, 10, reads, wins, T.crafted_dp_jobs(origin, wins, rng), T.crafted_ll_jobs(wins, contigs, rng),
            ol.simple_mat(a, b, sc_ambi), (q, e, q2, e2), budget=case["budget"])
''' % TESTS


@pytest.fixture(scope="module")
def tee_so(tmp_path_factory):
    return T.build(str(tmp_path_factory.mktemp("tee")))


def _run(tee_so, case, tmp_path, env=None):
    rep = str(tmp_path / "report.txt")
    t0 = time.time()
    out = subprocess.run([sys.executable, "-c", _CHILD, tee_so, json.dumps(case), rep], env=dict(os.environ, **(env or {})),
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=1200)
    assert out.returncode == 0, out.stdout[-3000:].decode(errors="replace")
    r = T.Report(rep)
    print(f"[{case.get('name', case['kind'])}] {time.time() - t0:.1f} s\n{r.text()}")
    return r


def _map_case(name, tmp_path):
    hpc = name.startswith("hpc_")
    m = (HPC_MANIFEST if hpc else MANIFEST)[name]
    ref, reads, wfile = (make_golden.make_hpc_inputs if hpc else make_golden.make_inputs)(name, str(tmp_path))
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"], "synthetic input generator drifted"
    return dict(kind="map", name=name, ref=ref, reads=reads, w=wfile, preset=m["params"]["preset"], scoring=make_golden.scoring_override(m["params"]),
                hpc=int(hpc), budget=BUDGET, out=str(tmp_path / "out.paf"))


def _check_map(r, case):
    assert r.n_mismatch == 0, r.text()
    got = open(case["out"], "rb").read()
    assert got == gzip.open(os.path.join(TESTS, "golden", case["name"] + ".paf.gz")).read(), "PAF differs from the golden"
    for key in ["dp.scan_zdrop_jobs", "dp.rounds_3plus_chunks"] + SHAPES[case["name"]]:
        assert r[key] > 0, key


@pytest.mark.parametrize("name", sorted(MANIFEST) + ["hpc_clr", "hpc_ont_small"])
def test_whole_path_matches_oracle_call_by_call(tee_so, name, tmp_path):
    case = _map_case(name, tmp_path)
    _check_map(_run(tee_so, case, tmp_path), case)


def test_whole_path_matches_oracle_under_tuning_switches(tee_so, tmp_path):
    """The same with every big DP job on the cooperative sweep, and more chaining tasks on the tile kernel and the CTA
    backtrack."""
    case = _map_case("ont_sv", tmp_path)
    r = _run(tee_so, case, tmp_path, env={"WM_DP_COOP_MIN_CELLS": "1", "WM_CHAIN_TILE_MIN": "256", "WM_CHAIN_BT_CTA_MIN": "512"})
    _check_map(r, case)
    # the switches moved work: chaining tasks of at most 2048 anchors onto the tile kernel and the CTA backtrack
    assert r["chain.tile_tasks"] > r["chain.le4096"] + r["chain.gt4096"], r.text()
    assert r["chain.bt_cta_tasks"] > r["chain.gt4096"], r.text()


# One CTA for the medium sort, the giant sort and the chaining tile kernel, with low thresholds for the giant classes: a
# worker that takes two tasks carries its state (mbarrier phases, work lists, rings, masks) from the first into the second.
TASK_LOOP_ENV = {"WM_SORT_MEDIUM_CTAS": "1", "WM_SORT_GIANT_MIN": "4096", "WM_SORT_GIANT_CTAS": "1", "WM_CHAIN_TILE_MIN": "256",
                 "WM_CHAIN_TILE_CTAS": "1", "WM_CHAIN_BT_CTA_MIN": "256"}
# The classes (tasks of one launch, peak over launches) each run reaches more than once under TASK_LOOP_ENV.  No run has two
# arrays of 2049-4096 anchors in one sort launch, so the medium sort's second array is left to tests/test_gpu_task_loops.py.
TASK_LOOP_PEAKS = {
    "ont_highocc": ["peak.chain_tile", "peak.chain_bt_cta", "peak.sort_giant"],
    "ont_tandem": ["peak.chain_tile", "peak.chain_bt_cta"],  # no anchor array above 2048
    "hpc_ont_small": [],  # at most one task above 256 anchors per call, no array above 2048: zero mismatches and the golden only
    "seed": ["peak.chain_tile", "peak.chain_bt_cta", "peak.sort_giant"],
    "seed_hpc": ["peak.chain_tile", "peak.chain_bt_cta", "peak.sort_giant"],
}


@pytest.mark.parametrize("name", ["ont_highocc", "ont_tandem", "hpc_ont_small"])
def test_whole_path_task_loops_match_oracle(tee_so, name, tmp_path):
    """Whole mapping runs with single-CTA grids for the sorts and the tile kernel: zero mismatches, the golden output, and
    some worker of each forced class took a second task."""
    case = _map_case(name, tmp_path)
    r = _run(tee_so, case, tmp_path, env=TASK_LOOP_ENV)
    _check_map(r, case)
    for key in TASK_LOOP_PEAKS[name]:
        assert r[key] > 1, (key, r.text())


@pytest.mark.parametrize("hpc", [False, True])
def test_crafted_seed_chain_task_loops_match_oracle(tee_so, hpc, tmp_path):
    """The crafted stage-1 / stage-2 seed batches of test_crafted_seed_chain_matches_oracle under the same single-CTA grids."""
    r = _run(tee_so, dict(kind="seed", ref=str(tmp_path / "ref.fa"), k=15, w=10, hpc=int(hpc)), tmp_path, env=TASK_LOOP_ENV)
    assert r.n_mismatch == 0, r.text()
    for key in TASK_LOOP_PEAKS["seed_hpc" if hpc else "seed"]:
        assert r[key] > 1, (key, r.text())


@pytest.mark.parametrize("hpc", [False, True])
def test_crafted_seed_chain_matches_oracle(tee_so, hpc, tmp_path):
    """A stage-1 call: windows at odd starts and at the read end, lengths around k, w + k - 1, 128 and 1024 and tens of kb;
    N runs, lower case and IUPAC codes.  Then the stage-2 call over whole reads, built as host_map.cpp builds it: stage-1
    anchors from the first call's chains in read coordinates, masked intervals at both read ends, across 32-base groups and
    around a single unmasked base, a read covered by its stage-1 windows (not sketched), stage-1 merges of every sort size
    class, and both chain sets.  max_occ is an occurrence count the index has, next to count - 1; chaining tasks of every
    class."""
    r = _run(tee_so, dict(kind="seed", ref=str(tmp_path / "ref.fa"), k=15, w=10, hpc=int(hpc)), tmp_path)
    assert r.n_mismatch == 0, r.text()
    assert r["seed.mixed_set_calls"] == 1 and r["seed.masked"] >= 4 and r["seed.no_sketch"] >= 1
    for key in ("sort3.le64", "sort3.le2048", "sort3.gt2048", "chain.le128", "chain.le2048", "chain.le4096", "chain.gt4096"):
        assert r[key] > 0, key


@pytest.mark.parametrize("scoring", sorted(T.SCORINGS))
def test_crafted_dp_and_ll_match_oracle(tee_so, scoring, tmp_path):
    """Query slices of both strands and reference slices, reversed or not, at odd offsets, at window and contig ends and
    through N; the flag sets of host_align.cpp; sizes on both sides of the shared-memory, long-diagonal and cooperative
    thresholds; jobs out of size order under a budget that cuts the round into chunks; ksw_ll on slices of both strands."""
    r = _run(tee_so, dict(kind="align", ref=str(tmp_path / "ref.fa"), scoring=scoring, budget=2 << 20), tmp_path)
    assert r.n_mismatch == 0, r.text()
    assert r["dp.scan_zdrop_jobs"] > 0 and r["dp.flag_0xc2"] > 0 and r["ll.jobs"] > 0 and r["dp.max_chunks"] >= 3
    a, b, q, e, q2, e2, sc_ambi = T.SCORINGS[scoring]
    if (q, e) != (q2, e2):  # the single-affine sweep has no cooperative form
        assert r["dp.coop_jobs"] > 0


def _blob_index(blob):
    from test_gpu_hpc import _blob_index as parse
    return parse(blob)


def test_plain_device_index_matches_reference(tmp_path):
    """The index Mapper builds on the device without -H (csrc/index_dev.cu) equals the reference's flattened index."""
    from winnowmap_b200.mapper import Mapper
    name = "ont_tandem"
    ref, _, wfile = make_golden.make_inputs(name, str(tmp_path))
    mp = Mapper(ref, wfile, preset=MANIFEST[name]["params"]["preset"])
    keys, poff, pos, flag = _blob_index(mp.index_blob())
    mp.close()
    fx = np.load(os.path.join(TESTS, "golden", name + ".refidx.npz"))
    assert flag == 0
    assert np.array_equal(keys, fx["keys"])
    assert np.array_equal(np.diff(poff), fx["n_pos"].astype(np.uint64))
    assert np.array_equal(pos, fx["pos"])
