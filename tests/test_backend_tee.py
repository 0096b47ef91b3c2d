"""The tee backend's comparator (tests/hostsim/tee_backend.cpp) without a GPU: two oracle backends behind the tee must agree
everywhere, and a backend that changes exactly one value must be reported at exactly that call, index and field.  This is
what makes a clean GPU report (tests/test_backend_parity.py) mean something."""
import gzip
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import make_golden  # noqa: E402
import oracle_lib as ol  # noqa: E402
import tee_lib as T  # noqa: E402

MANIFEST = json.load(open(os.path.join(ROOT, "tests", "golden", "manifest.json")))


@pytest.fixture(scope="module")
def tee(tmp_path_factory):
    return T.load(T.build(str(tmp_path_factory.mktemp("tee"))))


@pytest.fixture(scope="module")
def crafted(tmp_path_factory):
    d = tmp_path_factory.mktemp("crafted")
    ref = str(d / "ref.fa")
    contigs = T.crafted_reference(ref)
    return ref, contigs, T.crafted_reads(contigs)


def test_identical_backends_report_nothing(tee, tmp_path):
    """A whole mapping run (ont_sv: masked tasks, stage-1 anchors, both chain sets, Z-drop walks, ksw_ll) through two
    oracle backends: no mismatch, the golden output, and the counters saw those shapes."""
    name = "ont_sv"
    m = MANIFEST[name]
    ref, reads, wfile = make_golden.make_inputs(name, str(tmp_path))
    out, rep = str(tmp_path / "o.paf"), str(tmp_path / "report.txt")
    rc = tee.wmt_tee_map_file(ref.encode(), None, m["params"]["preset"].encode(), reads.encode(), out.encode(), 8, 0, 4 << 20, T.DEV_ORACLE, 0, rep.encode())
    assert rc == 0
    r = T.Report(rep)
    assert r.n_mismatch == 0, r.text()
    assert open(out, "rb").read() == gzip.open(os.path.join(ROOT, "tests", "golden", name + ".paf.gz")).read()
    for key in ("seed.masked", "seed.pre", "seed.mixed_set_calls", "dp.scan_zdrop_jobs", "ll.jobs", "dp.rounds_3plus_chunks"):
        assert r[key] > 0, key


def _seed_case(tee, crafted, tmp_path, dev, mutation):
    ref, contigs, reads = crafted
    k, w = 15, 10
    rows, reads2 = T.crafted_seed_tasks(reads, k, w)
    return T.seed_chain(tee, str(tmp_path / "rep.txt"), ref, k, w, reads, rows, reads2, T.CHAIN_SETS,
                        T.max_occ_with_neighbours(contigs, k, w), dev=dev, mutation=mutation)


def _align_case(tee, crafted, tmp_path, dev, mutation):
    ref, contigs, reads = crafted
    rng = np.random.default_rng(3)
    wins = T.crafted_dp_windows(reads)
    a, b, q, e, q2, e2, sc_ambi = T.SCORINGS["map-ont"]
    rows = T.crafted_dp_jobs(T.crafted_reads_with_origin(contigs)[1], wins, rng, sizes=T.BOUNDARY_SIZES[:4])
    return T.align(tee, str(tmp_path / "rep.txt"), ref, 15, 10, reads, wins, rows, T.crafted_ll_jobs(wins, contigs, rng, n=12),
                   ol.simple_mat(a, b, sc_ambi), (q, e, q2, e2), budget=1 << 20, dev=dev, mutation=mutation)


def test_identical_backends_agree_on_crafted_batches(tee, crafted, tmp_path):
    r = _seed_case(tee, crafted, tmp_path, T.DEV_ORACLE, 0)
    assert r.n_mismatch == 0 and r["seed.tasks"] > 0 and r["seed.masked"] > 0 and r["seed.no_sketch"] > 0, r.text()
    r = _align_case(tee, crafted, tmp_path, T.DEV_ORACLE, 0)
    assert r.n_mismatch == 0 and r["dp.jobs"] > 0 and r["ll.jobs"] > 0 and r["dp.scan_zdrop_jobs"] > 0, r.text()


@pytest.mark.parametrize("mutation", sorted(T.MUTATIONS))
def test_each_change_is_reported_where_it_was_made(tee, crafted, tmp_path, mutation):
    case = _seed_case if mutation in ("rep_len", "kept", "u", "b") else _align_case
    r = case(tee, crafted, tmp_path, T.DEV_MUTANT, T.MUTATIONS[mutation])
    assert r.mutated is not None, f"the mutant found nothing to change for {mutation}"
    assert r.n_mismatch == 1, r.text()
    got = r.mismatches[0]
    assert {k: got[k] for k in r.mutated} == r.mutated, (got, r.mutated)
    assert got["expected"] != got["got"] and got["desc"]


# mismatch and gap costs far above what the crafted reads' 2-5 % errors need: some fills are Z-dropped before their end
# (tests/test_gpu_scoring.py reaches every size at these scorings with low-error pairs)
HEAVY = ("asm5", "single_asm5", "limit")


@pytest.mark.parametrize("scoring", sorted(T.SCORINGS))
def test_crafted_dp_jobs_are_true_alignments(crafted, scoring):
    """Every crafted DP job pairs a query slice with the reference slice it was copied from, so the fill really runs to the
    sizes the batch is built around: each extension reaches the last row or column of its matrix, each gap fill is not
    Z-dropped (under the asm5-like scorings and, through the N run, --score-N 3: at least two thirds of them); some
    reference slices run through the N run.  Under
    the early-out scorings (a mismatch or N score above
    2(q + e)) no job is swept: each returns the initial ksw_extz_t without a CIGAR."""
    ref, contigs, reads = crafted
    wins = T.crafted_dp_windows(reads)
    rows = T.crafted_dp_jobs(T.crafted_reads_with_origin(contigs)[1], wins, np.random.default_rng(11))
    a, b, q, e, q2, e2, sc_ambi = T.SCORINGS[scoring]
    mat = ol.simple_mat(a, b, sc_ambi)
    early_out = max(b, sc_ambi) > 2 * min(q + e, q2 + e2)
    short = 0
    for r in rows:
        qs, ts = T.job_codes(reads, contigs, wins, r)
        assert (len(qs), len(ts)) == (r[4], r[9])
        if (q, e) == (q2, e2):
            ez, cig = ol.oracle_extz2(qs, ts, mat, q, e, r[11], r[12], r[13], r[14])
        else:
            ez, cig = ol.oracle_extd2(qs, ts, mat, q, e, q2, e2, r[11], r[12], r[13], r[14])
        if early_out:
            assert tuple(ez[[0, 1, 2, 3, 9, 10]]) == (0, 0, -1, -1, 0, 0) and len(cig) == 0, (r, ez)
        elif scoring in HEAVY or sc_ambi * int((ts == 4).sum()) > r[12]:  # or the N run alone costs more than the Z-drop
            short += not T.dp_job_reaches_end(r, ez, cig)
        else:
            assert T.dp_job_reaches_end(r, ez, cig), (r, ez)
    assert short <= len(rows) // 3, short
    assert sum(b"N" in contigs[r[7]][r[8]:r[8] + r[9]] for r in rows) >= 3
