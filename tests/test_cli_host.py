"""The command line (csrc/host_cli.cpp) end to end on the host, no GPU: the product's parser, index-part loop and file driver
over oracle backends (tests/hostsim/cli_backend.cpp) run the reference's own recorded command lines and reproduce its
goldens; the options the mapper does not build are refused with status 1 before any index is read."""
import gzip
import hashlib
import json
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]
import cli_lib  # noqa: E402
import make_golden  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
CLI = json.load(open(os.path.join(GOLD, "cli_manifest.json")))
MAIN = json.load(open(os.path.join(GOLD, "manifest.json")))
PARTS = json.load(open(os.path.join(GOLD, "parts_manifest.json")))["cases"]
# the oracle backend of this harness has neither -H indexes nor the self / dual seed filter of -X (their harnesses are
# overlap_backend.cpp and hpc_backend.cpp); the GPU test runs those command lines too
PARTS_CASES = sorted(n for n in PARTS if " -H " not in PARTS[n]["cmd"] and " -X " not in PARTS[n]["cmd"])


def first_diff(a, b):
    la, lb = a.split(b"\n"), b.split(b"\n")
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return f"line {i}: exp {x[:200]!r} got {y[:200]!r}"
    return f"line count {len(la)} vs {len(lb)}"


def cli_case(name, td):
    """argv[1..] of command-line golden `name`, its inputs written to td"""
    has_w = make_golden.make_cli_inputs(CLI[name]["inputs"], td)
    args = make_golden.cli_args(name, has_w)
    assert make_golden.md5(os.path.join(td, "ref.fa")) == CLI[name]["ref_md5"], "input generator drifted"
    assert make_golden.md5(os.path.join(td, "reads.fa")) == CLI[name]["reads_md5"], "input generator drifted"
    return args


def check_cli_output(name, out):
    exp = gzip.open(os.path.join(GOLD, name + (".sam.stripped.gz" if CLI[name]["sam"] else ".paf.gz"))).read()
    got = make_golden.cli_golden_bytes(out, CLI[name]["sam"])
    assert got == exp, first_diff(exp, got)
    assert hashlib.md5(out).hexdigest() == CLI[name]["out_md5"], "SEQ/QUAL differ"


def main_case(name, td):
    """argv[1..] of the recorded command of golden `name` of manifest.json, its inputs written to td"""
    make_golden.make_inputs(name, td)
    return [a.replace("/tmp/wm_golden/", "") for a in MAIN[name]["cmd"].split()[1:]]


def parts_case(name, td):
    m = PARTS[name]
    ref, reads, wfile = make_golden.make_parts_inputs(m["inputs"], os.path.join(td, "gen"))
    shutil.copy(ref, os.path.join(td, "ref.fa"))
    shutil.copy(reads, os.path.join(td, "reads.fa"))
    if wfile:
        shutil.copy(wfile, os.path.join(td, "rep.txt"))
    a = m["cmd"].split()[1:]
    return [("rep.txt" if a[i - 1] == "-W" else "tmp_split") if x == "<prefix>" else x for i, x in enumerate(a)]


def check_parts_output(name, out):
    m = PARTS[name]
    if m["lib"].get("sam"):
        got = make_golden.sam_without_pg(out)
        if hashlib.md5(got).hexdigest() != m["sam_md5"]:
            exp = gzip.open(os.path.join(GOLD, name + ".sam.stripped.gz")).read()
            got = make_golden.sam_strip_seq(got)
            assert got == exp, first_diff(exp, got)
            pytest.fail("SEQ/QUAL differ")
    else:
        exp = gzip.open(os.path.join(GOLD, name + ".paf.gz")).read()
        assert out == exp, first_diff(exp, out)


@pytest.mark.parametrize("name", sorted(CLI))
def test_cli_goldens(name, tmp_path):
    """--cap-sw-mem, --max-qlen, -R, several query files and -I with several files, against the reference's output"""
    args = cli_case(name, str(tmp_path))
    rc, out, err = cli_lib.cli_main_host(args, str(tmp_path))
    assert rc == 0, err[-2000:]
    check_cli_output(name, out)


@pytest.mark.parametrize("name", sorted(MAIN))
def test_recorded_commands(name, tmp_path):
    """the reference's recorded command of every mapping golden"""
    args = main_case(name, str(tmp_path))
    rc, out, err = cli_lib.cli_main_host(args, str(tmp_path))
    assert rc == 0, err[-2000:]
    exp = gzip.open(os.path.join(GOLD, name + ".paf.gz")).read()
    assert out == exp, first_diff(exp, out)


@pytest.mark.parametrize("name", PARTS_CASES)
def test_recorded_parts_commands(name, tmp_path):
    """-I, --split-prefix and -f command lines of the parts goldens (SAM but for the @PG line, which names other files)"""
    args = parts_case(name, str(tmp_path))
    rc, out, err = cli_lib.cli_main_host(args, str(tmp_path))
    assert rc == 0, err[-2000:]
    check_parts_output(name, out)
    assert not any(f.startswith("tmp_split") for f in os.listdir(tmp_path)), "the merge runs in memory"


REFUSED = [
    ["--heap-sort=yes"], ["--heap-sort", "y"], ["--sr"], ["-T", "20"], ["--frag=yes"], ["-x", "splice", "-c"], ["-x", "splice", "-a"],
    ["-x", "splice:hq", "--cs"], ["-x", "cdna", "--MD"], ["--splice", "-c"], ["-u", "f", "-c"], ["-u", "b", "--MD"], ["--split-prefix", "p", "reads2.fa"],
]


@pytest.mark.parametrize("extra", REFUSED, ids=lambda a: "_".join(a))
def test_refused_options(extra, tmp_path):
    """refused with status 1, naming the option, before the index is read: the reference file does not even exist"""
    rc, out, err = cli_lib.cli_main_host(["-x", "map-ont"] + extra + ["missing_ref.fa", "reads.fa"], str(tmp_path))
    assert rc == 1 and out == b""
    assert b"support" in err and b"missing_ref.fa" not in err


def test_refusals_undone_later_are_accepted(tmp_path):
    """--heap-sort=yes undone by --heap-sort=no and -u f undone by -u n are not refused: the reference file is then opened"""
    for extra in (["--heap-sort=yes", "--heap-sort=no"], ["-u", "f", "-u", "n", "-c"], ["--frag=yes", "--frag=no"], ["-T", "0"]):
        rc, out, err = cli_lib.cli_main_host(["-x", "map-ont"] + extra + ["missing_ref.fa", "reads.fa"], str(tmp_path))
        assert rc == 1 and b"failed to open file 'missing_ref.fa'" in err, (extra, err)


def test_unreadable_query_file_is_skipped(tmp_path):
    """like mm_map_file, a query file that cannot be opened is reported and skipped; the others are mapped, status 0"""
    args = cli_case("cli_two_files_paf", str(tmp_path))
    rc, out, err = cli_lib.cli_main_host(args[:-1] + ["absent.fa", args[-1]], str(tmp_path))
    assert rc == 0 and b"absent.fa" in err
    exp = gzip.open(os.path.join(GOLD, "cli_two_files_paf.paf.gz")).read()
    assert out and exp.endswith(out)


def test_output_file_and_version(tmp_path):
    args = cli_case("cli_sv_maxqlen", str(tmp_path))
    rc, out, err = cli_lib.cli_main_host(["-o", "out.paf"] + args, str(tmp_path))
    assert rc == 0 and out == b""
    check_cli_output("cli_sv_maxqlen", open(tmp_path / "out.paf", "rb").read())
    rc, out, _ = cli_lib.cli_main_host(["--version"], str(tmp_path))
    assert rc == 0 and out == b"2.03\n"
