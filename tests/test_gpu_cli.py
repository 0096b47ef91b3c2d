"""The built executable winnowmap_b200/winnowmap-b200 on the H100, as a subprocess: the command-line goldens (--cap-sw-mem,
--max-qlen, -R, several query files, -I with several files), the reference's recorded command of every mapping and parts
golden, and the exit statuses of refused options, byte for byte and status for status."""
import gzip
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]
import make_golden  # noqa: E402
import test_cli_host as th  # noqa: E402

EXE = os.path.join(ROOT, "winnowmap_b200", "winnowmap-b200")
pytestmark = pytest.mark.gpu


def run(args, cwd):
    p = subprocess.run([EXE] + list(args), cwd=cwd, capture_output=True, timeout=1800)
    return p.returncode, p.stdout, p.stderr


@pytest.mark.parametrize("name", sorted(th.CLI))
def test_gpu_cli_goldens(name, tmp_path):
    args = th.cli_case(name, str(tmp_path))
    rc, out, err = run(args, str(tmp_path))
    assert rc == 0, err[-2000:]
    th.check_cli_output(name, out)


@pytest.mark.parametrize("name", sorted(th.MAIN))
def test_gpu_recorded_commands(name, tmp_path):
    args = th.main_case(name, str(tmp_path))
    rc, out, err = run(args, str(tmp_path))
    assert rc == 0, err[-2000:]
    exp = gzip.open(os.path.join(th.GOLD, name + ".paf.gz")).read()
    assert out == exp, th.first_diff(exp, out)


@pytest.mark.parametrize("name", sorted(th.PARTS))
def test_gpu_recorded_parts_commands(name, tmp_path):
    args = th.parts_case(name, str(tmp_path))
    rc, out, err = run(args, str(tmp_path))
    assert rc == 0, err[-2000:]
    th.check_parts_output(name, out)


@pytest.mark.parametrize("extra", th.REFUSED, ids=lambda a: "_".join(a))
def test_gpu_refused_options(extra, tmp_path):
    rc, out, err = run(["-x", "map-ont"] + extra + ["missing_ref.fa", "reads.fa"], str(tmp_path))
    assert rc == 1 and out == b"" and b"support" in err


def test_gpu_cli_output_file_and_sam_header_once(tmp_path):
    args = th.cli_case("cli_two_files_sam", str(tmp_path))
    rc, out, err = run(["-o", "o.sam"] + args, str(tmp_path))
    assert rc == 0 and out == b"", err[-2000:]
    got = open(tmp_path / "o.sam", "rb").read()
    exp = gzip.open(os.path.join(th.GOLD, "cli_two_files_sam.sam.stripped.gz")).read()
    # the @PG line records the command, which now has -o
    assert make_golden.sam_without_pg(make_golden.sam_strip_seq(got)) == make_golden.sam_without_pg(exp)
    assert got.count(b"@PG\t") == 1 and b"\tCL:winnowmap -o o.sam " in got
