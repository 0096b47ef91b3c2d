"""The command-line parser (csrc/host_cli.cpp) against the reference's own main(), on the host: for every command line of
the table, what the product would map with -- mm_idxopt_t and mm_mapopt_t byte for byte outside their pointer fields, the
strings of those, the thread count, the -R line of a SAM run and the files -- and the exit status must equal what the
reference's main() hands to its index reader and mapper (oracle/cli_ref_dump.c, linked with the reference's main.o).  Where
that binary is absent the recorded digests of its dumps (tests/golden/cli_ref_digests.json) stand in; WM_RECORD_REF=1
rewrites them from the live reference.  Command lines with an option the mapper does not build must give status 1 instead."""
import hashlib
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import cli_lib  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
DIGESTS = os.path.join(GOLD, "cli_ref_digests.json")
F = ["ref.fa", "reads.fa"]


def golden_lines():
    """every recorded `cmd` of the golden manifests, with its files renamed"""
    out = []
    for fn in sorted(os.listdir(GOLD)):
        if not fn.endswith("manifest.json"):
            continue
        m = json.load(open(os.path.join(GOLD, fn)))
        for v in (m.get("cases", m)).values():
            if not isinstance(v, dict) or "cmd" not in v:
                continue
            a = v["cmd"].split()[1:]
            out.append(" ".join(os.path.basename(x) if "/" in x else ("p" if x == "<prefix>" else x) for x in a))
    return sorted(set(out))


HANDMADE = [
    # permuted positionals, -x after -k / -w / -O, repeated -x
    "ref.fa -x map-ont reads.fa -c", "ref.fa reads.fa -x map-pb -a", "-k 17 -x map-ont ref.fa reads.fa", "-w 30 -x asm5 ref.fa reads.fa",
    "-O 5,30 -x asm10 -c ref.fa reads.fa", "-x asm5 -x map-ont ref.fa reads.fa", "-x map-ont -x asm20 -c ref.fa reads.fa",
    "-x map-pb-clr -x map-pb ref.fa reads.fa", "-ax map-ont ref.fa reads.fa", "-cx asm20 ref.fa reads.fa", "-t8 -x map-ont ref.fa reads.fa",
    "-t 2 ref.fa reads.fa", "--sv-off ref.fa reads.fa", "-t 3 --sv-off ref.fa reads.fa", "--sv-off -t 3 ref.fa reads.fa",
    # comma pairs and number suffixes
    "-O4,24 -E2,1 -z400,200 ref.fa reads.fa", "-O6 -E3 -z300 -c ref.fa reads.fa", "-z 500,100 ref.fa reads.fa", "-O4,24 -E2 ref.fa reads.fa",
    "-I 4G -K 500M --cap-sw-mem 1.5M ref.fa reads.fa", "-I 250k -K 1k ref.fa reads.fa", "-I 1.5g --cap-sw-mem 50M ref.fa reads.fa",
    "--cap-sw-mem 5m -c ref.fa reads.fa", "--cap-sw-mem=100 -c ref.fa reads.fa", "--max-qlen 8000 ref.fa reads.fa", "--max-qlen=2.5k -c ref.fa reads.fa",
    "-r 1k -g 2k -F 900 ref.fa reads.fa", "-G 20k ref.fa reads.fa", "--max-intron-len 5k -x splice ref.fa reads.fa",
    # --cs, -S, --MD, secondary and -N
    "--cs -c ref.fa reads.fa", "--cs=long ref.fa reads.fa", "--cs=short -a ref.fa reads.fa", "--cs=none ref.fa reads.fa", "--cs=bogus ref.fa reads.fa",
    "-S ref.fa reads.fa", "--MD -c ref.fa reads.fa", "--MD ref.fa reads.fa", "-N 0 -c ref.fa reads.fa", "-N 0 ref.fa reads.fa", "-N 3 ref.fa reads.fa",
    "-N 10 -p 0.5 ref.fa reads.fa", "--secondary=no ref.fa reads.fa", "--secondary=yes -c ref.fa reads.fa", "--secondary=n -a ref.fa reads.fa",
    "--secondary=maybe ref.fa reads.fa", "--dual=no ref.fa reads.fa", "--dual=yes -X ref.fa reads.fa", "-X -c ref.fa ref.fa", "-D -P ref.fa reads.fa",
    "--for-only -c ref.fa reads.fa", "--rev-only ref.fa reads.fa", "-Q -L -Y -y -a ref.fa reads.fa", "--eqx -c ref.fa reads.fa",
    "--paf-no-hit ref.fa reads.fa", "--sam-hit-only -a ref.fa reads.fa", "--no-end-flt --hard-mask-level -M 0.7 ref.fa reads.fa",
    "--end-bonus 10 --min-dp-len 100 --end-seed-pen 4 -c ref.fa reads.fa", "--max-chain-skip 10 --max-chain-iter 1000 ref.fa reads.fa",
    "--max-clip-ratio 0.5 --lj-min-ratio 0.3 --score-N 2 -c ref.fa reads.fa", "--min-occ-floor 100 ref.fa reads.fa", "--min-occ-floor 9000 ref.fa reads.fa",
    "-n 5 -m 30 -s 50 -A 1 -B 3 -c ref.fa reads.fa", "--seed 7 --bucket-bits 12 ref.fa reads.fa", "--no-long-join ref.fa reads.fa",
    "-f 0.0002 ref.fa reads.fa", "-f 2 ref.fa reads.fa", "-f 0 ref.fa reads.fa", "-H -c ref.fa reads.fa", "-W rep.txt ref.fa reads.fa",
    "--split-prefix pre -c ref.fa reads.fa", "--split-prefix pre --cs ref.fa reads.fa", "-R @RG\\tID:rg1\\tSM:s1 -a ref.fa reads.fa",
    "-R @RG\\tID:rg1 ref.fa reads.fa", "-o out.paf ref.fa reads.fa", "-o - -c ref.fa reads.fa", "ref.fa reads.fa reads2.fa", "-a ref.fa a.fa b.fa c.fa",
    # -u and -G around -x splice (-u turns on splicing through mm_mapopt_update)
    "-x map-ont -u f ref.fa reads.fa", "-u b ref.fa reads.fa", "-u r -x map-ont ref.fa reads.fa", "-u n -x splice ref.fa reads.fa", "-u x ref.fa reads.fa",
    "-G 20k -x splice ref.fa reads.fa", "-x splice -G 20k ref.fa reads.fa", "-G 20k --splice ref.fa reads.fa", "--splice -G 20k ref.fa reads.fa",
    "-x splice:hq ref.fa reads.fa", "-x cdna ref.fa reads.fa", "-x splice -C 5 --junc-bonus 3 --splice-flank=no ref.fa reads.fa",
    "-x splice --junc-bed j.bed ref.fa reads.fa", "--splice-flank=yes ref.fa reads.fa",
    # accepted without effect
    "-2 -v 1 --no-kalloc --print-qname ref.fa reads.fa", "--dbg-polish --print-seeds --print-aln-seq ref.fa reads.fa", "--no-pairing ref.fa reads.fa",
    "--heap-sort=no ref.fa reads.fa", "--frag=no ref.fa reads.fa", "-T 0 ref.fa reads.fa", "--vers", "-V -x map-ont", "-x map-ont -V ref.fa",
    # errors of the reference
    "-x bogus ref.fa reads.fa", "--bogus ref.fa reads.fa", "-Z ref.fa reads.fa", "ref.fa reads.fa -k", "-x", "--split-prefix", "", "ref.fa",
    "-k 0 ref.fa reads.fa", "-w 0 ref.fa reads.fa", "-N -1 ref.fa reads.fa", "-p 1.5 ref.fa reads.fa", "--for-only --rev-only ref.fa reads.fa",
    "-O 0 ref.fa reads.fa", "-O 4,24 -E 1,2 ref.fa reads.fa", "-O 60,60 -E 10,5 ref.fa reads.fa", "-z 100,200 ref.fa reads.fa",
    "-X --secondary=no ref.fa reads.fa", "--splice --frag=yes ref.fa reads.fa", "--idx-no-seq -c ref.fa reads.fa", "--idx-no-seq ref.fa reads.fa",
]
# command lines the reference maps and the product refuses (with status 1): options it does not build
REFUSED = [
    "--heap-sort=yes ref.fa reads.fa", "--sr ref.fa reads.fa", "-T 20 ref.fa reads.fa", "--frag=yes ref.fa reads.fa",
    "-x splice -c ref.fa reads.fa", "-x splice -a ref.fa reads.fa", "-x cdna --cs ref.fa reads.fa", "-x splice --MD ref.fa reads.fa",
    "-u f -c -x map-ont ref.fa reads.fa", "--split-prefix pre ref.fa a.fa b.fa", "-k 29 ref.fa reads.fa", "-w 300 ref.fa reads.fa",
]
LINES = golden_lines() + HANDMADE


def argv(line):
    return line.split() if line else []


def digest(rec):
    status, dump = rec
    return {"status": status, "dump_md5": hashlib.md5(dump.encode()).hexdigest() if dump is not None else None}


def reference(line, tmp_path):
    live = cli_lib.parse_ref(argv(line), str(tmp_path / "ref.dump"), str(tmp_path))
    if live is not None:
        return live, digest(live)
    rec = json.load(open(DIGESTS)).get(line)
    if rec is None:
        pytest.skip("the reference's main() is not built here and the line has no recorded digest")
    return None, rec


def test_table_size():
    assert len(LINES) >= 100 and len(set(LINES)) == len(LINES)


@pytest.mark.parametrize("line", LINES)
def test_parse_matches_reference(line, tmp_path):
    live, rec = reference(line, tmp_path)
    ours = cli_lib.parse_host(argv(line), str(tmp_path / "ours.dump"))
    if live is not None:
        assert ours[0] == live[0], (ours, live)
        assert ours[1] == live[1]
    assert digest(ours) == rec


@pytest.mark.parametrize("line", REFUSED)
def test_parse_refuses(line, tmp_path):
    live, rec = reference(line, tmp_path)
    assert rec["status"] == 0 and rec["dump_md5"] is not None, "the reference maps this command line"
    assert cli_lib.parse_host(argv(line), str(tmp_path / "ours.dump")) == (1, None)


def test_record_reference_digests(tmp_path):
    if os.environ.get("WM_RECORD_REF") != "1":
        pytest.skip("WM_RECORD_REF=1 records the reference's digests")
    assert os.path.exists(cli_lib.REF_DUMP), "oracle/_ref/winnowmap_cli_dump is not built (oracle/build_cli_ref.sh)"
    rec = {}
    for line in LINES + REFUSED:
        rec[line] = digest(cli_lib.parse_ref(argv(line), str(tmp_path / "ref.dump"), str(tmp_path)))
    json.dump(rec, open(DIGESTS, "w"), indent=1, sort_keys=True)
