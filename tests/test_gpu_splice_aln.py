"""Spliced base-level alignment on the GPU: every splice_aln_* golden (-c / -a with the splice presets, --splice, --cs, --MD,
--eqx -Y, -u f / r / n, --splice-flank=no, -C, -H, -I --split-prefix, --cap-sw-mem, -G) reproduced by
Mapper(..., spliced_alignment=True).map_file, whose DP runs on the ksw_exts2 kernel."""
import pytest

from test_splice_aln_cpu import MANIFEST, check_output, inputs

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(MANIFEST))
def test_gpu_spliced_alignment_matches_reference(name, tmp_path):
    from winnowmap_b200.mapper import Mapper
    lo = MANIFEST[name]["lib"]
    ref, reads, wfile = inputs(name, str(tmp_path))
    mp = Mapper(ref, wfile, preset=lo["preset"], cigar=True, sam=lo.get("sam", False), hpc=lo.get("hpc", False), splice=lo.get("splice", False),
                max_intron_len=lo.get("max_intron_len"), part_bases=lo.get("part_bases"), split=lo.get("split", False), spliced_alignment=True)
    try:
        mp.mo.flag = (mp.mo.flag | lo.get("set_flags", 0)) & ~lo.get("clear_flags", 0)
        if lo.get("noncan", -1) >= 0:
            mp.mo.noncan = lo["noncan"]
        mp.mo.max_sw_mat = lo.get("max_sw_mat", 0)
        out = str(tmp_path / "o.out")
        mp.map_file(reads, out)
        assert mp.stats()["n_dp_jobs"] > 0
    finally:
        mp.close()
    check_output(name, out)
