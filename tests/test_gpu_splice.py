"""Spliced mapping without base alignment on the GPU: the cDNA instantiations of every chaining formulation through the C ABI
(wm_chain_dp_batch_cdna) against the oracle's mm_chain_dp(is_cdna = 1), under each launch configuration of
test_gpu_task_loops.py; every splice_* golden reproduced by Mapper.map_file; one spliced run through the CUDA-vs-oracle tee."""
import os
import subprocess
import sys

import numpy as np
import pytest

import splice_lib as S
import tee_lib as T
from test_gpu_task_loops import CHAIN_CONFIGS, ROOT_DIR, _cfg_id, _pack, _unpack
from test_oracle_vs_ref import make_anchors
from test_splice_cpu import MANIFEST, SPLICE_CHAIN, check_golden, giant_spliced, spliced_anchors, splice_inputs

pytestmark = pytest.mark.gpu

_CHILD = r'''
import sys
sys.path.insert(0, %r)
import numpy as np
from winnowmap_b200 import kernels
src, dst = sys.argv[1:3]
z = np.load(src)
cat, off = z["a"], z["a_off"]
arrays = [cat[off[i]:off[i + 1]].reshape(-1, 2) for i in range(len(off) - 1)]
out = {}
for k, (mx, mn, my, bw, skip, it) in enumerate(z["prm"].tolist()):
    got = kernels.chain_dp_batch(arrays, mx, mn, my, bw, max_skip=skip, max_iter=it, is_cdna=True)
    for p, lst in (("u%%d" %% k, [u for u, _ in got]), ("b%%d" %% k, [b for _, b in got])):
        out[p] = np.concatenate([np.asarray(x).reshape(-1) for x in lst])
        out[p + "_off"] = np.cumsum([0] + [np.asarray(x).size for x in lst])
np.savez(dst, **out)
print("child ok")
''' % ROOT_DIR


@pytest.fixture(scope="module")
def cdna_case(tmp_path_factory):
    """Giant spliced tasks whose 200 kb windows reach more than 4096 anchors back (the tile kernel's deep path), medium and small
    transcript-like and random tasks (the rings), in one call."""
    rng = np.random.default_rng(97)
    giant = [giant_spliced(rng) for _ in range(3)] + [make_anchors(rng, 5000, repeats=True)]
    for a in giant[:3]:
        x = a[:, 0].astype(np.int64)
        assert (np.searchsorted(x, x - 200000) < np.arange(len(a)) - 4096).any()
    medium = [spliced_anchors(rng, int(rng.integers(5, 60)), noise=int(rng.integers(0, 300))) for _ in range(300)]
    small = [spliced_anchors(rng, int(rng.integers(1, 4))) for _ in range(600)] + [make_anchors(rng, int(n)) for n in rng.integers(0, 129, 300)]
    arrays = giant + medium + small
    sizes = np.array([len(a) for a in arrays])
    assert (sizes > 2048).sum() >= 4 and ((sizes > 128) & (sizes <= 2048)).sum() > 100 and (sizes <= 128).sum() > 500
    arrays = [arrays[i] for i in rng.permutation(len(arrays))]
    src = str(tmp_path_factory.mktemp("cdna") / "in.npz")
    inp = {"prm": np.array(SPLICE_CHAIN, dtype=np.int64)}
    _pack(inp, "a", arrays)
    np.savez(src, **inp)
    exp = [[S.oracle_chain_cdna(a, mx, mn, my, bw, max_skip=skip, max_iter=it) for a in arrays] for mx, mn, my, bw, skip, it in SPLICE_CHAIN]
    return src, arrays, exp


@pytest.mark.parametrize("env", CHAIN_CONFIGS, ids=_cfg_id)
def test_cdna_chain_matches_oracle(cdna_case, env, tmp_path):
    src, arrays, exp = cdna_case
    dst = str(tmp_path / "out.npz")
    out = subprocess.run([sys.executable, "-c", _CHILD, src, dst], env=dict(os.environ, **env), stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, timeout=900)
    assert out.returncode == 0 and b"child ok" in out.stdout, out.stdout[-3000:].decode(errors="replace")
    z = np.load(dst)
    for k, prm in enumerate(SPLICE_CHAIN):
        us, bs = _unpack(z, f"u{k}"), _unpack(z, f"b{k}")
        for i, a in enumerate(arrays):
            ue, be = exp[k][i]
            assert np.array_equal(np.asarray(ue).reshape(-1), us[i]), (prm, i, len(a), "u")
            assert np.array_equal(np.asarray(be).reshape(-1), bs[i]), (prm, i, len(a), "b")


@pytest.mark.parametrize("name", sorted(MANIFEST))
def test_splice_golden_on_gpu(name, tmp_path):
    from winnowmap_b200.mapper import Mapper
    ref, reads, wfile = splice_inputs(name, tmp_path)
    mp = Mapper(ref, wfile, **MANIFEST[name]["lib"])
    out = str(tmp_path / "o.paf")
    mp.map_file(reads, out)
    mp.close()
    check_golden(name, open(out, "rb").read())


def test_splice_through_the_tee(tmp_path):
    """-x splice -W mapped by the CUDA backend and the oracle backend side by side, call by call: no call differs."""
    L = S.tee()
    ref, reads, wfile = splice_inputs("splice_W", tmp_path)
    out, rep = str(tmp_path / "o.paf"), str(tmp_path / "tee.txt")
    rc = L.wmt_tee_map_file_splice(ref.encode(), wfile.encode(), b"splice", 0, 0, reads.encode(), out.encode(), 8, 4 << 20, T.DEV_GPU, rep.encode())
    assert rc == 0
    r = T.Report(rep)
    assert r.n_mismatch == 0, r.text()
    assert r["seed.calls"] > 0
    check_golden("splice_W", open(out, "rb").read())
