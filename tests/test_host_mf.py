"""CPU suite: the host writers with the most-frequent-base consensus (-a 1) on oracle-aligned graphs of the golden inputs,
against the reference CLI's output (md5s in tests/golden/reference_runs_mf.json, see tests/mf_reference.py), as
test_host_layer.py::test_writers_match_reference_cli_md5 does for heaviest bundling; and the values that keep aborting."""
import ctypes as C
import subprocess
import sys

import pytest

from abpoa_b200 import capi
from abpoa_b200.aligner import PoaConfig, PoaSession
from gfa_reference import md5, reference_cli_md5, with_file
from helpers import INPUTS, read_fasta
from mf_reference import mf_cfg, mf_reference, set_outputs
from oracle_binding import oracle_align


@pytest.fixture(scope="module")
def reference():
    ref = mf_reference()
    yield ref
    ref.save()


def _fasta_names(path):
    return [ln[1:].split()[0] for ln in path.read_text().splitlines() if ln.startswith(">")]


@pytest.mark.parametrize("r", [0, 2, 4, 5])
@pytest.mark.parametrize("fname", ["seq.fa", "test.fa", "heter.fa"])
def test_host_mf_writers_match_reference_cli(product_lib, reference, fname, r):
    reads = read_fasta(INPUTS / fname)
    names = _fasta_names(INPUTS / fname)
    with PoaSession(mf_cfg(), product_lib) as s:
        set_outputs(s.lib, s.abpt, r)
        s.reset(max(len(x) for x in reads))
        abs_ = s.ab.contents.abs.contents
        for x in reads:
            _, res = oracle_align(s, x)
            s.add(x, res, len(reads))
        for i, nm in enumerate(names):           # names as abpoa_msa() would have stored them
            b = nm.encode()
            buf = capi.libc_realloc(None, len(b) + 1)
            C.memmove(buf, b + b"\0", len(b) + 1)
            abs_.name[i].s = C.cast(buf, C.c_char_p)
            abs_.name[i].l = len(b)
            abs_.name[i].m = len(b) + 1
        got = with_file(lambda fp: product_lib.abpoa_output(s.ab, s.abpt, fp))
    assert md5(got) == reference_cli_md5(reference, ["-a", "1", "-r", str(r)], [INPUTS / fname]), f"-a 1 -r {r} {fname}"


@pytest.mark.parametrize("setting,message", [("a.max_n_cons = 2", "max_n_cons > 1"), ("a.cons_algrm = 2", "unknown consensus algorithm")])
def test_other_consensus_settings_still_abort(setting, message, tmp_path):
    """-d 2 (with or without -a 1) and -a 2 still end in poa_die: a clean exit with a message."""
    code = (
        "import sys; sys.path.insert(0, 'tests')\n"
        "from abpoa_b200.aligner import PoaSession\n"
        "from abpoa_b200.capi import product\n"
        "from mf_reference import mf_cfg\n"
        "from oracle_binding import oracle_align\n"
        "from helpers import INPUTS, read_fasta\n"
        "reads = read_fasta(INPUTS / 'seq.fa')\n"
        "with PoaSession(mf_cfg(), product()) as s:\n"
        "    a = s.abpt.contents\n"
        "    s.reset(max(len(x) for x in reads))\n"
        "    for x in reads:\n"
        "        _, res = oracle_align(s, x)\n"
        "        s.add(x, res, len(reads))\n"
        f"    {setting}\n"
        "    s.lib.abpoa_generate_consensus(s.ab, s.abpt)\n"
    )
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    p = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=300)
    assert p.returncode != 0 and message in p.stderr, (p.returncode, p.stderr[-2000:])
