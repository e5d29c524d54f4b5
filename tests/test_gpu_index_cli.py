"""GPU end-to-end: mapping with homopolymer-compressed (map-pb, ava-pb, -H), even-k and wide-window (w + k > 64) indexes, an HPC
index in -I parts, and an HPC index file this library wrote with -d, on homopolymer-rich inputs, against the reference binary's
recorded output (tests/golden/expected/reference_lines.json). With HPC a seed's span differs from k; the span reaches chaining,
mm_align1's anchor coordinates and mm_est_err, which only a whole mapping run compares."""
import os
import subprocess
import pytest
import index_cases as IC
import oracle_lib as O

pytestmark = pytest.mark.gpu
MINE = os.path.join(O.ROOT, "minimap2_b200", "minimap2-b200")


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("hpc_cli"))
    return d, IC.cli_inputs(d, "hpc", 240_000, 60, 17)


def run(args, cwd):
    p = subprocess.run([MINE, "-t", "8"] + args, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=1200)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    return p.stdout.decode().splitlines()


@pytest.mark.parametrize("i", range(7))
def test_index_options_match_reference(inputs, i):
    d, (rf, qf) = inputs
    args = IC.cli_lines(rf, qf)[i]
    ref = O.reference_lines(args, d)
    O.assert_matches_reference(run(args, d), ref)
    assert len(ref) >= 20


def test_mapping_through_an_hpc_index_file_written_here(inputs):
    """`-x map-pb -d` of this library, then mapping through that file, gives the reference's output of mapping against the FASTA"""
    d, (rf, qf) = inputs
    run(["-x", "map-pb", "-d", "hpc.mmi", rf], d)
    part, = IC.parse_mmi(open(os.path.join(d, "hpc.mmi"), "rb").read())
    assert part.hdr[:2] == (10, 19) and part.hdr[4] & IC.MM_I_HPC
    O.assert_matches_reference(run(["-x", "map-pb", "-c", "--cs", "hpc.mmi", qf], d), O.reference_lines(IC.cli_lines(rf, qf)[0], d))
