"""GPU end-to-end: the chaining options at their edges through the CLI, on the committed fixtures, against the reference binary's
recorded output (tests/golden/expected/reference_lines.json): --max-chain-iter 0 (every window emptied by the iteration cut),
--max-chain-skip 0, a skip penalty (--chain-skip-scale), and -r bandwidth pairs under which the long-join rescue re-chains reads:
the reference's recorded output for those differs from its output with --no-long-join, which the test checks."""
import os
import subprocess
import pytest
import oracle_lib as O

pytestmark = pytest.mark.gpu
MINE = os.path.join(O.ROOT, "minimap2_b200", "minimap2-b200")
DATA = os.path.join(O.ROOT, "tests", "golden", "data")
ONT = [os.path.join(DATA, "synth-ref.fa"), os.path.join(DATA, "synth-ont.fa")]
MT = [os.path.join(DATA, "MT-human.fa"), os.path.join(DATA, "MT-orang.fa")]

LINES = [["-x", "map-ont", "-c", "--max-chain-iter", "0"] + ONT,
         ["-x", "map-ont", "-c", "--max-chain-iter", "0"] + MT,
         ["-x", "map-ont", "--max-chain-skip", "0"] + ONT,
         ["-x", "map-ont", "-c", "--chain-skip-scale", "1"] + ONT,
         ["-x", "map-ont", "-c", "-r", "10,2000"] + ONT,
         ["-x", "map-hifi", "-c", "-r", "50,20000", os.path.join(DATA, "synth-ref.fa"), os.path.join(DATA, "synth-hifi.fa")]]
RESCUED = {4, 5}


@pytest.mark.parametrize("i", range(len(LINES)))
def test_chain_options_match_reference(i):
    ref = O.reference_lines(LINES[i])
    p = subprocess.run([MINE, "-t", "8"] + LINES[i], stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=1200)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    O.assert_matches_reference(p.stdout.decode().splitlines(), ref)
    assert len(ref) > 0
    if i in RESCUED:
        assert O.reference_lines(LINES[i][:-2] + ["--no-long-join"] + LINES[i][-2:]).all != ref.all
