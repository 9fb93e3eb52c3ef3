"""The math the device and the oracle must compute alike has one text, in structure-plp-slam_b200/csrc/, and the oracle
compiles those files.  A header of the same name under oracle/ would shadow the shared one without any error, because a
quoted include searches the including file's directory first."""
from pathlib import Path

import oracle_api

ROOT = Path(__file__).resolve().parent.parent
ORACLE = ROOT / "oracle"
CSRC = ROOT / "structure-plp-slam_b200" / "csrc"
HEADER_SUFFIXES = (".h", ".cuh", ".hpp", ".inc")
SHARED = {"cammath.h", "detmath.h", "essmath.h", "planemath.h", "pnpmath.h", "sim3math.h", "sim3optmath.h", "rectmath.h",
          "brief_pattern.inc"}


def test_no_oracle_file_has_the_name_of_a_library_header():
    headers = {p.name for p in CSRC.iterdir() if p.suffix in HEADER_SUFFIXES}
    assert not headers & {p.name for p in ORACLE.iterdir()}


def test_oracle_compiles_the_library_headers():
    """The dependency lists g++ wrote (-MMD) while oracle/Makefile compiled each object with its own flags."""
    oracle_api.lib()
    found = set()
    for d in sorted((ORACLE / "_build").glob("*.d")):
        rule = d.read_text().replace("\\\n", " ").split("\n", 1)[0]
        for dep in rule.split(":", 1)[1].split()[1:]:  # the first prerequisite is the .cc itself
            path = (ORACLE / dep).resolve()
            if (CSRC / path.name).exists():
                assert path == CSRC / path.name, f"{d.name}: {dep}"
                found.add(path.name)
    assert SHARED <= found, SHARED - found
