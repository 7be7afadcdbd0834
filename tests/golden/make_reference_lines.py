"""Writes tests/golden/reference_lines.json: the line count of every file of a pbs-plus checkout (the commit the
documents cite, 26d6969) whose name the documents cite, keyed by path relative to the checkout.  The citation test
(tests/test_citations_cpu.py) checks every file:line citation of the documents against it; rerun this when a
document starts citing another file.

    python tests/golden/make_reference_lines.py <pbs-plus checkout>
"""
import importlib.util
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]


def main():
    ref = Path(sys.argv[1]).resolve()
    spec = importlib.util.spec_from_file_location("cites", ROOT / "tests" / "test_citations_cpu.py")
    t = importlib.util.module_from_spec(spec)
    (HERE / "reference_lines.json").write_text("{}")   # the test module reads it on import
    spec.loader.exec_module(t)
    names = {m.group(1).split("/")[-1] for doc in t.DOCS for m in t.CITE.finditer((ROOT / doc).read_text())}
    names |= {p.split("/")[-1] for p in t.ALIASES.values()}
    lines = {str(p.relative_to(ref)): sum(1 for _ in p.open(errors="replace"))
             for p in sorted(ref.rglob("*")) if p.is_file() and p.name in names}
    body = ",\n".join(f'"{k}": {v}' for k, v in lines.items())
    (HERE / "reference_lines.json").write_text("{\n" + body + "\n}\n")


if __name__ == "__main__":
    main()
