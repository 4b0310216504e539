"""Writes tests/golden/sampling_sigmas.json: the reference's `get_sampling_sigmas` (fastvideo/sample/sample_5b.py, extracted with
`ast` because the script itself cannot be imported) evaluated at the (steps, shift) pairs the samplers use.
Usage: python tools/make_golden_sigmas.py <reference root>"""
import ast
import json
import sys
from pathlib import Path

import numpy as np

CASES = ((4, 7.0), (50, 3.0), (50, 5.0), (1, 7.0), (30, 1.0))


def main(ref_root: Path) -> None:
    src = ref_root / "fastvideo" / "sample" / "sample_5b.py"
    tree = ast.parse(src.read_text())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "get_sampling_sigmas")
    ns = {"np": np}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), str(src), "exec"), ns)
    out = [{"steps": s, "shift": sh, "sigmas": [float(x) for x in ns["get_sampling_sigmas"](s, sh)]} for s, sh in CASES]
    dst = Path(__file__).resolve().parents[1] / "tests" / "golden" / "sampling_sigmas.json"
    dst.write_text(json.dumps(out, indent=1) + "\n")
    print(f"wrote {dst}")


if __name__ == "__main__":
    main(Path(sys.argv[1]))
