"""Run an UNMODIFIED reference script on the CUDA engine.

    python -m drawingspinup_b200.run /path/to/3_style_translator/test_stage1.py --uid <uid>

Changes into the script's folder (the scripts use relative ``configs/...`` paths,
test_stage1.py:23), imports the reference's ``training.models``, rebinds ``GeneratorJ_RIC`` and
``GeneratorJ`` to the engine classes (see :func:`drawingspinup_b200.install`) and executes the script
as ``__main__``.  Everything else in the script - YAML parsing, ``torch.load``,
``load_state_dict``, the DataLoader, PNG writing - is the reference's own code.
"""
from __future__ import annotations

import os
import runpy
import sys


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        print(__doc__)
        return 2
    script = os.path.abspath(argv[0])
    folder = os.path.dirname(script)
    os.chdir(folder)
    if folder not in sys.path:
        sys.path.insert(0, folder)
    import drawingspinup_b200
    drawingspinup_b200.install()
    sys.argv = [script] + argv[1:]
    runpy.run_path(script, run_name="__main__")
    return 0


if __name__ == "__main__":
    sys.exit(main())
