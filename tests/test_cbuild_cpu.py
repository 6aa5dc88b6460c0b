"""The oracles' cache key follows #include "...": a stale shared object built from an old included file is never loaded."""
import os
import shutil

import cbuild

HERE = os.path.dirname(os.path.abspath(__file__))


def test_key_covers_included_files_only(tmp_path):
    for name in ("transform_oracle.c", "pgo_oracle.c"):
        shutil.copy(os.path.join(HERE, name), tmp_path / name)
    (tmp_path / "unrelated.c").write_text("int unrelated;\n")
    src = str(tmp_path / "transform_oracle.c")
    k0 = cbuild.key(src)
    with open(tmp_path / "unrelated.c", "a") as f:
        f.write("int edited;\n")
    assert cbuild.key(src) == k0
    with open(tmp_path / "pgo_oracle.c", "a") as f:
        f.write("\n/* edited */\n")
    assert cbuild.key(src) != k0
