"""The table of test_shim_args_gpu.py has one row for every entry point the four torch modules export, so a new entry
point without a row fails here, on a machine without a GPU."""
import dpvo_b200
from test_shim_args_gpu import MODULES, ROWS


def test_the_argument_table_covers_every_entry_point():
    exported = {"%s.%s" % (name, fn) for name, mod in zip(MODULES, dpvo_b200.extensions()) for fn in dir(mod) if not fn.startswith("_")}
    assert set(ROWS) == exported, {"without a row": sorted(exported - set(ROWS)), "not exported": sorted(set(ROWS) - exported)}
