"""Print the PLANS and LAST_READER tables of test_layer_accesses_cpu.py from the library as built in this tree:

    python tests/make_layer_accesses_pins.py > pins.py

and paste them over the tables at the end of the test.  No device is needed."""
import sys
import tempfile
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from test_layer_accesses_cpu import deploy_nets, last_readers, plan_hashes  # noqa: E402

with tempfile.TemporaryDirectory() as tmp:
    nets = deploy_nets(Path(tmp))
    print("PLANS = {")
    for rel, f in nets.items():
        print(f"    {rel!r}: {{")
        for case, digest in plan_hashes(rel, f).items():
            print(f"        {case!r}: {digest!r},")
        print("    },")
    print("}")
    print("LAST_READER = {")
    for rel, reader in zip(nets, last_readers(Path(tmp), list(nets.values()))):
        print(f"    {rel!r}: {reader!r},")
    print("}")
