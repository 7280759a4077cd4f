"""`ptgnn_b200.overlay.install()` without the reference's packages on the path: only the torch_scatter shim is installed.
Runs in a fresh interpreter because the point is import order."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_overlay_without_reference_installs_only_the_shim():
    code = ("import sys; sys.path.insert(0, %r)\nimport ptgnn_b200.overlay as ov\nr = ov.install(force_torch_scatter=True)\n"
            "import torch_scatter\nassert torch_scatter.__name__ == 'ptgnn_b200.torch_scatter_shim'\n"
            "assert r['layers'] is False and 'note' in r, r\nprint('SHIM-OK')\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "SHIM-OK" in r.stdout, r.stdout + r.stderr[-3000:]
