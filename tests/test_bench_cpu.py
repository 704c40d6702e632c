"""bench.py host logic that can run without a GPU: the reference (CPU) arm and its isolation from the product."""
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_runs_the_staged_reference_and_never_maps_the_product_library():
    """`bench.py --impl reference` must time the reference's own code (kind "reference" when tools/ref_import.py
    finds a checkout of it, else the oracle port) and must not dlopen libstylesinger_b200.so (VERDICT r1: the
    round-1 arm imported stylesinger_b200.dist -> engine -> _lib)."""
    code = (
        "import sys, json, io, contextlib\n"
        f"sys.path.insert(0, {REPO!r}); sys.argv = ['bench.py', '--impl', 'reference', '--steps', '1', '--warmup', '1', '--T', '2', "
        "'--cpu-sample-seconds', '0.3']\n"
        "import bench\n"
        "buf = io.StringIO()\n"
        "with contextlib.redirect_stdout(buf):\n"
        "    bench.main()\n"
        "line = [l for l in buf.getvalue().splitlines() if l.startswith('{')][-1]\n"
        "maps = open('/proc/self/maps').read()\n"
        "print('RESULT ' + json.dumps({'line': json.loads(line), 'mapped': 'libstylesinger_b200' in maps}))\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, cwd=REPO)
    assert r.returncode == 0, r.stderr[-2000:]
    res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])
    assert res["mapped"] is False
    line = res["line"]
    assert line["impl"] == "reference" and line["gpu_launches"] == 0 and line["value"] > 0
    assert line["cpu_baseline"]["kind"] in ("reference", "port")
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0
    have_ref = any(c and os.path.isdir(os.path.join(c, "modules", "StyleSinger"))  # tools/ref_import.py find_reference()
                   for c in (os.environ.get("STYLESINGER_REF"), os.path.join(REPO, "baseline", "_ref", "StyleSinger")))
    assert line["cpu_baseline"]["kind"] == ("reference" if have_ref else "port")
