"""Stack retirement in the C++ reporter mirror (Config::retireIdleBatches): retired traces register again on their next sighting,
live and zero-hash traces keep their handles, a cache entry replaced by a newer handle stays, and TraceCache deletion keeps every
other entry reachable across probe chains. CPU only, against a recording Sink."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reporter_retires_stacks():
    exe = os.path.join(ROOT, "tests", "cpp", "_build", "test_reporter_retire")
    src = os.path.join(ROOT, "tests", "cpp", "test_reporter_retire.cpp")
    so_dir = os.path.join(ROOT, "parca_agent_b200")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(src), os.path.getmtime(os.path.join(so_dir, "libparcaagg.so"))):
        subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, src, "-L" + so_dir, "-lparcaagg", "-Wl,-rpath," + so_dir, "-lpthread"], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "ok"
