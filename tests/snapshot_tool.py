"""The g++-built snapshot helper (tests/cpp/snapshot_test.cpp) and a Python restatement of the snapshot checksum
(fiesta_b200/csrc/fb_snapshot.h), shared by the CPU format tests and the GPU snapshot tests."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "snapshot_test.cpp")
_M = (1 << 64) - 1


def build(out_dir):
    """Compile the helper into out_dir and return its path."""
    exe = os.path.join(str(out_dir), "snapshot_test")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-Wextra", "-Werror", SRC, "-o", exe])
    return exe


def edit(exe, data, op, tmp_dir):
    """`data` (bytes) with the helper's edit `op` applied and every checksum recomputed."""
    src, dst = os.path.join(str(tmp_dir), "in.snap"), os.path.join(str(tmp_dir), "out.snap")
    with open(src, "wb") as f:
        f.write(data)
    subprocess.check_call([exe, "edit", src, dst, op])
    with open(dst, "rb") as f:
        return f.read()


def _mix(z):
    z = (z + 0x9E3779B97F4A7C15) & _M
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M
    return z ^ (z >> 31)


def checksum(data):
    """mix(n + sum_j mix(w_j ^ (j * K))) over the n little-endian 64-bit words of data."""
    n = len(data) // 8
    s = 0
    for j in range(n):
        w = int.from_bytes(data[8 * j:8 * j + 8], "little")
        s = (s + _mix(w ^ ((j * 0xD1B54A32D192ED03) & _M))) & _M
    return _mix((s + n) & _M)


def header(data):
    """mode, grid and stored tile count of a snapshot (offsets of fb_snapshot.h)."""
    mode = int.from_bytes(data[12:16], "little")
    grid = tuple(int.from_bytes(data[72 + 4 * i:76 + 4 * i], "little", signed=True) for i in range(3))
    return mode, grid, int.from_bytes(data[312:320], "little")


def cobs_words(data):
    """Every stored closest-obstacle record of a snapshot, tile after tile."""
    import numpy as np
    mode, g, n = header(data)
    tn = [(x + 7) // 8 for x in g]
    lst = np.frombuffer(data, np.uint32, n, 384)
    off = 384 + (4 * n + 7) // 8 * 8
    out = []
    for t in lst.tolist():
        tc = (t // (tn[2] * tn[1]), (t // tn[2]) % tn[1], t % tn[2])
        nv = int(np.prod([min(8, g[i] - 8 * tc[i]) for i in range(3)]))
        nf = 3 if mode == 0 else 2
        out.append(np.frombuffer(data, np.uint32, nv, off + 8 * nf * nv))
        off += 8 * (nf * nv + (nv + 1) // 2 + 1)
    return np.concatenate(out) if out else np.zeros(0, np.uint32)
