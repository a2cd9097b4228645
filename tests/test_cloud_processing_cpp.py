"""The C++ mirror of cloudProcessing in include/srlivo_b200_lio.hpp (srl::cloudProcessing): it builds at the reference's language
level (-std=c++14) against the library, throws without a GPU instead of falling back to anything, and on the GPU decodes a
message, cuts it and reports the queue's front / back / size as the restated handler does."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cloud_processing_ref as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROGRAM = r'''
#include <cstdio>
#include <fstream>
#include <iterator>
#include <vector>
#include "srlivo_b200_lio.hpp"
int main(int argc, char** argv) {
    srl_ctx* ctx = nullptr;
    try {
        if (srl_ctx_create(0, nullptr, &ctx) != SRL_OK) throw std::runtime_error("srl_ctx_create: no CUDA device (no CPU fallback)");
        // Ouster at config/ntu.yaml's parameters: 16 rings, 20 Hz, ns, blind 4, point_filter_num 4
        srl::cloudProcessing cp(ctx, 3, 16, 20, 3, 4.0, 4, 64);
        std::ifstream f(argv[1], std::ios::binary);
        std::vector<uint8_t> data((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        srl_cloud2_layout y{48, 0, 4, 8, 20, 26, 0, 0};
        const double stamp = 1.7e9;
        const int64_t appended = cp.process(data.data(), data.size() / 48, y, stamp);
        std::vector<double> xyz, rel, ts;
        cp.download(xyz, rel, ts);
        const double front = cp.frontTimestamp(), back = cp.backTimestamp();
        const size_t size = cp.size();
        const double* d_xyz = nullptr;
        const double* d_ts = nullptr;
        const int64_t popped = cp.cut(ts[ts.size() / 2], &d_xyz, &d_ts);
        std::printf("appended=%lld size=%zu given=%d interval=%.17g type=%d front=%.17g back=%.17g popped=%lld left=%zu ptr=%d\n",
                    (long long)appended, size, (int)cp.isPointTimeEnable(), cp.getSweepInterval(), cp.getLidarType(), front, back,
                    (long long)popped, cp.size(), d_xyz != nullptr && d_ts != nullptr);
        srl_ctx_destroy(ctx);
        return 0;
    } catch (const std::exception& e) {
        std::printf("threw: %s\n", e.what());
        if (ctx) srl_ctx_destroy(ctx);
        return 3;
    }
}
'''


@pytest.fixture(scope="module")
def program(tmp_path_factory):
    from sr_livo_b200 import capi
    d = tmp_path_factory.mktemp("cp_cpp")
    src, exe = d / "cp.cpp", d / "cp"
    src.write_text(PROGRAM)
    libdir = os.path.dirname(capi.LIB_PATH)
    subprocess.check_call(["g++", "-std=c++14", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                           "-L", libdir, "-lsrlivo_b200", f"-Wl,-rpath,{libdir}"])
    msg = R.cloud2(R.OUST, 11, 16, 128, scan_rate=20)
    (d / "msg.bin").write_bytes(msg.tobytes())
    return exe, d / "msg.bin", msg


def test_cpp_mirror_compiles_and_throws_without_a_gpu(program):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the GPU test runs the program")
    exe, path, _ = program
    r = subprocess.run([str(exe), str(path)], capture_output=True, text=True)
    assert r.returncode == 3 and "no CPU fallback" in r.stdout, r.stdout


@pytest.mark.gpu
def test_cpp_mirror_runs_the_handler_and_the_cut(program):
    exe, path, msg = program
    r = subprocess.run([str(exe), str(path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = dict(kv.split("=") for kv in r.stdout.split())
    ref = R.CloudProcessingRef(R.OUST, 16, 20, R.NS, 4.0, 4)
    appended = ref.process(msg, 1.7e9)
    ts = [q[4] for q in ref.queue]
    assert int(got["appended"]) == appended == int(got["size"]) and got["given"] == "1" and got["type"] == "3"
    assert float(got["interval"]) == ref.getSweepInterval()
    assert float(got["front"]) == ts[0] and float(got["back"]) == ts[-1]
    popped = ref.cut(ts[len(ts) // 2])
    assert int(got["popped"]) == len(popped) and int(got["left"]) == len(ref.queue) and got["ptr"] == "1"
