"""The device-memory layout helper (structure-plp-slam_b200/csrc/layout.h) placed at fake device and host bases on the CPU:
alignment, no overlaps, inputs as the copied prefix, null inputs, a job struct patched before it is copied, aliases."""
import json
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

DRIVER = r"""
#include <stdio.h>
#include <stdint.h>
#include <vector>
#include "layout.h"

struct Job {
    int n;
    const float *a;
    const int32_t *b;
    const uint8_t *none;
    float *o1;
    uint32_t *o2;
    const float *alias;
};

static const uintptr_t kDev = 0x7f0000000000ull;

static long long off(const void *p) { return p ? (long long)((uintptr_t)p - kDev) : -1; }

int main() {
    float a[10];
    int32_t b[3];
    for (int i = 0; i < 10; ++i) a[i] = 0.5f * i;
    for (int i = 0; i < 3; ++i) b[i] = 100 + i;
    Job J = {};
    J.n = 7;
    J.none = (const uint8_t *)&J;  // must be overwritten with null
    const Job *dj = nullptr;
    plp::DevLayout L;
    L.in(J.a, a, 10);
    L.out(J.o1, 100);
    L.in(J.none, (const uint8_t *)nullptr, 5);
    L.in(J.b, b, 3, 70);
    L.out(J.o2, 1);
    L.same(J.alias, J.o1);
    L.in(dj, &J, 1);
    std::vector<uint8_t> host(L.bytes(), 0xCD);
    const size_t copied = L.place((uint8_t *)kDev, host.data());
    const Job *img = (const Job *)(host.data() + off(dj));
    const float *ha = (const float *)(host.data() + off(J.a));
    const int32_t *hb = (const int32_t *)(host.data() + off(J.b));
    bool data_ok = true;
    for (int i = 0; i < 10; ++i) data_ok = data_ok && ha[i] == a[i];
    for (int i = 0; i < 3; ++i) data_ok = data_ok && hb[i] == b[i];
    printf("{\"bytes\": %zu, \"in_bytes\": %zu, \"copied\": %zu, \"data_ok\": %d, \"host_of_o2\": %lld,\n",
           L.bytes(), L.in_bytes(), copied, data_ok ? 1 : 0, (long long)((uint8_t *)L.host(J.o2) - host.data()));
    printf(" \"pieces\": {\"a\": [%lld, %zu, \"in\"], \"b\": [%lld, %zu, \"in\"], \"job\": [%lld, %zu, \"in\"],"
           " \"o1\": [%lld, %zu, \"out\"], \"o2\": [%lld, %zu, \"out\"]},\n",
           off(J.a), sizeof(float) * 10, off(J.b), sizeof(int32_t) * 70, off(dj), sizeof(Job), off(J.o1),
           sizeof(float) * 100, off(J.o2), sizeof(uint32_t));
    printf(" \"b_copied\": %zu, \"job_bytes\": %zu, \"none\": %lld, \"alias\": %lld,\n", sizeof(int32_t) * 3, sizeof(Job),
           off(J.none), off(J.alias));
    printf(" \"image\": {\"n\": %d, \"a\": %lld, \"b\": %lld, \"none\": %lld, \"o1\": %lld, \"o2\": %lld, \"alias\": %lld}}\n",
           img->n, off(img->a), off(img->b), off(img->none), off(img->o1), off(img->o2), off(img->alias));
    return 0;
}
"""


@pytest.fixture(scope="module")
def placed(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    d = tmp_path_factory.mktemp("layout")
    (d / "driver.cc").write_text(DRIVER)
    exe = d / "driver"
    cmd = ["g++", "-O1", "-std=c++17", "-Wall", "-Werror", f"-I{ROOT / 'structure-plp-slam_b200' / 'csrc'}",
           str(d / "driver.cc"), "-o", str(exe)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[:3000]
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    return json.loads(out)


def test_pieces_are_aligned_and_disjoint(placed):
    spans = sorted((off, off + size) for off, size, _ in placed["pieces"].values())
    for lo, _ in spans:
        assert lo % 256 == 0
    for (_, hi), (lo, _) in zip(spans, spans[1:]):
        assert hi <= lo
    assert spans[-1][1] <= placed["bytes"]
    assert placed["bytes"] % 256 == 0


def test_inputs_form_the_copied_prefix(placed):
    p = placed["pieces"]
    ins = [v for v in p.values() if v[2] == "in"]
    outs = [v for v in p.values() if v[2] == "out"]
    assert max(off + size for off, size, _ in ins) <= min(off for off, _, _ in outs)
    # the copy ends at the last input's copied bytes: the job struct, declared last
    assert placed["copied"] == placed["in_bytes"] == p["job"][0] + placed["job_bytes"]
    assert p["b"][0] + placed["b_copied"] <= placed["in_bytes"]
    assert placed["data_ok"] == 1


def test_outputs_lie_outside_the_copy(placed):
    for off, _, kind in placed["pieces"].values():
        if kind == "out":
            assert off >= placed["in_bytes"]
    assert placed["host_of_o2"] == placed["pieces"]["o2"][0]


def test_null_source_gives_null_field_and_no_bytes(placed):
    assert placed["none"] == -1
    # a (10 floats), b (70 int32), the job, o1 (100 floats), o2: one 256-byte granule each except b (280 B -> 512)
    assert placed["bytes"] == 256 + 512 + 256 + 512 + 256


def test_struct_input_holds_patched_addresses(placed):
    img, p = placed["image"], placed["pieces"]
    assert img["n"] == 7
    assert img["a"] == p["a"][0] and img["b"] == p["b"][0]
    assert img["o1"] == p["o1"][0] and img["o2"] == p["o2"][0]
    assert img["none"] == -1
    assert img["alias"] == placed["alias"] == p["o1"][0]
