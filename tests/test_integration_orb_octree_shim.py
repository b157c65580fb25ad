"""The strategy-10 shim (integration/ORB_OCTREE_B200.cpp) is real C++: compiled -Werror against the stand-ins of the reference headers
(integration/stubs) and include/lcd_b200.h, linked against liblcd_b200.so, and on the GPU run through Feature2D's own entry points: it
detects what lcd_orb_detect_describe detects with ORB-OCTREE selected, and what the restatement (oracle/orb_octree_py.py) detects."""
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
LIB = ROOT / "rtabmap_b200" / "lib"
INC = ["-I", str(ROOT / "integration" / "stubs"), "-I", str(ROOT / "include")]

DRIVER = r"""
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <rtabmap/core/Features2d.h>
namespace rtabmap { Feature2D * createOrbOctreeB200(const ParametersMap & parameters); }
int main(int argc, char ** argv)
{
	const int w = std::atoi(argv[2]), h = std::atoi(argv[3]);
	std::vector<unsigned char> img(static_cast<size_t>(w) * h);
	FILE * f = std::fopen(argv[1], "rb");
	if (!f || std::fread(img.data(), 1, img.size(), f) != img.size()) return 2;
	std::fclose(f);
	rtabmap::ParametersMap p{{"Kp/MaxFeatures", "700"}, {"ORB/ScaleFactor", "1.2"}, {"ORB/NLevels", "8"}, {"FAST/MinThreshold", "9"}};
	rtabmap::Feature2D * d = rtabmap::createOrbOctreeB200(p);
	if (d->getType() != rtabmap::Feature2D::kFeatureOrbOctree) return 3;
	cv::Mat m(h, w, CV_8U);
	std::copy(img.begin(), img.end(), m.data);
	std::vector<cv::KeyPoint> kps = d->generateKeypoints(m);
	cv::Mat desc = d->generateDescriptors(m, kps);
	FILE * o = std::fopen(argv[4], "wb");
	for (const cv::KeyPoint & k : kps)
	{
		const float row[6] = {k.pt.x, k.pt.y, k.size, k.angle, k.response, static_cast<float>(k.octave)};
		std::fwrite(row, sizeof(float), 6, o);
	}
	std::fclose(o);
	o = std::fopen(argv[5], "wb");
	if (!kps.empty()) std::fwrite(desc.data, 1, kps.size() * 32, o);
	std::fclose(o);
	delete d;
	std::printf("octree shim ok %d\n", static_cast<int>(kps.size()));
	return 0;
}
"""


def test_orb_octree_shim_compiles_and_links_against_the_c_abi(tmp_path):
    import rtabmap_b200

    rtabmap_b200.load_library()
    obj = tmp_path / "ORB_OCTREE_B200.o"
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-fPIC", *INC, "-c", str(ROOT / "integration" / "ORB_OCTREE_B200.cpp"),
                        "-o", str(obj)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run(["g++", "-shared", "-o", str(tmp_path / "liboctree_shim.so"), str(obj), "-L", str(LIB), "-llcd_b200", "-Wl,--no-undefined",
                        f"-Wl,-rpath,{LIB}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


@pytest.mark.gpu
def test_orb_octree_shim_runs_against_the_engine(tmp_path):
    from oracle import orb_octree_py as oc
    from rtabmap_b200 import Engine, synth

    (tmp_path / "driver.cpp").write_text(DRIVER)
    exe = tmp_path / "octree_driver"
    r = subprocess.run(["g++", "-std=c++17", "-O1", *INC, str(tmp_path / "driver.cpp"), str(ROOT / "integration" / "ORB_OCTREE_B200.cpp"), "-o", str(exe),
                        "-L", str(LIB), "-llcd_b200", f"-Wl,-rpath,{LIB}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    img = synth.make_image(480, 640, 77)
    img.tofile(tmp_path / "img.raw")
    r = subprocess.run([str(exe), str(tmp_path / "img.raw"), "640", "480", str(tmp_path / "kp.bin"), str(tmp_path / "desc.bin")], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0 and "octree shim ok" in r.stdout, r.stdout + r.stderr
    kp = np.fromfile(tmp_path / "kp.bin", np.float32).reshape(-1, 6)
    desc = np.fromfile(tmp_path / "desc.bin", np.uint8).reshape(-1, 32)
    p = oc.OctreeParams(n_features=700, scale_factor=1.2, n_levels=8, fast_min_threshold=9)
    want_kp, want_desc, _ = oc.detect_describe_octree(img, None, synth.CAMERA_K4, p)
    eng = Engine()
    eng.set_detector_orb_octree(9)
    got_kp, got_desc, _ = eng.orb_detect_describe(img[None], None, Engine.orb_params(synth.CAMERA_K4, n_features=700, n_levels=8,
                                                                                         scale_factor=1.2))[0]
    assert len(kp) == 700
    assert np.array_equal(kp.view(np.uint32), got_kp.view(np.uint32)) and np.array_equal(desc, got_desc)
    assert np.array_equal(kp.view(np.uint32), want_kp.view(np.uint32)) and np.array_equal(desc, want_desc)
