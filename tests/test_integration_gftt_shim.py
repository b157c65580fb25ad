"""The strategy-8 shim (integration/GFTT_ORB_B200.cpp) is real C++: compiled -Werror against the stand-ins of the reference headers
(integration/stubs) and include/lcd_b200.h, linked against liblcd_b200.so, and on the GPU run through Feature2D's own entry points
against cv::GFTTDetector + cv::ORB::compute (oracle/gftt_py.py)."""
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
namespace rtabmap { Feature2D * createGfttOrbB200(const ParametersMap & parameters); }
int main(int argc, char ** argv)
{
	const int w = std::atoi(argv[2]), h = std::atoi(argv[3]);
	std::vector<unsigned char> img(static_cast<size_t>(w) * h);
	FILE * f = std::fopen(argv[1], "rb");
	if (!f || std::fread(img.data(), 1, img.size(), f) != img.size()) return 2;
	std::fclose(f);
	rtabmap::ParametersMap p{{"Kp/MaxFeatures", "700"}, {"GFTT/MinDistance", "5"}, {"GFTT/QualityLevel", "0.002"}};
	rtabmap::Feature2D * d = rtabmap::createGfttOrbB200(p);
	if (d->getType() != rtabmap::Feature2D::kFeatureGfttOrb) return 3;
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
	std::printf("gftt shim ok %d\n", static_cast<int>(kps.size()));
	return 0;
}
"""


def test_gftt_shim_compiles_and_links_against_the_c_abi(tmp_path):
    import rtabmap_b200

    rtabmap_b200.load_library()
    obj = tmp_path / "GFTT_ORB_B200.o"
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-fPIC", *INC, "-c", str(ROOT / "integration" / "GFTT_ORB_B200.cpp"),
                        "-o", str(obj)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run(["g++", "-shared", "-o", str(tmp_path / "libgftt_shim.so"), str(obj), "-L", str(LIB), "-llcd_b200", "-Wl,--no-undefined",
                        f"-Wl,-rpath,{LIB}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


@pytest.mark.gpu
def test_gftt_shim_runs_against_the_engine(tmp_path):
    from oracle import feature2d_py as f2d
    from oracle import gftt_py as gf
    from rtabmap_b200 import synth

    (tmp_path / "driver.cpp").write_text(DRIVER)
    exe = tmp_path / "gftt_driver"
    r = subprocess.run(["g++", "-std=c++17", "-O1", *INC, str(tmp_path / "driver.cpp"), str(ROOT / "integration" / "GFTT_ORB_B200.cpp"), "-o", str(exe),
                        "-L", str(LIB), "-llcd_b200", f"-Wl,-rpath,{LIB}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    img = synth.make_image(480, 640, 77)
    img.tofile(tmp_path / "img.raw")
    r = subprocess.run([str(exe), str(tmp_path / "img.raw"), "640", "480", str(tmp_path / "kp.bin"), str(tmp_path / "desc.bin")], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0 and "gftt shim ok" in r.stdout, r.stdout + r.stderr
    kp = np.fromfile(tmp_path / "kp.bin", np.float32).reshape(-1, 6)
    desc = np.fromfile(tmp_path / "desc.bin", np.uint8).reshape(-1, 32)
    want_kp, want_desc, _ = gf.detect_describe_gftt(img, None, synth.CAMERA_K4, f2d.OrbParams(n_features=700),
                                                    gf.GfttParams(quality_level=0.002, min_distance=5.0))
    assert len(kp) > 300
    assert np.array_equal(kp.view(np.uint32), want_kp.view(np.uint32))
    assert np.array_equal(desc, want_desc)
