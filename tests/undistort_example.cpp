// A C++ caller of FrameView::UndistortKeyPoints / ComputeImageBounds (include/orb_b200/orb_slam3.hpp), built with plain g++ by
// tests/test_undistort_gpu.py: reads a rows x cols image and a camera (fx fy cx cy k1 k2 p1 p2 k3) from the directory the test wrote,
// extracts it with ORBextractor(1000, 1.2, 8, 20, 7), undistorts the keypoints and computes the bounds, then writes mvKeysUn to kpsUn.raw
// and prints the bounds' bit patterns and the keypoint count.
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "orb_b200/orb_slam3.hpp"

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const std::string dir = argv[1];
    int rows = 0, cols = 0;
    OrbPinholeCamera cam;
    {
        std::ifstream f(dir + "/dims.txt");
        f >> rows >> cols >> cam.fx >> cam.fy >> cam.cx >> cam.cy >> cam.k1 >> cam.k2 >> cam.p1 >> cam.p2 >> cam.k3;
    }
    std::ifstream fi(dir + "/image.raw", std::ios::binary);
    std::vector<uint8_t> img((std::istreambuf_iterator<char>(fi)), std::istreambuf_iterator<char>());
    if ((int)img.size() != rows * cols) return 3;
    ORB_SLAM3::ORBextractor ex(1000, 1.2f, 8, 20, 7, cols, rows);
    ORB_SLAM3::Image im;
    im.data = img.data(); im.rows = rows; im.cols = cols; im.step = (size_t)cols;
    std::vector<ORB_SLAM3::KeyPoint> mvKeys;
    ORB_SLAM3::Descriptors desc;
    std::vector<int> lap = {0, 1000};
    ex(im, ORB_SLAM3::Image(), mvKeys, desc, lap);
    ORB_SLAM3::FrameView F;
    F.UndistortKeyPoints(ex, cam, mvKeys);
    F.ComputeImageBounds(cam, cols, rows);
    std::ofstream fo(dir + "/kpsUn.raw", std::ios::binary);
    fo.write((const char*)F.mvKeysUn.data(), (std::streamsize)(F.mvKeysUn.size() * sizeof(ORB_SLAM3::KeyPoint)));
    const float b[4] = {F.mnMinX, F.mnMaxX, F.mnMinY, F.mnMaxY};
    uint32_t u[4];
    std::memcpy(u, b, sizeof(u));
    std::printf("n %zu\nbounds %08x,%08x,%08x,%08x\n", F.mvKeysUn.size(), u[0], u[1], u[2], u[3]);
    return 0;
}
