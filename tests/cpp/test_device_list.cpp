// test_device_list.cpp -- w2xc::gpuRuntime's W2X_DEVICES parsing and GPU count (host/w2xc.hpp); needs no device.
// Exit code 0 on success; prints CHECK lines.
#include <cstdio>
#include <cstdlib>

#include "w2xc.hpp"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("CHECK FAILED line %d: %s\n", __LINE__, #c); fails++; } } while (0)

int main() {
    using w2xc::gpuRuntime;
    std::vector<int> ids;
    CHECK(gpuRuntime::parseDeviceList("0", ids) && ids == std::vector<int>({0}));
    CHECK(gpuRuntime::parseDeviceList("0,0", ids) && ids == std::vector<int>({0, 0}));
    CHECK(gpuRuntime::parseDeviceList("3,0,12", ids) && ids == std::vector<int>({3, 0, 12}));
    for (const char *bad : {"", ",", "0,", ",0", "0,,1", "a", "1,b", "-1", "+1", " 1", "1 ", "1, 2", "1;2", "99999999999"})
        CHECK(!gpuRuntime::parseDeviceList(bad, ids));
    CHECK(!gpuRuntime::parseDeviceList(nullptr, ids));
    std::string many = "0";
    for (int i = 1; i < 64; i++) many += ",0";
    CHECK(gpuRuntime::parseDeviceList(many.c_str(), ids) && ids.size() == 64);
    CHECK(!gpuRuntime::parseDeviceList((many + ",0").c_str(), ids));

    unsetenv("W2X_DEVICES");
    unsetenv("W2X_GPUS");
    CHECK(gpuRuntime::plannedNumberOfGpus(0) == 1);
    CHECK(gpuRuntime::plannedNumberOfGpus(3) == 3);
    setenv("W2X_GPUS", "2", 1);
    CHECK(gpuRuntime::plannedNumberOfGpus(0) == 2);
    CHECK(gpuRuntime::plannedNumberOfGpus(1) == 2);
    CHECK(gpuRuntime::plannedNumberOfGpus(4) == 4);
    setenv("W2X_DEVICES", "5,1,5", 1);                     // the list overrides both
    CHECK(gpuRuntime::plannedNumberOfGpus(0) == 3);
    CHECK(gpuRuntime::plannedNumberOfGpus(2) == 3);
    setenv("W2X_DEVICES", "5", 1);
    CHECK(gpuRuntime::plannedNumberOfGpus(0) == 1);
    std::printf(fails ? "FAILED\n" : "ALL OK\n");
    return fails ? 1 : 0;
}
