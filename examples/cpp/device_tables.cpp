// The same program on the GPUs: tables live in HBM, Add / Get are the fused sm_90a kernels,
// all pointers are device pointers (include/multiverso/device/device.h). One process per GPU.
//
//   g++ -std=c++17 -Iinclude examples/cpp/device_tables.cpp -o device_tables \
//       -Lmultiverso_b200/_lib -lmvdevice -lmultiverso -lmvb200 -Wl,-rpath,$PWD/multiverso_b200/_lib
//   python tools/mvrun.py -n 8 -- ./device_tables -sync=true
#include <cstdio>
#include <vector>

#include "multiverso/device/device.h"
#include "multiverso/multiverso.h"

namespace dev = multiverso::device;

int main(int argc, char* argv[]) {
  dev::Init(&argc, argv);
  const int W = multiverso::MV_NumWorkers();
  const int64_t rows = 1 << 16, cols = 64;
  {
    dev::MatrixTable<float> table(rows, cols, dev::TableInit::Fill(0.0), "sgd");   // collective
    std::vector<float> host(rows * cols, 0.25f);
    float* d_grad = static_cast<float*>(dev::DeviceAlloc(host.size() * sizeof(float)));
    float* d_w = static_cast<float*>(dev::DeviceAlloc(host.size() * sizeof(float)));
    dev::CopyToDevice(d_grad, host.data(), host.size() * sizeof(float));

    const int h = table.AddAsync(d_grad);     // reduce-scatter over NVLink fused with the SGD updater
    table.Wait(h);
    dev::Barrier();
    table.Get(d_w);                            // all-gather by P2P pull
    dev::CopyToHost(host.data(), d_w, host.size() * sizeof(float));
    printf("rank %d/%d on GPU %d: w[0] = %g (expected %g)\n", dev::Rank(), dev::Size(), dev::DeviceId(), host[0],
           -0.25 * W);

    float one = 1.0f, *d_one = static_cast<float*>(dev::DeviceAlloc(sizeof(float)));
    dev::CopyToDevice(d_one, &one, sizeof one);
    dev::Aggregate(d_one, 1);                  // MV_Aggregate: in-place SUM all-reduce
    dev::CopyToHost(&one, d_one, sizeof one);
    printf("rank %d: aggregate(1) = %g\n", dev::Rank(), one);
    dev::Barrier();
    dev::DeviceFree(d_grad);
    dev::DeviceFree(d_w);
    dev::DeviceFree(d_one);
  }                                            // tables are destroyed (collectively) before ShutDown
  dev::ShutDown();
  return 0;
}
