// Topology detection for one NVLink/NVSwitch server.
//
// The reference infers the intra-server topology by *timing*: TCP loopback under
// numa_run_on_node to find the NIC's NUMA node, pairwise D2H bandwidth drops to find GPUs
// behind one PCIe switch, H2D under NIC load to find the GPU closest to the NIC, then dumps
// topology/topo_detect_<rank>.xml as <cpu><pcie>[<nic/>]<gpu id/>…
// (/root/reference/csrc/detect.cu:209-427). On an NVSwitch box none of that has to be guessed: NVML,
// the CUDA P2P attributes and sysfs report it. We emit the same XML schema (so the control
// plane's gather step is unchanged) plus attributes the synthesizer uses on NVSwitch
// systems: NVLink link counts, P2P performance rank, native atomics, multicast (NVLS).
#include <dirent.h>
#include <dlfcn.h>
#include <nvml.h>
#include <unistd.h>

#include <algorithm>
#include <fstream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "common.h"
#include "driver_api.h"

namespace adapcc {
namespace {

struct Nvml {
  void* lib = nullptr;
  nvmlReturn_t (*Init)() = nullptr;
  nvmlReturn_t (*Shutdown)() = nullptr;
  nvmlReturn_t (*DeviceGetHandleByPciBusId)(const char*, nvmlDevice_t*) = nullptr;
  nvmlReturn_t (*DeviceGetNvLinkState)(nvmlDevice_t, unsigned, nvmlEnableState_t*) = nullptr;
  nvmlReturn_t (*DeviceGetNvLinkRemotePciInfo)(nvmlDevice_t, unsigned, nvmlPciInfo_t*) = nullptr;
  nvmlReturn_t (*DeviceGetNvLinkRemoteDeviceType)(nvmlDevice_t, unsigned, nvmlIntNvLinkDeviceType_t*) = nullptr;
  nvmlReturn_t (*DeviceGetTopologyCommonAncestor)(nvmlDevice_t, nvmlDevice_t, nvmlGpuTopologyLevel_t*) = nullptr;
  bool ok = false;

  template <typename F> void sym(F& f, const char* n) { f = reinterpret_cast<F>(dlsym(lib, n)); }
  bool load() {
    lib = dlopen("libnvidia-ml.so.1", RTLD_NOW | RTLD_LOCAL);
    if (!lib) return false;
    sym(Init, "nvmlInit_v2");
    sym(Shutdown, "nvmlShutdown");
    sym(DeviceGetHandleByPciBusId, "nvmlDeviceGetHandleByPciBusId_v2");
    sym(DeviceGetNvLinkState, "nvmlDeviceGetNvLinkState");
    sym(DeviceGetNvLinkRemotePciInfo, "nvmlDeviceGetNvLinkRemotePciInfo_v2");
    sym(DeviceGetNvLinkRemoteDeviceType, "nvmlDeviceGetNvLinkRemoteDeviceType");
    sym(DeviceGetTopologyCommonAncestor, "nvmlDeviceGetTopologyCommonAncestor");
    ok = Init && DeviceGetHandleByPciBusId && Init() == NVML_SUCCESS;
    return ok;
  }
  ~Nvml() {
    if (ok && Shutdown) Shutdown();
    if (lib) dlclose(lib);
  }
};

std::string read_line(const std::string& path) {
  std::ifstream f(path);
  std::string s;
  if (f) std::getline(f, s);
  return s;
}

std::string lower(std::string s) {
  std::transform(s.begin(), s.end(), s.begin(), ::tolower);
  return s;
}

// resolved sysfs path of a PCI device, e.g. /sys/devices/pci0000:15/0000:15:01.0/0000:17:00.0
std::string pci_sysfs_path(const std::string& bdf) {
  char buf[4096];
  std::string p = "/sys/bus/pci/devices/" + lower(bdf);
  ssize_t n = readlink(p.c_str(), buf, sizeof(buf) - 1);
  if (n <= 0) return std::string();
  buf[n] = 0;
  return std::string(buf);
}

size_t common_prefix_depth(const std::string& a, const std::string& b) {
  size_t depth = 0, i = 0;
  while (i < a.size() && i < b.size() && a[i] == b[i]) {
    if (a[i] == '/') ++depth;
    ++i;
  }
  return depth;
}

struct Gpu {
  int dev = 0;
  std::string bdf, name, sysfs;
  int numa = -1;
  int nvlinks = 0, nvlinks_to_switch = 0;
  int multicast = 0;
  std::string nic;      // closest NIC (by PCIe ancestry), may be empty
};

struct Nic { std::string name, sysfs; int numa = -1; };

std::vector<Nic> list_nics() {
  std::vector<Nic> out;
  DIR* d = opendir("/sys/class/infiniband");
  if (!d) return out;
  while (dirent* e = readdir(d)) {
    if (e->d_name[0] == '.') continue;
    Nic n;
    n.name = e->d_name;
    char buf[4096];
    std::string p = std::string("/sys/class/infiniband/") + e->d_name + "/device";
    ssize_t k = readlink(p.c_str(), buf, sizeof(buf) - 1);
    if (k > 0) { buf[k] = 0; n.sysfs = buf; }
    std::string numa = read_line(p + "/numa_node");
    n.numa = numa.empty() ? -1 : atoi(numa.c_str());
    out.push_back(n);
  }
  closedir(d);
  std::sort(out.begin(), out.end(), [](const Nic& a, const Nic& b) { return a.name < b.name; });
  return out;
}

}  // namespace
}  // namespace adapcc

using namespace adapcc;

extern "C" {

// Writes the detect XML for all GPUs visible to this process into `out` (NUL terminated).
// `first_rank` is the world rank of local device 0 (gpu ids in the XML are LOCAL indices, as
// in the reference's topo_detect_<rank>.xml). Returns the XML length, or -1.
int adapcc_detect_topology(int first_rank, char* out, int cap) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    (void)cudaGetLastError();
    set_error("detect: no CUDA device visible");
    return -1;
  }
  Nvml nvml;
  nvml.load();
  const DriverApi& drv = driver();
  std::vector<Gpu> gpus(ndev);
  std::vector<Nic> nics = list_nics();
  for (int d = 0; d < ndev; ++d) {
    Gpu& g = gpus[d];
    g.dev = d;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, d) == cudaSuccess) g.name = prop.name;
    char bdf[32] = {0};
    if (cudaDeviceGetPCIBusId(bdf, sizeof(bdf), d) == cudaSuccess) g.bdf = bdf;
    g.sysfs = pci_sysfs_path(g.bdf);
    std::string numa = read_line("/sys/bus/pci/devices/" + lower(g.bdf) + "/numa_node");
    g.numa = numa.empty() ? -1 : atoi(numa.c_str());
    if (drv.ok) {
      CUdevice cd;
      int v = 0;
      if (drv.DeviceGet(&cd, d) == CUDA_SUCCESS &&
          drv.DeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, cd) == CUDA_SUCCESS)
        g.multicast = v;
    }
    if (nvml.ok) {
      nvmlDevice_t h;
      if (nvml.DeviceGetHandleByPciBusId(g.bdf.c_str(), &h) == NVML_SUCCESS && nvml.DeviceGetNvLinkState) {
        for (unsigned l = 0; l < NVML_NVLINK_MAX_LINKS; ++l) {
          nvmlEnableState_t st;
          if (nvml.DeviceGetNvLinkState(h, l, &st) != NVML_SUCCESS || st != NVML_FEATURE_ENABLED) continue;
          ++g.nvlinks;
          nvmlIntNvLinkDeviceType_t ty;
          if (nvml.DeviceGetNvLinkRemoteDeviceType &&
              nvml.DeviceGetNvLinkRemoteDeviceType(h, l, &ty) == NVML_SUCCESS &&
              ty == NVML_NVLINK_DEVICE_TYPE_SWITCH)
            ++g.nvlinks_to_switch;
        }
      }
    }
    size_t best = 0;
    for (const Nic& n : nics) {
      size_t depth = common_prefix_depth(g.sysfs, n.sysfs);
      if (depth > best) { best = depth; g.nic = n.name; }
    }
  }

  // group: NUMA node -> (PCIe root complex = 4th path component) -> gpus
  std::map<int, std::map<std::string, std::vector<int>>> tree;
  for (const Gpu& g : gpus) {
    std::string root = "pci";
    size_t a = g.sysfs.find("/pci");
    if (a != std::string::npos) {
      size_t b = g.sysfs.find('/', a + 1);
      root = g.sysfs.substr(a + 1, b == std::string::npos ? std::string::npos : b - a - 1);
    }
    tree[g.numa][root].push_back(g.dev);
  }

  std::ostringstream x;
  x << "<?xml version=\"1.0\" encoding=\"utf-8\"?>\n";
  x << "<topology first_rank=\"" << first_rank << "\" gpus=\"" << ndev << "\" nvml=\"" << (nvml.ok ? 1 : 0)
    << "\">\n";
  for (auto& numa : tree) {
    x << "  <cpu numa=\"" << numa.first << "\">\n";
    for (auto& rc : numa.second) {
      x << "    <pcie root=\"" << rc.first << "\">\n";
      std::vector<std::string> seen;
      for (int d : rc.second) {
        const Gpu& g = gpus[d];
        if (!g.nic.empty() && std::find(seen.begin(), seen.end(), g.nic) == seen.end()) {
          seen.push_back(g.nic);
          x << "      <nic name=\"" << g.nic << "\"/>\n";
        }
        x << "      <gpu id=\"" << d << "\" bdf=\"" << g.bdf << "\" name=\"" << g.name << "\" nvlinks=\""
          << g.nvlinks << "\" nvswitch_links=\"" << g.nvlinks_to_switch << "\" multicast=\"" << g.multicast
          << "\"/>\n";
      }
      x << "    </pcie>\n";
    }
    x << "  </cpu>\n";
  }
  // P2P matrix (what cudaSend/cudaRecv silently assumed in the reference)
  for (int a = 0; a < ndev; ++a)
    for (int b = 0; b < ndev; ++b) {
      if (a == b) continue;
      int can = 0, perf = 0, atomics = 0;
      cudaDeviceCanAccessPeer(&can, a, b);
      cudaDeviceGetP2PAttribute(&perf, cudaDevP2PAttrPerformanceRank, a, b);
      cudaDeviceGetP2PAttribute(&atomics, cudaDevP2PAttrNativeAtomicSupported, a, b);
      (void)cudaGetLastError();
      x << "  <p2p src=\"" << a << "\" dst=\"" << b << "\" access=\"" << can << "\" perf_rank=\"" << perf
        << "\" atomics=\"" << atomics << "\"/>\n";
    }
  x << "</topology>\n";
  std::string s = x.str();
  if ((int)s.size() + 1 > cap) { set_error("detect: output buffer too small (%zu needed)", s.size() + 1); return -1; }
  memcpy(out, s.c_str(), s.size() + 1);
  return (int)s.size();
}

}  // extern "C"
