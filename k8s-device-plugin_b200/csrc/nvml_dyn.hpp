// nvml_dyn.hpp -- NVML, resolved at run time with dlopen (the library has no link-time NVML dependency).
//
// NVML is the H100 counterpart of what the reference reads from sysfs/kfd and libdrm: PCI identity, device minor,
// firmware versions, and -- for MIG-partitioned GPUs -- the instance table that plays the role of the
// /sys/devices/platform/amdgpu_xcp_* devices (amdgpu.go:221-265).  Structs below restate the public nvml.h layouts
// the entry points take (no NVML header is needed to build).
#pragma once
#include <dlfcn.h>

#include <cstdlib>
#include <cstring>

namespace b2dp {

struct NvmlPciInfo {            // nvmlPciInfo_t (v3)
    char busIdLegacy[16];
    unsigned int domain, bus, device, pciDeviceId, pciSubSystemId;
    char busId[32];
};
struct NvmlDeviceAttributes {   // nvmlDeviceAttributes_t
    unsigned int multiprocessorCount, sharedCopyEngineCount, sharedDecoderCount, sharedEncoderCount, sharedJpegCount,
        sharedOfaCount, gpuInstanceSliceCount, computeInstanceSliceCount;
    unsigned long long memorySizeMB;
};
struct NvmlMemory { unsigned long long total, free, used; };  // nvmlMemory_t

struct Nvml {
    void* lib = nullptr;
    int (*init)() = nullptr;
    int (*shutdown)() = nullptr;
    int (*driver_version)(char*, unsigned) = nullptr;
    int (*handle_by_bus_id)(const char*, void**) = nullptr;
    int (*minor_number)(void*, unsigned*) = nullptr;
    int (*vbios)(void*, char*, unsigned) = nullptr;
    int (*mig_mode)(void*, unsigned*, unsigned*) = nullptr;
    int (*running_procs)(void*, unsigned*, void*) = nullptr;        // nvmlDeviceGetComputeRunningProcesses_v3
    int (*ecc_total)(void*, int, int, unsigned long long*) = nullptr;  // nvmlDeviceGetTotalEccErrors
    int (*remapped_rows)(void*, unsigned*, unsigned*, unsigned*, unsigned*) = nullptr;  // nvmlDeviceGetRemappedRows
    struct EventData { void* device; unsigned long long type, data; unsigned gi, ci; };  // nvmlEventData_t
    int (*event_set_create)(void**) = nullptr;
    int (*register_events)(void*, unsigned long long, void*) = nullptr;
    int (*event_wait)(void*, EventData*, unsigned) = nullptr;          // nvmlEventSetWait_v2
    int (*event_set_free)(void*) = nullptr;
    int (*index_of)(void*, unsigned*) = nullptr;                       // nvmlDeviceGetIndex
    int (*uuid_of)(void*, char*, unsigned) = nullptr;                  // nvmlDeviceGetUUID
    int (*inforom_image)(void*, char*, unsigned) = nullptr;            // nvmlDeviceGetInforomImageVersion
    int (*inforom_object)(void*, int, char*, unsigned) = nullptr;      // nvmlDeviceGetInforomVersion(OEM 0 / ECC 1 / POWER 2)
    int (*gsp_firmware)(void*, char*) = nullptr;                       // nvmlDeviceGetGspFirmwareVersion
    // enumeration without CUDA (probe=off / probe=helpers / MIG)
    int (*device_count)(unsigned*) = nullptr;                          // nvmlDeviceGetCount_v2
    int (*handle_by_index)(unsigned, void**) = nullptr;                // nvmlDeviceGetHandleByIndex_v2
    int (*pci_info)(void*, NvmlPciInfo*) = nullptr;                    // nvmlDeviceGetPciInfo_v3
    int (*name_of)(void*, char*, unsigned) = nullptr;                  // nvmlDeviceGetName
    int (*memory_info)(void*, NvmlMemory*) = nullptr;                  // nvmlDeviceGetMemoryInfo
    int (*num_cores)(void*, unsigned*) = nullptr;                      // nvmlDeviceGetNumGpuCores
    int (*cuda_cc)(void*, int*, int*) = nullptr;                       // nvmlDeviceGetCudaComputeCapability
    // MIG (the amdgpu_xcp_* analogue)
    int (*max_mig_count)(void*, unsigned*) = nullptr;                  // nvmlDeviceGetMaxMigDeviceCount
    int (*mig_handle)(void*, unsigned, void**) = nullptr;              // nvmlDeviceGetMigDeviceHandleByIndex
    int (*gi_id)(void*, unsigned*) = nullptr;                          // nvmlDeviceGetGpuInstanceId
    int (*ci_id)(void*, unsigned*) = nullptr;                          // nvmlDeviceGetComputeInstanceId
    int (*parent_of_mig)(void*, void**) = nullptr;                     // nvmlDeviceGetDeviceHandleFromMigDeviceHandle
    int (*attributes)(void*, NvmlDeviceAttributes*) = nullptr;         // nvmlDeviceGetAttributes_v2
    int (*nvlink_state)(void*, unsigned, unsigned*) = nullptr;         // nvmlDeviceGetNvLinkState
    int (*p2p_status)(void*, void*, int, int*) = nullptr;              // nvmlDeviceGetP2PStatus
    // PCIe link (the host-link self-test reports these; none of them is judged)
    int (*pcie_gen)(void*, unsigned*) = nullptr;                       // nvmlDeviceGetCurrPcieLinkGeneration
    int (*pcie_width)(void*, unsigned*) = nullptr;                     // nvmlDeviceGetCurrPcieLinkWidth
    int (*pcie_max_gen)(void*, unsigned*) = nullptr;                   // nvmlDeviceGetMaxPcieLinkGeneration
    int (*pcie_max_width)(void*, unsigned*) = nullptr;                 // nvmlDeviceGetMaxPcieLinkWidth
    int (*pcie_replays)(void*, unsigned*) = nullptr;                   // nvmlDeviceGetPcieReplayCounter
    bool ok = false;

    ~Nvml() {
        if (ok && shutdown) shutdown();  // nvmlInit/nvmlShutdown are reference counted
        if (lib) dlclose(lib);
    }
    template <class F>
    void sym(F& f, const char* name) { f = reinterpret_cast<F>(dlsym(lib, name)); }
    void load() {
        // B2DP_NVML_LIBRARY: an alternative NVML (tests: tests/native/nvml_stub.cpp describes a MIG-partitioned node)
        const char* alt = getenv("B2DP_NVML_LIBRARY");
        lib = dlopen(alt && *alt ? alt : "libnvidia-ml.so.1", RTLD_NOW | RTLD_LOCAL);
        if (!lib) return;
        sym(init, "nvmlInit_v2");
        sym(shutdown, "nvmlShutdown");
        sym(driver_version, "nvmlSystemGetDriverVersion");
        sym(handle_by_bus_id, "nvmlDeviceGetHandleByPciBusId_v2");
        sym(minor_number, "nvmlDeviceGetMinorNumber");
        sym(vbios, "nvmlDeviceGetVbiosVersion");
        sym(mig_mode, "nvmlDeviceGetMigMode");
        sym(running_procs, "nvmlDeviceGetComputeRunningProcesses_v3");
        sym(ecc_total, "nvmlDeviceGetTotalEccErrors");
        sym(remapped_rows, "nvmlDeviceGetRemappedRows");
        sym(event_set_create, "nvmlEventSetCreate");
        sym(register_events, "nvmlDeviceRegisterEvents");
        sym(event_wait, "nvmlEventSetWait_v2");
        sym(event_set_free, "nvmlEventSetFree");
        sym(index_of, "nvmlDeviceGetIndex");
        sym(uuid_of, "nvmlDeviceGetUUID");
        sym(inforom_image, "nvmlDeviceGetInforomImageVersion");
        sym(inforom_object, "nvmlDeviceGetInforomVersion");
        sym(gsp_firmware, "nvmlDeviceGetGspFirmwareVersion");
        sym(device_count, "nvmlDeviceGetCount_v2");
        sym(handle_by_index, "nvmlDeviceGetHandleByIndex_v2");
        sym(pci_info, "nvmlDeviceGetPciInfo_v3");
        sym(name_of, "nvmlDeviceGetName");
        sym(memory_info, "nvmlDeviceGetMemoryInfo");
        sym(num_cores, "nvmlDeviceGetNumGpuCores");
        sym(cuda_cc, "nvmlDeviceGetCudaComputeCapability");
        sym(max_mig_count, "nvmlDeviceGetMaxMigDeviceCount");
        sym(mig_handle, "nvmlDeviceGetMigDeviceHandleByIndex");
        sym(gi_id, "nvmlDeviceGetGpuInstanceId");
        sym(ci_id, "nvmlDeviceGetComputeInstanceId");
        sym(parent_of_mig, "nvmlDeviceGetDeviceHandleFromMigDeviceHandle");
        sym(attributes, "nvmlDeviceGetAttributes_v2");
        sym(nvlink_state, "nvmlDeviceGetNvLinkState");
        sym(p2p_status, "nvmlDeviceGetP2PStatus");
        sym(pcie_gen, "nvmlDeviceGetCurrPcieLinkGeneration");
        sym(pcie_width, "nvmlDeviceGetCurrPcieLinkWidth");
        sym(pcie_max_gen, "nvmlDeviceGetMaxPcieLinkGeneration");
        sym(pcie_max_width, "nvmlDeviceGetMaxPcieLinkWidth");
        sym(pcie_replays, "nvmlDeviceGetPcieReplayCounter");
        ok = init && init() == 0;
    }
};

}  // namespace b2dp
