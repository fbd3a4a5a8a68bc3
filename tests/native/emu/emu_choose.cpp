// TEST INFRASTRUCTURE: the shared-subscription choice (relations.cuh k_relations<true> through launch_relations, the launch
// behind gm_relations_choose_device) over HOST memory, on the CPU emulation in cuda_runtime.h.  It builds from relations.cuh
// alone, without the host tries of emu_driver.cpp.  Exposed as a small C interface for
// tests/test_shared_choice_cpu.py, which compares the results with a Python model.  Build (the test does it):
//   g++ -O1 -g -std=c++17 -DGM_CPU_EMU -Itests/native/emu -Irmqtt_b200/csrc -shared -fPIC -pthread tests/native/emu/emu_choose.cpp \
//       -o <out>.so     (+ -fsanitize=address,undefined for the ASan run)
#include <cuda_runtime.h>      // the emulation (this directory is first on the include path)

#include "relations.cuh"

using namespace gm;

namespace {
constexpr u32 EMU_SMS = 2;               // as the driver of the other kernels: several CTAs, grid-stride loops exercised
}  // namespace

extern "C" {

// gm_relations_choose_device over host arrays; online = null: every client online
int32_t emu_relations_choose(const gm_span* spans, const uint32_t* ids, uint64_t n, const uint32_t* pubs, const gm_rel* rels, uint64_t n_rels,
                             const gm_span* groups, uint32_t n_groups, const uint32_t* members, const uint32_t* online, uint32_t n_online_bits, uint64_t seed,
                             gm_span* out_spans, gm_sub_relation* out_rels, uint64_t cap_rels, uint32_t* out_sub_ids, uint64_t cap_sub_ids, uint64_t* needed3,
                             int32_t* status) {
    needed3[0] = needed3[1] = needed3[2] = 0;
    if (n == 0) return 0;
    const gm_rel_groups g{groups, n_groups, members, online, n_online_bits, seed};
    launch_relations(spans, ids, n, pubs, rels, n_rels, &g, gm_rel_out{out_spans, out_rels, cap_rels, out_sub_ids, cap_sub_ids, needed3, status}, EMU_SMS, nullptr);
    return 0;
}

// the kernel's own key function, compiled for the host
uint64_t emu_share_key(uint64_t seed, uint32_t row, uint32_t group, uint32_t occ, uint32_t client_key) { return share_key(seed, row, group, occ, client_key); }

}  // extern "C"
