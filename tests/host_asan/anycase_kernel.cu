// Compile-only check (tests/test_host_asan_cpu.py): the predicates of csrc/vl_anycase.cuh build for sm_90a as device code, i.e. the row
// kernels can call them as they are.  One thread per value; not part of libvlscan.so.
#include "vl_anycase.cuh"

extern "C" __global__ void k_next_predicates(const uint8_t* values, const uint32_t* offs, uint32_t n, const uint8_t* needle, uint32_t needle_len,
                                             const uint8_t* list, uint32_t list_len, uint8_t* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* s = values + offs[i]; const uint32_t len = offs[i + 1] - offs[i];
    uint8_t bits = 0;
    bits |= vl::any_case_match(s, len, needle, needle_len, false) ? 1 : 0;
    bits |= vl::any_case_match(s, len, needle, needle_len, true) ? 2 : 0;
    bits |= vl::match_sequence(s, len, vl::PhraseList{list, list_len}) ? 4 : 0;
    bits |= vl::match_all_phrases(s, len, vl::PhraseList{list, list_len}) ? 8 : 0;
    bits |= vl::match_any_phrase(s, len, vl::PhraseList{list, list_len}) ? 16 : 0;
    out[i] = bits;
}
