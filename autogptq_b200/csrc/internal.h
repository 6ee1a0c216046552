// Shared between the translation units of libautogptq_b200.so (not part of the ABI).
#pragma once
// Records `msg` as the calling thread's last error (agb200_last_error) and returns `code`.  Defined in abi.cu.
int agb_internal_fail(int code, const char* msg);
// out[m, perm[j]] = in[m, j] for 16-bit [M, K] rows (the act-order dx of the dgrad paths) on `stream`; 2 K bytes of a
// row must fit in shared memory.  Returns 0 or the failure code (recorded as above).  Defined in abi.cu.
int agb_internal_unpermute_columns(const void* in, const int* perm, void* out, int M, int K, void* stream);
