// dedup_cli_main.cpp — TEST-ONLY command line: the product's host code (star_cli_main_engine of libstar_b200.so) with the CPU oracle
// engine (oracle/_build/liboracle.so), and for duplicate marking the sequential restatement of bamRemoveDuplicates or, with
// STAR_DEDUP_EMUL=1, the emulated kernels of dedup_kernels.cuh (dedup_check.cpp).  Runs --runMode inputAlignmentsFromBAM without a GPU.
#include <cstdlib>

#include "../../oracle/star_oracle.h"

extern "C" {
int dedup_oracle_open(void** h, int device, uint64_t mate2basesN);
int dedup_oracle_batch(void* h, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* groups, uint64_t n, uint8_t* unmark, float* ms);
void dedup_oracle_close(void* h);
int dedup_emul_open(void** h, int device, uint64_t mate2basesN);
int dedup_emul_batch(void* h, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* groups, uint64_t n, uint8_t* unmark, float* ms);
void dedup_emul_close(void* h);
}

int main(int argc, char** argv) {
    star_engine_vtbl_t vt = *star_oracle_engine();
    const char* e = getenv("STAR_DEDUP_EMUL");
    if (e && atoi(e)) { vt.dedup_open = dedup_emul_open; vt.dedup_batch = dedup_emul_batch; vt.dedup_close = dedup_emul_close; }
    else { vt.dedup_open = dedup_oracle_open; vt.dedup_batch = dedup_oracle_batch; vt.dedup_close = dedup_oracle_close; }
    return star_cli_main_engine(argc, argv, &vt);
}
