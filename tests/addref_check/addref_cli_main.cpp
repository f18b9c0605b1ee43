// addref_cli_main.cpp — TEST-ONLY command line: the product's host code (star_cli_main_engine of libstar_b200.so) with the CPU oracle
// engine (oracle/_build/liboracle.so), and for adding references the sequential restatement of insertSeqSA or, with STAR_ADDREF_EMUL=1,
// the emulated kernels of addref_kernels.cuh (addref_check.cpp).  Runs --genomeFastaFiles at the mapping stage without a GPU.
#include <cstdlib>

#include "../../oracle/star_oracle.h"

extern "C" {
int addref_oracle_open(void** h, int device, const star_index_view_t* grown, uint64_t nG, uint64_t nG1, uint64_t nG2, float* ms);
int addref_oracle_search(void* h, const uint8_t* seq, uint64_t* indArray, float* ms);
int addref_oracle_merge_sa(void* h, const uint64_t* indSorted, uint64_t nInd, uint8_t* SAnew, uint64_t nSAnewByte, float* ms);
void addref_oracle_close(void* h);
int addref_emul_open(void** h, int device, const star_index_view_t* grown, uint64_t nG, uint64_t nG1, uint64_t nG2, float* ms);
int addref_emul_search(void* h, const uint8_t* seq, uint64_t* indArray, float* ms);
int addref_emul_merge_sa(void* h, const uint64_t* indSorted, uint64_t nInd, uint8_t* SAnew, uint64_t nSAnewByte, float* ms);
void addref_emul_close(void* h);
}

int main(int argc, char** argv) {
    star_engine_vtbl_t vt = *star_oracle_engine();
    const char* e = getenv("STAR_ADDREF_EMUL");
    if (e && atoi(e)) { vt.addref_open = addref_emul_open; vt.addref_search = addref_emul_search; vt.addref_merge_sa = addref_emul_merge_sa; vt.addref_close = addref_emul_close; }
    else { vt.addref_open = addref_oracle_open; vt.addref_search = addref_oracle_search; vt.addref_merge_sa = addref_oracle_merge_sa; vt.addref_close = addref_oracle_close; }
    return star_cli_main_engine(argc, argv, &vt);
}
