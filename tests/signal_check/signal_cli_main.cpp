// signal_cli_main.cpp — TEST-ONLY command line: the product's host code (star_cli_main_engine of libstar_b200.so) driven by the CPU oracle
// engine (oracle/_build/liboracle.so) for mapping, and for the signal tracks by the sequential restatement of signalFromBAM, or, with
// STAR_SIGNAL_EMUL=1, by the emulated kernels of signal_kernels.cuh (signal_check.cpp).  Runs --outWigType mapping runs and
// --runMode inputAlignmentsFromBAM without a GPU.
#include <cstdlib>

#include "../../oracle/star_oracle.h"

extern "C" {
int signal_oracle_open(void** h, int device, uint32_t nStrands);
int signal_oracle_segment(void* h, uint32_t chrLen, const star_signal_block_t* blocks, uint64_t nBlocks, int mode, star_signal_track_t* tracks, float* ms);
void signal_oracle_close(void* h);
int signal_emul_open(void** h, int device, uint32_t nStrands);
int signal_emul_segment(void* h, uint32_t chrLen, const star_signal_block_t* blocks, uint64_t nBlocks, int mode, star_signal_track_t* tracks, float* ms);
void signal_emul_close(void* h);
}

int main(int argc, char** argv) {
    star_engine_vtbl_t vt = *star_oracle_engine();
    const char* e = getenv("STAR_SIGNAL_EMUL");
    if (e && atoi(e)) { vt.signal_open = signal_emul_open; vt.signal_segment = signal_emul_segment; vt.signal_close = signal_emul_close; }
    else { vt.signal_open = signal_oracle_open; vt.signal_segment = signal_oracle_segment; vt.signal_close = signal_oracle_close; }
    return star_cli_main_engine(argc, argv, &vt);
}
