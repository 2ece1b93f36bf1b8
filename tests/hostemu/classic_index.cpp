// classic_label_index (chess_dev.cuh) on a board of the host emulation (test scaffolding, built by
// tests/test_classic_index_hostemu.py like tests/hostemu/hostemu.cpp).
#include "chess_dev.cuh"

extern "C" int he_classic_index(const void* board, unsigned short move, int mode) {
    const ara::Board& b = *static_cast<const ara::Board*>(board);
    return ara::classic_label_index(move, b.stm, b.chess960, mode);
}
