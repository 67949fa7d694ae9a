// kernel_shape() (sha256_kernels.cuh) on the host: which kernel each (streams per warp, jobs to pair, variant) runs.
// The rows are the choices the engine's launch paths made before the choice moved into that one function: the pump
// passes the co-resident job count, an unsplit dm_ingest_device its batch size, the long half of a split batch its own
// size, the rest of a split batch 0.
#include <cstdio>
#include "sha256_kernels.cuh"

static int failures = 0;

static void expect(int spw, uint32_t pair_jobs, int wide, int deep, int want_spw, bool want_pairs, int want_form)
{
    const dm::KernelShape s = dm::kernel_shape(spw, pair_jobs, wide, deep);
    if (s.spw != want_spw || s.pairs != want_pairs || s.form != want_form) {
        std::printf("kernel_shape(%d, %u, %d, %d) = {%d, %d, %d}, want {%d, %d, %d}\n", spw, pair_jobs, wide, deep,
                    s.spw, (int)s.pairs, s.form, want_spw, (int)want_pairs, want_form);
        ++failures;
    }
}

int main()
{
    const int W = dm::kDefaultWideVariant;
    // the default (9): pairs at every S <= 16 while ceil(jobs / S) <= 264
    expect(1, 264, W, 9, 1, true, 7);
    expect(1, 265, W, 9, 1, false, 7);
    expect(2, 528, W, 9, 2, true, 7);
    expect(2, 529, W, 9, 2, false, 7);
    expect(16, 4224, W, 9, 16, true, 7);
    expect(16, 4225, W, 9, 16, false, 7);
    expect(16, 8448, W, 9, 16, false, 7);
    // 8: pairs at S = 1 only
    expect(1, 264, W, 8, 1, true, 7);
    expect(1, 265, W, 8, 1, false, 7);
    expect(2, 2, W, 8, 2, false, 7);
    expect(16, 16, W, 8, 16, false, 7);
    // 10: pairs at S = 1 whatever the count, never at S > 1
    expect(1, 265, W, 10, 1, true, 7);
    expect(1, 5000, W, 10, 1, true, 7);
    expect(4, 4, W, 10, 4, false, 7);
    // pair count 0 (the rest of a split batch): never pairs
    for (int d = 8; d <= 10; ++d)
        for (int s = 1; s <= 16; s *= 2) expect(s, 0, W, d, s, false, 7);
    // 0..7 never pair; deep 1 and 3 -> form 1, 2 -> 2 at S = 1; group 1..3 -> form 0
    for (int d = 0; d <= 7; ++d) {
        const int f1 = d == 3 ? 1 : d;
        const int fs = d <= 3 ? 0 : d;
        expect(1, 1, W, d, 1, false, f1);
        expect(1, 264, W, d, 1, false, f1);
        for (int s = 2; s <= 16; s *= 2) expect(s, s, W, d, s, false, fs);
    }
    // variant numbers outside the table run form 0
    expect(1, 1, W, 11, 1, false, 0);
    expect(2, 2, W, -1, 2, false, 0);
    // spw = 32: the wide variant if it is built, else the default; the deep variant and the pair count do not matter
    for (int w = 0; w < 24; ++w) {
        const bool built = (w < 20 && w % 4 != 3) || w == 21;
        expect(32, 100000, w, 9, 32, false, built ? w : W);
        expect(32, 0, w, 0, 32, false, built ? w : W);
    }
    expect(32, 1, 3, 9, 32, false, 9);
    expect(32, 1, 21, 9, 32, false, 21);
    if (failures) {
        std::printf("%d kernel_shape rows wrong\n", failures);
        return 1;
    }
    std::printf("KERNEL SHAPE OK\n");
    return 0;
}
