"""Writes train_data_golden.npz: the key orders of the reference's CustomData layer, made by libstdc++ itself.

A ten-line C++ program (standard library only) calls std::srand(seed) unless the seed is <= 0, then std::random_shuffle on
each given [lo, hi) of 0 .. n-1, and prints the vector.  This script applies the range cut and the block off-by-one
(custom_data_layer.cpp:28-41, 394-470) around it and stores only the resulting permutations, which pin
flownet2_b200.data.permutation.  Needs g++ with glibc; run from anywhere:

    python tests/golden/make_train_data_golden.py
"""
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SHUFFLE_CPP = r"""
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>
int main(int argc, char** argv) {
    int n = atoi(argv[1]), seed = atoi(argv[2]);
    std::vector<int> v(n);
    for (int i = 0; i < n; i++) v[i] = i;
    if (seed > 0) std::srand(unsigned(seed));
    for (int a = 3; a + 1 < argc; a += 2) std::random_shuffle(v.begin() + atoi(argv[a]), v.begin() + atoi(argv[a + 1]));
    for (int i = 0; i < n; i++) printf("%d\n", v[i]);
}
"""

N = 22872                                       # FlyingChairs
# name -> (n, seed, block_size, range_start, range_end, order)
CASES = {
    "full_seed77": (N, 77, 0, 0, -1, "FIRST_PERMUTE_THEN_RANGE"),
    "full_seed1": (N, 1, 0, 0, -1, "FIRST_PERMUTE_THEN_RANGE"),
    "full_seed0": (N, 0, 0, 0, -1, "FIRST_PERMUTE_THEN_RANGE"),
    "block1000_seed77": (N, 77, 1000, 0, -1, "FIRST_PERMUTE_THEN_RANGE"),
    "permute_then_range": (N, 77, 0, 640, 22231, "FIRST_PERMUTE_THEN_RANGE"),
    "range_then_permute": (N, 77, 0, 640, 22231, "FIRST_RANGE_THEN_PERMUTE"),
    "range_then_permute_block": (N, 77, 333, 17, 9000, "FIRST_RANGE_THEN_PERMUTE"),
    "small20_seed77": (20, 77, 0, 0, -1, "FIRST_PERMUTE_THEN_RANGE"),
}


def shuffled(exe, n, seed, spans):
    args = [exe, str(n), str(seed)] + [str(x) for lo, hi in spans for x in (lo, hi)]
    return np.array(subprocess.run(args, check=True, capture_output=True, text=True).stdout.split(), np.int32)


def case(exe, n, seed, block, rs, re_, order):
    rs = min(max(rs, 0), n - 1)
    re_ = n - 1 if re_ < 0 or re_ >= n else re_
    m = re_ - rs + 1 if order == "FIRST_RANGE_THEN_PERMUTE" else n
    spans = [(b * block, min((b + 1) * block, m) - 1) for b in range((m + block - 1) // block)] if block else [(0, m)]
    v = shuffled(exe, m, seed, spans)
    return v + rs if order == "FIRST_RANGE_THEN_PERMUTE" else v[rs:re_ + 1]


def main():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "shuffle.cpp"), os.path.join(d, "shuffle")
        with open(src, "w") as f:
            f.write(SHUFFLE_CPP)
        subprocess.run(["g++", "-O1", "-std=c++11", src, "-o", exe], check=True)
        out = {name: case(exe, *spec) for name, spec in CASES.items()}
    np.savez_compressed(os.path.join(HERE, "train_data_golden.npz"), **{k: v.astype(np.int16) for k, v in out.items()})     # n < 2^15
    print("wrote %d permutations" % len(out))


if __name__ == "__main__":
    main()
