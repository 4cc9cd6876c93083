#!/bin/bash
# Builds the product library (sm_90a only), the CPU oracle and the synthetic-input generator, in-tree.
set -e
cd "$(dirname "$0")"
make -s -j8 -C skani_b200/csrc
make -s -C oracle
/usr/bin/g++ -O2 -std=c++17 -o skani_b200/skani-b200 skani_b200/cli/skani_b200_cli.cpp -Lskani_b200 -lskani_b200 -lz -lpthread -Wl,-rpath,'$ORIGIN'
/usr/bin/g++ -O2 -std=c++17 -o skani_b200/skani-db-tool skani_b200/cli/skani_db_tool.cpp -lz
/usr/bin/g++ -O3 -march=x86-64-v3 -std=c++17 -fPIC -fopenmp -shared -o bench_support/libsynth.so bench_support/synth.cpp
echo build ok
