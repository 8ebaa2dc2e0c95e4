# ORACLE build for sharded input (test infrastructure only), next to oracle/Makefile:
#   shard_oracle       the reference's sharded reader (shard_bam_reader.rs) restated: writes the winners as one BAM
#   coverm_shardcheck  the product's host code linked against the CPU device emulator with the cmb_shard_* entry points
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -ffp-contract=off -Wall -Wextra -Wno-unused-parameter
HOST = ../coverm_b200/csrc/host
all: shard_oracle coverm_shardcheck
shard_oracle: shard_oracle.cpp oracle_core.hpp oracle_bam.hpp
	$(CXX) $(CXXFLAGS) -o $@ shard_oracle.cpp -lz -lpthread
coverm_shardcheck: shard_emulator.cpp device_emulator.cpp $(HOST)/host_api.cpp $(HOST)/coverm_main.cpp $(wildcard $(HOST)/*.hpp) ../include/coverm_b200.h
	$(CXX) $(CXXFLAGS) -o $@ shard_emulator.cpp $(HOST)/host_api.cpp $(HOST)/coverm_main.cpp -lz -lpthread
clean:
	rm -f shard_oracle coverm_shardcheck
