# TEST-ONLY: host emulation of whmec_realign_kmerald and whmec_kmer_align_batch (emul_kmerald.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_kmerald.cpp $(C)/realign_plan.cpp $(C)/hostpool.cpp
libwhemul_kmerald.so: $(SRC) $(C)/kmerald.h $(C)/realign.h $(C)/realign_plan.h $(C)/hostpool.h ../../include/whmec.h
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ $(SRC)
clean:
	rm -f libwhemul_kmerald.so
