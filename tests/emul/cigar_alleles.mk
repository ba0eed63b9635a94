# TEST-ONLY: host emulation of whmec_detect_alleles_cigar (emul_cigar_alleles.cpp); whmec_realign_release comes with the realign
# emulation's sources.
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_cigar_alleles.cpp $(C)/cigar_alleles_plan.cpp emul_realign.cpp $(C)/realign_plan.cpp $(C)/hostpool.cpp
libwhemul_cigar_alleles.so: $(SRC) $(C)/cigar_alleles.h $(C)/cigar_alleles_plan.h $(C)/realign.h $(C)/realign_plan.h $(C)/hostpool.h ../../include/whmec.h
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ $(SRC)
clean:
	rm -f libwhemul_cigar_alleles.so
