# TEST-ONLY: host emulation of whmec_merge_reads (emul_merge.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_merge.cpp $(C)/merge_plan.cpp
libwhemul_merge.so: $(SRC) $(C)/merge.h $(C)/merge_plan.h ../../include/whmec.h
	$(CXX) -std=c++17 -O2 -Wall -fPIC -shared -o $@ $(SRC)
clean:
	rm -f libwhemul_merge.so
