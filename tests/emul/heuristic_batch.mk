# TEST-ONLY: host emulation of whmec_heuristic_batch (emul_heuristic_batch.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_heuristic_batch.cpp $(C)/heuristic_batch.cpp $(C)/heuristic.cpp
libwhemul_heuristic_batch.so: $(SRC) $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -o $@ $(SRC)
clean:
	rm -f libwhemul_heuristic_batch.so
