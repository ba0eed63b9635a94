# TEST-ONLY: host emulation of whmec_realign (emul_realign.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_realign.cpp $(C)/realign_plan.cpp $(C)/hostpool.cpp
libwhemul_realign.so: $(SRC) $(C)/realign.h $(C)/realign_plan.h $(C)/hostpool.h ../../include/whmec.h
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ $(SRC)
clean:
	rm -f libwhemul_realign.so
