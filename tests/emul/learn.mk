# TEST-ONLY: host emulation of whmec_learn (emul_learn.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_learn.cpp $(C)/learn_plan.cpp $(C)/hostpool.cpp
libwhemul_learn.so: $(SRC) $(C)/learn.h $(C)/learn_plan.h $(C)/hostpool.h ../../include/whmec.h
	$(CXX) -std=c++17 -O2 -Wall -fPIC -shared -pthread -o $@ $(SRC)
clean:
	rm -f libwhemul_learn.so
