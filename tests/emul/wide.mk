# TEST-ONLY: host emulation of the wide column sweep (emul_wide.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
libwhemul_wide.so: emul_wide.cpp $(C)/col_plan.cpp $(C)/pack.cpp $(C)/hostpool.cpp $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ emul_wide.cpp $(C)/col_plan.cpp $(C)/pack.cpp $(C)/hostpool.cpp
clean:
	rm -f libwhemul_wide.so
