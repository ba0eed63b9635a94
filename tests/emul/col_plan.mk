# TEST-ONLY: plan inspector of the column-kernel paths (emul_col_plan.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
libwhemul_col_plan.so: emul_col_plan.cpp $(C)/col_plan.cpp $(C)/pack.cpp $(C)/hostpool.cpp $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ emul_col_plan.cpp $(C)/col_plan.cpp $(C)/pack.cpp $(C)/hostpool.cpp
clean:
	rm -f libwhemul_col_plan.so
