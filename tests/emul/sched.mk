# TEST-ONLY: host emulation of the tile kernel's schedule (emul_sched.cpp), with 2^14-entry tiles and with 2^4-entry ones.
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_sched.cpp $(C)/pack.cpp $(C)/tile_plan.cpp $(C)/hostpool.cpp
all: libwhemul_sched.so libwhemul_sched_small.so
libwhemul_sched.so: $(SRC) $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ $(SRC)
libwhemul_sched_small.so: $(SRC) $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -DWHMEC_TILE_SMAX=4 -fPIC -shared -pthread -o $@ $(SRC)
clean:
	rm -f libwhemul_sched.so libwhemul_sched_small.so
