# TEST-ONLY: host emulation of the groups of whmec_solve_batch: a tile group (emul_batch.cpp, with 2^14-entry tiles and with 2^4-entry
# ones) and a fused-trio group (emul_fused_batch.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_batch.cpp $(C)/pack.cpp $(C)/tile_plan.cpp $(C)/hostpool.cpp
all: libwhemul_batch.so libwhemul_batch_small.so libwhemul_fused_batch.so
libwhemul_batch.so: $(SRC) emul_sched.cpp $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ $(SRC)
libwhemul_batch_small.so: $(SRC) emul_sched.cpp $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -DWHMEC_TILE_SMAX=4 -fPIC -shared -pthread -o $@ $(SRC)
libwhemul_fused_batch.so: emul_fused_batch.cpp emul.cpp $(C)/pack.cpp $(C)/hostpool.cpp $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ emul_fused_batch.cpp $(C)/pack.cpp $(C)/hostpool.cpp
clean:
	rm -f libwhemul_batch.so libwhemul_batch_small.so libwhemul_fused_batch.so
