# TEST-ONLY: emulation of the tile kernel's narrow steady-state panels (emul_narrow.cpp, which includes emul_tile.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_narrow.cpp $(C)/pack.cpp $(C)/tile_plan.cpp $(C)/hostpool.cpp
all: libwhemul_narrow.so
libwhemul_narrow.so: $(SRC) emul_tile.cpp $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ $(SRC)
clean:
	rm -f libwhemul_narrow.so
