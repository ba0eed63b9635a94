# TEST-ONLY: census of the tile planner's schedule (emul_census.cpp), with the library's 2^14-entry tiles.
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_census.cpp $(C)/pack.cpp $(C)/tile_plan.cpp $(C)/hostpool.cpp
all: libwhemul_census.so
libwhemul_census.so: $(SRC) $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ $(SRC)
clean:
	rm -f libwhemul_census.so
