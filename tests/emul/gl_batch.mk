# TEST-ONLY: host emulation of whmec_genotype_batch (emul_gl_batch.cpp; tables that fit no group: emul_gl_bounded.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_gl_batch.cpp emul_gl_bounded.cpp $(C)/gl_batch.cpp $(C)/gl_pack.cpp $(C)/pack.cpp $(C)/hostpool.cpp
libwhemul_gl_batch.so: $(SRC) $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ $(SRC)
clean:
	rm -f libwhemul_gl_batch.so
