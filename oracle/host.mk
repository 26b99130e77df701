# oracle/host.mk -- builds the UNMODIFIED reference host programs that load our plugin through GGML_BACKEND_PATH:
#
#   _ref/host/libggml-base.so libggml-cpu.so libggml.so libllama.so      the reference's own libraries
#   _ref/host/test-backend-ops                                           its per-op differential test
#   _ref/host/llama-bench                                                its benchmark tool (SURVEY 8d: the metric's definition)
#   _ref/host/libllama_host.so                                           our small driver over its public API (tools/llama_host.cpp)
#
# Everything is compiled with plain gcc/g++ from the sources where they lie under $(REF) (nothing is copied, no cmake);
# the one generated file the reference's build system would write, common/build-info.cpp, is produced from its template
# with sed.  Outputs go only into oracle/_ref/host (git-ignored; built where the reference sources exist, used as built elsewhere).
#
# The product (the plugin) names the host's libggml-base by soname only and never links, loads or rpaths anything here.
REF      ?= /root/reference
HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref/host
OBJ      := $(HERE)_ref/obj/host
$(shell mkdir -p $(OUT))
CC       := gcc
CXX      := g++

GGML_INC := -I$(REF)/ggml/include -I$(REF)/ggml/src
COMMON_D := -DNDEBUG -D_GNU_SOURCE -D_XOPEN_SOURCE=600 -DGGML_SCHED_MAX_COPIES=4 -DGGML_SHARED -DGGML_BACKEND_SHARED
CFLAGS   := -O3 -std=gnu11 -fPIC -w
CXXFLAGS := -O3 -std=gnu++17 -fPIC -w
# x86-64-v3 (AVX2+FMA+F16C): the objects must also run on the GPU box's host CPU
CPU_ARCH := -march=x86-64-v3

.PHONY: all libs tools clean
all: libs tools $(OUT)/libllama_host.so

# ------------------------------------------------------------------ ggml-base
BASE_C   := ggml.c ggml-alloc.c ggml-quants.c
BASE_CXX := ggml.cpp ggml-backend.cpp ggml-backend-meta.cpp ggml-opt.cpp ggml-threading.cpp gguf.cpp
BASE_OBJ := $(addprefix $(OBJ)/base/,$(BASE_C:.c=.c.o) $(BASE_CXX:.cpp=.cpp.o))
BASE_D   := $(COMMON_D) -DGGML_BUILD -DGGML_VERSION=\"0.21.0\" -DGGML_COMMIT=\"unknown\"
$(OBJ)/base/%.c.o: $(REF)/ggml/src/%.c
	@mkdir -p $(dir $@)
	$(CC) $(CFLAGS) $(BASE_D) $(GGML_INC) -c $< -o $@
$(OBJ)/base/%.cpp.o: $(REF)/ggml/src/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) $(BASE_D) $(GGML_INC) -c $< -o $@
$(OUT)/libggml-base.so: $(BASE_OBJ)
	$(CXX) -shared -Wl,-soname,libggml-base.so -o $@ $^ -lm -lpthread -ldl

# ------------------------------------------------------------------ ggml-cpu (a user's default build: repack + llamafile on)
CPU_DIR  := $(REF)/ggml/src/ggml-cpu
CPU_C    := ggml-cpu.c quants.c arch/x86/quants.c
CPU_CXX  := ggml-cpu.cpp binary-ops.cpp unary-ops.cpp ops.cpp traits.cpp vec.cpp repack.cpp hbm.cpp \
            arch/x86/repack.cpp arch/x86/cpu-feats.cpp amx/amx.cpp amx/mmq.cpp llamafile/sgemm.cpp
CPU_OBJ  := $(addprefix $(OBJ)/cpu/,$(CPU_C:.c=.c.o) $(CPU_CXX:.cpp=.cpp.o))
CPU_D    := $(COMMON_D) -DGGML_BACKEND_BUILD -DGGML_USE_CPU_REPACK -DGGML_USE_LLAMAFILE -DGGML_USE_OPENMP
CPU_INC  := $(GGML_INC) -I$(CPU_DIR)
$(OBJ)/cpu/%.c.o: $(CPU_DIR)/%.c
	@mkdir -p $(dir $@)
	$(CC) $(CFLAGS) $(CPU_ARCH) -fopenmp $(CPU_D) $(CPU_INC) -c $< -o $@
$(OBJ)/cpu/%.cpp.o: $(CPU_DIR)/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) $(CPU_ARCH) -fopenmp $(CPU_D) $(CPU_INC) -c $< -o $@
$(OUT)/libggml-cpu.so: $(CPU_OBJ) $(OUT)/libggml-base.so
	$(CXX) -shared -fopenmp -Wl,-soname,libggml-cpu.so -o $@ $(CPU_OBJ) -L$(OUT) -lggml-base -Wl,-rpath,'$$ORIGIN' -lm -lpthread

# ------------------------------------------------------------------ registry (libggml.so: CPU statically registered + the dl loader)
REG_OBJ  := $(OBJ)/reg/ggml-backend-reg.cpp.o $(OBJ)/reg/ggml-backend-dl.cpp.o
$(OBJ)/reg/%.cpp.o: $(REF)/ggml/src/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) $(COMMON_D) -DGGML_BUILD -DGGML_USE_CPU $(GGML_INC) -c $< -o $@
$(OUT)/libggml.so: $(REG_OBJ) $(OUT)/libggml-cpu.so
	$(CXX) -shared -Wl,-soname,libggml.so -o $@ $(REG_OBJ) -L$(OUT) -lggml-cpu -lggml-base -Wl,-rpath,'$$ORIGIN' -ldl

# ------------------------------------------------------------------ libllama
LLAMA_SRC := $(wildcard $(REF)/src/*.cpp) $(wildcard $(REF)/src/models/*.cpp)
LLAMA_OBJ := $(patsubst $(REF)/src/%.cpp,$(OBJ)/llama/%.cpp.o,$(LLAMA_SRC))
LLAMA_D   := $(COMMON_D) -DGGML_USE_CPU -DLLAMA_BUILD -DLLAMA_SHARED -DLLAMA_VERSION=\"0.2.0-dev\" -DLLAMA_COMMIT=\"unknown\"
$(OBJ)/llama/%.cpp.o: $(REF)/src/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) $(LLAMA_D) -I$(REF)/src -I$(REF)/include -I$(REF)/ggml/include -c $< -o $@
$(OUT)/libllama.so: $(LLAMA_OBJ) $(OUT)/libggml.so
	$(CXX) -shared -Wl,-soname,libllama.so -o $@ $(LLAMA_OBJ) -L$(OUT) -lggml -lggml-cpu -lggml-base -Wl,-rpath,'$$ORIGIN' -lpthread

libs: $(OUT)/libggml-base.so $(OUT)/libggml-cpu.so $(OUT)/libggml.so $(OUT)/libllama.so

# ------------------------------------------------------------------ test-backend-ops
$(OUT)/test-backend-ops: $(REF)/tests/test-backend-ops.cpp $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) $(COMMON_D) -DGGML_USE_CPU $(GGML_INC) $< -o $@ \
	    -L$(OUT) -lggml -lggml-cpu -lggml-base -Wl,-rpath,'$$ORIGIN' -lpthread

# ------------------------------------------------------------------ llama-bench (libllama-common + tools/llama-bench, unmodified)
COMMON_DIR := $(REF)/common
COMMON_SRC := $(filter-out $(COMMON_DIR)/llguidance.cpp,$(wildcard $(COMMON_DIR)/*.cpp)) $(wildcard $(COMMON_DIR)/jinja/*.cpp)
COMMON_OBJ := $(patsubst $(COMMON_DIR)/%.cpp,$(OBJ)/common/%.cpp.o,$(COMMON_SRC)) $(OBJ)/common/llguidance.cpp.o
COMMON_INC := -I$(COMMON_DIR) -I$(REF)/include -I$(REF)/ggml/include -I$(REF)/vendor -I$(REF)/vendor/cpp-httplib -I$(REF)/vendor/nlohmann -I$(REF)/vendor/sheredom -I$(REF)/src
COMMON_DEF := $(COMMON_D) -DLLAMA_SHARED -DCPPHTTPLIB_NO_EXCEPTIONS_DISABLED
$(OBJ)/common/%.cpp.o: $(COMMON_DIR)/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) $(COMMON_DEF) $(COMMON_INC) -c $< -o $@
# the file the reference's cmake would configure from common/build-info.cpp.in
$(OBJ)/common/build-info.cpp: $(COMMON_DIR)/build-info.cpp.in
	@mkdir -p $(dir $@)
	sed -e 's/@LLAMA_BUILD_NUMBER@/0/' -e 's/@LLAMA_BUILD_COMMIT@/unknown/' -e 's/@BUILD_COMPILER@/gcc/' -e 's/@BUILD_TARGET@/x86_64-linux-gnu/' $< > $@
$(OBJ)/common/build-info.cpp.o: $(OBJ)/common/build-info.cpp
	$(CXX) $(CXXFLAGS) -I$(COMMON_DIR) -c $< -o $@
HTTPLIB_OBJ := $(OBJ)/common/httplib.cpp.o
$(HTTPLIB_OBJ): $(REF)/vendor/cpp-httplib/httplib.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -I$(REF)/vendor/cpp-httplib -c $< -o $@
$(OUT)/libllama-common.so: $(COMMON_OBJ) $(OBJ)/common/build-info.cpp.o $(HTTPLIB_OBJ) $(OUT)/libllama.so
	$(CXX) -shared -Wl,-soname,libllama-common.so -o $@ $(COMMON_OBJ) $(OBJ)/common/build-info.cpp.o $(HTTPLIB_OBJ) -L$(OUT) -lllama -lggml -lggml-base -Wl,-rpath,'$$ORIGIN' -lpthread
$(OUT)/llama-bench: $(REF)/tools/llama-bench/llama-bench.cpp $(REF)/tools/llama-bench/main.cpp $(OUT)/libllama-common.so
	$(CXX) $(CXXFLAGS) $(COMMON_DEF) $(COMMON_INC) $(REF)/tools/llama-bench/llama-bench.cpp $(REF)/tools/llama-bench/main.cpp -o $@ \
	    -L$(OUT) -lllama-common -lllama -lggml -lggml-base -Wl,-rpath,'$$ORIGIN' -lpthread

tools: $(OUT)/test-backend-ops $(OUT)/llama-bench

# ------------------------------------------------------------------ our driver over the public API (ctypes entry points for tests, smoke, bench)
$(OUT)/libllama_host.so: $(abspath $(HERE)../tools/llama_host.cpp) $(OUT)/libllama.so
	$(CXX) -O2 -std=c++17 -fPIC -shared -I$(REF)/include -I$(REF)/ggml/include $< -o $@ -L$(OUT) -lllama -lggml -lggml-base -Wl,-rpath,'$$ORIGIN'

clean:
	rm -rf $(OUT)
