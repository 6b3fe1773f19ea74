# TEST INFRASTRUCTURE.  Builds oracle/_ref/libdbow_ref.so from the reference's own, unmodified DBoW2 sources in a pl-slam
# checkout (make -f dbow.mk REF=/path/to/pl-slam; __graft_entry__.build() passes oracle.refbin.reference_dir()):
# 3rdparty/DBoW2/include/DBoW2/TemplatedVocabulary.h, src/DBoW2/{BowVector,FeatureVector,ScoringObject,FORB}.cpp and src/DUtils, against
# the OpenCV stand-in of opencv_stub/, with the array-filling subclass of ref_wrap_dbow.cpp.  Outputs are git-ignored.
OUT := ../_ref
CXX ?= g++

ifeq ($(REF),)
all:
	@echo "oracle/ref_build/dbow.mk: set REF to a pl-slam checkout" >&2; exit 1
else
DB  := $(REF)/3rdparty/DBoW2
SRC := ref_wrap_dbow.cpp $(DB)/src/DBoW2/BowVector.cpp $(DB)/src/DBoW2/FeatureVector.cpp $(DB)/src/DBoW2/ScoringObject.cpp $(DB)/src/DBoW2/FORB.cpp \
       $(DB)/src/DUtils/Random.cpp $(DB)/src/DUtils/Timestamp.cpp
all: $(OUT)/libdbow_ref.so

$(OUT)/libdbow_ref.so: $(SRC) opencv_stub/opencv2/core.hpp $(DB)/include/DBoW2/TemplatedVocabulary.h
	mkdir -p $(OUT)
	$(CXX) -std=c++11 -O2 -fPIC -w -ffp-contract=off -fno-fast-math -Iopencv_stub -I$(DB)/include -I$(DB)/include/DBoW2 \
	       -I$(DB)/include/DUtils -shared -o $@ $(SRC) -lm
endif

.PHONY: all
