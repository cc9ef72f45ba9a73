// Reader of the self-contained model file of dd3d_create_from_file (format: include/dd3d_b200.h).  Host code only: it
// makes no CUDA call, so a defective file is refused before any device work.
#pragma once

#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/dd3d_b200.h"

namespace dd3d {

constexpr char kModelFileMagic[8] = {'D', 'D', '3', 'D', 'B', '2', '0', '0'};
constexpr uint32_t kModelFileVersion = 1;
constexpr int kModelFileMaxNdim = 8;  // dd3d_load_weight's limit

struct ModelFileTensor {
    std::string name;
    std::vector<int64_t> shape;
    size_t data_offset = 0;  // byte offset of the fp32 data in ModelFile::bytes
    size_t count = 0;        // number of floats
};

struct ModelFile {
    std::vector<uint8_t> bytes;  // the whole file
    dd3d_model_desc desc{};
    dd3d_layout_desc layout{};
    int32_t backbone_norm = 0;
    int32_t fpn_channels = 0;
    std::vector<int32_t> fpn_inputs;   // empty: dd3d_set_fpn_inputs is not called
    std::vector<int32_t> in_features;  // empty: dd3d_set_in_features is not called
    int32_t canon_classes = 0;         // 0: dd3d_set_canonical_sizes is not called
    std::vector<float> canon;          // [canon_classes][3]
    std::vector<ModelFileTensor> tensors;
};

// Reads `path` and validates all of it (size, magic, version, struct sizes, checksum, every record inside the file, no
// name twice).  Returns false with *err naming the first defect.
bool read_model_file(const char* path, ModelFile* out, std::string* err);

}  // namespace dd3d
