// Host-only dump of a part's block directory as part_dir.cc builds it, for tests/test_part_schema_mix.py (built there with
// g++, no CUDA).  Usage: part_dir_dump <dir with the part's files> < keys; stdin holds one interned key per line
// ("f:<field>" / "t:<family>/<tag>").  Prints
//   RC <rc> <error>
//   FILES <name> ...                              the part's file table
//   B <sid> <count> <n_cols>                      per block, then per column
//   C <name_id> <value_type> <off> <size> <file_id>
//   K <id> <key>                                  NameTable::find of every key on stdin (0: never interned)
//   SLICED <0|1>                                  the directory parsed in as many slices as primary frames, merged, is the same
#include <dirent.h>

#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <iterator>
#include <string>
#include <vector>

#include "part_dir.hpp"

using namespace bydb;

int main(int argc, char **argv) {
    if (argc != 2) return 2;
    std::vector<std::string> names;
    std::vector<std::vector<uint8_t>> data;
    DIR *d = opendir(argv[1]);
    if (!d) return 2;
    while (dirent *e = readdir(d)) {
        if (e->d_name[0] == '.') continue;
        std::ifstream in(std::string(argv[1]) + "/" + e->d_name, std::ios::binary);
        names.push_back(e->d_name);
        data.emplace_back(std::istreambuf_iterator<char>(in), std::istreambuf_iterator<char>());
    }
    closedir(d);
    std::vector<FileImage> files;
    for (size_t i = 0; i < names.size(); ++i) files.push_back(FileImage{names[i], data[i].data(), data[i].size()});
    NameTable table;
    PartDir dir;
    std::string err;
    const int rc = build_part_dir(files, table, dir, err);
    std::printf("RC %d %s\n", rc, err.c_str());
    if (rc) return 0;
    std::printf("FILES");
    for (const auto &f : dir.files) std::printf(" %s", f.c_str());
    std::printf("\n");
    for (const DevBlock &b : dir.blocks) {
        std::printf("B %llu %u %u\n", static_cast<unsigned long long>(b.sid), b.count, b.n_cols);
        for (uint32_t c = 0; c < b.n_cols; ++c) {
            const DevCol &col = dir.cols[b.col_begin + c];
            std::printf("C %u %u %llu %u %u\n", col.name_id, col.value_type, static_cast<unsigned long long>(col.off), col.size, col.file_id);
        }
    }
    std::string key;
    while (std::getline(std::cin, key)) std::printf("K %u %s\n", table.find(key), key.c_str());
    // slices start with empty positional caches: the merged slices must give the same directory (file ids compared by
    // name: parser threads number the .tf files in the order they meet them)
    size_t n_primary = 0;
    bool same = count_primary_blocks(files, &n_primary, err) == 0;
    std::vector<PartDir> pieces(n_primary);
    for (size_t t = 0; same && t < n_primary; ++t) same = build_part_dir(files, table, pieces[t], err, t, n_primary) == 0;
    PartDir merged;
    same = same && merge_part_dirs(pieces, merged, err) == 0 && merged.blocks.size() == dir.blocks.size() && merged.cols.size() == dir.cols.size() &&
           (dir.blocks.empty() || std::memcmp(merged.blocks.data(), dir.blocks.data(), dir.blocks.size() * sizeof(DevBlock)) == 0);
    for (size_t i = 0; same && i < dir.cols.size(); ++i) {
        const DevCol &a = merged.cols[i], &b = dir.cols[i];
        same = a.off == b.off && a.size == b.size && a.name_id == b.name_id && a.value_type == b.value_type &&
               merged.files[a.file_id] == dir.files[b.file_id];
    }
    std::printf("SLICED %d\n", same ? 1 : 0);
    return 0;
}
