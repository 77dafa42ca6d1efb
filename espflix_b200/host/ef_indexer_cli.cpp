// ef_indexer_cli video.ts fwd.ts rev.ts out_dir — the index half of the reference tool's main()
// (indexer/indexer.cpp:318-333) without the ffmpeg calls: three make_index() + merge_index().
// ef_indexer_cli title_dir [qscale] — a title directory that holds only video.ts: the tool's make_video() fwd and rwd steps
// (indexer.cpp:308-309) on the GPU (ef_trick_build, no ffmpeg) write title_dir/video_fwd.ts and title_dir/video_rwd.ts, then
// make_index() + merge_index() of the three files write title_dir/video.idx.
// ef_indexer_cli --encode pictures.i420 title_dir [qscale_i qscale_p] — the whole make_video() from decoded pictures: the 352 x 192
// I420 pictures of pictures.i420 are encoded on the GPU (ef_encode_build at espflix_b200.capi.ENCODE_DEFAULTS, no ffmpeg) into
// title_dir/video.ts, then the title_dir path above writes video_fwd.ts, video_rwd.ts and video.idx.
#include <stdio.h>
#include <stdlib.h>

#include <exception>
#include <stdexcept>
#include <string>
#include <vector>

#include "espflix_b200.h"
#include "ef_indexer.h"

static std::vector<uint8_t> read_file(const std::string& path)
{
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) throw std::runtime_error("cannot open " + path);
    std::vector<uint8_t> data;
    uint8_t buf[1 << 16];
    size_t n;
    while ((n = fread(buf, 1, sizeof(buf), f)) > 0) data.insert(data.end(), buf, buf + n);
    fclose(f);
    return data;
}

static void write_file(const std::string& path, const uint8_t* data, size_t n)
{
    FILE* f = fopen(path.c_str(), "wb");
    if (!f || fwrite(data, 1, n, f) != n || fclose(f) != 0) throw std::runtime_error("cannot write " + path);
}

// video_fwd.ts and video_rwd.ts of dir/video.ts
static void make_trick_files(const std::string& dir, int qscale)
{
    const std::vector<uint8_t> main = read_file(dir + "/video.ts");
    const uint64_t off[2] = { 0, main.size() };
    uint64_t fo[2] = { 0, 0 }, ro[2] = { 0, 0 }, cap = main.size() + 188 * 1024;
    std::vector<uint8_t> fwd, rwd;
    for (int attempt = 0;; attempt++) {
        fwd.resize(cap); rwd.resize(cap);
        const int rc = ef_trick_build(0, main.data(), off, 1, qscale, fwd.data(), cap, fo, rwd.data(), cap, ro);
        if (rc == EF_ENOMEM && attempt == 0 && (fo[1] > cap || ro[1] > cap)) { cap = fo[1] > ro[1] ? fo[1] : ro[1]; continue; }
        if (rc != EF_OK) throw std::runtime_error(std::string("ef_trick_build: ") + ef_last_error());
        break;
    }
    write_file(dir + "/video_fwd.ts", fwd.data(), fo[1]);
    write_file(dir + "/video_rwd.ts", rwd.data(), ro[1]);
}

// title_dir/video.ts of the pictures in `pictures` (I420, 101,376 bytes each)
static void make_video(const std::string& pictures, const std::string& dir, int qscale_i, int qscale_p)
{
    const std::vector<uint8_t> pics = read_file(pictures);
    if (pics.empty() || pics.size() % 101376) throw std::runtime_error(pictures + ": not a whole number of 352 x 192 I420 pictures");
    const uint64_t off[2] = { 0, pics.size() / 101376 };
    const ef_encode_params p = { 12, qscale_i, qscale_p, 7, 1, 2, 0, 3750 };
    uint64_t to[2] = { 0, 0 };
    std::vector<uint8_t> ts(pics.size() / 4);
    int rc = ef_encode_build(0, pics.data(), off, 1, &p, ts.data(), ts.size(), to);
    if (rc == EF_ENOMEM && to[1] > ts.size()) {
        ts.resize(to[1]);
        rc = ef_encode_build(0, pics.data(), off, 1, &p, ts.data(), ts.size(), to);
    }
    if (rc != EF_OK) throw std::runtime_error(std::string("ef_encode_build: ") + ef_last_error());
    write_file(dir + "/video.ts", ts.data(), to[1]);
}

int main(int argc, char** argv)
{
    const bool encode = argc >= 2 && std::string(argv[1]) == "--encode";
    if (encode ? (argc != 4 && argc != 6) : (argc != 5 && argc != 2 && argc != 3)) {
        fprintf(stderr, "usage: %s video.ts fwd.ts rev.ts out_dir\n       %s title_dir [qscale]   (title_dir/video.ts -> video_fwd.ts, video_rwd.ts, video.idx)\n"
                        "       %s --encode pictures.i420 title_dir [qscale_i qscale_p]   (-> title_dir/video.ts, then as title_dir)\n",
                argv[0], argv[0], argv[0]);
        return 2;
    }
    try {
        std::vector<idx> all;
        if (argc == 5 && !encode) {
            make_index(argv[1], all);
            make_index(argv[2], all);
            make_index(argv[3], all);
            merge_index(all, argv[4]);
        } else {
            const std::string dir = encode ? argv[3] : argv[1];
            const int qscale = !encode && argc == 3 ? atoi(argv[2]) : 8;
            if (encode) make_video(argv[2], dir, argc == 6 ? atoi(argv[4]) : 8, argc == 6 ? atoi(argv[5]) : 8);
            make_trick_files(dir, qscale);
            make_index(dir + "/video.ts", all);
            make_index(dir + "/video_fwd.ts", all);
            make_index(dir + "/video_rwd.ts", all);
            merge_index(all, dir);
        }
    } catch (const std::exception& e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}
