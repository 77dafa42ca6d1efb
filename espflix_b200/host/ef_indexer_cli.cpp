// ef_indexer_cli video.ts fwd.ts rev.ts out_dir — the index half of the reference tool's main()
// (indexer/indexer.cpp:318-333) without the ffmpeg calls: three make_index() + merge_index().
// ef_indexer_cli title_dir [qscale] — a title directory that holds only video.ts: the tool's make_video() fwd and rwd steps
// (indexer.cpp:308-309) on the GPU (ef_trick_build, no ffmpeg) write title_dir/video_fwd.ts and title_dir/video_rwd.ts, then
// make_index() + merge_index() of the three files write title_dir/video.idx.
// ef_indexer_cli --encode pictures.i420 title_dir [qscale_i qscale_p] — the whole make_video() from decoded pictures: the 352 x 192
// I420 pictures of pictures.i420 are encoded on the GPU (ef_encode_build at espflix_b200.capi.ENCODE_DEFAULTS, no ffmpeg) into
// title_dir/video.ts, then the title_dir path above writes video_fwd.ts, video_rwd.ts and video.idx.
// ef_indexer_cli --encode pictures.i420 title_dir --rate bit_rate vbv_bits — the same, with video.ts encoded to a bit rate and buffer
// size (ef_encode_build_rate at espflix_b200.capi.ENCODE_RATE_DEFAULTS' quantisers 3..31) in place of the fixed quantisers.
//   --audio pcm.s16le (last) gives the title its sound: mono 16-bit little-endian PCM at 48 kHz, encoded to SBC (ef_sbc_encode at
//   espflix_b200.capi.AUDIO_ENCODE_DEFAULTS: the reference's 48 kHz, 192 kbit/s) and interleaved on PID 0x102 (ef_mux_audio). The
//   trick files stay audio-free, as the reference's "-an" makes them.
//   --poster poster.i420 (last) also writes title_dir/poster.ts, what make_video()'s "ffmpeg ... -bf 0 -q 2 poster.ts" makes
//   (indexer.cpp:306): the one 352 x 192 I420 picture of poster.i420 as an I picture at quantiser scale 2 (ef_encode_build with gop 1
//   and qscale_i 2, the rest as video.ts; espflix_b200.capi.encode_poster).
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

// the video transport stream `ts` with the SBC of the PCM in `pcm_path` interleaved
static std::vector<uint8_t> add_audio(const std::vector<uint8_t>& ts, const std::string& pcm_path)
{
    const std::vector<uint8_t> raw = read_file(pcm_path);
    if (raw.size() % 2) throw std::runtime_error(pcm_path + ": not a whole number of 16-bit samples");
    std::vector<int16_t> pcm(raw.size() / 2 + 1, 0);
    for (size_t i = 0; i + 1 < pcm.size(); i++) pcm[i] = (int16_t)(raw[2 * i] | raw[2 * i + 1] << 8);
    const ef_audio_params p = { 3, 0, 28, 0, 0 };
    const uint64_t po[2] = { 0, raw.size() / 2 };
    uint64_t so[2] = { 0, 0 };
    if (ef_sbc_encode(0, pcm.data(), po, 1, &p, nullptr, 0, so) != EF_ENOMEM && so[1]) throw std::runtime_error("ef_sbc_encode: sizing failed");
    std::vector<uint8_t> sbc(so[1] + 1);
    if (ef_sbc_encode(0, pcm.data(), po, 1, &p, sbc.data(), so[1], so) != EF_OK) throw std::runtime_error(std::string("ef_sbc_encode: ") + ef_last_error());
    const uint64_t to[2] = { 0, ts.size() };
    uint64_t oo[2] = { 0, 0 };
    const int rc = ef_mux_audio(0, ts.data(), to, sbc.data(), so, 1, &p, nullptr, 0, oo);
    if (rc != EF_ENOMEM) throw std::runtime_error(std::string("ef_mux_audio: ") + ef_last_error());
    std::vector<uint8_t> out(oo[1]);
    if (ef_mux_audio(0, ts.data(), to, sbc.data(), so, 1, &p, out.data(), out.size(), oo) != EF_OK)
        throw std::runtime_error(std::string("ef_mux_audio: ") + ef_last_error());
    return out;
}

// the transport stream of the I420 pictures `pics` encoded with `p` (and to `rate` when it is not NULL)
static std::vector<uint8_t> encode(const std::vector<uint8_t>& pics, const ef_encode_params& p, const ef_rate_params* rate)
{
    const uint64_t off[2] = { 0, pics.size() / 101376 };
    uint64_t to[2] = { 0, 0 };
    std::vector<uint8_t> ts(pics.size() / 4);
    auto build = [&]() {
        return rate ? ef_encode_build_rate(0, pics.data(), off, 1, &p, rate, ts.data(), ts.size(), to, nullptr, nullptr)
                    : ef_encode_build(0, pics.data(), off, 1, &p, ts.data(), ts.size(), to);
    };
    int rc = build();
    if (rc == EF_ENOMEM && to[1] > ts.size()) {
        ts.resize(to[1]);
        rc = build();
    }
    if (rc != EF_OK) throw std::runtime_error(std::string(rate ? "ef_encode_build_rate: " : "ef_encode_build: ") + ef_last_error());
    ts.resize(to[1]);
    return ts;
}

// title_dir/video.ts of the pictures in `pictures` (I420, 101,376 bytes each), with the sound of `pcm_path` when it is not empty
static void make_video(const std::string& pictures, const std::string& dir, int qscale_i, int qscale_p, const ef_rate_params* rate,
                       const std::string& pcm_path)
{
    const std::vector<uint8_t> pics = read_file(pictures);
    if (pics.empty() || pics.size() % 101376) throw std::runtime_error(pictures + ": not a whole number of 352 x 192 I420 pictures");
    std::vector<uint8_t> ts = encode(pics, ef_encode_params{ 12, qscale_i, qscale_p, 7, 1, 2, 0, 3750 }, rate);
    if (!pcm_path.empty()) ts = add_audio(ts, pcm_path);
    write_file(dir + "/video.ts", ts.data(), ts.size());
}

// title_dir/poster.ts of the one picture in `picture`: gop 1, qscale_i 2 (ffmpeg's -q 2)
static void make_poster(const std::string& picture, const std::string& dir)
{
    const std::vector<uint8_t> pic = read_file(picture);
    if (pic.size() != 101376) throw std::runtime_error(picture + ": not one 352 x 192 I420 picture");
    const std::vector<uint8_t> ts = encode(pic, ef_encode_params{ 1, 2, 8, 7, 1, 2, 0, 3750 }, nullptr);
    write_file(dir + "/poster.ts", ts.data(), ts.size());
}

int main(int argc, char** argv)
{
    const bool encode = argc >= 2 && std::string(argv[1]) == "--encode";
    std::string pcm_path, poster_path;
    if (encode && argc >= 6 && std::string(argv[argc - 2]) == "--poster") { poster_path = argv[argc - 1]; argc -= 2; }
    if (encode && argc >= 6 && std::string(argv[argc - 2]) == "--audio") { pcm_path = argv[argc - 1]; argc -= 2; }
    const bool rated = encode && argc == 7 && std::string(argv[4]) == "--rate";
    ef_rate_params rate = { 1500000, 250000, 3, 31 };
    if (rated) {
        rate.bit_rate = (uint32_t)strtoul(argv[5], nullptr, 10);
        rate.vbv_bits = (uint32_t)strtoul(argv[6], nullptr, 10);
    }
    if (encode ? (argc != 4 && argc != 6 && !rated) : (argc != 5 && argc != 2 && argc != 3)) {
        fprintf(stderr, "usage: %s video.ts fwd.ts rev.ts out_dir\n       %s title_dir [qscale]   (title_dir/video.ts -> video_fwd.ts, video_rwd.ts, video.idx)\n"
                        "       %s --encode pictures.i420 title_dir [qscale_i qscale_p | --rate bit_rate vbv_bits] [--audio pcm.s16le] [--poster poster.i420]   "
                        "(-> title_dir/video.ts, then as title_dir)\n",
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
            if (encode) make_video(argv[2], dir, argc == 6 ? atoi(argv[4]) : 8, argc == 6 ? atoi(argv[5]) : 8, rated ? &rate : nullptr, pcm_path);
            if (!poster_path.empty()) make_poster(poster_path, dir);
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
