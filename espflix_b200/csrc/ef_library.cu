// espflix_b200/csrc/ef_library.cu — titles held in device memory (ef_library_*): every stream's place in its title resolved on the
// device from the title's video.idx, and every stream's run of packets gathered from the title into one TS submit.
//
// The reference's player reads a title through Streamer::get(url, offset) and 8-packet Buffers (espflix.cpp:723-747, 787-798) and
// seeks with the video.idx sample at idx_hdr::pts2offset (espflix.cpp:607-629, 823-829). Here the titles live in HBM: a command is
// a few bytes from the host, the offset arithmetic and the sample read run on the device, and a submit is a device-to-device gather.
// The poster menu (nav(), menu(), load_poster(), espflix.cpp:704-720, 778-785, 1060-1069) runs here too: the scroll mode of each
// stream's latest nav, the saved positions nv_read() / nv_write() keep in NVS, and the mode a submit carries to the present calls.
#include "../../include/espflix_b200.h"
#include "ef_common.cuh"

namespace {

// idx_hdr::pts2offset (espflix.cpp:607-629): the byte offset in video.idx of the sample for main pts `pts` at `speed`. The casts and
// unsigned divisions are the reference's: at speed 1 (uint32) applies to the difference before the two divisions, at -1 first_pts
// is subtracted a second time (and wraps), and every min() is unsigned.
__device__ __forceinline__ uint32_t lib_pts2offset(const EfLibTitle& t, int64_t pts, int speed)
{
    uint32_t offset;
    pts = max(min(pts, t.v_last), t.v_first);
    if (speed == 1) {
        offset = (uint32_t)(pts - t.v_first) / t.f_trick / t.f_bin;
        offset = min(t.f_n - 1u, offset);
        offset += t.v_n;
    } else if (speed == -1) {
        offset = (uint32_t)((t.v_last - pts) - t.v_first) / t.r_trick / t.r_bin;
        offset = min(t.r_n - 1u, offset);
        offset += t.v_n + t.f_n;
    } else {
        offset = (uint32_t)((pts - t.v_first) / (int64_t)t.v_bin);
        offset = min(t.v_n - 1u, offset);
    }
    return offset * 4u + 104u;                                             // sizeof(idx_hdr)
}

// play(i, speed, get_index(speed, pos) * 188) (espflix.cpp:800-811, 823-829): the stream reads its title's file speed + 1 from the
// packet the sample names. A sample that points at or past the end of its file leaves the cursor there (the stream ends at its next
// submit); the reference's uint32 product would wrap only for such samples.
__device__ __forceinline__ void lib_play(EfLibStream& v, const EfLibTitle& t, int speed)
{
    const uint32_t at = lib_pts2offset(t, v.pos, speed);
    const uint32_t sample = *(const uint32_t*)(t.idx + at);                 // 4-byte aligned: 104 + 4k into a cudaMalloc'd image
    v.speed = speed;
    v.file = speed + 1;
    v.cursor = (uint64_t)sample * 188u;
    v.state = EF_LIB_PLAYING;
}

// nav(s, i) (espflix.cpp:704-720, 1060-1069): the scroll mode load_poster() flushes the poster's last picture with, from the old title
// (_nav - i; 0 before the first nav), pos = nv_read() of title i, and the poster's bytes from byte 0. hide_progress() stages a blend of
// 0 on a presenting context (ovl), as ef_present_overlay stages it. _speed stays.
__device__ __forceinline__ void lib_nav(EfLibStream& v, int s, int i, uint8_t* mode, const int64_t* nv, int n_streams, EfOverlayState* ovl)
{
    const int dir = v.title == -1 ? 0 : v.title - i;
    mode[s] = dir == 0 ? 1 : dir < 0 ? 2 : 3;
    v.title = i;
    v.pos = nv[(size_t)i * n_streams + s];
    v.state = EF_LIB_POSTER;
    v.file = EF_LIB_POSTER_FILE;
    v.cursor = 0;
    if (ovl) {
        ovl[s].p_blend = 0;
        ovl[s].pending |= 2u;
    }
}

}  // namespace

// One thread per commanded stream of [first, first + count): the ESPFlix method the command names (espflix.cpp:704-720, 778-859,
// 906-939). Every command but PLAY_AT, RESUME, NAV and NAV_STEP first saves pos = pts2pts(get_pts(), _speed) on a PLAYING stream
// (save_pos, espflix.cpp:843-852); get_pts() is the stream's last_pts after the current submit. The host has checked the arguments
// against every stream's state. mode / nv / ovl: the poster modes, the saved positions (nv[title][stream]) and the overlay states
// (NULL off a presenting context); only the poster commands use them.
__global__ void ef_library_resolve_kernel(EfLibStream* __restrict__ ls, const EfLibTitle* __restrict__ titles, const int64_t* __restrict__ pts_last,
                                          int first, int count, int cmd, int title, int64_t arg, uint8_t* __restrict__ mode, int64_t* __restrict__ nv,
                                          int n_streams, int n_titles, EfOverlayState* __restrict__ ovl)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const int s = first + k;
    EfLibStream v = ls[s];
    if (cmd == EF_LIB_PLAY_AT) {                                        // nav(i) with pos, then play_pause() from NAV
        v.title = title;
        v.pos = arg;
        lib_play(v, titles[title], 0);
    } else if (cmd == EF_LIB_NAV) {
        lib_nav(v, s, title, mode, nv, n_streams, ovl);
    } else if (cmd == EF_LIB_NAV_STEP) {                                // the left / right keys in NAV: nav(_nav +- 1)
        const int64_t i = (int64_t)v.title + arg;
        if (i < 0 || i >= n_titles) return;                             // nav()'s early return
        lib_nav(v, s, (int)i, mode, nv, n_streams, ovl);
    } else {
        const EfLibTitle& t = titles[v.title];
        if (cmd != EF_LIB_RESUME && v.state == EF_LIB_PLAYING) v.pos = ef_lib_pts2pts(t, pts_last[s], v.speed);
        switch (cmd) {
        case EF_LIB_PLAY: lib_play(v, t, 0); break;
        case EF_LIB_SKIP:                                               // n.pos += s * 90000: an int product
            v.pos += (int32_t)((uint32_t)(int32_t)arg * 90000u);
            lib_play(v, t, 0);
            break;
        case EF_LIB_FAST_FORWARD: lib_play(v, t, 1); break;
        case EF_LIB_REWIND: lib_play(v, t, -1); break;
        case EF_LIB_PAUSE: if (v.state == EF_LIB_PLAYING) v.state = EF_LIB_PAUSED; break;
        case EF_LIB_RESUME: v.state = EF_LIB_PLAYING; break;
        case EF_LIB_MENU:                                               // menu(), then loop()'s pending-NAV branch
            if (v.state == EF_LIB_POSTER) break;                        // set_state(NAV) from NAV
            if (v.state == EF_LIB_PLAYING) {                            // save_pos(pts, true)
                nv[(size_t)v.title * n_streams + s] = v.pos;
                if (v.speed) { lib_play(v, t, 0); break; }              // trick mode: play_pause() from NAV, no poster
            }
            lib_nav(v, s, v.title, mode, nv, n_streams, ovl);           // set_state(NAV): nav(_nav), mode 1
            break;
        default: v.state = EF_LIB_STOPPED; break;                           // STOP
        }
    }
    ls[s] = v;
}

// One thread per stream: one iteration of ESPFlix::loop() (espflix.cpp:886-1010) with keys[s] (0: none). First the pause branch of a
// stream whose title ended (_pending == DONE): nav(s, title) as EF_LIB_MENU does on ENDED; a title without a poster stays ENDED and
// ignores the key. Then the key on the state that left, its pending action resolved at once (the library pauses at the submit
// boundary): the EF_LIB_* command it runs as, by the rules of ef_library_resolve_kernel. A command ef_library_command would refuse
// (a missing trick file, no poster at the target) does nothing. done[s] (may be NULL) = that command or EF_KEY_DONE_NOTHING, with
// EF_KEY_DONE_ENDED when the DONE branch ran; ops[s] = the restart op of the iteration. ovl (NULL off a presenting context): the blend
// play(), the pause, the resume and nav() leave, staged as ef_present_overlay stages it. clk (NULL before ef_present_clock): on a
// stream whose clock is on, speed and the paused bit follow the stream, _last_seconds = 0 where play_pause() and the pause zero it
// (espflix.cpp:819, 935), and a nav to another title writes that title's records.
__global__ void ef_library_keys_kernel(EfLibStream* __restrict__ ls, const EfLibTitle* __restrict__ titles, const int64_t* __restrict__ pts_last,
                                       const uint8_t* __restrict__ keys, uint8_t* __restrict__ done, uint8_t* __restrict__ ops, uint8_t* __restrict__ mode,
                                       int64_t* __restrict__ nv, int n_streams, int n_titles, EfOverlayState* __restrict__ ovl, EfClockState* __restrict__ clk)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_streams) return;
    EfLibStream v = ls[s];
    const int key = keys[s], title0 = v.title;
    uint32_t d = EF_KEY_DONE_NOTHING;
    int op = 0, blend = -2;                                             // -2: no blend of its own staged
    bool zero_seconds = false;
    if (v.state != EF_LIB_IDLE && !(v.state == EF_LIB_ENDED && !titles[v.title].ts[EF_LIB_POSTER_FILE])) {
        if (v.state == EF_LIB_ENDED) {                                  // the DONE branch: set_state(NAV)
            lib_nav(v, s, v.title, mode, nv, n_streams, ovl);
            d |= EF_KEY_DONE_ENDED;
            op = 1;
        }
        const bool play = key == EF_KEY_PLAY || key == EF_KEY_SELECT, side = key == EF_KEY_RIGHT || key == EF_KEY_LEFT;
        const bool vert = key == EF_KEY_UP || key == EF_KEY_DOWN;
        const int sign = key == EF_KEY_RIGHT || key == EF_KEY_UP ? 1 : -1;
        int cmd = -1, arg = 0;
        if (v.state == EF_LIB_POSTER) {
            if (play) cmd = EF_LIB_PLAY;                                // play_pause() from NAV
            else if (side) { cmd = EF_LIB_NAV_STEP; arg = sign; }       // nav(_nav +- 1)
            zero_seconds = play;
        } else if (v.state == EF_LIB_PLAYING) {                         // the key pauses with _pending set; the pause branch
            if (key == EF_KEY_MENU) cmd = EF_LIB_MENU;
            else if (v.speed && (play || side || vert)) cmd = EF_LIB_PLAY;   // trick mode: play_pause() from NAV
            else if (play) cmd = EF_LIB_PAUSE;
            else if (side) cmd = sign > 0 ? EF_LIB_FAST_FORWARD : EF_LIB_REWIND;
            else if (vert) { cmd = EF_LIB_SKIP; arg = 30 * sign; }
            zero_seconds = cmd >= 0 && (play || v.speed);               // play_pause(), or the NONE case of the pause branch
        } else if (v.state == EF_LIB_PAUSED) {
            if (key == EF_KEY_MENU) cmd = EF_LIB_MENU;
            else if (play) cmd = EF_LIB_RESUME;
            else if (side) cmd = sign > 0 ? EF_LIB_FAST_FORWARD : EF_LIB_REWIND;
            zero_seconds = play;
        } else if (v.state == EF_LIB_STOPPED) {
            if (key == EF_KEY_MENU) cmd = EF_LIB_MENU;
            zero_seconds = play;                                        // play_pause() does nothing else there
        }
        const EfLibTitle& t = titles[v.title];
        int nav_to = -1;                                                // the title whose poster the command shows
        if (cmd == EF_LIB_NAV_STEP) {
            nav_to = v.title + arg;
            if (nav_to < 0 || nav_to >= n_titles) cmd = -1;             // nav()'s early return
        } else if (cmd == EF_LIB_MENU && !(v.state == EF_LIB_PLAYING && v.speed)) nav_to = v.title;
        if (cmd >= 0 && nav_to >= 0 && !titles[nav_to].ts[EF_LIB_POSTER_FILE]) cmd = -1;
        if ((cmd == EF_LIB_FAST_FORWARD && !t.ts[2]) || (cmd == EF_LIB_REWIND && !t.ts[0])) cmd = -1;
        if (cmd >= 0) {
            if (cmd != EF_LIB_RESUME && v.state == EF_LIB_PLAYING) v.pos = ef_lib_pts2pts(t, pts_last[s], v.speed);   // save_pos
            d = (d & ~0xFu) | (uint32_t)cmd;
            switch (cmd) {
            case EF_LIB_PLAY: lib_play(v, t, 0); break;
            case EF_LIB_SKIP:
                v.pos += (int32_t)((uint32_t)arg * 90000u);
                lib_play(v, t, 0);
                break;
            case EF_LIB_FAST_FORWARD: lib_play(v, t, 1); break;
            case EF_LIB_REWIND: lib_play(v, t, -1); break;
            case EF_LIB_PAUSE: v.state = EF_LIB_PAUSED; blend = 180; break;    // show_progress(), then video_pause(1)
            case EF_LIB_RESUME: v.state = EF_LIB_PLAYING; blend = 180; op = 2; break;
            case EF_LIB_NAV_STEP: lib_nav(v, s, nav_to, mode, nv, n_streams, ovl); op = 1; break;
            default:                                                    // MENU
                if (v.state == EF_LIB_PLAYING) {                        // save_pos(pts, true)
                    nv[(size_t)v.title * n_streams + s] = v.pos;
                    if (v.speed) { lib_play(v, t, 0); break; }
                }
                lib_nav(v, s, v.title, mode, nv, n_streams, ovl);
                op = 1;
                break;
            }
            if (v.state == EF_LIB_PLAYING && cmd != EF_LIB_RESUME) {     // play(): show_progress(speed == 0 ? 180 : -1)
                blend = v.speed == 0 ? 180 : -1;
                op = 1;
            }
        }
        if (ovl && blend != -2) {
            ovl[s].p_blend = blend;
            ovl[s].pending |= 2u;
        }
        if (clk && (clk[s].flags & 1u)) {
            EfClockState& k = clk[s];
            k.speed = v.speed;
            k.flags = (k.flags & ~2u) | (v.state == EF_LIB_PAUSED ? 2u : 0u);
            if (zero_seconds) k.last_seconds = 0;
            if (v.title != title0) {
                const EfLibTitle& u = titles[v.title];
                k.v_first = u.v_first; k.v_last = u.v_last; k.f_first = u.f_first; k.f_last = u.f_last; k.r_first = u.r_first; k.r_last = u.r_last;
            }
        }
        ls[s] = v;
    }
    if (done) done[s] = (uint8_t)d;
    ops[s] = (uint8_t)op;
}

// One CTA: every PLAYING stream, and every POSTER stream with poster bytes left, takes min(its budget, packets left in its file)
// packets from its cursor; the exclusive prefix of the run lengths gives each stream's place in the submit (off[n_streams + 1],
// EfBlockScan). A stream whose cursor reaches the end of its file ends with this submit: end[s] = 1. A PLAYING stream becomes ENDED
// with pos = pts2pts(0, _speed) (save_pos(0) at DONE, espflix.cpp:906-911); a POSTER stream stays POSTER with its pos (the poster
// stays on screen), and its mode travels with the submit: smode[s] (NULL on a context without posters) = mode[s] there, else 0.
// src[s] = where the stream's run starts.
__global__ void __launch_bounds__(1024)
ef_library_count_kernel(EfLibStream* __restrict__ ls, const EfLibTitle* __restrict__ titles, const uint32_t* __restrict__ budget, uint32_t packets,
                        int n_streams, const uint8_t** __restrict__ src, uint64_t* __restrict__ off, uint8_t* __restrict__ end,
                        const uint8_t* __restrict__ mode, uint8_t* __restrict__ smode)
{
    __shared__ EfBlockScan<uint64_t, 1024> scan;
    scan.init();
    for (int base = 0; base < n_streams; base += 1024) {
        const int k = base + threadIdx.x;
        uint64_t v = 0;
        if (k < n_streams) {
            EfLibStream q = ls[k];
            uint8_t e = 0, m = 0;
            if (q.state == EF_LIB_PLAYING || q.state == EF_LIB_POSTER) {
                const EfLibTitle& t = titles[q.title];
                const uint64_t size = t.bytes[q.file];
                if (q.state == EF_LIB_PLAYING || q.cursor < size) {
                    const uint64_t left = q.cursor < size ? (size - q.cursor) / 188u : 0;
                    const uint64_t b = budget ? budget[k] : packets;
                    const uint64_t take = b < left ? b : left;
                    v = take * 188u;
                    src[k] = t.ts[q.file] + (q.cursor < size ? q.cursor : 0);
                    q.cursor += v;
                    if (take == left) {
                        e = 1;
                        if (q.state == EF_LIB_POSTER) m = mode[k];
                        else {
                            q.state = EF_LIB_ENDED;
                            q.pos = ef_lib_pts2pts(t, 0, q.speed);
                        }
                    }
                    ls[k] = q;
                }
            }
            end[k] = e;
            if (smode) smode[k] = m;
        }
        const uint64_t excl = scan.exclusive(v);
        if (k < n_streams) off[k] = excl;
    }
    if (threadIdx.x == 0) off[n_streams] = scan.carry;
}

// The gather: the submit is one flat range of 16-byte units, EF_LIB_UNITS of them per thread, a CTA's units contiguous. Every stream's
// run is one contiguous range of its file copied to one contiguous range of the submit; both ends are multiples of 188 (4-byte
// aligned, not 16). Each unit is stored with one aligned 16-byte store, its four words loaded from whichever runs they belong to
// (a unit may straddle runs). Thread 0 finds the CTA's first run by binary search over off[]; each thread then walks forward.
// Words past the end of the submit are stored as 0 (the staging buffer has room for the last unit).
#define EF_LIB_GATHER_THREADS 256
#define EF_LIB_UNITS 4
__global__ void __launch_bounds__(EF_LIB_GATHER_THREADS)
ef_library_gather_kernel(const uint8_t* const* __restrict__ src, const uint64_t* __restrict__ off, int n_streams, uint8_t* __restrict__ dst)
{
    __shared__ int s0;
    const uint64_t total = off[n_streams];
    const uint64_t unit0 = (uint64_t)blockIdx.x * (EF_LIB_GATHER_THREADS * EF_LIB_UNITS);
    if (unit0 * 16 >= total) return;
    if (threadIdx.x == 0) {                                                 // the last run with off[s] <= the CTA's first byte
        int lo = 0, hi = n_streams - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (off[mid] <= unit0 * 16) lo = mid; else hi = mid - 1;
        }
        s0 = lo;
    }
    __syncthreads();
    int s = s0;
    uint64_t s_lo = off[s], s_hi = off[s + 1];
    uint4 out[EF_LIB_UNITS];
#pragma unroll
    for (int j = 0; j < EF_LIB_UNITS; j++) {
        const uint64_t b0 = (unit0 + (uint64_t)j * EF_LIB_GATHER_THREADS + threadIdx.x) * 16;
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint64_t b = b0 + 4 * i;
            w[i] = 0;
            if (b < total) {
                while (b >= s_hi) { s++; s_lo = s_hi; s_hi = off[s + 1]; }
                w[i] = __ldg((const uint32_t*)(src[s] + (b - s_lo)));
            }
        }
        out[j] = make_uint4(w[0], w[1], w[2], w[3]);
    }
#pragma unroll
    for (int j = 0; j < EF_LIB_UNITS; j++) {
        const uint64_t b0 = (unit0 + (uint64_t)j * EF_LIB_GATHER_THREADS + threadIdx.x) * 16;
        if (b0 < total) *(uint4*)(dst + b0) = out[j];
    }
}

cudaError_t ef_launch_library_resolve(EfLibStream* ls, const EfLibTitle* titles, const int64_t* pts_last, int first, int count, int cmd, int title,
                                      int64_t arg, uint8_t* mode, int64_t* nv, int n_streams, int n_titles, EfOverlayState* ovl)
{
    ef_library_resolve_kernel<<<(count + 127) / 128, 128>>>(ls, titles, pts_last, first, count, cmd, title, arg, mode, nv, n_streams, n_titles, ovl);
    return cudaGetLastError();
}

cudaError_t ef_launch_library_keys(EfLibStream* ls, const EfLibTitle* titles, const int64_t* pts_last, const uint8_t* keys, uint8_t* done, uint8_t* ops,
                                   uint8_t* mode, int64_t* nv, int n_streams, int n_titles, EfOverlayState* ovl, EfClockState* clk, cudaStream_t st)
{
    ef_library_keys_kernel<<<(n_streams + 127) / 128, 128, 0, st>>>(ls, titles, pts_last, keys, done, ops, mode, nv, n_streams, n_titles, ovl, clk);
    return cudaGetLastError();
}

// count, then gather over at most max_bytes of submit (the host's bound: its grid follows it, CTAs past the submit's end exit)
cudaError_t ef_launch_library_gather(EfLibStream* ls, const EfLibTitle* titles, const uint32_t* budget, uint32_t packets, int n_streams,
                                     const uint8_t** src, uint64_t* off, uint8_t* end, const uint8_t* mode, uint8_t* smode, uint8_t* dst,
                                     uint64_t max_bytes, cudaStream_t st, uint64_t* launches)
{
    ef_library_count_kernel<<<1, 1024, 0, st>>>(ls, titles, budget, packets, n_streams, src, off, end, mode, smode);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    ++*launches;
    const uint64_t per_cta = (uint64_t)EF_LIB_GATHER_THREADS * EF_LIB_UNITS * 16;
    const uint64_t ctas = (max_bytes + per_cta - 1) / per_cta;
    if (!ctas) return cudaSuccess;
    ef_library_gather_kernel<<<(unsigned)ctas, EF_LIB_GATHER_THREADS, 0, st>>>(src, off, n_streams, dst);
    ++*launches;
    return cudaGetLastError();
}
