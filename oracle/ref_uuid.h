/* oracle/ref_uuid.h — TEST INFRASTRUCTURE: the part of libuuid's <uuid/uuid.h> the reference's
 * Uuid::generate uses (backends/uuids.cc, HAVE_UUID_UUID_H branch).  oracle/build_ref.sh installs it as
 * oracle/_ref/gen/uuid/uuid.h.  The default /proc/sys/kernel/random/uuid source is missing in sandboxes
 * and containers that hide /proc/sys, where every WritableDatabase would then fail to open.
 * Random version-4 UUIDs from getrandom(2); a database UUID only has to differ between databases.
 */
#ifndef XGM_REF_UUID_H
#define XGM_REF_UUID_H
#include <stdint.h>
#include <string.h>
#include <sys/random.h>
#include <time.h>
#include <unistd.h>

typedef unsigned char uuid_t[16];

static inline void uuid_generate(uuid_t out) {
    size_t got = 0;
    while (got < 16) {
        ssize_t n = getrandom(out + got, 16 - got, 0);
        if (n <= 0) break;
        got += (size_t)n;
    }
    if (got < 16) { /* no entropy source: splitmix64 over the clock, the pid and a counter */
        static uint64_t counter = 0;
        struct timespec ts;
        clock_gettime(CLOCK_REALTIME, &ts);
        uint64_t x = (uint64_t)ts.tv_sec * 1000000007ull ^ (uint64_t)ts.tv_nsec ^ ((uint64_t)getpid() << 32) ^ ++counter;
        for (int i = 0; i < 2; ++i) {
            uint64_t z = (x += 0x9e3779b97f4a7c15ull);
            z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
            z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
            z ^= z >> 31;
            memcpy(out + 8 * i, &z, 8);
        }
    }
    out[6] = (unsigned char)((out[6] & 0x0f) | 0x40); /* version 4 */
    out[8] = (unsigned char)((out[8] & 0x3f) | 0x80); /* RFC 4122 variant */
}
#endif
