/* oracle/ref_config.h — TEST INFRASTRUCTURE, not product code.
 *
 * Hand-written stand-in for the header the reference's CMake would generate from
 * /root/reference/config.h.in (cmakedefines at config.h.in:11-532, rare()/usual() at :587-588).
 * Only used by oracle/build_ref.sh to compile the reference's vendored Xapian
 * (/root/reference/src/xapian) where it lies; no reference source is copied into this repo.
 */
#ifndef XGM_REF_CONFIG_H
#define XGM_REF_CONFIG_H

#define HAVE_STRINGS_H 1
#define HAVE_STRING_H 1
#define HAVE_FLOAT_H 1
#define HAVE_STDLIB_H 1
#define HAVE_STDDEF_H 1
#define HAVE_STDINT_H 1
#define HAVE_INTTYPES_H 1
#define HAVE_SYS_STAT_H 1
#define HAVE_SYS_TYPES_H 1
#define HAVE_FCNTL_H 1
#define HAVE_LIMITS_H 1
#define HAVE_NETINET_IN_H 1
#define HAVE_POLL_H 1
#define HAVE_SYS_SELECT_H 1
#define HAVE_SYS_SOCKET_H 1
#define HAVE_SYS_TIME_H 1
#define HAVE_UNISTD_H 1
#define HAVE_SYS_RESOURCE_H 1
#define HAVE_SYS_UIO_H 1
#define HAVE_SYS_UTSNAME_H 1
#define HAVE_ZLIB_H 1
#define STDC_HEADERS 1
#define HAVE_ZLIB 1
#define HAVE_PTHREADS 1

#define HAVE_CLOCK_GETTIME 1
#define HAVE_POLL 1
#define HAVE_FDATASYNC 1
#define HAVE_FSYNC 1
#define HAVE_GETTIMEOFDAY 1
#define HAVE_NANOSLEEP 1
#define HAVE_POSIX_FADVISE 1
#define HAVE_PREAD 1
#define HAVE_PWRITE 1
#define HAVE_SELECT 1
#define HAVE_SOCKET 1
#define HAVE_FORK 1
#define HAVE_FTRUNCATE 1
#define HAVE_GETHOSTNAME 1
#define HAVE_GETRLIMIT 1
#define HAVE_GETRUSAGE 1
#define HAVE_LINK 1
#define HAVE_NFTW 1
#define HAVE_RANDOM 1
#define HAVE_SETENV 1
#define HAVE_SIGACTION 1
#define HAVE_SIGSETJMP 1
#define HAVE_SLEEP 1
#define HAVE_SOCKETPAIR 1
#define HAVE_SRANDOM 1
#define HAVE_STRERROR_R 1
#define HAVE_SYSCONF 1
#define HAVE_TIMER_CREATE 1
#define HAVE_TIMES 1
#define HAVE_WRITEV 1
#define HAVE_CLOSEFROM 1
#define HAVE_STD_IS_TRIVIALLY_COPYABLE 1
#define HAVE___BUILTIN_EXPECT 1

#define HAVE_DECL_EXP10 1
#define HAVE_DECL_LOG2 1
#define HAVE_DECL_STRERROR_R 1
#define HAVE_DECL___BUILTIN_ADD_OVERFLOW 1
#define HAVE_DECL___BUILTIN_MUL_OVERFLOW 1
#define HAVE_DECL___BUILTIN_BSWAP16 1
#define HAVE_DECL___BUILTIN_BSWAP32 1
#define HAVE_DECL___BUILTIN_BSWAP64 1
#define HAVE_DECL___BUILTIN_CLZ 1
#define HAVE_DECL___BUILTIN_CLZL 1
#define HAVE_DECL___BUILTIN_CLZLL 1
#define HAVE_DECL___BUILTIN_CTZ 1
#define HAVE_DECL___BUILTIN_CTZL 1
#define HAVE_DECL___BUILTIN_CTZLL 1
#define HAVE_DECL___BUILTIN_POPCOUNT 1
#define HAVE_DECL___BUILTIN_POPCOUNTL 1
#define HAVE_DECL___BUILTIN_POPCOUNTLL 1
#define HAVE_DECL___BUILTIN_EXPECT 1
#define HAVE_DECL__BYTESWAP_UINT64 0
#define HAVE_DECL__BYTESWAP_ULONG 0
#define HAVE_DECL__BYTESWAP_USHORT 0
#define HAVE_DECL__PUTENV_S 0
#define HAVE_DECL___EXP10 0
#define HAVE_DECL___POPCNT 0
#define HAVE_DECL___POPCNT64 0

#define XAPIAN_MOVE_SEMANTICS 1
#define DIR_SEPS '/'
#define DIR_SEPS_LIST {'/'}
#define FLINTLOCK_USE_FLOCK 1
#define PACKAGE "xapiand"
#define PACKAGE_STRING "xapian-core 1.5.0"
#define SNPRINTF snprintf
#define SNPRINTF_ISO snprintf
#define FOLLOWS_IEEE 1
#define SOCKLEN_T socklen_t
#define STRERROR_R_CHAR_P 1
#define HAVE_UUID_UUID_H 1 /* oracle/ref_uuid.h, not /proc/sys/kernel/random/uuid */
#define XAPIAN_LIB_BUILD 1
#define SIZEOF_SHORT 2
#define SIZEOF_INT 4
#define SIZEOF_LONG 8
#define SIZEOF_LONG_LONG 8

#define rare(COND) __builtin_expect(!!(COND), 0)
#define usual(COND) __builtin_expect(!!(COND), 1)

#endif
